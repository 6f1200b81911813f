"""Adaptive projected guidance under `method="adaptive"` on the H100: the device controller feeds the words pass and the
APG step from its coefficient block (dev_coef[9..10]) while the host passes (1, 0). Against the host controller on the
device and against the CPU executor, on a discrete, a linear and a flow schedule, both algorithms and orders 2 and 3,
eta and a norm threshold (momentum is refused with the adaptive method): the same number of network evaluations, and y
within ADAPTIVE_TOL relative."""
import contextlib
import io

import numpy as np
import pytest
import torch

from apg_oracle import APGOracle
from cases import make_betas
from gpu_configs import backend, rel_err

pytestmark = pytest.mark.gpu
# Measured on an H100 80GB HBM3 (700 W power limit) over the 8 runs of each schedule below, the largest relative
# distance of the device controller's y: discrete 9.1e-7 from the host controller and 1.0e-6 from the CPU executor,
# linear 1.35e-6 from both, flow 0. The controllers sum the error norm in other orders, so an accepted step size can move
# by an ulp and the trajectories then differ by rounding; the NFE never differed. Asserted at 1.5 times the largest.
ADAPTIVE_TOL = 2.0e-6
SHAPE = (2, 4, 16, 16)


def schedule(name):
    import dpm_solver_b200 as new
    if name == "flow":
        return new.NoiseScheduleFlow(shift=3.0)
    if name == "linear":
        return new.NoiseScheduleVP("linear")
    return new.NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))


def run(name, algo, order, device, controller="device", scales=None):
    """(y, NFE) of one adaptive APG run: the NFE the solver prints (the device controller enqueues iterations in
    chunks between two reads of its `done` flag, so it calls the network past the end of the run)."""
    import dpm_solver_b200 as new
    ns = schedule(name)
    def net(x, t, c):        # exact IEEE multiplies and adds: the CPU and the device evaluate it to the same bits
        one = (-1,) + (1,) * (x.dim() - 1)
        o = 0.1 * x + ((t * 0.001) * 0.05 - 0.02).reshape(one)
        return o * (1. + 0.25 * c.reshape(one)) + 0.05 * c.reshape(one)

    B = SHAPE[0]
    w = 5.0 if scales is None else torch.tensor(scales, device=device)
    fn = new.model_wrapper(net, ns, model_type="flow" if name == "flow" else "noise", guidance_type="classifier-free",
                           condition=torch.ones(B, 1, device=device), unconditional_condition=torch.zeros(B, 1, device=device),
                           guidance_scale=w, apg_eta=0.3, apg_norm_threshold=25.0)
    s = new.DPM_Solver(fn, ns, algorithm_type=algo)
    s.adaptive_controller = controller
    x = torch.randn(SHAPE, generator=torch.Generator().manual_seed(4)).to(device)
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        y = s.sample(x, order=order, method="adaptive", atol=0.0078, rtol=0.05)
    return y.cpu(), int(out.getvalue().split()[-1])


@pytest.mark.parametrize("name", ["discrete", "linear", "flow"])
def test_device_controller_vs_host_and_executor(cuda_backend, name):
    worst_host = worst_cpu = 0.0
    for algo in ("dpmsolver++", "dpmsolver"):
        for order in (2, 3):
            for scales in (None, [4.0, 1.0]):
                y, n = run(name, algo, order, "cuda", scales=scales)
                yh, nh = run(name, algo, order, "cuda", "host", scales)
                with backend(APGOracle(exact=True)):
                    yc, nc = run(name, algo, order, "cpu", scales=scales)
                what = (algo, order, scales)
                assert n == nh == nc, (what, n, nh, nc)
                assert np.isfinite(y.numpy()).all(), what
                worst_host = max(worst_host, rel_err(y, yh))
                worst_cpu = max(worst_cpu, rel_err(y, yc))
    print("\n%s: device controller vs host %.3g, vs CPU executor %.3g" % (name, worst_host, worst_cpu))
    assert worst_host <= ADAPTIVE_TOL and worst_cpu <= ADAPTIVE_TOL, (worst_host, worst_cpu)
