"""UniPC on the device: every kind of dpm_step_unipc launch against the numpy executor bit for bit, sample() against the
executor over seeded configurations (first call, second call, fresh solver, graph replay, intermediates), full-size
launches against separate torch CUDA ops, and the bf16-state distance to the fp64 transcription."""
import math
import random

import numpy as np
import pytest
import torch

from cases import make_betas
from dpm_solver_b200 import NoiseScheduleFlow, NoiseScheduleVP, UniPC, model_wrapper, ops, plan as P
from dpm_solver_b200._lib import PARAM_FLOW, PARAM_NOISE, PARAM_SCORE, PARAM_V, PARAM_X_START
from dpm_solver_b200.ops import StepArgs
from unipc_oracle import UniPCOracle, unipc_fp64

pytestmark = pytest.mark.gpu

PAIRS = [(torch.float32, torch.float32), (torch.bfloat16, torch.bfloat16), (torch.float16, torch.float16),
         (torch.bfloat16, torch.float32), (torch.float16, torch.float32)]
ORDERS = [(pc, pp) for pc in range(4) for pp in range(4) if pc or pp]


def same(a, b):
    a, b = a.detach().cpu().float(), b.detach().cpu().float()
    return a.shape == b.shape and bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


def _tensor(shape, dt, g, dev, edge=False):
    v = torch.randn(shape, generator=g) * 2
    if edge:       # IEEE edges: zeros of both signs, infinities, NaN, huge and tiny values
        flat = v.view(-1)
        k = flat.numel()
        idx = torch.randint(0, k, (max(1, k // 50),), generator=g)
        vals = torch.tensor([0.0, -0.0, float("inf"), -float("inf"), float("nan"), 3e38, -3e38, 1e-30, 6e4])
        flat[idx] = vals[torch.randint(0, len(vals), idx.shape, generator=g)]
    return v.to(dt).to(dev)


def launch_case(rng, g):
    pc, pp = rng.choice(ORDERS)
    te, ts = rng.choice(PAIRS)
    ne = rng.choice([0, 1, 2]) if te == ts else rng.choice([1, 2])
    param = rng.choice([PARAM_NOISE, PARAM_NOISE, PARAM_FLOW, PARAM_X_START, PARAM_V, PARAM_SCORE])
    predict_x0 = rng.random() < 0.6
    thr = ne > 0 and predict_x0 and rng.random() < 0.3
    B = rng.choice([1, 2, 3])
    per = rng.choice([4096, 64, 13, 1024 + 5])
    layout = rng.choice(["c", "c", "c", "view", "cl"])
    edge = rng.random() < 0.2
    return dict(pc=pc, pp=pp, te=te, ts=ts, ne=ne, param=param, predict_x0=predict_x0, thr=thr, B=B, per=per,
                layout=layout, out2=pp > 0 and rng.random() < 0.4, out_c=pp == 0 or rng.random() < 0.4, edge=edge,
                words=P.UniCoeffs(pc, pp, (rng.uniform(-1, 1), rng.uniform(-1, 1)), rng.uniform(-1, 1),
                                  rng.uniform(0.5, 1.5), rng.uniform(-1, 1), (rng.uniform(-1, 1), rng.uniform(-1, 1))))


def build_args(c, dev, g):
    B, per = c["B"], c["per"]
    if c["layout"] == "cl":
        shape = (B, 4, 8, per // 32 if per >= 32 else 1) if per % 32 == 0 else (B, per)
    else:
        shape = (B, per)
    ts_, te_ = c["ts"], c["te"]
    gen = lambda dt: _tensor(shape, dt, g, "cpu", c["edge"])
    host = dict(x=gen(ts_), m0=gen(ts_), m1=gen(ts_), m2=gen(ts_), m3=gen(ts_), ec=gen(te_), eu=gen(te_))
    dv = {}
    for k, v in host.items():
        if dev == "cpu":
            dv[k] = v
        elif c["layout"] == "view":          # unaligned: a view one element into a larger buffer
            buf = torch.empty(v.numel() + 1, dtype=v.dtype, device=dev)
            buf[1:].copy_(v.reshape(-1).to(dev))
            dv[k] = buf[1:].view(v.shape)
        elif c["layout"] == "cl" and v.dim() == 4:
            dv[k] = v.to(dev).contiguous(memory_format=torch.channels_last)
        else:
            dv[k] = v.to(dev)
    ne = c["ne"]
    a = StepArgs(form=1, n_model=ne, x=dv["x"], xe=dv["x"], m0=dv["m0"] if ne == 0 else None, m1=dv["m1"], m2=dv["m2"],
                 e_cond=dv["ec"] if ne else None, e_uncond=dv["eu"] if ne == 2 else None, param=c["param"],
                 predict_x0=c["predict_x0"], guidance=3.5, alpha_e=0.6, sigma_e=0.8, want_m_out=ne > 0,
                 state_dtype=ts_, unipc=c["words"], m3=dv["m3"])
    n = dv["x"].numel()
    if c["thr"]:
        a.per_sample = n // B
        a.thr = (torch.rand(B, generator=g) * 2 + 0.5).to(dev)
    if c["out2"]:
        a.out2 = torch.empty_like(dv["x"])
    if c["out_c"]:
        a.out_c = torch.empty_like(dv["x"])
    return a


@pytest.mark.parametrize("tuning", [(2, 0, 0), (0, 128, 0), (0, 64, 2), (2, 256, 1)])
def test_every_launch_kind_matches_the_executor(cuda_backend, tuning):
    rng = random.Random(1000 + tuning[1] + tuning[2])
    ora = UniPCOracle()
    cuda_backend.set_tuning(*tuning)
    try:
        seen = set()
        for k in range(300):
            c = launch_case(rng, None)
            seen.add((c["pc"], c["pp"], c["ne"]))
            a_d = build_args(c, "cuda", torch.Generator().manual_seed(k))
            a_h = build_args(c, "cpu", torch.Generator().manual_seed(k))
            if c["thr"]:
                a_d.thr = a_h.thr.cuda()
            m_d, o_d = cuda_backend.step(a_d)
            m_h, o_h = ora.step(a_h)
            if c["ne"] > 0:
                assert same(m_d, m_h), c
            if c["pp"] > 0:
                assert same(o_d, o_h), c
                if c["out2"]:
                    assert same(a_d.out2, o_h), c
            if c["out_c"]:
                assert same(a_d.out_c, a_h.out_c), c
        torch.cuda.synchronize()
        assert len(seen) >= 35
    finally:
        cuda_backend.set_tuning(2, 0, 0)


def test_rejected_launches_launch_nothing(cuda_backend):
    x = torch.zeros(64, device="cuda")
    before = cuda_backend.launch_count()
    for w in (P.UniCoeffs(4, 1), P.UniCoeffs(0, 0), P.UniCoeffs(1, -1)):
        with pytest.raises(Exception):
            cuda_backend.step(StepArgs(form=1, n_model=1, x=x, e_cond=x, m1=x, m2=x, unipc=w))
    with pytest.raises(Exception):      # pc == 3 without m_{i-3}
        cuda_backend.step(StepArgs(form=1, n_model=1, x=x, e_cond=x, m1=x, m2=x, unipc=P.UniCoeffs(3, 1)))
    with pytest.raises(Exception):      # raw_round
        cuda_backend.step(StepArgs(form=1, n_model=1, x=x, e_cond=x, m1=x, unipc=P.UniCoeffs(1, 1), raw_round=1))
    assert cuda_backend.launch_count() == before


# ---- sample() ----------------------------------------------------------------------------------------------------------

def draw(rng):
    sched = rng.choice(["discrete", "discrete", "linear", "flow"])
    steps = rng.randint(1, 12)
    sd = rng.choice([None, None, torch.bfloat16, torch.float16])
    params = ["noise", "noise", "x_start", "flow"] if sched == "flow" else ["noise", "noise", "x_start", "v", "score"]
    return dict(sched=sched, steps=steps, order=rng.randint(1, min(3, steps)), variant=rng.choice(["bh1", "bh2"]),
                alg=rng.choice(["dpmsolver++", "dpmsolver"]), corr=rng.random() < 0.8, lof=rng.random() < 0.5,
                d2z=rng.random() < 0.2, sd=sd, param=rng.choice(params), cfg=rng.random() < 0.4,
                thr=rng.random() < 0.25, shape=rng.choice([(4, 64, 64), (3, 8, 8), (4, 128, 128), (1, 7, 5)]),
                B=rng.choice([1, 2, 3]), skip=rng.choice(["logSNR", "time_uniform", "time_quadratic"]),
                hook=rng.random() < 0.15)


def make(c, dev):
    ns = NoiseScheduleFlow(shift=3.0) if c["sched"] == "flow" else (
        NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1])) if c["sched"] == "discrete"
        else NoiseScheduleVP("linear"))

    def net(x, t, cc=None):        # exact IEEE multiplies and adds: the same bits on CPU and CUDA
        out = 0.1 * x + ((t * 0.001) * 0.05 - 0.02).reshape(-1, *([1] * (x.dim() - 1)))
        return out if cc is None else out + 0.05 * cc.reshape(-1, *([1] * (x.dim() - 1)))

    B = c["B"]
    kw = dict(model_type=c["param"])
    if c["cfg"]:
        kw.update(guidance_type="classifier-free", condition=torch.ones(B, device=dev),
                  unconditional_condition=torch.zeros(B, device=dev), guidance_scale=4.5)
    hook = (lambda x, t, s: x * 0.5 + x * 0.5) if c["hook"] else None
    return UniPC(model_wrapper(net, ns, **kw), ns, algorithm_type=c["alg"], variant=c["variant"], state_dtype=c["sd"],
                 correcting_x0_fn="dynamic_thresholding" if c["thr"] and c["alg"] == "dpmsolver++" else None,
                 correcting_xt_fn=hook)


def kwargs(c):
    return dict(steps=c["steps"], order=c["order"], skip_type=c["skip"], lower_order_final=c["lof"],
                use_corrector=c["corr"], denoise_to_zero=c["d2z"])


@pytest.mark.parametrize("chunk", range(4))
def test_sample_matches_the_executor(chunk):
    rng = random.Random(77 + chunk)
    old = ops._backend
    try:
        for k in range(25):
            c = draw(rng)
            x = torch.randn(c["B"], *c["shape"], generator=torch.Generator().manual_seed(k))
            ops.set_backend(UniPCOracle())
            y_h, inter_h = make(c, "cpu").sample(x, return_intermediate=True, **kwargs(c))
            ops.set_backend(ops.CudaBackend())
            s = make(c, "cuda")
            xd = x.cuda()
            y1, inter_d = s.sample(xd, return_intermediate=True, **kwargs(c))
            assert same(y1, y_h), c
            assert len(inter_d) == len(inter_h) and all(same(u, v) for u, v in zip(inter_d, inter_h)), c
            assert same(s.sample(xd, **kwargs(c)), y_h), c                 # second call
            assert same(make(c, "cuda").sample(xd, **kwargs(c)), y_h), c  # fresh solver
            if not c["hook"]:
                g = make(c, "cuda").capture(xd, **kwargs(c))
                assert same(g(xd), y_h), c
            torch.cuda.synchronize()
    finally:
        ops.set_backend(old)


def test_one_fused_launch_per_evaluation(cuda_backend):
    ns = NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))
    net = lambda x, t: 0.1 * x
    x = torch.randn(2, 4, 64, 64, device="cuda")
    for thr, per_eval in ((False, 1), (True, 2)):
        s = UniPC(model_wrapper(net, ns), ns, correcting_x0_fn="dynamic_thresholding" if thr else None)
        s.sample(x, steps=10, order=3)
        torch.cuda.synchronize()
        before = cuda_backend.launch_count()
        s.sample(x, steps=10, order=3)
        torch.cuda.synchronize()
        n = cuda_backend.launch_count() - before
        if thr:
            assert 10 * 2 <= n <= 10 * 4, n       # one quantile (one or two kernels) and one step per evaluation
        else:
            assert n == 10, n


# ---- full size -----------------------------------------------------------------------------------------------------------

def _torch_chain(x, ec, m1, m2, w, dt):
    T = ec.float()
    c = x.float() + w.cd[0] * (m2.float() - m1.float())
    c = (c + w.ct * (T - m1.float())).to(dt).float()
    o = w.a * c + w.c0 * T
    o = o + w.cp[0] * (m1.float() - T)
    return o.to(dt), c.to(dt)


W2 = P.UniCoeffs(2, 2, (0.4375, 0.0), -0.8125, 0.96875, -0.15625, (0.3125, 0.0))


def test_c2_shape_bf16_equals_torch_ops(cuda_backend):
    g = torch.Generator(device="cuda").manual_seed(0)
    sh, dt = (4096, 4, 64, 64), torch.bfloat16
    x, ec, m1, m2 = (torch.randn(sh, device="cuda", generator=g).to(dt) for _ in range(4))
    out_c = torch.empty_like(x)
    m, o = cuda_backend.step(StepArgs(form=1, n_model=1, x=x, e_cond=ec, m1=m1, m2=m2, want_m_out=True, state_dtype=dt,
                                      unipc=W2, out_c=out_c))
    o_ref, c_ref = _torch_chain(x, ec, m1, m2, W2, dt)
    assert torch.equal(o, o_ref) and torch.equal(out_c, c_ref) and torch.equal(m, ec)


def test_one_launch_beyond_2_31_elements(cuda_backend):
    n = (1 << 31) + 1003
    g = torch.Generator(device="cuda").manual_seed(1)
    dt = torch.bfloat16
    x, ec, m1, m2 = (torch.randn(n, device="cuda", generator=g).to(dt) for _ in range(4))
    _, o = cuda_backend.step(StepArgs(form=1, n_model=1, x=x, e_cond=ec, m1=m1, m2=m2, state_dtype=dt, unipc=W2))
    step = 1 << 28
    for s0 in range(0, n, step):
        sl = slice(s0, min(n, s0 + step))
        o_ref, _ = _torch_chain(x[sl], ec[sl], m1[sl], m2[sl], W2, dt)
        assert torch.equal(o[sl], o_ref), s0


# ---- bf16 distance -------------------------------------------------------------------------------------------------------

# max |x_N(bf16 state) - x_N(fp64)| / max |x_N(fp64)| on the configuration below, measured on an H100 (DESIGN.md §8.10)
BF16_DISTANCE = 1.85e-2


def test_bf16_state_distance_to_the_fp64_transcription(cuda_backend):
    """c2-like: SD's discrete schedule, noise network, dpmsolver++, UniPC-2 bh2 with the corrector, 20 steps."""
    ns = NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))
    net = lambda x, t: 0.1 * x + ((t * 0.001) * 0.05 - 0.02).reshape(-1, 1, 1, 1)
    x = torch.randn(8, 4, 64, 64, generator=torch.Generator().manual_seed(2))
    y = UniPC(model_wrapper(net, ns), ns, state_dtype=torch.bfloat16).sample(x.cuda(), steps=20, order=2)
    s = UniPC(model_wrapper(net, ns), ns)
    ts = s.get_time_steps("time_uniform", ns.T, 1. / ns.total_N, 20, "cpu")
    marg = P.Marginals(ns, ts)
    lam, al, sg = (v.double().numpy() for v in (marg.lam, marg.alpha, marg.sigma))
    tin = ((ts.double() - 1. / ns.total_N) * 1000.).numpy()

    def model(xx, i):
        eps = 0.1 * xx + ((tin[i] * 0.001) * 0.05 - 0.02)
        return (xx - sg[i] * eps) / al[i]

    x64 = unipc_fp64(model, al, sg, lam, x.double().numpy(), 2)
    d = float(np.abs(y.double().cpu().numpy() - x64).max() / np.abs(x64).max())
    print("bf16 state distance to fp64:", d)
    assert d <= 1.5 * BF16_DISTANCE, d
