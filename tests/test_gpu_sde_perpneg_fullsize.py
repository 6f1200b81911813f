"""SDE-DPM-Solver++ and Perp-Neg sample() at full size on the H100, checked on row slices against the numpy executor.

The network acts element by element (exact IEEE multiplies and adds, the same bits on the CPU and the device), so each
row of a run depends on that row's inputs alone: a slice of rows run through the executor must give the device run's
rows bit for bit. An SDE slice is fed the matching rows of the full run's draws (the contract's draw,
torch.empty_like(x, dtype=float32).normal_(generator=g) at each update, replayed on the device from the same seed).

  * SDE at c2's bf16 [4096, 4, 64, 64]: 2M with CFG, 3M unguided;
  * SDE beyond 2^29 elements (bf16 [48094, 3, 61, 61]): the noise of each update is drawn as ATen draws it, in two
    launches, and half of the size is odd, so the second segment starts off a packet boundary (the element path);
  * Perp-Neg at bf16 [2048, 4, 64, 64] with K = 3 and 4: 16384 elements per sample, so the words pass merges two
    chunks per sample.
"""
import pytest
import torch

from gpu_configs import backend
from perpneg_oracle import PerpNegOracle
from sde_oracle import SdeOracle

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def net(x, t, c=None):
    """An element-wise network: 0.1*x plus a time term; with a condition c, (1 + c/4)*o + (c*c/20)*x*x (so that the
    conditional differences of several conditions are not parallel)."""
    one = (-1,) + (1,) * (x.dim() - 1)
    xf = x.float()
    o = 0.1 * xf + ((t * 0.001) * 0.05 - 0.02).reshape(one)
    if c is not None:
        cc = c.reshape(one).float()
        o = o * (1. + 0.25 * cc) + ((0.05 * cc) * cc) * (xf * xf)
    return o


def solve(x, kind, gen=None, K=0, scales=None, **skw):
    """sample() of x: kind "sde" (unguided), "sde_cfg" (scale 7.5) or "perp" (K conditions, `scales`), bf16 state."""
    import dpm_solver_b200 as new
    B, dev = x.shape[0], x.device
    ns = new.NoiseScheduleVP("discrete", betas=torch.linspace(1e-4, 2e-2, 1000))
    uc = torch.zeros(B, 1, device=dev)
    if kind == "sde":
        fn = new.model_wrapper(lambda xx, tt: net(xx, tt), ns, model_type="noise")
    elif kind == "sde_cfg":
        fn = new.model_wrapper(net, ns, model_type="noise", guidance_type="classifier-free",
                               condition=torch.ones(B, 1, device=dev), unconditional_condition=uc, guidance_scale=7.5)
    else:
        fn = new.model_wrapper(net, ns, model_type="noise", guidance_type="classifier-free",
                               condition=[torch.full((B, 1), float(k + 1), device=dev) for k in range(K)],
                               unconditional_condition=uc, guidance_scale=list(scales), perp_neg=True)
    algo = "dpmsolver++" if kind == "perp" else "sde-dpmsolver++"
    s = new.DPM_Solver(fn, ns, algorithm_type=algo, state_dtype=BF)
    if kind != "perp":
        skw = dict(skw, generator=gen)
    return s.sample(x, **skw)


def draws_of_rows(shape, seed, updates, slices):
    """The rows `slices` of each update's draw, replayed on the device from `seed`: ([[z_1[sl], ...] for sl in slices]
    on the CPU, the generator's offset after the draws)."""
    g = torch.Generator("cuda").manual_seed(seed)
    out = [[] for _ in slices]
    for _ in range(updates):
        z = torch.empty(shape, dtype=torch.float32, device="cuda").normal_(generator=g)
        for rows, sl in zip(out, slices):
            rows.append(z[sl].cpu())
        del z
    return out, g.get_offset()


class FedDraws(SdeOracle):
    """SdeOracle whose launches take their noise from `draws` in order (the rows of the full run's draws) instead of
    drawing it."""

    def __init__(self, draws):
        super().__init__()
        self.fed = iter(draws)

    def draw(self, a):
        return next(self.fed).to(a.x.device).reshape(a.x.shape)


def executor_with_draws(run, draws):
    """run() on the CPU with FedDraws(draws)."""
    with backend(FedDraws(draws)):
        return run()


def check_sde_rows(x, kind, seed, slices, order, steps, eta):
    """The device run of x from `seed` against the executor on each slice of rows; the generator ends where the
    contract's draws leave it."""
    skw = dict(steps=steps, order=order, eta=eta, solver_type="taylor" if order == 3 else "dpmsolver")
    g = torch.Generator("cuda").manual_seed(seed)
    y = solve(x, kind, g, **skw)
    ys = [y[sl].cpu() for sl in slices]
    del y
    draws, offset = draws_of_rows(x.shape, seed, steps, slices)
    assert g.get_offset() == offset
    for sl, got, zs in zip(slices, ys, draws):
        xs = x[sl].cpu()
        want = executor_with_draws(lambda: solve(xs, kind, torch.Generator(), **skw), zs)
        assert torch.equal(got, want), (kind, sl, float((got.float() - want.float()).abs().max()))


def _memory_under(gib):
    return torch.cuda.max_memory_allocated() <= gib * 2 ** 30


@pytest.mark.parametrize("kind,order", [("sde_cfg", 2), ("sde", 3)])
def test_sde_sample_at_c2_size(cuda_backend, kind, order):
    torch.cuda.reset_peak_memory_stats()
    shape = (4096, 4, 64, 64)
    x = torch.randn(shape, generator=torch.Generator("cuda").manual_seed(1), device="cuda").to(BF)
    slices = [slice(0, 3), slice(2047, 2050), slice(4093, 4096)]
    check_sde_rows(x, kind, 40 + order, slices, order, steps=5, eta=1.0)
    assert _memory_under(12), torch.cuda.max_memory_allocated()


def test_sde_sample_beyond_2_29_elements(cuda_backend):
    """n = 48094*3*61*61 > 2^29: each update's noise is two launches of n/2 (odd) elements; the rows around the split
    and at both ends against the executor."""
    from dpm_solver_b200 import ops
    torch.cuda.reset_peak_memory_stats()
    shape = (48094, 3, 61, 61)
    ps = 3 * 61 * 61
    n = shape[0] * ps
    assert n > 1 << 29 and (n // 2) % 8
    x = torch.empty(shape, dtype=BF, device="cuda")
    x.copy_(torch.randn(shape, generator=torch.Generator("cuda").manual_seed(2), device="cuda"))
    torch.cuda.empty_cache()
    split = (n // 2) // ps
    slices = [slice(0, 2), slice(split - 1, split + 2), slice(shape[0] - 2, shape[0])]
    assert ops.backend().name == "cuda-sm90a"
    check_sde_rows(x, "sde", 77, slices, order=2, steps=2, eta=0.5)
    assert _memory_under(16), torch.cuda.max_memory_allocated()


@pytest.mark.parametrize("K,scales", [(3, [5.0, -2.0, -1.5]), (4, [4.0, -1.0, 0.0, -2.5])])
def test_perp_neg_sample_at_full_size(cuda_backend, K, scales):
    """bf16 [2048, 4, 64, 64]: 16384 elements per sample (two words chunks each), rows against the executor."""
    torch.cuda.reset_peak_memory_stats()
    shape = (2048, 4, 64, 64)
    x = torch.randn(shape, generator=torch.Generator("cuda").manual_seed(K), device="cuda")
    skw = dict(steps=4, order=2)
    y = solve(x, "perp", K=K, scales=scales, **skw)
    assert _memory_under(12), torch.cuda.max_memory_allocated()
    for sl in (slice(0, 2), slice(1023, 1026), slice(2046, 2048)):
        with backend(PerpNegOracle(exact=True)):
            want = solve(x[sl].cpu(), "perp", K=K, scales=scales, **skw)
        assert torch.equal(y[sl].cpu(), want), (K, sl)
