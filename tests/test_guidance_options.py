"""Which classifier-free guidance options combine, and in which solver contexts each one runs, through the public API
on the CPU: every option alone and every pair of options through model_wrapper, then every accepted wrapper through
each solver context. A refusal is a ValueError before any network call and any launch; an accepted combination
completes a small run on the numpy executor."""
import itertools

import pytest
import torch

from perpneg_oracle import PerpNegOracle
from sde_oracle import SdeOracle

B, SHAPE = 2, (2, 2, 8, 8)


class Oracle(SdeOracle, PerpNegOracle):
    """The numpy executor with every guidance form and the SDE step."""


@pytest.fixture()
def backend():
    from dpm_solver_b200 import ops
    be = Oracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


def net(x, t, c):
    cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
    return 0.5 * torch.sin(1.3 * x) + 0.4 * x + 0.25 * cc * torch.cos(0.7 * x + cc) - 0.1


def _conds(kw):
    return len(kw["condition"]) if isinstance(kw["condition"], list) else 1


def _per_sample(kw):
    s = torch.tensor(kw["guidance_scale"], dtype=torch.float32)
    kw["guidance_scale"] = torch.stack([s * (1.0 + 0.1 * b) for b in range(B)])     # [B], or [B, K] with K conditions


# Each option edits model_wrapper's keyword arguments; a pair applies both edits in this order.
OPTIONS = {
    "fdg": lambda kw: kw.update(fdg_scales=[2.0, 3.0], guidance_scale=1.0),
    "several": lambda kw: kw.update(condition=[torch.full((B, 1), 1.0), torch.full((B, 1), 2.0)],
                                    guidance_scale=[7.5, -2.0]),
    "perp": lambda kw: kw.update(condition=[torch.full((B, 1), 1.0), torch.full((B, 1), 2.0)],
                                 guidance_scale=[7.5, -2.0], perp_neg=True),
    "mask": lambda kw: kw.update(guidance_mask=[torch.ones(8, 8)] * _conds(kw)),
    "per_sample": _per_sample,
    "rescale": lambda kw: kw.update(guidance_rescale=0.7),
    "apg": lambda kw: kw.update(apg_eta=0.0),
    "apg_momentum": lambda kw: kw.update(apg_eta=0.0, apg_momentum=-0.5),
    "cfgzero": lambda kw: kw.update(cfg_zero_star=True),
    "cfgzero_init": lambda kw: kw.update(cfg_zero_star=True, cfg_zero_init_steps=1),
    "cfgpp": lambda kw: kw.update(cfg_pp=True),
    "tcfg": lambda kw: kw.update(tcfg=True),
}

# Every option alone is accepted. These pairs are accepted; every other pair is refused.
ACCEPTED_PAIRS = {
    ("several", "perp"), ("several", "mask"), ("per_sample", "rescale"), ("per_sample", "apg"),
    ("per_sample", "apg_momentum"), ("per_sample", "cfgzero"), ("per_sample", "cfgzero_init"), ("per_sample", "cfgpp"),
    ("per_sample", "tcfg"), ("apg", "apg_momentum"), ("cfgzero", "cfgzero_init"),
}

# The solver contexts, in the column order of CONTEXT_TABLE.
CONTEXTS = ["reference_rounding", "sde", "unipc", "adaptive", "dpmsolver", "thresholding", "x0_fn", "singlestep",
            "singlestep_fixed", "order3", "direct"]

# Per accepted wrapper: x where the context refuses it, . where it runs.
CONTEXT_TABLE = """
                            rr sde unipc adaptive dpmsolver thr x0_fn singlestep fixed order3 direct
plain                       .  .   .     .        .         .   .     .          .     .      .
fdg                         x  .   .     .        .         .   .     .          .     .      .
several                     x  x   x     .        .         .   .     .          .     .      .
perp                        x  x   x     .        .         .   .     .          .     .      .
mask                        x  x   x     .        .         .   .     .          .     .      .
per_sample                  x  .   x     .        .         .   .     .          .     .      .
rescale                     x  .   x     .        .         .   .     .          .     .      .
apg                         x  x   .     .        .         .   .     .          .     .      .
apg_momentum                x  x   .     x        .         .   .     .          .     .      .
cfgzero                     x  .   .     .        .         .   .     .          .     .      .
cfgzero_init                x  .   .     x        .         .   .     .          .     .      .
cfgpp                       x  x   x     x        x         x   x     x          x     x      x
tcfg                        x  .   .     .        .         .   .     .          .     .      .
several+perp                x  x   x     .        .         .   .     .          .     .      .
several+mask                x  x   x     .        .         .   .     .          .     .      .
per_sample+rescale          x  .   x     .        .         .   .     .          .     .      .
per_sample+apg              x  x   x     .        .         .   .     .          .     .      .
per_sample+apg_momentum     x  x   x     x        .         .   .     .          .     .      .
per_sample+cfgzero          x  .   x     .        .         .   .     .          .     .      .
per_sample+cfgzero_init     x  .   x     x        .         .   .     .          .     .      .
per_sample+cfgpp            x  x   x     x        x         x   x     x          x     x      x
per_sample+tcfg             x  .   x     .        .         .   .     .          .     .      .
apg+apg_momentum            x  x   .     x        .         .   .     .          .     .      .
cfgzero+cfgzero_init        x  .   .     x        .         .   .     .          .     .      .
"""


def _table():
    rows = [r.split() for r in CONTEXT_TABLE.strip().splitlines()[1:]]
    return {tuple(r[0].split("+")) if r[0] != "plain" else (): dict(zip(CONTEXTS, (v == "x" for v in r[1:])))
            for r in rows}


TABLE = _table()


def _order(names):
    return tuple(n for n in OPTIONS if n in names)


def _kwargs(names):
    kw = dict(guidance_type="classifier-free", condition=torch.full((B, 1), 1.0),
              unconditional_condition=torch.zeros(B, 1), guidance_scale=7.5)
    for n in _order(names):
        OPTIONS[n](kw)
    return kw


def _wrap(names, calls):
    import dpm_solver_b200 as new

    def model(x, t, c):
        calls.append(tuple(x.shape))
        return net(x, t, c)
    return new.model_wrapper(model, new.NoiseScheduleVP("linear"), **_kwargs(names))


def _x():
    return torch.randn(SHAPE, generator=torch.Generator().manual_seed(0))


def _refused(backend, calls, call):
    n = backend.launch_count()
    with pytest.raises(ValueError):
        call()
    assert backend.launch_count() == n and calls == []


def test_the_table_covers_every_accepted_wrapper():
    singles = {(n,) for n in OPTIONS}
    assert set(TABLE) == {()} | singles | {_order(p) for p in ACCEPTED_PAIRS}
    assert all(_order(p) == p for p in ACCEPTED_PAIRS)


@pytest.mark.parametrize("pair", list(itertools.combinations(OPTIONS, 2)), ids="+".join)
def test_pairs(backend, pair):
    calls = []
    if pair in ACCEPTED_PAIRS:
        _wrap(pair, calls)
    else:
        _refused(backend, calls, lambda: _wrap(pair, calls))


def _direct_updates(s, x):
    t = lambda v: torch.tensor([v])
    ms, ts = [x * 0.9, x * 0.8, x * 0.7], [t(0.9), t(0.8), t(0.7)]
    return [
        lambda: s.dpm_solver_first_update(x, t(1.0), t(0.6)),
        lambda: s.singlestep_dpm_solver_second_update(x, t(1.0), t(0.6)),
        lambda: s.singlestep_dpm_solver_third_update(x, t(1.0), t(0.6)),
        lambda: s.singlestep_dpm_solver_update(x, t(1.0), t(0.6), order=2),
        lambda: s.multistep_dpm_solver_second_update(x, ms[1:], ts[1:], t(0.6)),
        lambda: s.multistep_dpm_solver_third_update(x, ms, ts, t(0.6)),
        lambda: s.multistep_dpm_solver_update(x, ms[1:], ts[1:], t(0.6), order=2),
        lambda: s.dpm_solver_adaptive(x, order=2, t_T=1.0, t_0=0.2, atol=1.0, rtol=1.0),
    ]


@pytest.mark.parametrize("names", list(TABLE), ids=lambda n: "+".join(n) or "plain")
def test_solver_contexts(backend, names, capsys):
    import dpm_solver_b200 as new
    ns = new.NoiseScheduleVP("linear")
    two = dict(steps=2, order=2)
    cases = {
        "reference_rounding": (dict(reference_rounding=True), dict(two)),
        "sde": (dict(algorithm_type="sde-dpmsolver++"), dict(two)),
        "adaptive": ({}, dict(method="adaptive", order=2, t_end=0.2, atol=1.0, rtol=1.0)),
        "dpmsolver": (dict(algorithm_type="dpmsolver"), dict(two)),
        "thresholding": (dict(correcting_x0_fn="dynamic_thresholding"), dict(two)),
        "x0_fn": (dict(correcting_x0_fn=lambda x0, t: x0), dict(two)),
        "singlestep": ({}, dict(two, method="singlestep")),
        "singlestep_fixed": ({}, dict(two, method="singlestep_fixed")),
        "order3": ({}, dict(steps=3, order=3)),
    }
    for ctx, refused in TABLE[names].items():
        calls = []
        fn = _wrap(names, calls)
        if ctx == "unipc":
            run = [lambda: new.UniPC(fn, ns).sample(_x(), **two)]
        elif ctx == "direct":
            run = _direct_updates(new.DPM_Solver(fn, ns), _x())
        else:
            skw, kw = cases[ctx]
            run = [lambda: new.DPM_Solver(fn, ns, **skw).sample(_x(), **kw)]
        for r in run:
            if refused:
                _refused(backend, calls, r)
            else:
                r()
                calls.clear()
    capsys.readouterr()
