"""dpm_step_unipc and DPM_PARAM_FLOW launches across many CTAs and every tuning.

k_step_unipc walks its tiles in a grid-stride loop: with a CTA cap (ctas_per_sm > 0) every CTA runs several tiles, and
each later tile reads its per-sample threshold by packet index (pk / pk_per_sample on the FAST kernels, (e + i) /
per_sample on the generic ones). The launches here are sized to about 3.5 x sm_count x 4 x 256 x 16 elements (3.5
passes of the largest capped grid: 4 CTAs per SM, 256 threads, 2 packets of 8 each), so at every (threads, ctas) in
{0, 32, 64, 256} x {0, 1, 2, 4} the loop iterates; odd per-sample sizes add a tail for the scalar kernel. Every
(corrector order, predictor order) and number of network outputs, the five dtype pairs of k_step_unipc, FAST (NOISE,
FLOW) and generic (X_START, or thresholds with a per-sample size that is not a multiple of 8) launches are compared
with the numpy executor bit for bit at the default tuning and must give identical bits at every other one.
k_step_unipc_scalar (grid capped at sm_count x 8 CTAs of 256 threads) loops over an unaligned view above 600k
elements. FLOW launches on the direct, TMA ring and multi-condition kernels get the same tuning invariance."""
import dataclasses
import random

import numpy as np
import pytest
import torch

from dpm_solver_b200 import plan as P
from dpm_solver_b200._lib import FORM_DIFF2, FORM_LIN1, FORM_LIN2, FORM_MS3, PARAM_FLOW, PARAM_NOISE, PARAM_X_START
from dpm_solver_b200.ops import StepArgs
from flow_oracle import FlowOracle
from step_edges import assert_bits_equal
from unipc_oracle import UniPCOracle

pytestmark = pytest.mark.gpu
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
PAIRS = [(F32, F32), (BF16, BF16), (F16, F16), (BF16, F32), (F16, F32)]     # (model, state) of k_step_unipc
ORDERS = [(pc, pp) for pc in range(4) for pp in range(4) if pc or pp]
TUNINGS = [(t, c) for t in (0, 32, 64, 256) for c in (0, 1, 2, 4)]
B = 5


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 12 * 2 ** 30


def per_sample_sizes():
    """(a multiple of 8, an odd size) per sample, B samples making about 3.5 passes of the largest capped grid."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per8 = int(3.5 * sms * 4 * 256 * 16) // (8 * B) * 8
    return per8, per8 + 3


def _bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a.contiguous()), _bits(b.contiguous()))


def _data(rng, n, dt):
    return torch.from_numpy(rng.standard_normal(n, dtype=np.float32) * np.float32(2)).to(dt)


def _to(a, dev, offset=0):
    """StepArgs `a` with every tensor on `dev`; offset > 0: each a view that many elements into a larger buffer."""
    d = dataclasses.replace(a)
    for f in dataclasses.fields(a):
        v = getattr(a, f.name)
        if torch.is_tensor(v):
            if offset and f.name != "thr":
                buf = torch.empty(v.numel() + offset, dtype=v.dtype, device=dev)
                buf[offset:].copy_(v.reshape(-1))
                v = buf[offset:].view(v.shape)
            else:
                v = v.to(dev)
            setattr(d, f.name, v)
        elif isinstance(v, tuple) and v and torch.is_tensor(v[0]):
            setattr(d, f.name, tuple(t.to(dev) for t in v))
    return d


# ---- k_step_unipc -----------------------------------------------------------------------------------------------
def unipc_cases():
    """Every (pc, pp) x number of network outputs, each with a seeded dtype pair, parameterisation, solver space and
    threshold layout."""
    rng = random.Random(4242)
    cases = []
    for k, ((pc, pp), ne) in enumerate((o, ne) for o in ORDERS for ne in (0, 1, 2)):
        md, sd = rng.choice(PAIRS if ne else PAIRS[:3])
        param = rng.choice([PARAM_NOISE, PARAM_FLOW, PARAM_X_START])
        px0 = ne > 0 and rng.random() < 0.7
        thr = px0 and rng.random() < 0.7
        mult8 = rng.random() < 0.5
        fast = ne == 0 or (param in (PARAM_NOISE, PARAM_FLOW) and not (thr and not mult8))
        words = P.UniCoeffs(pc, pp, (rng.uniform(-1, 1), rng.uniform(-1, 1)), rng.uniform(-1, 1), rng.uniform(0.5, 1.5),
                            rng.uniform(-1, 1), (rng.uniform(-1, 1), rng.uniform(-1, 1)))
        cases.append(dict(seed=k, pc=pc, pp=pp, ne=ne, md=md, sd=sd, param=param, px0=px0, thr=thr, mult8=mult8,
                          fast=fast, words=words))
    return cases


def unipc_args(c, per):
    """The launch of case `c` on the host, B samples of `per` elements."""
    rng = np.random.default_rng(c["seed"])
    n = B * per
    md, sd, ne = c["md"], c["sd"], c["ne"]
    x = _data(rng, n, sd)
    a = StepArgs(form=FORM_LIN1, n_model=ne, x=x, xe=x, m0=_data(rng, n, sd) if ne == 0 else None,
                 m1=_data(rng, n, sd), m2=_data(rng, n, sd), m3=_data(rng, n, sd),
                 e_cond=_data(rng, n, md) if ne else None, e_uncond=_data(rng, n, md) if ne == 2 else None,
                 param=c["param"], predict_x0=c["px0"], guidance=3.5, alpha_e=0.6, sigma_e=0.8, want_m_out=ne > 0,
                 state_dtype=sd, unipc=c["words"])
    if c["thr"]:
        a.per_sample = per
        a.thr = torch.from_numpy(rng.random(B, dtype=np.float32) * np.float32(0.3) + np.float32(0.3))
    return a


def _nan_like(t):
    return torch.full_like(t, float("nan"))


def _fresh_outputs(d):
    """d with NaN-filled outputs, so that an element a launch fails to write never matches (not recycled memory)."""
    d = dataclasses.replace(d)
    if d.n_model > 0:
        d.m_out = _nan_like(d.x)
    if d.unipc is None or d.unipc.pp > 0:
        d.out = _nan_like(d.x)
    if d.unipc is not None:
        d.out_c = _nan_like(d.x)
        d.out2 = _nan_like(d.x) if d.unipc.pp > 0 else None
    return d


def _launch(be, d, tuning=(2, 0, 0)):
    """One launch into fresh outputs; returns (m_out, out, out2, out_c) (None where not written)."""
    d = _fresh_outputs(d)
    be.set_tuning(*tuning)
    try:
        m, o = be.step(d)
    finally:
        be.set_tuning(2, 0, 0)
    return m, o, d.out2, d.out_c


def test_unipc_launches_across_ctas_and_tunings(cuda_backend):
    per8, per_odd = per_sample_sizes()
    seen = set()
    for c in unipc_cases():
        per = per8 if c["mult8"] else per_odd
        host = unipc_args(c, per)
        host.out_c = torch.empty_like(host.x)
        with np.errstate(all="ignore"):
            wm, wo = UniPCOracle().step(host)
        d = _to(host, "cuda")
        m0, o0, o20, oc0 = _launch(cuda_backend, d)
        what = {k: c[k] for k in ("pc", "pp", "ne", "md", "sd", "param", "px0", "thr", "mult8")}
        if c["ne"]:
            assert_bits_equal(m0, wm, "m_out %s" % what)
        if c["pp"]:
            assert_bits_equal(o0, wo, "out %s" % what)
            assert_bits_equal(o20, wo, "out2 %s" % what)
        assert_bits_equal(oc0, host.out_c, "out_c %s" % what)
        del wm, wo, host
        for threads, ctas in TUNINGS:
            got = _launch(cuda_backend, d, (2, threads, ctas))
            for g, w, name in zip(got, (m0, o0, o20, oc0), ("m_out", "out", "out2", "out_c")):
                assert (g is None) == (w is None) and (g is None or _same(g, w)), (name, threads, ctas, what)
            del got
        seen |= {"fast" if c["fast"] else "generic", "pair:%s/%s" % (c["md"], c["sd"]), "ne:%d" % c["ne"],
                 "thr:%s:%s" % ("fast" if c["fast"] else "generic", "mult8" if c["mult8"] else "odd") if c["thr"] else
                 "no thr", "param:%d" % c["param"] if c["ne"] else "m0"}
        del d, m0, o0, o20, oc0
    want = {"fast", "generic", "ne:0", "ne:1", "ne:2", "thr:fast:mult8", "thr:generic:odd", "thr:generic:mult8",
            "param:%d" % PARAM_NOISE, "param:%d" % PARAM_FLOW, "param:%d" % PARAM_X_START}
    want |= {"pair:%s/%s" % p for p in PAIRS}
    assert want <= seen, want - seen


@pytest.mark.parametrize("pair", PAIRS + [(F32, BF16), (BF16, F16)], ids=lambda p: "%s/%s" % p)
def test_unipc_scalar_kernel_loops_over_an_unaligned_view(cuda_backend, pair):
    """A view one element into its buffer runs k_step_unipc_scalar over the whole range (as do the dtype pairs no
    packet kernel serves): above 600k elements its capped grid loops, and each element reads its threshold by
    (i + elem_offset) / per_sample."""
    md, sd = pair
    rng = random.Random(str(pair))
    for per in (140000, 140001):                        # B * per > 600k: 2.6 passes of sm_count x 8 x 256 on 132 SMs
        for (pc, pp), ne in (((3, 3), 2), ((2, 1), 1), ((1, 0), 1), ((3, 2), 0)):
            if ne == 0 and md != sd:
                continue
            c = dict(seed=per + 10 * pc + pp, pc=pc, pp=pp, ne=ne, md=md, sd=sd,
                     param=rng.choice([PARAM_NOISE, PARAM_FLOW, PARAM_X_START]), px0=ne > 0, thr=ne > 0,
                     words=P.UniCoeffs(pc, pp, (0.4375, -0.21875), -0.8125, 0.96875, -0.15625, (0.3125, 0.59375)))
            host = unipc_args(c, per)
            host.out_c = torch.empty_like(host.x)
            if pp:
                host.out2 = torch.empty_like(host.x)
            with np.errstate(all="ignore"):
                wm, wo = UniPCOracle().step(host)
            d = _to(host, "cuda", offset=1)            # (outputs too: out_c and out2 are unaligned views)
            assert d.x.data_ptr() % 16 != 0 and d.out_c.data_ptr() % 16 != 0
            d.out_c.fill_(float("nan"))
            if pp:
                d.out2.fill_(float("nan"))
            m, o = cuda_backend.step(d)
            if ne:
                assert_bits_equal(m, wm, "m_out %s" % c)
            if pp:
                assert_bits_equal(o, wo, "out %s" % c)
                assert_bits_equal(d.out2, wo, "out2 %s" % c)
            assert_bits_equal(d.out_c, host.out_c, "out_c %s" % c)


# ---- FLOW launches: direct, TMA ring, multi-condition --------------------------------------------------------------
def flow_cases():
    cases = []
    for k, (md, sd) in enumerate(PAIRS):
        cases += [dict(path="direct", form=FORM_DIFF2, ne=2, px0=True, thr="mult8"),
                  dict(path="direct", form=FORM_LIN2, ne=1, px0=True, thr="odd"),
                  dict(path="direct", form=FORM_MS3, ne=1, px0=False, thr=None),
                  dict(path="tma", form=FORM_DIFF2, ne=2, px0=True, thr=None),
                  dict(path="tma", form=FORM_LIN1, ne=1, px0=False, thr=None),
                  dict(path="multi", form=FORM_DIFF2, ne=2, px0=True, thr="mult8"),
                  dict(path="multi", form=FORM_MS3, ne=2, px0=False, thr=None)]
        for c in cases[-7:]:
            c.update(md=md, sd=sd)
    for i, c in enumerate(cases):
        c["seed"] = 500 + i
    return cases


def flow_args(c, per8, per_odd):
    rng = np.random.default_rng(c["seed"])
    per = per_odd if c["thr"] == "odd" else per8
    n = B * per
    md, sd = c["md"], c["sd"]
    x = _data(rng, n, sd)
    coef = {k: float(np.float32(rng.uniform(-1, 1))) for k in ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3")}
    a = StepArgs(form=c["form"], n_model=c["ne"], x=x, xe=x, m1=_data(rng, n, sd), m2=_data(rng, n, sd),
                 e_cond=_data(rng, n, md), e_uncond=_data(rng, n, md) if c["ne"] == 2 else None, param=PARAM_FLOW,
                 predict_x0=c["px0"], guidance=3.5, alpha_e=0.4, sigma_e=0.6, want_m_out=True, state_dtype=sd, **coef)
    if c["path"] == "multi":
        a.e_conds = (a.e_cond, _data(rng, n, md), _data(rng, n, md))
        a.scales = (4.0, -1.5, 7.5)
    if c["thr"]:
        a.per_sample = per
        a.thr = torch.from_numpy(rng.random(B, dtype=np.float32) * np.float32(0.3) + np.float32(0.3))
    return a


def test_flow_launches_across_ctas_and_tunings(cuda_backend):
    per8, per_odd = per_sample_sizes()
    for c in flow_cases():
        host = flow_args(c, per8, per_odd)
        with np.errstate(all="ignore"):
            wm, wo = FlowOracle().step(host)
        d = _to(host, "cuda")
        variant = 1 if c["path"] == "tma" else 2
        m0, o0 = (t.clone() for t in _launch_flow(cuda_backend, d, (variant, 0, 0)))
        assert_bits_equal(m0, wm, "m_out %s" % c)
        assert_bits_equal(o0, wo, "out %s" % c)
        del wm, wo, host
        for threads, ctas in TUNINGS:
            m, o = _launch_flow(cuda_backend, d, (variant, threads, ctas))
            assert _same(m, m0) and _same(o, o0), (threads, ctas, c)
            del m, o
        del d, m0, o0


def _launch_flow(be, d, tuning):
    d = _fresh_outputs(d)
    be.set_tuning(*tuning)
    try:
        return be.step(d)
    finally:
        be.set_tuning(2, 0, 0)
