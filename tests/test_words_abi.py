"""The C ABI of the per-sample guidance words passes, without a GPU: every dpm_*_workspace size over a grid of
(n_samples, per_sample), and the return code and message of each argument error of each words entry. All of these are
decided before any CUDA call, so the pointers below are never dereferenced, and no error advances dpm_launch_count."""
import ctypes as C

import pytest

from dpm_solver_b200 import _lib

ARG, UNSUPPORTED = -1, -2
F32, BAD_DTYPE = _lib.DPM_F32, 7
P, MISALIGNED = 1 << 20, (1 << 20) + 4    # fake device addresses: aligned, and not 8-byte aligned
SUMS = {"dpm_cfg_rescale_workspace": 4, "dpm_apg_workspace": 3, "dpm_cfgzero_workspace": 2, "dpm_tcfg_workspace": 3,
        "dpm_perpneg_workspace": 4}
GRID = [0, 1, 8191, 8192, 8193, 3 * 256 * 256, 1 << 33]


@pytest.fixture(scope="module")
def L():
    return _lib.lib()


@pytest.mark.parametrize("fn", sorted(SUMS))
def test_workspace_sizes(L, fn):
    for nb in GRID:
        for ps in GRID:
            want = 0 if nb == 0 or ps == 0 else nb * (-(-ps // 8192)) * SUMS[fn] * 8 % 2 ** 64
            assert getattr(L, fn)(nb, ps) == want, (nb, ps)


def _pair_cases(L, ws_fn, prefix):
    """The argument errors the pair passes share, as ((out, e_cond, e_uncond, dtype, per_sample, n, ws, ws_bytes),
    return code, message); message None: not set."""
    ws = getattr(L, ws_fn)(2, 8192)
    return [
        ((P, None, P, F32, 8, 16, P, ws), ARG, prefix + ": NULL tensor"),
        ((None, P, P, BAD_DTYPE, 8, 16, P, ws), ARG, prefix + ": NULL tensor"),
        ((P, P, P, BAD_DTYPE, 8, 16, P, ws), ARG, prefix + ": bad dtype or sizes"),
        ((P, P, P, F32, 0, 16, P, ws), ARG, prefix + ": bad dtype or sizes"),
        ((P, P, P, F32, 3, 16, P, ws), ARG, prefix + ": bad dtype or sizes"),
        ((P, P, P, F32, 8192, 16384, None, ws), ARG, prefix + ": workspace too small or not 8-byte aligned"),
        ((P, P, P, F32, 8192, 16384, P, ws - 1), ARG, prefix + ": workspace too small or not 8-byte aligned"),
        ((P, P, P, F32, 8192, 16384, MISALIGNED, ws), ARG, prefix + ": workspace too small or not 8-byte aligned"),
        ((P, P, P, F32, 1, 1 << 31, P, 1 << 40), UNSUPPORTED, prefix + ": too many chunks"),
        ((None, None, None, BAD_DTYPE, 0, 0, None, 0), 0, None),     # n == 0: nothing to do, nothing checked
    ]


def _call(L, fn, args, rc, msg):
    before = L.dpm_launch_count()
    assert fn(*args, None) == rc, (args, L.dpm_last_error())
    if msg is not None:
        assert L.dpm_last_error().decode() == msg, args
    assert L.dpm_launch_count() == before


def test_rescale_errors(L):
    for (o, c, u, dt, ps, n, w, wb), rc, msg in _pair_cases(L, "dpm_cfg_rescale_workspace", "cfg rescale"):
        _call(L, L.dpm_cfg_rescale_ratio, (o, c, u, 3.5, ps, n, dt, w, wb), rc, msg)
        _call(L, L.dpm_cfg_rescale_ratio_guided, (o, c, u, P if o else None, ps, n, dt, w, wb), rc, msg)
    _call(L, L.dpm_cfg_rescale_ratio_guided, (P, P, P, None, 8, 16, F32, P, 1 << 20), ARG, "cfg rescale: NULL tensor")


@pytest.mark.parametrize("entry,ws,prefix", [("dpm_cfgzero_scale", "dpm_cfgzero_workspace", "cfg-zero* scale"),
                                             ("dpm_tcfg_words", "dpm_tcfg_workspace", "tcfg words")])
def test_pair_pass_errors(L, entry, ws, prefix):
    for args, rc, msg in _pair_cases(L, ws, prefix):
        _call(L, getattr(L, entry), args, rc, msg)


def _apg_desc(**kw):
    d = _lib.StepDesc()
    d.x = d.xe = d.e_cond = d.e_uncond = P
    d.n, d.per_sample, d.n_model, d.guidance, d.alpha_e, d.sigma_e = 16384, 8192, 2, 3.5, 0.8, 0.6
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_apg_errors(L):
    ws = L.dpm_apg_workspace(2, 8192)
    need = "apg words: needs words, n_model == 2, raw_round == 0 and per_sample dividing n"
    small = "apg words: workspace too small or not 8-byte aligned"
    for desc, words, w, wb, rc, msg in [
            (None, P, P, ws, ARG, need),
            (_apg_desc(), None, P, ws, ARG, need),
            (_apg_desc(n_model=1), P, P, ws, ARG, need),
            (_apg_desc(per_sample=3), P, P, ws, ARG, need),
            (_apg_desc(per_sample=0), P, P, ws, ARG, need),
            (_apg_desc(param=_lib.PARAM_EDM, dev_coef=P), P, P, ws, ARG,
             "apg words: DPM_PARAM_EDM takes its words by value, not from dev_coef"),
            (_apg_desc(model_dtype=BAD_DTYPE), P, P, ws, ARG, "bad dtype (state 0, model 7)"),
            (_apg_desc(), P, None, ws, ARG, small),
            (_apg_desc(), P, P, ws - 1, ARG, small),
            (_apg_desc(), P, MISALIGNED, ws, ARG, small),
            (_apg_desc(n=1 << 31, per_sample=1), P, P, 1 << 40, UNSUPPORTED, "apg words: too many chunks"),
            (_apg_desc(n=0, n_model=0), None, None, 0, 0, None)]:
        _call(L, L.dpm_apg_words, (words, None if desc is None else C.byref(desc), None, 0.0, 0.0, 0.0, None, None,
                                   w, wb), rc, msg)


def test_perpneg_errors(L):
    ws = L.dpm_perpneg_workspace(2, 8192)
    conds = (C.c_void_p * 4)(P, P, P, P)
    scales = (C.c_float * 4)(7.5, -1.0, -1.0, -1.0)
    small = "perpneg words: workspace too small or not 8-byte aligned"

    def call(rc, msg, out=P, eu=P, ec=conds, sc=scales, k=2, dt=F32, ps=8192, n=16384, w=P, wb=ws):
        _call(L, L.dpm_perpneg_words, (out, eu, ec, sc, k, dt, ps, n, w, wb), rc, msg)

    # n_cond is checked first, before n == 0 and before every pointer; the dtype too comes before n == 0
    for k in (0, 1, 5):
        call(ARG, "perpneg words: n_cond must be 2..4, got %d" % k, k=k, out=None, n=0)
    call(ARG, "perpneg words: NULL pointer", out=None, dt=BAD_DTYPE)
    call(ARG, "perpneg words: NULL pointer", eu=None)
    call(ARG, "perpneg words: NULL pointer", ec=None)
    call(ARG, "perpneg words: NULL pointer", sc=None)
    call(ARG, "perpneg words: NULL e_conds[2]", ec=(C.c_void_p * 4)(P, P, None, P), k=3, dt=BAD_DTYPE)
    call(0, None, ec=(C.c_void_p * 4)(P, P, None, P), k=2, n=0)      # only the first n_cond entries are read
    call(ARG, "perpneg words: bad dtype", dt=BAD_DTYPE, n=0)
    call(0, None, n=0, ps=0)
    call(ARG, "perpneg words: per_sample must divide n", ps=0)
    call(ARG, "perpneg words: per_sample must divide n", ps=3)
    for k in (2, 3, 4):     # one workspace size, whatever K is
        call(ARG, small, k=k, w=None)
        call(ARG, small, k=k, wb=ws - 1)
        call(ARG, small, k=k, w=MISALIGNED)
    call(UNSUPPORTED, "perpneg words: too many chunks", ps=1, n=1 << 31, wb=1 << 40)
