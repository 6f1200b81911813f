"""The SDE and UniPC edge cases without a GPU: the dispatch mirror over the full case lists reaches every required
kernel and path, and on the same edge operands the two executors reduce to the plain executor bit for bit --
SdeOracle with cz = 0 to dpm_step's LIN1 / DIFF2 / MS3 update, UniPCOracle with (pc, pp) = (0, 1) to its LIN1 update.
test_step_edges_vs_reference.py holds that plain executor to the unmodified reference, which has neither SDE nor
UniPC; these identities carry it over to the new oracles at the edges."""
import dataclasses
from collections import Counter

import numpy as np
import pytest
import torch

from dpm_solver_b200._lib import FORM_LIN1
from oracle_backend import OracleBackend
from sde_oracle import SdeOracle
from sde_unipc_edges import (GivenNoise, build_sde, build_unipc, guard_hits, planted_hits, required, required_hits,
                             sde_specs, tally_launch, unipc_specs)
from step_edges import assert_bits_equal
from unipc_oracle import UniPCOracle

f32 = np.float32


def test_mirror_reaches_every_required_path():
    tally, hits = Counter(), Counter()
    for spec in sde_specs():
        a, info = build_sde(spec)
        guard_hits(hits, spec, a, info, tally_launch(tally, spec, a, info))
    for spec in unipc_specs():
        a, info = build_unipc(spec)
        guard_hits(hits, spec, a, info, tally_launch(tally, spec, a, info))
        planted_hits(hits, spec, info)
    missing = [k for k in required() if tally[k] == 0]
    # (the SDE pin and fp16 lanes are planted once z is drawn, on the device)
    missing += [k for k in required_hits() if (k[0] == "unipc" or k[1] in ("alpha", "thr")) and hits[k] == 0]
    assert not missing, missing


@pytest.mark.parametrize("chunk", range(4))
def test_sde_with_zero_cz_is_the_plain_update(chunk):
    """cz = 0: out = fl_S(o + 0*z) with o the plain update in fp32. o + (+-0) is o for every o but one: an update of
    -0 plus +0 (z >= 0, so 0*z = +0) is +0. So SdeOracle's out equals the executor's, except that where the fp32
    update is -0 and z >= 0 it is +0."""
    rng = np.random.default_rng(chunk)
    flipped = 0
    for spec in sde_specs()[chunk::4]:
        a, info = build_sde(spec)
        z = torch.from_numpy(rng.standard_normal(info["n"]).astype(f32))
        z[::5] = 0.0
        a.sde = dataclasses.replace(a.sde, cz=0.0)
        b = dataclasses.replace(a, sde=None)
        with np.errstate(all="ignore"):
            m_s, o_s = GivenNoise(z).step(dataclasses.replace(a, out2=None))
            m_p, o_p = SdeOracle().step(dataclasses.replace(b, out2=None))
            # the fp32 update: the same expression with an fp32 state over the operands as the launch reads them
            T0 = a.m0 if a.n_model == 0 else m_p
            o32 = OracleBackend().step(dataclasses.replace(
                b, n_model=0, m0=T0.float(), x=a.x.float(), m1=None if a.m1 is None else a.m1.float(),
                m2=None if a.m2 is None else a.m2.float(), state_dtype=torch.float32, e_cond=None, e_uncond=None,
                xe=None, thr=None, ratio=None, guidance_b=None, cfgzero_s=None, tcfg_w=None, out2=None))[1]
        neg0 = (o32.reshape(-1) == 0) & torch.signbit(o32.reshape(-1)) & (z >= 0)
        want = o_p.reshape(-1).clone()
        want[neg0] = 0.0
        flipped += int(neg0.sum())
        assert_bits_equal(o_s, want, "out of %s" % spec)
        assert (m_s is None) == (m_p is None)
        if m_s is not None:
            assert_bits_equal(m_s, m_p, "m_out of %s" % spec)
    assert flipped > 0


@pytest.mark.parametrize("chunk", range(4))
def test_unipc_predictor_alone_is_the_lin1_update(chunk):
    """(pc, pp) = (0, 1): c = x~ and out = a*c + c0*m_i, the LIN1 update of dpm_step with its words a, c0."""
    specs = [s for s in unipc_specs() if (s["pc"], s["pp"]) == (0, 1)]
    for spec in specs[chunk::4]:
        a, info = build_unipc(spec)
        a.out_c = a.out2 = None
        with np.errstate(all="ignore"):
            m_u, o_u = UniPCOracle().step(a)
            m_p, o_p = UniPCOracle().step(dataclasses.replace(a, unipc=None, m1=None, m2=None, m3=None,
                                                              form=FORM_LIN1, a=a.unipc.a, c0=a.unipc.c0))
        assert_bits_equal(o_u, o_p, "out of %s" % spec)
        assert (m_u is None) == (m_p is None)
        if m_u is not None:
            assert_bits_equal(m_u, m_p, "m_out of %s" % spec)
