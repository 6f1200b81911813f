"""The CPU side of tests/test_gpu_guidance_random_configs.py, pinned where there is no device: the exact executor's
result for every CFG-Zero*, CFG++, regional-guidance, TCFG, FDG and Perp-Neg configuration the device test draws,
against the unmodified reference wherever it can express the configuration (CFG-Zero*, masks, TCFG, FDG and Perp-Neg bit
for bit, CFG++ within CFGPP_TOL of the fp64 transcription, plus the rounding bound of an x_start network's x0
conversion, each with as many evaluations); an FDG run with equal scales is its one-level run; the refused
configurations are exactly the documented ones (each of Perp-Neg's refusals met); and the fixed seeds reach every path
the device test must meet."""
import pytest

from guidance_configs import CHUNKS, FEATURES, PERP_REFUSALS, REQUIRED, configurations, cpu_oracle, \
    perp_refusal_reached, reference_expressible, refused, tally_static
from oracle import ref_loader

pytestmark = pytest.mark.skipif(not ref_loader.available(), reason="oracle/_ref not built and no reference tree")
TALLY = {}
CHUNKS_RUN = set()


@pytest.mark.parametrize("chunk", range(CHUNKS))
def test_oracle_of_every_drawn_configuration(chunk):
    for c in configurations(chunk):
        out = cpu_oracle(c)
        assert ("error" in out) == refused(c), (c, out.get("error"))
        if "error" in out:
            assert isinstance(out["error"], ValueError), (c, out["error"])
            TALLY["rejected"] = TALLY.get("rejected", 0) + 1
            if perp_refusal_reached(c):
                TALLY["perp:refused:" + c["perp_refusal"]] = TALLY.get("perp:refused:" + c["perp_refusal"], 0) + 1
            continue
        assert all(t.dtype == out["y"].dtype for t in out["inter"]), c
        assert ("pinned" in out) == reference_expressible(c), c
        for k in tally_static(c) + (["pinned:" + c["feature"]] if "pinned" in out else []):
            TALLY[k] = TALLY.get(k, 0) + 1
    CHUNKS_RUN.add(chunk)


def test_tally_of_the_drawn_configurations():
    """After the chunks: every path the device test requires, a refused draw, each of Perp-Neg's refusals and a pinned
    draw of each feature."""
    if len(CHUNKS_RUN) < CHUNKS:
        pytest.skip("needs every chunk of test_oracle_of_every_drawn_configuration in the same session")
    print("\ntally: %s" % dict(sorted(TALLY.items())))
    pinned = ["pinned:" + f for f in FEATURES]
    refusals = ["perp:refused:" + why for why in PERP_REFUSALS]
    assert not [k for k in REQUIRED + pinned + refusals + ["rejected"] if not TALLY.get(k)]
