"""The CPU side of tests/test_gpu_flow_unipc_random_configs.py, pinned where there is no device: the oracle of every
configuration the device test draws is built here -- the numpy executor, equal to the unmodified reference bit for bit
(flow DPM_Solver) or to its multistep DPM-Solver(++)(2M) within UNIPC_2M_TOL (UniPC bh2, order <= 2, no corrector)
wherever the reference can express the configuration -- the refused ones are exactly the documented ones, and the
fixed seeds reach every path the device test must meet."""
import pytest

from flow_unipc_configs import (CHUNKS, REQUIRED, REQUIRED_PINNED, configurations, cpu_oracle, flow_reference_expressible,
                                refused, tally_static, unipc_is_2m)
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
            continue
        assert out["calls"] and all(t.dtype == out["y"].dtype for t in out["inter"]), c
        assert ("pinned" in out) == (flow_reference_expressible(c) or unipc_is_2m(c)), c
        for k in tally_static(c) + (["pinned:" + out["pinned"]] if "pinned" in out else []):
            TALLY[k] = TALLY.get(k, 0) + 1
    CHUNKS_RUN.add(chunk)


def test_tally_of_the_drawn_configurations():
    """After the chunks: every path the device test requires, both pinnings and a refused draw were met."""
    if len(CHUNKS_RUN) < CHUNKS:
        pytest.skip("needs every chunk of test_oracle_of_every_drawn_configuration in the same session")
    print("\ntally: %s" % dict(sorted(TALLY.items())))
    assert not [k for k in REQUIRED + REQUIRED_PINNED + ["rejected"] if not TALLY.get(k)]
