"""The CPU side of tests/test_gpu_sde_random_configs.py, pinned where there is no device: every SDE-DPM-Solver++
configuration the device test draws, run on the numpy executor with the CPU generator. The refused configurations are
exactly the documented ones and launch and draw nothing; an eta = 0 run is the "dpmsolver++" run bit for bit and
leaves its generator untouched; where k-diffusion's DPM++ 2M / 3M SDE loop can express a draw, the executor lies within
KDIFF_TOL of it in float64, fed the same noise; and the fixed seeds reach every path the device test must meet."""
import pytest

from sde_configs import CHUNKS, REQUIRED, REQUIRED_PINNED, REQUIRED_REFUSED, configurations, kdiff_expressible, \
    oracle, refused, tally_static

TALLY = {}
CHUNKS_RUN = set()


def hit(key):
    TALLY[key] = TALLY.get(key, 0) + 1


@pytest.mark.parametrize("chunk", range(CHUNKS))
def test_oracle_of_every_drawn_configuration(chunk):
    for c in configurations(chunk):
        out = oracle(c)
        assert ("error" in out) == refused(c), (c, out.get("error"))
        if "error" in out:
            assert isinstance(out["error"], ValueError), (c, out["error"])
            hit("refused:" + (c["refusal"] or "base"))
            continue
        assert all(t.dtype == out["y"].dtype for t in out["inter"]), c
        assert out["draws"] == (c["steps"] if c["eta"] else 0), c
        pinned = out.get("pinned")
        assert (pinned is not None and pinned != "eta=0") == kdiff_expressible(c), c
        for k in tally_static(c):
            hit(k)
        if pinned is not None:
            hit("pinned:" + ("eta=0" if pinned == "eta=0" else "kdiff"))
    CHUNKS_RUN.add(chunk)


def test_tally_of_the_drawn_configurations():
    """After the chunks: every path the device test requires, each refusal, and both pins."""
    if len(CHUNKS_RUN) < CHUNKS:
        pytest.skip("needs every chunk of test_oracle_of_every_drawn_configuration in the same session")
    print("\ntally: %s" % dict(sorted(TALLY.items())))
    assert not [k for k in REQUIRED + REQUIRED_PINNED + REQUIRED_REFUSED if not TALLY.get(k)]
