"""The CPU side of tests/test_gpu_random_configs.py, pinned where there is no device: the fixed seeds reach every path
the device test must meet, and the oracle of the device runs -- the numpy executor on the extended draws -- equals the
unmodified reference wherever the reference can express the configuration."""
import random

import pytest

from gpu_configs import CHUNKS, REQUIRED, SEED, configurations, cpu_oracle, draw_gpu, reference_expressible, tally_static
from oracle import ref_loader

needs_reference = pytest.mark.skipif(not ref_loader.available(), reason="oracle/_ref not built and no reference tree")


def test_the_fixed_seeds_cover_every_path():
    """The static part of the tally, from the draws alone: runs without a device."""
    seen = {k for chunk in range(CHUNKS) for c in configurations(chunk) for k in tally_static(c)}
    assert not [k for k in REQUIRED if k not in seen]


@needs_reference
def test_extended_draws_reference_equals_executor():
    """The oracle of the device runs, pinned where there is no device: of the extended draws, 30 the reference can
    express must come out of the numpy executor bit for bit (intermediates and call trace included); the others on
    the way (16-bit state, per-sample scales, rescale, several conditions) must run on the executor or be rejected."""
    rng = random.Random(SEED - 1)
    checked = others = 0
    while checked < 30:
        c = draw_gpu(rng)
        if c["shape"] == (4, 64, 64) and c["B"] == 4 and c["steps"] > 24:
            continue                                    # (keep the CPU run short)
        out = cpu_oracle(c)
        if reference_expressible(c) and c["method"] != "adaptive" and "error" not in out:
            assert out.get("reference"), c
            checked += 1
        else:
            others += 1
    assert others >= 30
