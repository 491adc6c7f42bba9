"""The demod kernel's wide tiles (1984 outputs per pass on d = 1 and the d = 2 fast path, 31 RSSI segments of 64) against
the oracle, bit for bit, at batch lengths that end a tile one segment in (M = 2048), one segment short of full
(M = 61440 = 30 * 1984 + 1920) and exactly on a tile boundary (M = 63488 = 32 * 1984); the narrow tile of the mixer
at d = 2 beside them (CPU build)."""
import numpy as np
import pytest

import pipeline_checks as pc
from conftest import load_fixture


@pytest.mark.parametrize("blocks", [1, 30, 31])
@pytest.mark.parametrize("flags", ["-v", "-v -a -p S", "-v -d 1", "-v -d 1 -s", "-v -s"])
def test_demod_stages_at_tile_edges(pkg, hostsim_lib, flags, blocks):
    cu8 = load_fixture("synth_mixed_1m6.cu8")
    d = 1 if "-d 1" in flags else 2
    n = 4096 * d * blocks                        # check_stages' batch granule: 2048 decimated samples
    assert len(cu8) >= n
    pc.check_stages(pkg, hostsim_lib, np.ascontiguousarray(cu8[:n]), flags)
