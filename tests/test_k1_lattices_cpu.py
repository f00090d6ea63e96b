"""The dot lattices the K1 warp-segment tests are built from, checked on the CPU oracle: each must reach the bound it is built for,
so that a later edit of a generator cannot quietly turn its GPU test into an easy case.

K1 (pyr_fast_kernel) collects a tile's corners in one shared-memory segment of kWarpCorners slots per warp, with no guard: a
warp's corner kWarpCorners + 1 would land in the next warp's first slot.  A segment filled exactly to kWarpCorners while the next
warp of the same tile holds a corner is the case where a segment one slot short shows in the raw corners."""
import numpy as np
import pytest

from extract_cases import (boundary_lattice, boundary_lattice_target, cams_for, fullest_segment, segments_before_corners,
                           warp_fill_lattice)
from k1_geometry import K1

FILL_SIZES = [(1280, 720), (1279, 720)]          # cells of 31 px: one tile column whose rows hold 34 maxima
LATTICE_SIZES = [(754, 480), (1280, 720), (764, 480), (641, 479)]


def oracle_corners(oa, cams, img):
    """level-0 raw corners of the oracle (x, y, score)"""
    h, w = img.shape
    oe = oa.OracleExtractor(nfeatures=1000, nlevels=1)
    oe.extract(img, np.ones((h, w), np.uint8), cams_for(cams, w, h)[0])
    return oe.debug_read(0, 3)


@pytest.mark.parametrize("w,h", FILL_SIZES)
def test_warp_fill_lattice_fills_segments(oa, cams, w, h):
    """phases 0 and 1 together fill segments of at least two different warps to exactly kWarpCorners before a non-empty one"""
    full = set()
    for phase in (0, 1):
        raw = oracle_corners(oa, cams, warp_fill_lattice(w, h, phase))
        seg = segments_before_corners(raw)
        assert max(seg.values()) == K1["kWarpCorners"], f"phase {phase}: fullest segment {max(seg.values())}"
        full |= {k[2] for k, v in seg.items() if v == K1["kWarpCorners"]}
    print(f"{w}x{h}: segments of {K1['kWarpCorners']} corners before a non-empty warp, warps {sorted(full)}")
    assert len(full) >= 2 and max(full) < K1["kThreads"] // 32 - 1


@pytest.mark.parametrize("w,h", LATTICE_SIZES)
def test_boundary_lattice_reaches_its_target(oa, cams, w, h):
    for v in range(3):
        assert fullest_segment(oracle_corners(oa, cams, boundary_lattice(w, h, v))) == boundary_lattice_target(w), (w, h, v)
    print(f"{w}x{h}: boundary_lattice fills {boundary_lattice_target(w)} of {K1['kWarpCorners']} slots before a non-empty warp")
    if w == 1280:
        assert boundary_lattice_target(w) == K1["kWarpCorners"] - 1
