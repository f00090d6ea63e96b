"""GPU parity of K1 (pyr_fast_kernel) at the boundaries between its code paths, every stage against the CPU oracle at every level.

K1 copies level 0 word by word where a tile's columns and ring need no reflection, and scores FAST without per-pixel cell tests
where the tile and its ring lie inside the cell grid; the other tiles take the general paths.  Level-0 widths (769, 767, 641,
703) and heights (449, 511) one pixel above and below a multiple of the 64x64 tile put a tile of one or 63 columns / rows at the
right and bottom edges (tests/test_k1_tile64_gpu.py covers heights at every level), and the first and last
tiles of each level touch exactly one image edge and the edge of the cell grid.  Binary noise makes every pixel pair of such a
tile matter: corners everywhere, saturated margins, and maxima on both sides of every cell edge."""
import numpy as np
import pytest

from extract_cases import boundary_lattice, cams_for, run_batch

pytestmark = pytest.mark.gpu


def noise(w, h, seed):
    return (np.random.default_rng(seed).integers(0, 2, (h, w)) * 255).astype(np.uint8)


@pytest.mark.parametrize("w,h", [(769, 479), (767, 481), (641, 449), (703, 511)])
def test_tile_size_boundaries(api, oa, cams, w, h):
    cs = cams_for(cams, w, h)
    imgs = np.stack([noise(w, h, 1), boundary_lattice(w, h, 1), noise(w, h, 2)[::-1].copy()])
    masks = np.stack([np.ones((h, w), np.uint8)] * 3)
    res = run_batch(api, oa, imgs, masks, cs, [0, 1, 2], 2000, "mdbrief")
    for _, raw in res:
        assert len(raw) > 0


def test_mirror_masks_at_path_boundaries(api, oa, cams):
    """camera mirror masks: tiles on the mask border consult the level-0 mask per corner, on both K1 paths"""
    from multicol_slam_b200 import synth
    w, h = 769, 479
    cs = [synth.scaled_cam(c, w, h) for c in cams]
    imgs = np.stack([noise(w, h, 3), noise(w, h, 4), boundary_lattice(w, h, 2)])
    masks = np.stack([np.ascontiguousarray(api.mirror_mask(c)) for c in cs])
    run_batch(api, oa, imgs, masks, cs, [0, 1, 2], 2000, "mdbrief")
