"""GPU parity of K1 (pyr_fast_kernel) on 64x64 tiles, every stage against the CPU oracle at every level.

Level heights one row above and below a multiple of 64 leave a bottom tile of one or 63 rows; the 420x269 pyramid ends in levels of
75 and 90 rows, a full tile over a short one, and its level 7 is as short as a level can be (the FAST cell grid needs 74 rows).
FAST cells are about 30 px, so every 64-row tile crosses two or three cell edges in each direction; binary noise puts maxima on
both sides of each.  Mirror masks give tiles on the mask border (flag 1), and a tight device batch of an odd width stages its
rows without TMA."""
import numpy as np
import pytest

from extract_cases import boundary_lattice, cams_for, run_batch

pytestmark = pytest.mark.gpu

SIZES = [(705, 577), (833, 383), (420, 269)]


def noise(w, h, seed):
    return (np.random.default_rng(seed).integers(0, 2, (h, w)) * 255).astype(np.uint8)


@pytest.mark.parametrize("w,h", SIZES)
def test_tile_rows_at_level_edges(api, oa, cams, w, h):
    cs = cams_for(cams, w, h)
    imgs = np.stack([noise(w, h, 11), boundary_lattice(w, h, 5), noise(w, h, 12)[:, ::-1].copy()])
    masks = np.stack([np.ones((h, w), np.uint8)] * 3)
    res = run_batch(api, oa, imgs, masks, cs, [0, 1, 2], 1000, "mdbrief")
    for _, raw in res:
        assert len(raw) > 0


@pytest.mark.parametrize("w,h", SIZES)
def test_mask_border_tiles(api, oa, cams, w, h):
    from multicol_slam_b200 import synth
    cs = [synth.scaled_cam(c, w, h) for c in cams]
    imgs = np.stack([noise(w, h, 13), synth.frame(cs[1], 7), boundary_lattice(w, h, 2)])
    masks = np.stack([np.ascontiguousarray(api.mirror_mask(c)) for c in cs])
    assert all(0 < (m != 0).mean() < 1 for m in masks)
    run_batch(api, oa, imgs, masks, cs, [0, 1, 2], 1000, "mdbrief")


def test_unaligned_device_batch(api, oa, cams):
    """a tight device batch of width 705 (rows not 16-byte aligned): level 0 is staged with byte loads instead of TMA"""
    import torch
    w, h = 705, 577
    cs = cams_for(cams, w, h)
    imgs = np.stack([noise(w, h, 14), boundary_lattice(w, h, 1), noise(w, h, 15)])
    masks = np.stack([np.ones((h, w), np.uint8)] * 3)
    ex = api.mdBRIEFextractorOct(nfeatures=1000, do_dBrief=True, learnMasks=True)
    oe = oa.OracleExtractor(nfeatures=1000, do_dbrief=True, learn_masks=True)
    dev = torch.device("cuda", 0)
    tight = torch.from_numpy(imgs).to(dev)
    st = torch.cuda.Stream(dev)
    with torch.cuda.stream(st):
        out = ex.extract_batch_device(tight, masks, cs, [0, 1, 2], stream=st)
    ex.check_status(st)
    counts = out["counts"].cpu().numpy()
    kps = out["kps"].cpu().numpy().view(api.KEYPOINT_DTYPE).reshape(3, -1)
    for i in range(3):
        ok, od, om = oe.extract(imgs[i], masks[i], cs[i])
        for l in range(ex.GetLevels()):
            assert np.array_equal(ex.debug_read(l, 0, i), oe.debug_read(l, 0)), f"image {i}: pyramid level {l}"
            assert np.array_equal(ex.debug_read(l, 3, i), oe.debug_read(l, 3)), f"image {i}: raw corners level {l}"
        n = counts[i]
        assert n == len(ok) and kps[i, :n].tobytes() == ok.tobytes()
        assert np.array_equal(out["desc"][i, :n].cpu().numpy(), od)
        assert np.array_equal(out["dmask"][i, :n].cpu().numpy(), om)
