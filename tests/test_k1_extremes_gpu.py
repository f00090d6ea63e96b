"""GPU parity of K1 (pyr_fast_kernel) at the bounds of its 64x64 tiles, every stage against the CPU oracle at every level.

Corner segments: warp w of a CTA collects the strict maxima of tile rows w, w + 8, .., w + 56 in its own shared-memory segment of
kWarpCorners = 8 x 34 slots, with no guard; corner kWarpCorners + 1 would land in the next warp's first slot.  warp_fill_lattice
fills segments to exactly kWarpCorners while the next warp of the tile holds a corner, so a segment one slot short loses or
duplicates a raw corner.  The checks run on a pitched host batch (rows staged by TMA) and on a tight device batch of an odd width
(level 0 staged byte by byte).

Staging: the source rows of a tile are staged in dynamic shared memory of max(box_h * kSrcWB, kStagingMin) bytes, box_h being the
level's tallest source region.  The geometries reach the tallest box the host accepts, a source / level ratio above 2, and box
heights on both sides of kStagingMin; level_boxes (the host's arithmetic) shows that each reaches its edge.  Every batch holds binary
noise, a dense lattice, a synthetic frame under the camera's mirror mask (tiles on the mask border at every level) and a seam: an
image whose last rows are black before one whose first rows are saturated.  The bottom tiles' boxes reach past their image, where
the 3-D tensor map zero-fills; a row taken from the next image would change the resized and blurred rows at the seam."""
import numpy as np
import pytest

from extract_cases import MODES, boundary_lattice, cams_for, run_batch, segments_before_corners, warp_fill_lattice
from k1_geometry import K1, level_boxes, staging_bytes

pytestmark = pytest.mark.gpu


def full_warps(raw):
    """warps whose segment holds exactly kWarpCorners level-0 corners while the next warp of the same tile holds corners too"""
    return {k[2] for k, v in segments_before_corners(raw).items() if v == K1["kWarpCorners"]}


def run_device_batch(api, oa, imgs, masks, cams, coi, nf, mode="mdbrief", **kw):
    """extract_batch_device of a tight device batch (row stride = width) against the oracle, every stage at every level; returns
    the device's level-0 raw corners per image"""
    import torch
    m = MODES[mode]
    ex = api.mdBRIEFextractorOct(nfeatures=nf, do_dBrief=m["do_dbrief"], learnMasks=m["learn_masks"], **kw)
    oe = oa.OracleExtractor(nfeatures=nf, **m, nlevels=kw.get("nlevels", 8), scale_factor=kw.get("scaleFactor", 1.2))
    dev = torch.device("cuda", 0)
    tight = torch.from_numpy(np.ascontiguousarray(imgs)).to(dev)
    st = torch.cuda.Stream(dev)
    with torch.cuda.stream(st):
        out = ex.extract_batch_device(tight, masks, cams, coi, stream=st)
    ex.check_status(st)
    counts = out["counts"].cpu().numpy()
    kps = out["kps"].cpu().numpy().view(api.KEYPOINT_DTYPE).reshape(len(imgs), -1)
    raws = []
    for i, c in enumerate(coi):
        ok, od, om = oe.extract(imgs[i], masks[c], cams[c])
        for l in range(ex.GetLevels()):
            for what, name in enumerate(("pyramid", "blurred", "mask", "raw corners")):
                if what != 1 or np.any(ok["octave"] == l):          # the oracle blurs only levels with keypoints
                    assert np.array_equal(ex.debug_read(l, what, i), oe.debug_read(l, what)), f"image {i}: {name} level {l}"
        n = counts[i]
        assert n == len(ok) and kps[i, :n].tobytes() == ok.tobytes(), f"image {i}: keypoints"
        assert np.array_equal(out["desc"][i, :n].cpu().numpy(), od), f"image {i}: descriptors"
        assert np.array_equal(out["dmask"][i, :n].cpu().numpy(), om), f"image {i}: descriptor masks"
        raws.append(ex.debug_read(0, 3, i))
    return raws


# ---- corner segments filled to kWarpCorners ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["orb", "mdbrief"])
@pytest.mark.parametrize("nlevels", [1, 8])
def test_warp_segments_filled(api, oa, cams, nlevels, mode):
    w, h = 1280, 720
    cs = cams_for(cams, w, h)
    imgs = np.stack([warp_fill_lattice(w, h, phase) for phase in (0, 1)])
    masks = np.stack([np.ones((h, w), np.uint8)] * 3)
    res = run_batch(api, oa, imgs, masks, cs, [0, 1], 2000, mode, nlevels=nlevels)
    warps = set().union(*(full_warps(raw) for _, raw in res))       # run_batch asserted these raw corners on the device's
    assert len(warps) >= 2, f"segments of {K1['kWarpCorners']} corners before a non-empty warp in warps {sorted(warps)}"


def test_warp_segments_filled_device_unaligned(api, oa, cams):
    w, h = 1279, 720
    cs = cams_for(cams, w, h)
    imgs = np.stack([warp_fill_lattice(w, h, phase) for phase in (0, 1)])
    masks = np.stack([np.ones((h, w), np.uint8)] * 3)
    raws = run_device_batch(api, oa, imgs, masks, cs, [0, 1], 2000)
    warps = set().union(*(full_warps(raw) for raw in raws))
    assert len(warps) >= 2, f"segments of {K1['kWarpCorners']} corners before a non-empty warp in warps {sorted(warps)}"


# ---- staging at its extremes ------------------------------------------------------------------------------------------------------
STAGING = {     # (W, H, scale factor, levels), and the edge its level boxes reach
    "tallest_box": ((1001, 997, 2.0, 4), lambda boxes: max(b.box_h for b in boxes) >= K1["kSrcH"] - 8),
    "ratio_above_2": ((999, 963, 2.0, 4), lambda boxes: max(b.ratio for b in boxes) > 2.0),
    "staging_min_both_sides": ((754, 480, 1.385, 6), lambda boxes: {100, 101} <= {int(b.box_h) for b in boxes}
                               and staging_bytes(100) == K1["kStagingMin"] < staging_bytes(101)),
}


def staging_batch(api, cams, w, h):
    """(cameras, images, masks per camera, camera of each image): noise, a dense lattice, a synthetic frame under camera 2's mirror
    mask, and the seam pair (images 3 and 4)"""
    from multicol_slam_b200 import synth
    cs = [synth.scaled_cam(c, w, h) for c in cams]
    rng = np.random.default_rng(w * h)
    noise = [(rng.integers(0, 2, (h, w)) * 255).astype(np.uint8) for _ in range(3)]
    seam = h // 4
    noise[1][-seam:] = 0
    noise[2][:seam] = 255
    imgs = np.stack([noise[0], boundary_lattice(w, h, 4), synth.frame(cs[2], 9), noise[1], noise[2]])
    masks = np.stack([np.ones((h, w), np.uint8), np.ones((h, w), np.uint8), np.ascontiguousarray(api.mirror_mask(cs[2]))])
    assert 0 < (masks[2] != 0).mean() < 1
    return cs, imgs, masks, [0, 1, 2, 0, 1]


@pytest.mark.parametrize("edge", list(STAGING))
def test_staging_extremes(api, oa, cams, edge):
    (w, h, sf, nl), reached = STAGING[edge]
    boxes = level_boxes(w, h, sf, nl)
    assert reached(boxes), boxes
    assert all(b.past > 0 for b in boxes), boxes                  # every level's bottom box reaches past its source
    cs, imgs, masks, coi = staging_batch(api, cams, w, h)
    run_batch(api, oa, imgs, masks, cs, coi, 1000, "mdbrief", scaleFactor=sf, nlevels=nl)


def test_staging_scale2_device_unaligned(api, oa, cams):
    """a tight device batch of width 1001: level 0 is staged byte by byte, the levels above it (pitched pyramid) by TMA"""
    (w, h, sf, nl), _ = STAGING["tallest_box"]
    cs, imgs, masks, coi = staging_batch(api, cams, w, h)
    run_device_batch(api, oa, imgs, masks, cs, coi, 1000, scaleFactor=sf, nlevels=nl)
