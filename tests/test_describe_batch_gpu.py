"""K3 (describe_kernel) works on warp batches: a warp takes 32 consecutive selected slots of one image, sets up one keypoint per lane
and then walks the batch.  These tests put keypoint counts around the batch edge, batches across pyramid levels and batches that
mix the descriptor tiers through the kernel, for every descriptor type and size, and compare every output bit with the CPU
oracle."""
import numpy as np
import pytest

from extract_cases import extract_and_compare

pytestmark = pytest.mark.gpu


# (nlevels, nfeatures, mask, keypoints of the first image): 0 on a flat image, 1 through a 6 x 6 mask window, and 31 / 32 / 33
# selected keypoints (one level holds them all for 32, so the batch edge falls exactly after the last one)
@pytest.mark.parametrize("nl,nf,kind,expect", [(1, 200, "flat", 0), (1, 200, "window", 1), (2, 31, "full", 31), (1, 31, "full", 32),
                                               (3, 32, "full", 33)])
def test_counts_around_the_batch_edge(api, oa, cams, nl, nf, kind, expect):
    from multicol_slam_b200 import synth
    cam = cams[0]
    mask = synth.mirror_mask(cam)
    img = synth.frame(cam, 0)
    if kind == "flat":
        img = np.full_like(img, 128)
    if kind == "window":
        mask = np.zeros_like(mask)
        mask[240:246, 377:383] = 1
    # the second image (full mask, another camera) shares the launch: batches of images with different counts side by side
    counts = extract_and_compare(api, oa, [img, synth.frame(cams[1], 5)], [mask, synth.mirror_mask(cams[1])], [cam, cams[1]],
                                 [0, 1], nf, nlevels=nl)
    assert counts[0] == expect


@pytest.mark.parametrize("ds", [16, 32, 64])
@pytest.mark.parametrize("mode", ["orb", "dbrief", "mdbrief"])
def test_batches_across_levels_every_descriptor(api, oa, cams, mode, ds):
    """8 levels with 300 features: the level's slot ranges (quota + 3 slots each) do not start on multiples of 32, so most batches
    hold keypoints of two levels"""
    from multicol_slam_b200 import synth
    imgs = [synth.frame(cams[c], 40 + c) for c in range(3)]
    extract_and_compare(api, oa, imgs, [synth.mirror_mask(c) for c in cams], list(cams), [0, 1, 2], 300, mode, descSize=ds)


def test_batches_mixing_tiers(api, oa, cams):
    """Full-size frames: tier-2 keypoints (closer than 40 px to the distortion centre, or undecided by tier 1) and tier-3 patterns
    sit in batches whose other keypoints take tier 1"""
    from multicol_slam_b200 import synth
    imgs = [synth.frame(cams[c], 300 + c) for c in range(3)]
    masks = [synth.mirror_mask(c) for c in cams]
    ex = api.mdBRIEFextractorOct(nfeatures=2000, do_dBrief=True, learnMasks=True)
    ex.tier_stats(True)
    counts = extract_and_compare(api, oa, imgs, masks, list(cams), [0, 1, 2], 2000, ex=ex)
    t = ex.tier_stats(False)
    assert t.sum() == 3 * counts.sum()
    assert t[0] > 0 and t[1] > 0 and t[2] > 0 and t[3] > 0, t.tolist()
