"""K3 (describe_kernel) on fisheye calibrations other than Lafida's (tests/golden/synthetic_cams.json, written by
tests/golden/make_synthetic_cams.py).  The kernel's tiers rest on camera-dependent premises -- where the table's tier-1 forms
start, the fp32 error budget, the staged 51x51 patch, the table's extent -- and each synthetic camera drives it down one path the
Lafida cameras barely reach.  Every output bit is compared with the CPU oracle, which tests/test_ref_pin_cpu.py pins to the
reference on the same cameras through the ref_extract_syn_* fixtures."""
import json
import pathlib

import numpy as np
import pytest

from device_frames import on_device
from extract_cases import extract_and_compare

pytestmark = pytest.mark.gpu
SYNTHETIC = {c["name"]: c for c in json.loads((pathlib.Path(__file__).resolve().parent / "golden" / "synthetic_cams.json").read_text())}
# cameras whose patterns must reach the exact tier: keypoints beyond the table or at 90 degrees incidence and more (wide), pattern
# offsets beyond the staged patch (magnify)
EXACT = {"wide1920x1080_195", "magnify130"}


def features(cam):
    return 4000 if cam["width"] == 1920 else 2000


def frames(cam, seeds):
    from multicol_slam_b200 import synth
    return [synth.frame(cam, s) for s in seeds], [synth.mirror_mask(cam)]


@pytest.mark.parametrize("mode,ds", [("orb", 32), ("dbrief", 32), ("mdbrief", 16), ("mdbrief", 64)])
@pytest.mark.parametrize("name", list(SYNTHETIC))
def test_camera_every_descriptor(api, oa, name, mode, ds):
    cam = SYNTHETIC[name]
    imgs, masks = frames(cam, [700, 701])
    extract_and_compare(api, oa, imgs, masks, [cam], [0, 0], features(cam), mode, descSize=ds)


@pytest.mark.parametrize("name", list(SYNTHETIC))
def test_camera_mdbrief_tiers(api, oa, name):
    """mdBRIEF-256 on three frames per camera, with the patterns each tier took: tier 1 and its repair run on every camera (all of
    them have tier-1 rows), the exact tier on the wide and the magnifying one"""
    cam = SYNTHETIC[name]
    imgs, masks = frames(cam, [710, 711, 712])
    nf = features(cam)
    ex = api.mdBRIEFextractorOct(nfeatures=nf, do_dBrief=True, learnMasks=True)
    ex.tier_stats(True)
    counts = extract_and_compare(api, oa, imgs, masks, [cam], [0, 0, 0], nf, ex=ex)
    t = ex.tier_stats(False)
    print(f"\n{name}: keypoints {counts.sum()}  patterns tier 1 {t[0]}  repaired {t[1]}  tier 2 {t[2]}  exact {t[3]}")
    assert t.sum() == 3 * counts.sum()
    assert t[0] > 0 and t[1] > 0, t.tolist()
    if name in EXACT:
        assert t[3] > 0, t.tolist()


def test_mixed_launch_with_lafida(api, oa, cams):
    """one launch over the 754x480 synthetic cameras and the Lafida ones: per-image tables and camera constants via cam_of_image"""
    from multicol_slam_b200 import synth
    allcams = list(cams) + [c for c in SYNTHETIC.values() if (c["width"], c["height"]) == (754, 480)]
    coi = list(range(len(allcams)))[::-1] + [3, 0]
    imgs = [synth.frame(allcams[c], 720 + i) for i, c in enumerate(coi)]
    extract_and_compare(api, oa, imgs, [synth.mirror_mask(c) for c in allcams], allcams, coi, 2000)


def test_packed_device_buffer(api, oa):
    """extract_batch_packed_device on the 1280x720 camera: the same bytes as the oracle in the packed exchange buffer"""
    import torch
    from multicol_slam_b200 import rig
    cam = SYNTHETIC["narrow1280x720_120"]
    imgs, masks = frames(cam, [730, 731])
    ex = api.mdBRIEFextractorOct(nfeatures=2000, do_dBrief=True, learnMasks=True)
    packed = torch.zeros(rig.packed_layout(2, ex.capacity, 32)[1], dtype=torch.uint8, device="cuda")
    v = ex.extract_batch_packed_device(on_device(np.stack(imgs)), np.stack(masks), [cam], [0, 0], packed)
    torch.cuda.synchronize()
    counts = v["counts"].cpu().numpy()
    kps = v["kps"].cpu().numpy().view(api.KEYPOINT_DTYPE).reshape(2, ex.capacity)
    oe = oa.OracleExtractor(nfeatures=2000, do_dbrief=True, learn_masks=True)
    for i, img in enumerate(imgs):
        ok, od, om = oe.extract(img, masks[0], cam)
        n = int(counts[i])
        assert n == len(ok) and kps[i, :n].tobytes() == ok.tobytes()
        assert np.array_equal(v["desc"][i, :n].cpu().numpy(), od) and np.array_equal(v["dmask"][i, :n].cpu().numpy(), om)
