"""CPU: the magnifying synthetic camera (tests/golden/synthetic_cams.json "magnify130", inv_pol 1.3x pol) exists to push distorted
pattern offsets beyond the 51x51 patch K3 stages.  Beyond its 25 px ring the reference reads raw buffer bytes that the kernel's
clamped sample_px cannot reproduce, so the comparison is only meaningful where every sample of every keypoint the oracle keeps
stays inside its level image.  This checks both halves on the oracle's own keypoints: offsets beyond the patch occur, and no
sample leaves the level."""
import importlib.util
import json
import pathlib

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
CAM = next(c for c in json.loads((ROOT / "tests" / "golden" / "synthetic_cams.json").read_text()) if c["name"] == "magnify130")


def test_magnifying_camera_samples_stay_inside_the_level(oa):
    from multicol_slam_b200 import synth
    spec = importlib.util.spec_from_file_location("k3_fp32_model", ROOT / "tools" / "k3_fp32_model.py")
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    pat = m.pattern()
    a0 = CAM["pol"][0]
    beyond = 0
    for seed in (60, 710):
        e = oa.OracleExtractor(nfeatures=1000, do_dbrief=True, learn_masks=True)
        k, _, _ = e.extract(synth.frame(CAM, seed), synth.mirror_mask(CAM), CAM)
        for kp in k:
            lv = int(kp["octave"])
            scale = float(e.info.scale_factor[lv])
            h, w = e.debug_read(lv, 0).shape
            kx, ky = int(round(float(kp["x"]) / scale)), int(round(float(kp["y"]) / scale))
            ukx, uky = m.undistort(CAM, np.float64(np.float32(kx) * np.float32(scale)), np.float64(np.float32(ky) * np.float32(scale)))
            base = float(kp["angle"]) / 57.2957763671875
            for rot in (0.0, np.radians(20), -np.radians(20)):
                ca, sa = np.cos(base + rot), np.sin(base + rot)
                u, v = m.world_to_img(CAM, pat[:, 0] * ca - pat[:, 1] * sa + ukx, pat[:, 0] * sa + pat[:, 1] * ca + uky, -a0)
                du, dv = np.rint(u - u.mean()), np.rint(v - v.mean())
                beyond += max(np.abs(du).max(), np.abs(dv).max()) > 25
                assert (kx + du >= 0).all() and (kx + du < w).all() and (ky + dv >= 0).all() and (ky + dv < h).all(), (lv, kx, ky)
    assert beyond > 0
