"""make_ref_extract_golden.py -- writes tests/golden/ref_extract_*.npz from outputs of the REFERENCE'S OWN extractor
(oracle/_ref/libmcs_ref.so = /root/reference/src/mdBRIEFextractorOct.cpp + cam_model_omni.cpp + misc.cpp compiled in place,
`make -C oracle ref`).  Run in the build container:   python tests/golden/make_ref_extract_golden.py

Every fixture stores the synthetic-image seed, the camera, the constructor arguments and what the reference returned:
keypoints (cv::KeyPoint bytes), descriptors and masks -- in full for the small cases, as count + CRC32 for the large ones --
plus CRC32s of the reference's pyramid levels (as operator() leaves them: blurred where a level produced keypoints) and of
its mask pyramid.  tests/test_ref_pin_cpu.py checks the oracle restatement against them, tests/test_ref_pin_gpu.py the CUDA
path.  The reference runs under a monotonic allocator (oracle/ref_mcs/wrap.cpp) so that its pointer tie-break is creation order.
"""
import json
import pathlib
import sys
import zlib

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))
import ref_mcs_api as ra  # noqa: E402
from multicol_slam_b200 import synth  # noqa: E402

GOLD = ROOT / "tests" / "golden"
ORB, DBRIEF, MDBRIEF = dict(), dict(do_dbrief=True), dict(do_dbrief=True, learn_masks=True)

# (name, camera spec, seed, constructor arguments, store full outputs?)
#   camera spec: Lafida index, or (index, width, height) for a rescaled sensor, or (index, "nomask") for mirrorMask 0, or the name
#   of a calibration in tests/golden/synthetic_cams.json
CASES = [
    # the configuration the reference ships: plain ORB, 400 features (Examples/Lafida/Slam_Settings_indoor1.yaml:12-27)
    ("shipped_orb400_cam0", 0, 11, dict(nfeatures=400, **ORB), True),
    ("shipped_orb400_cam1", 1, 12, dict(nfeatures=400, **ORB), True),
    ("shipped_orb400_cam2", 2, 13, dict(nfeatures=400, **ORB), True),
    # the tracker's init extractor of that configuration: 2 x nFeatures, FAST threshold 5 (src/cTracking.cpp:152-158)
    ("shipped_init_orb800_th5_cam0", 0, 14, dict(nfeatures=800, fast_threshold=5, **ORB), False),
    # BASELINE.json config 1 / 2: mdBRIEF-256 with masks at 1000 / 2000 features, all three cameras
    ("cfg1_mdbrief1000_cam0", 0, 21, dict(nfeatures=1000, **MDBRIEF), False),
    ("cfg1_mdbrief1000_cam1", 1, 22, dict(nfeatures=1000, **MDBRIEF), False),
    ("cfg1_mdbrief1000_cam2", 2, 23, dict(nfeatures=1000, **MDBRIEF), False),
    ("cfg2_mdbrief2000_cam0", 0, 24, dict(nfeatures=2000, **MDBRIEF), False),
    ("cfg2_mdbrief2000_cam1", 1, 25, dict(nfeatures=2000, **MDBRIEF), False),
    ("dbrief1000_cam1", 1, 26, dict(nfeatures=1000, **DBRIEF), False),
    ("mdbrief400_cam2", 2, 27, dict(nfeatures=400, **MDBRIEF), True),
    # parameter corners
    ("mdbrief_desc16_cam0", 0, 31, dict(nfeatures=500, desc_size=16, **MDBRIEF), False),
    ("mdbrief_desc64_cam1", 1, 32, dict(nfeatures=500, desc_size=64, **MDBRIEF), False),
    ("orb_sf15_l5_cam2", 2, 33, dict(nfeatures=600, scale_factor=1.5, nlevels=5, **ORB), False),
    ("dbrief_sf11_l8_th40_cam0", 0, 34, dict(nfeatures=700, scale_factor=1.1, nlevels=8, fast_threshold=40, **DBRIEF), False),
    ("mdbrief_nomask_cam0", (0, "nomask"), 35, dict(nfeatures=600, **MDBRIEF), False),
    # BASELINE.json configs 3 / 4 sensor sizes
    ("cfg3_1280x720_mdbrief2000", (0, 1280, 720), 41, dict(nfeatures=2000, **MDBRIEF), False),
    ("cfg4_1920x1080_mdbrief4000", (1, 1920, 1080), 42, dict(nfeatures=4000, **MDBRIEF), False),
    ("small_333x211_l4_orb", (2, 333, 211), 43, dict(nfeatures=300, nlevels=4, **ORB), True),
    # fisheye calibrations other than Lafida's (tests/golden/synthetic_cams.json): each drives the descriptor kernel down another path
    ("syn_equidistant185_mdbrief1000", "equidistant185", 51, dict(nfeatures=1000, **MDBRIEF), False),
    ("syn_equisolid230_dbrief1000", "equisolid230", 52, dict(nfeatures=1000, **DBRIEF), False),
    ("syn_equisolid230_mdbrief300", "equisolid230", 53, dict(nfeatures=300, **MDBRIEF), True),
    ("syn_stereographic170_orb400", "stereographic170", 54, dict(nfeatures=400, **ORB), True),
    ("syn_stereographic170_mdbrief1000", "stereographic170", 55, dict(nfeatures=1000, **MDBRIEF), False),
    ("syn_affine185_mdbrief1000", "affine185", 56, dict(nfeatures=1000, **MDBRIEF), False),
    ("syn_affine185_mdbrief_desc16", "affine185", 57, dict(nfeatures=500, desc_size=16, **MDBRIEF), False),
    ("syn_wide1920x1080_195_mdbrief4000", "wide1920x1080_195", 58, dict(nfeatures=4000, **MDBRIEF), False),
    ("syn_narrow1280x720_120_dbrief2000", "narrow1280x720_120", 59, dict(nfeatures=2000, **DBRIEF), False),
    ("syn_magnify130_mdbrief1000", "magnify130", 60, dict(nfeatures=1000, **MDBRIEF), False),
    ("syn_magnify130_mdbrief_desc64", "magnify130", 61, dict(nfeatures=500, desc_size=64, **MDBRIEF), False),
    ("syn_magnify130_dbrief300", "magnify130", 62, dict(nfeatures=300, **DBRIEF), True),
]


def make_cam(spec):
    cams = synth.lafida_cams()
    if isinstance(spec, str):
        return next(c for c in json.loads((GOLD / "synthetic_cams.json").read_text()) if c["name"] == spec)
    if isinstance(spec, int):
        return dict(cams[spec])
    if spec[1] == "nomask":
        c = dict(cams[spec[0]])
        c["mirror_mask"] = 0
        return c
    return synth.scaled_cam(cams[spec[0]], spec[1], spec[2])


def crc(a):
    return zlib.crc32(np.ascontiguousarray(a).tobytes())


def main(only=None):
    for name, spec, seed, kw, full in CASES:
        if only and not name.startswith(only):
            continue
        cam = make_cam(spec)
        img = synth.frame(cam, seed)
        mask = ra.mirror_mask(cam)                       # the reference's own CreateMirrorMask (or all ones)
        assert np.array_equal(mask, synth.mirror_mask(cam))
        ex = ra.RefExtractor(**kw)
        k, d, m = ex.extract(img, mask, cam)
        k2, d2, m2 = ra.RefExtractor(**kw).extract(img, mask, cam)          # reproducible under the monotonic allocator
        assert k.tobytes() == k2.tobytes() and np.array_equal(d, d2) and np.array_equal(m, m2)
        L = kw.get("nlevels", 8)
        out = dict(cam_json=np.frombuffer(json.dumps(cam).encode(), np.uint8), params_json=np.frombuffer(json.dumps(kw).encode(), np.uint8),
                   seed=seed, image_crc=crc(img), n=len(k), kps_crc=crc(k), desc_crc=crc(d), dmask_crc=crc(m),
                   per_level=np.array([int((k["octave"] == l).sum()) for l in range(L)]),
                   level_after_crc=np.array([crc(ex.debug_read(l, 0)) for l in range(L)], np.int64),
                   mask_level_crc=np.array([crc(ex.debug_read(l, 1)) for l in range(L)], np.int64))
        if full:
            out.update(kps=k, desc=d, dmask=m)
        np.savez_compressed(GOLD / f"ref_extract_{name}.npz", **out)
        print(f"{name}: {len(k)} keypoints, per level {out['per_level'].tolist()}")


if __name__ == "__main__":
    if not ra.available():
        raise SystemExit("oracle/_ref/libmcs_ref.so is missing: run `make -C oracle ref` where /root/reference exists")
    main(sys.argv[1] if len(sys.argv) > 1 else None)
