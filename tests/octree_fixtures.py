"""The reference octree fixtures (tests/golden/ref_octree_*.npz) and what the extractor says about each fixture's geometry."""
import glob
import json
import pathlib

import numpy as np

GOLD = pathlib.Path(__file__).resolve().parent / "golden"
FIXTURES = sorted(glob.glob(str(GOLD / "ref_octree_*.npz")))
TOO_WIDE = "image too wide for nfeatures: the octree can return more keypoints than the capacity"
# what the extractor says about each fixture's geometry before any launch; every other fixture is extracted
REFUSED = {
    "wide_4095x600_orb100": TOO_WIDE,
    "wide_3000x400_orb200": TOO_WIDE,
    "wide_3000x400_mdbrief100": TOO_WIDE,
    "wide_1500x200_l4_orb40": TOO_WIDE,
    "wide_4095x244_l7_orb100": TOO_WIDE,
    "one_level_4095x600_orb10": TOO_WIDE,
    "wide_2000x250_orb50": "level too small for the 30 px cell grid",     # level 7 is 70 px high: no row of 30 px cells
}


def load(path):
    from multicol_slam_b200 import synth
    g = np.load(path)
    cam = json.loads(bytes(g["cam_json"]).decode())
    kw = json.loads(bytes(g["params_json"]).decode())
    img = synth.frame(cam, int(g["seed"]))
    assert zlib_crc(img) == int(g["image_crc"]), "synthetic image generator changed"
    return pathlib.Path(path).stem[len("ref_octree_"):], g, cam, kw, img


def zlib_crc(a):
    import zlib
    return zlib.crc32(np.ascontiguousarray(a).tobytes())
