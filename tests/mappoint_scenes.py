"""Seeded map-point scenes for mcs_update_mappoints_device (ComputeDistinctiveDescriptors / UpdateNormalAndDepth), shared by
tests/test_mappoint_update_device_cpu.py (host mirrors against the reference's own cMapPoint) and
tests/test_mappoint_update_device_gpu.py (the device against the host mirrors).

A scene is n_kf key frames of n_cams cameras with slot-indexed descriptors, masks and octaves (slot = c * capacity + j), and map
points whose observations are lists of (key frame, slot), each key frame's slots adjacent.  The points cover the observation counts
0, 1, 2, 3, an even and an odd count, 32, 33 and a few hundred, key frames seen in several cameras, bad key frames, bad points and
reference key frames that do not observe their point."""
import numpy as np

from device_frames import pack_frames
from multicol_slam_b200.ctypes_defs import KEYPOINT_DTYPE

EDGE_COUNTS = (0, 1, 2, 3, 6, 7, 32, 33, 300)


def scene(seed, dim=32, n_cams=3, capacity=16, n_kf=160, n_levels=8, scale=1.2, n_random=16, pool=6, flips=6, p_bad_kf=0.1,
          counts=EDGE_COUNTS):
    """descriptors are drawn from `pool` base rows with up to `flips` flipped bits, so that equal distances and equal medians are
    frequent; pool=1, flips=0 makes every descriptor equal"""
    rng = np.random.default_rng(seed)
    NS = n_cams * capacity
    base = rng.integers(0, 256, (pool, dim), dtype=np.uint8)
    desc = base[rng.integers(0, pool, (n_kf, NS))]
    for k in range(n_kf):
        for s in range(NS):
            for b in rng.integers(0, 8 * dim, rng.integers(0, flips + 1)):
                desc[k, s, b // 8] ^= np.uint8(1 << (b % 8))
    dmask = np.where(rng.random((n_kf, NS, dim)) < 0.85, 0xFF, rng.integers(0, 256, (n_kf, NS, dim))).astype(np.uint8)
    octave = rng.integers(0, n_levels, (n_kf, NS)).astype(np.int32)
    kf_counts = rng.integers(capacity // 2, capacity + 1, (n_kf, n_cams)).astype(np.int32)
    ow = rng.uniform(-5, 5, (n_kf, 3))
    kf_bad = (rng.random(n_kf) < p_bad_kf).astype(np.int32)
    sf = np.array([scale ** i for i in range(n_levels)])
    obs, ref, bad = [], [], []
    sizes = list(counts) + list(rng.integers(2, 13, n_random))
    for i, n in enumerate(sizes):
        o, left = [], int(n)
        for k in rng.permutation(n_kf):
            if left == 0:
                break
            live = [c * capacity + j for c in range(n_cams) for j in range(kf_counts[k, c])]
            m = min(left, int(rng.integers(1, 4)), len(live))              # several cameras of one key frame: one normal term
            o += [(int(k), int(s)) for s in rng.choice(live, m, replace=False)]
            left -= m
        obs.append(o)
        kfs_of = sorted({k for k, _ in o})
        if o and rng.random() > 0.15:
            ref.append(int(o[0][0]) if rng.random() < 0.5 else int(rng.choice(kfs_of)))
        else:                                                               # a ref key frame that does not observe the point
            ref.append(int(rng.choice([k for k in range(n_kf) if k not in kfs_of] or [0])))
        bad.append(i >= len(counts) and rng.random() < 0.08)
    X = rng.uniform(-20, 20, (len(obs), 3))
    return dict(dim=dim, n_cams=n_cams, capacity=capacity, n_levels=n_levels, sf=sf, desc=desc, dmask=dmask, octave=octave,
                kf_counts=kf_counts, ow=ow, kf_bad=kf_bad, obs=obs, ref=np.array(ref, np.int32), bad=np.array(bad, np.uint8), X=X)


def slot_rows(sc, k):
    """(kps, desc, dmask) per camera of key frame k, the images of a packed frame"""
    cap, out = sc["capacity"], []
    for c in range(sc["n_cams"]):
        n = int(sc["kf_counts"][k, c])
        kps = np.zeros(n, KEYPOINT_DTYPE)
        kps["octave"] = sc["octave"][k, c * cap:c * cap + n]
        kps["x"], kps["y"] = np.arange(n, dtype=np.float32), np.float32(c)
        out.append((kps, sc["desc"][k, c * cap:c * cap + n], sc["dmask"][k, c * cap:c * cap + n]))
    return out


def packed_frames(sc, layout, device="cuda"):
    """the key frames as packed-frame records (buffer, n_parts, part_images, first_image): "one" = every image in one layout,
    "parts" = one image per layout of one buffer, "separate" = one buffer per key frame; device None gives numpy buffers"""
    kw = {"one": dict(layout="joint"), "parts": dict(layout="parts"), "separate": dict(layout="single", first_image=0, after=0)}[layout]
    return pack_frames([slot_rows(sc, k) for k in range(len(sc["ow"]))], sc["capacity"], sc["dim"], device=device, **kw)


SCENES = {"d32": dict(seed=1), "d32_masks": dict(seed=2, masks=True), "d16_masks": dict(seed=3, dim=16, masks=True),
          "d64": dict(seed=4, dim=64), "ties": dict(seed=5, pool=2, flips=1, masks=True), "equal": dict(seed=6, pool=1, flips=0)}


def named_scene(name):
    """the scene SCENES[name] and whether it runs with masks"""
    kw = dict(SCENES[name])
    masks = kw.pop("masks", False)
    return scene(**kw), masks


def host_update(api, sc, ids, what, having_masks, obs=None, tables=None):
    """api.update_mappoints_host over the scene (obs: the observation lists to use, by default the scene's); returns (status,
    tables) with tables = (desc, dmask, normal, min_dist, max_dist) updated in place from `tables` or from fill values"""
    obs = sc["obs"] if obs is None else obs
    n, dim = len(obs), sc["dim"]
    off, okf, oslot = api.mappoint_obs_csr(obs)
    if tables is None:
        tables = fill_tables(n, dim)
    st = api.update_mappoints_host(sc["desc"], sc["dmask"], sc["octave"], sc["ow"], sc["kf_bad"], sc["n_cams"], sc["capacity"],
                                   sc["kf_counts"], sc["sf"], ids, off, okf, oslot, sc["ref"], sc["bad"], sc["X"], *tables,
                                   what=what, having_masks=having_masks)
    return st, tables


def fill_tables(n, dim):
    """recognisable initial table contents: rows a call does not write keep them"""
    return (np.full((n, dim), 0xA5, np.uint8), np.full((n, dim), 0x5A, np.uint8), np.full((n, 3), -7.25), np.full(n, -1.5),
            np.full(n, -2.5))
