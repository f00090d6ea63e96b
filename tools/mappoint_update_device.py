"""Time mcs_update_mappoints_device (ComputeDistinctiveDescriptors + UpdateNormalAndDepth for many map points) at config 3 sizes:
a rig of 3 cameras with 2 000-keypoint slots (capacity 2048, 32-byte masked descriptors, 8 levels), a local window of 20 key
frames, and two batches:
  - ProcessNewKeyFrame: 8 000 points, each observed by 2 to 12 key frames, in 1 or 2 cameras of each;
  - local BA: 30 000 points with the same observation counts.
The device call is timed with CUDA events around the Python call (median of --runs after one warm-up); the host mirror
(api.update_mappoints_host, the reference's methods restated in Python) is timed on --host-points points of the batch and reported
per point.  The device tables are compared with the host mirror's on those points.  The card's name and power limit are read in
the same run.

    python tools/mappoint_update_device.py [--runs 20] [--host-points 300] [--out /tmp/mappoint_update_device.json]
"""
import argparse
import json
import pathlib
import subprocess
import sys
import time

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # the measurement still stands; say that the card could not be read
        return f"unknown ({e})"


def batch(rng, n_points, n_kf, n_cams, capacity, counts):
    obs = []
    for _ in range(n_points):
        o = []
        for k in rng.choice(n_kf, int(rng.integers(2, 13)), replace=False):
            for c in rng.choice(n_cams, int(rng.integers(1, 3)), replace=False):
                o.append((int(k), int(c * capacity + rng.integers(0, counts[k, c]))))
        obs.append(o)
    ref = np.array([o[0][0] for o in obs], np.int32)
    return obs, ref, rng.uniform(-20, 20, (n_points, 3)), np.zeros(n_points, np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--host-points", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import multicol_slam_b200.api as api
    import mappoint_scenes as S
    rng = np.random.default_rng(0)
    n_kf, nc, cap, dim, nl = 20, 3, 2048, 32, 8
    counts = rng.integers(1900, 2001, (n_kf, nc)).astype(np.int32)
    NS = nc * cap
    base = dict(dim=dim, n_cams=nc, capacity=cap, n_levels=nl, sf=np.array([1.2 ** i for i in range(nl)]),
                desc=rng.integers(0, 256, (n_kf, NS, dim), dtype=np.uint8),
                dmask=np.where(rng.random((n_kf, NS, dim)) < 0.85, 0xFF, rng.integers(0, 256, (n_kf, NS, dim))).astype(np.uint8),
                octave=rng.integers(0, nl, (n_kf, NS)).astype(np.int32), kf_counts=counts, ow=rng.uniform(-5, 5, (n_kf, 3)),
                kf_bad=np.zeros(n_kf, np.int32))
    kfs = [(fr, base["ow"][k], 0) for k, fr in enumerate(S.packed_frames(base, "one"))]
    res = {"card": _card(), "n_kf": n_kf, "n_cams": nc, "capacity": cap, "dim": dim, "masks": True}
    for name, n_points in (("process_new_keyframe", 8000), ("local_ba", 30000)):
        obs, ref, X, bad = batch(rng, n_points, n_kf, nc, cap, counts)
        sc = dict(base, obs=obs, ref=ref, X=X, bad=bad)
        off, okf, oslot = api.mappoint_obs_csr(obs)
        T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        tables = [T(t) for t in S.fill_tables(n_points, dim)]
        ids_t, dev_in = T(np.arange(n_points, dtype=np.int32)), [T(off), T(okf), T(oslot)]
        ref_t, X_t, bad_t = T(ref), T(X), T(bad)

        def call():
            return api.update_mappoints_device(kfs, nc, cap, base["sf"], ids_t, *dev_in, what=3, having_masks=True, desc_t=tables[0],
                                               dmask_t=tables[1], normal_t=tables[2], min_dist_t=tables[3], max_dist_t=tables[4],
                                               ref_kf_t=ref_t, world_t=X_t, bad_t=bad_t)
        st = call()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.runs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        hp = min(args.host_points, n_points)
        t0 = time.perf_counter()
        _, th = S.host_update(api, dict(sc, obs=obs[:hp] + [[] for _ in range(n_points - hp)]), np.arange(hp), 3, True)
        host_s = time.perf_counter() - t0
        td = [t.cpu().numpy() for t in tables]
        same = all(a[:hp].tobytes() == b[:hp].tobytes() for a, b in zip(th, td))
        res[name] = {"points": n_points, "observations": int(off[-1]), "status": int(st.item()), "device_ms_median": float(np.median(ms)),
                     "device_ms_min": float(np.min(ms)), "host_mirror_ms_per_point": 1e3 * host_s / hp, "host_points_timed": hp,
                     "device_equals_host_on_timed_points": bool(same)}
        print(name, json.dumps(res[name]), flush=True)
    print(json.dumps(res))
    if args.out:
        pathlib.Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
