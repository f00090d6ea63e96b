"""Measure relocalisation's bag-of-words step on the device on a config-3-sized scene: (a) ComputeBoW of the current frame
(mcs_bow_vectors_device) and (b) SearchByBoW(KF_i, F) for 10 candidate key frames in one call (mcs_search_by_bow_device), each
against today's host route on the same data: device-to-host copy of the features, then mcs_bow_vectors, or 10 x mcs_search_by_bow
with the feature vectors already on the host.  The scene: bench.py's 1280x720 cameras (4, one frame), 2000 features, masks on; the
current frame and its 10 candidates are 11 consecutive frames of bench.make_stream extracted into one packed buffer; 70 % of every
key frame's keypoints carry a map point; the vocabulary is the small one in tests/golden (k = 9, L = 6, levelsup = 4).  Per call:
the device time (CUDA events and wall clock, runs alternated with the host route), whether both routes give the same containers /
assign the same matches, the largest (key-frame keypoints x frame keypoints) group the search met, and a per-kernel split
(torch.profiler, a separate run).

    python tools/relocalisation_bow_device.py [--runs 20] [--out /tmp/relocalisation_bow_device.json]
"""
import argparse
import json
import pathlib
import re
import subprocess
import sys
import time

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
N_KF = 10


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import bench
    import multicol_slam_b200.api as api
    from multicol_slam_b200 import rig as rigmod
    from multicol_slam_b200 import synth

    cfg = bench.CONFIGS[3]
    W, H, NF = cfg["w"], cfg["h"], cfg["nfeatures"]
    dev = torch.device("cuda", 0)
    cams = bench.rig_cams(cfg)
    nc, nfr = len(cams), N_KF + 1
    masks = np.stack([synth.mirror_mask(c) for c in cams])
    images = bench.make_stream(cams, list(range(nc)), nfr, 1000)                # [nfr, nc, H, W]
    pitch = (W + 63) // 64 * 64
    dev_images = torch.zeros((nfr * nc, H, pitch), dtype=torch.uint8, device=dev)
    dev_images[:, :, :W] = torch.from_numpy(images.reshape(nfr * nc, H, W)).to(dev)
    ex = api.mdBRIEFextractorOct(nfeatures=NF, nlevels=bench.NLEVELS, do_dBrief=True, learnMasks=True)
    cap, ds = ex.capacity, 32
    packed = torch.zeros(rigmod.packed_layout(nfr * nc, cap, ds)[1], dtype=torch.uint8, device=dev)
    views = ex.extract_batch_packed_device(dev_images, masks, cams, list(range(nc)) * nfr, packed, width=W)
    torch.cuda.synchronize()
    counts = views["counts"].cpu().numpy().reshape(nfr, nc)
    voc = api.ORBVocabulary(np.load(ROOT / "tests" / "golden" / "voc_small_9_6.npz"))
    max_nodes = voc.level_nodes(4)
    stream = torch.cuda.current_stream(dev)
    frame = lambda f: (packed, 1, nfr * nc, f * nc)  # noqa: E731
    CUR = N_KF // 2                                                             # the candidates are its neighbours on both sides
    kf_ids = [f for f in range(nfr) if f != CUR]

    def d2h(f):
        """today's route: the frame's descriptors and masks to the host, concatenated in camera order"""
        n = views["counts"][f * nc:(f + 1) * nc].cpu().numpy()
        d = np.concatenate([views["desc"][f * nc + c, :n[c]].cpu().numpy() for c in range(nc)])
        m = np.concatenate([views["dmask"][f * nc + c, :n[c]].cpu().numpy() for c in range(nc)])
        return d, m

    def slots_to_ids(slots, f):
        first = np.concatenate([[0], np.cumsum(counts[f])])
        slots = np.asarray(slots)
        return first[slots // cap] + slots % cap

    # ---- (a) ComputeBoW of the current frame ----
    def bow_device():
        return voc.transform_device(frame(CUR), nc, cap, 4, max_nodes, stream=stream)

    def bow_host():
        return voc.transform(d2h(CUR)[0], 4)

    # ---- (b) the 10-candidate search ----
    rng = np.random.default_rng(7)
    bows = {f: voc.transform_device(frame(f), nc, cap, 4, max_nodes, stream=stream) for f in range(nfr)}
    torch.cuda.synchronize()
    host_fv = {f: voc.transform(d2h(f)[0], 4)[2] for f in range(nfr)}
    mp, mp_t = {}, {}
    for f in kf_ids:
        n = int(counts[f].sum())
        mp[f] = np.where(rng.random(n) < 0.7, np.arange(n), -1).astype(np.int32)
        mp_t[f] = torch.from_numpy(api.contiguous_to_slots(mp[f], counts[f], cap)).to(dev)
    n_points = int(max(counts.sum(axis=1)))
    mt = api.cORBmatcher(0.75, False, ds, True)                                 # Relocalisation's matcher (ref src/cTracking.cpp:1155)
    ns = nc * cap
    outs = (torch.empty((N_KF, ns), dtype=torch.int32, device=dev), torch.empty((N_KF, ns), dtype=torch.int32, device=dev),
            torch.zeros(N_KF, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))

    def search_device():
        return mt.SearchByBoWDevice([(bows[f], mp_t[f]) for f in kf_ids], bows[CUR], n_points, stream=stream, out=outs)

    def search_host():
        dc, mc = d2h(CUR)
        res = []
        for f in kf_ids:
            dk, mk = d2h(f)
            res.append(mt.SearchByBoWFrame(dk, host_fv[f], dc, host_fv[CUR], mk, mc, (mp[f] >= 0).astype(np.uint8)))
        return res

    def same_bow(b, h):
        bw, bv, (fn, fo, ff) = b.host()
        return bool(np.array_equal(bw, h[0]) and np.array_equal(bv, h[1]) and np.array_equal(fn, h[2][0]) and np.array_equal(fo, h[2][1]) and
                    np.array_equal(slots_to_ids(ff, CUR), h[2][2]) and int(b.status.item()) == 0)

    def same_search(o, h):
        msl, nm = o[1].cpu().numpy(), o[2].cpu().numpy()
        for k, f in enumerate(kf_ids):
            sl = api.slots_to_contiguous(msl[k], counts[CUR], cap)
            idx = np.where(sl >= 0, slots_to_ids(np.maximum(sl, 0), f), -1)
            if int(nm[k]) != h[k][0] or not np.array_equal(idx, h[k][1]):
                return False
        return int(o[3].item()) == 0

    # the largest group: key-frame keypoints with a map point x frame keypoints of one common node
    groups = []
    cn, co, _ = host_fv[CUR]
    for f in kf_ids:
        kn, ko, kfeat = host_fv[f]
        for a, node in enumerate(kn):
            b = np.searchsorted(cn, node)
            if b < len(cn) and cn[b] == node:
                groups.append((int((mp[f][kfeat[ko[a]:ko[a + 1]]] >= 0).sum()), int(co[b + 1] - co[b])))
    work = np.array([q * c for q, c in groups])

    res = {"gpu": torch.cuda.get_device_name(dev), "cameras": nc, "image": f"{W}x{H}", "nfeatures": NF, "capacity": cap,
           "keypoints_current": int(counts[CUR].sum()), "keypoints_key_frames": [int(counts[f].sum()) for f in kf_ids],
           "vocabulary": "tests/golden/voc_small_9_6.npz", "levelsup": 4, "max_nodes": max_nodes, "key_frames": N_KF,
           "groups": len(groups), "largest_group_queries_x_candidates": list(groups[int(work.argmax())]),
           "median_group_queries_x_candidates": [int(np.median([g[0] for g in groups])), int(np.median([g[1] for g in groups]))],
           "share_of_distance_work_in_largest_group": float(work.max() / work.sum()), "calls": {}}
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                                            text=True, timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        res["power_limit"] = f"unknown ({e})"
    from torch.profiler import ProfilerActivity, profile
    for name, device_call, host_call, same in (("compute_bow", bow_device, bow_host, same_bow),
                                               ("search_by_bow_10_key_frames", search_device, search_host, same_search)):
        h = host_call()
        for _ in range(3):                                                      # warm-up: modules, the pool, the scratch cache
            o = device_call()
        torch.cuda.synchronize()
        identical = same(o, h)
        host_ms, dev_ms, dev_gpu_ms = [], [], []
        for _ in range(args.runs):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            host_call()
            host_ms.append((time.perf_counter() - t0) * 1e3)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record(stream)
            device_call()
            e1.record(stream)
            torch.cuda.synchronize()
            dev_ms.append((time.perf_counter() - t0) * 1e3)
            dev_gpu_ms.append(e0.elapsed_time(e1))
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            device_call()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            if e.device_type.name == "CUDA":
                hit = re.search(r"(\w+_kernel)(<[^>]*>)?", e.name)
                kname = hit.group(0) if hit else e.name.strip()
                k = kern.setdefault(kname, [0, 0.0])
                k[0] += 1
                k[1] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
        med = lambda x: float(np.median(x))  # noqa: E731
        res["calls"][name] = {
            "identical_results": bool(identical), "runs": args.runs,
            "host_route_wall_ms_median": med(host_ms), "host_route_wall_ms_min_max": [min(host_ms), max(host_ms)],
            "device_call_wall_ms_median": med(dev_ms), "device_call_wall_ms_min_max": [min(dev_ms), max(dev_ms)],
            "device_call_gpu_ms_median": med(dev_gpu_ms), "device_call_gpu_ms_min_max": [min(dev_gpu_ms), max(dev_gpu_ms)],
            "kernels_ms": {k: {"launches": c, "ms": round(ms, 4)} for k, (c, ms) in sorted(kern.items(), key=lambda x: -x[1][1])}}
    res["calls"]["search_by_bow_10_key_frames"]["matches_per_key_frame"] = outs[2].cpu().numpy().tolist()
    print(json.dumps(res, indent=1))
    if args.out:
        pathlib.Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        pathlib.Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
