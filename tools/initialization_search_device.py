"""Measure map initialisation's search on the device, SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, 50)
(mcs_search_for_initialization_device), against the host route an integrator has without it: both frames copied to the host, then
mcs_search_for_initialization.  The scene is bench.py's config 3 (four 1280x720 cameras) through the tracker's initialisation
extractor (2 x 2000 features, FAST threshold 5, masks on, ref src/cTracking.cpp:156-158): F1 = frame 0 and F2 = frames 1..5 of
bench.make_stream, all extracted into one packed buffer, with prev seeded by mcs_search_for_initialization_seed_device and carried
from call to call on each route.  Per F2 and route: the call time (CUDA events and wall clock for the device call, wall clock for
the host route, runs alternated), median and min-max; whether both routes give the same matches and prev; the device call's
rescans and a per-kernel split (torch.profiler, a separate run).  The card's name and power limit are read in the same run.

    python tools/initialization_search_device.py [--runs 20] [--out /tmp/initialization_search_device.json]
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
N_F2 = 5


def _stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "n": len(xs)}


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
    W, H, NF = cfg["w"], cfg["h"], 2 * cfg["nfeatures"]
    dev = torch.device("cuda", 0)
    cams = bench.rig_cams(cfg)
    nc, nfr = len(cams), 1 + N_F2
    masks = np.stack([synth.mirror_mask(c) for c in cams])
    images = bench.make_stream(cams, list(range(nc)), nfr, 1000)                # [frames, nc, H, W]
    pitch = (W + 63) // 64 * 64
    dev_images = torch.zeros((nfr * nc, H, pitch), dtype=torch.uint8, device=dev)
    dev_images[:, :, :W] = torch.from_numpy(images.reshape(nfr * nc, H, W)).to(dev)
    ex = api.mdBRIEFextractorOct(nfeatures=NF, nlevels=bench.NLEVELS, fastThreshold=5, do_dBrief=True, learnMasks=True)
    cap, ds = ex.capacity, 32
    packed = torch.zeros(rigmod.packed_layout(nfr * nc, cap, ds)[1], dtype=torch.uint8, device=dev)
    v = ex.extract_batch_packed_device(dev_images, masks, cams, list(range(nc)) * nfr, packed, width=W)
    torch.cuda.synchronize()
    counts = v["counts"].cpu().numpy()
    sf = [float(ex.info.scale_factor[l]) for l in range(bench.NLEVELS)]
    sizes = [(W, H)] * nc
    frame = lambda t: (packed, 1, nfr * nc, t * nc)  # noqa: E731
    mt = api.cORBmatcher(0.9, False, ds, True)
    stream = torch.cuda.current_stream(dev)

    def host_frame(t):
        """the host route's copy of frame t: keypoints, descriptors and masks to the host"""
        kps = v["kps"][t * nc:(t + 1) * nc].cpu().numpy().view(api.KEYPOINT_DTYPE).reshape(nc, cap)
        d, m = v["desc"][t * nc:(t + 1) * nc].cpu().numpy(), v["dmask"][t * nc:(t + 1) * nc].cpu().numpy()
        n = counts[t * nc:(t + 1) * nc]
        return api.Frame.from_cameras([(kps[c, :n[c]], d[c, :n[c]], m[c, :n[c]]) for c in range(nc)], sizes, sf)

    c1 = counts[:nc]
    prev_t = torch.zeros(nc * cap * 2, dtype=torch.float64, device=dev)
    m12_t = torch.full((nc * cap,), -1, dtype=torch.int32, device=dev)
    outs = (torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(2, dtype=torch.int32, device=dev))
    F1 = host_frame(0)
    res = {"gpu": torch.cuda.get_device_name(dev), "cameras": nc, "image": f"{W}x{H}", "nfeatures": NF, "fast_threshold": 5,
           "f1_keypoints": int(c1.sum()), "window": 50, "nnratio": 0.9, "th_low": mt.TH_LOW_, "runs": args.runs, "calls": []}
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                                            text=True, timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        res["power_limit"] = f"unknown ({e})"

    def seed():
        mt.SearchForInitializationSeedDevice(frame(0), nc, cap, prev_t, stream=stream)

    def device_call(t):
        return mt.SearchForInitializationDevice(frame(0), frame(t), cap, sizes, prev_t, 50, m12_t, stream=stream, out=outs, diag=True)

    def host_call(t, prev):
        F2 = host_frame(t)
        return mt.SearchForInitialization(host_frame(0), F2, prev, 50), F2

    def device_prev():
        p = prev_t.cpu().numpy().reshape(nc, cap, 2)
        return np.concatenate([p[c, :c1[c]] for c in range(nc)])

    # the chain once on each route, checked call by call
    seed()
    hprev = np.stack([F1.keys["x"], F1.keys["y"]], axis=1).astype(np.float64)
    torch.cuda.synchronize()
    identical = device_prev().tobytes() == hprev.tobytes()
    chain_prev = {}
    for t in range(1, nfr):
        chain_prev[t] = (prev_t.clone(), hprev.copy())
        (hn, hm12), F2 = host_call(t, hprev)
        dn, _, diag = device_call(t)
        torch.cuda.synchronize()
        off2 = np.concatenate([[0], np.cumsum(counts[t * nc:(t + 1) * nc])])
        m = api.slots_to_contiguous(m12_t.cpu().numpy(), c1, cap)
        s = np.maximum(m, 0)
        gm = np.where(m >= 0, off2[s // cap] + s % cap, -1)
        same = int(dn.item()) == hn and np.array_equal(gm, hm12) and device_prev().tobytes() == hprev.tobytes()
        identical &= same
        res["calls"].append({"f2": t, "matches": hn, "queries": int(diag[0].item()), "rescans": int(diag[1].item()), "identical": bool(same)})
    res["identical_matches_and_prev"] = bool(identical)

    # timing: each call from the prev it had in the chain, device and host alternated
    dev_ms, dev_gpu_ms, host_ms = [], [], []
    for r in range(args.runs):
        t = 1 + r % N_F2
        prev_t.copy_(chain_prev[t][0])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        device_call(t)
        e1.record(stream)
        torch.cuda.synchronize()
        dev_ms.append((time.perf_counter() - t0) * 1e3)
        dev_gpu_ms.append(e0.elapsed_time(e1))
        p = chain_prev[t][1].copy()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host_call(t, p)
        host_ms.append((time.perf_counter() - t0) * 1e3)
    res["device_call_gpu_ms"] = _stats(dev_gpu_ms)
    res["device_call_wall_ms"] = _stats(dev_ms)
    res["host_route_wall_ms"] = _stats(host_ms)

    from torch.profiler import ProfilerActivity, profile
    prev_t.copy_(chain_prev[1][0])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        device_call(1)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            hit = re.search(r"(\w+_kernel)(<[^>]*>)?", e.name)
            kname = hit.group(0) if hit else e.name.strip()
            k = kern.setdefault(kname, [0, 0.0])
            k[0] += 1
            k[1] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    res["kernels_ms_f2_1"] = {k: {"launches": c, "ms": round(ms, 4)} for k, (c, ms) in sorted(kern.items(), key=lambda x: -x[1][1])}
    print(json.dumps(res, indent=1))
    if args.out:
        pathlib.Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        pathlib.Path(args.out).write_text(json.dumps(res, indent=1))
    if not identical:
        sys.exit("the device call and the host route differ")


if __name__ == "__main__":
    main()
