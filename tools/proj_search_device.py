"""Measure SearchByProjection on the config-3 scene of bench.py: the host chain bench.py runs (D2H of the packed features, a
Python frame view, mcs_project_mappoints, mcs_search_by_projection) against the device chain (mcs_project_mappoints_device ->
mcs_search_by_projection_device straight from the packed buffer), alternated in one process, three runs each.  Also splits the
device chain per kernel with torch.profiler, reports the fixpoint rounds the data needed and whether the sequential walk ran, and
checks that both chains assign the same map points.

    python tools/proj_search_device.py [--frames 4] [--out /tmp/proj_search_device.json]
"""
import argparse
import json
import pathlib
import re
import sys
import time

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4, help="frames of bench.py's config-3 camera, searched as the cameras of one frame")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import bench
    import multicol_slam_b200.api as api
    from multicol_slam_b200 import rig, synth

    cfg = bench.CONFIGS[3]
    F, W, H, NF = args.frames, cfg["w"], cfg["h"], cfg["nfeatures"]
    dev = torch.device("cuda", 0)
    cams = bench.rig_cams(cfg)
    masks = np.stack([synth.mirror_mask(c) for c in cams])
    images = bench.make_stream(cams, [0], F, 1000)                                   # bench.py: rank 0's camera, seed 1000
    pitch = (W + 63) // 64 * 64
    dev_images = torch.zeros((F, H, pitch), dtype=torch.uint8, device=dev)
    dev_images[:, :, :W] = torch.from_numpy(images).to(dev).view(F, H, W)
    ex = api.mdBRIEFextractorOct(nfeatures=NF, nlevels=bench.NLEVELS, do_dBrief=True, learnMasks=True)
    cap, ds = ex.capacity, 32
    packed = torch.zeros(rig.packed_layout(F, cap, ds)[1], dtype=torch.uint8, device=dev)
    coi = np.zeros(F, np.int32)
    v = ex.extract_batch_packed_device(dev_images, masks, cams, coi, packed, width=W)
    torch.cuda.synchronize()
    n0 = int(v["counts"][0].item())
    f0 = (v["kps"][0, :n0].cpu().numpy().view(api.KEYPOINT_DTYPE).reshape(-1), v["desc"][0, :n0].cpu().numpy(), v["dmask"][0, :n0].cpu().numpy())
    scene = bench.make_scene(3, cfg, cams, 0, f0, F, 7)
    mtmc = np.ascontiguousarray(scene["poses"])
    mtmc_inv = np.ascontiguousarray(np.stack([np.linalg.inv(p) for p in scene["poses"]]))
    masks_f = np.ascontiguousarray(np.broadcast_to(masks[0], (F,) + masks[0].shape))
    sf = np.array([float(np.float32(1.2)) ** l for l in range(bench.NLEVELS)])
    nmp = len(scene["world"])
    mt = api.cORBmatcher(0.8, False, ds, True)

    h_feat = dict(counts=torch.empty(F, dtype=torch.int32).pin_memory(), kps=torch.empty((F, cap, 7), dtype=torch.int32).pin_memory(),
                  desc=torch.empty((F, cap, ds), dtype=torch.uint8).pin_memory(), dmask=torch.empty((F, cap, ds), dtype=torch.uint8).pin_memory())

    def host_chain():
        for k in h_feat:
            h_feat[k].copy_(v[k], non_blocking=True)
        torch.cuda.synchronize()
        counts = h_feat["counts"].numpy()
        kps = h_feat["kps"].numpy().view(api.KEYPOINT_DTYPE).reshape(F, cap)
        keys = np.concatenate([kps[f, :counts[f]] for f in range(F)])
        key_cam = np.concatenate([np.full(counts[f], f, np.int32) for f in range(F)])
        desc = np.concatenate([h_feat["desc"].numpy()[f, :counts[f]] for f in range(F)])
        dmask = np.concatenate([h_feat["dmask"].numpy()[f, :counts[f]] for f in range(F)])
        Fr = api.Frame(keys, key_cam, desc, dmask, [(W, H)] * F, sf)
        iv, lv, px, py, vc = api.project_mappoints(mtmc_inv, mtmc, [cams[0]] * F, masks_f, scene["world"], scene["normal"], scene["min_d"],
                                                   scene["max_d"], sf)
        mp = api.MapPoints(np.zeros(nmp, np.uint8), iv, lv, px, py, vc, scene["mp_desc"], scene["mp_dmask"])
        n, fmp = mt.SearchByProjection(Fr, mp, 3.0)
        return n, fmp, counts

    # map points resident on the device, as the cMapPoint members would be
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    masks_t, world_t, normal_t, mind_t, maxd_t = t(masks_f), t(scene["world"]), t(scene["normal"]), t(scene["min_d"]), t(scene["max_d"])
    proj = api.project_mappoints_device(mtmc_inv, mtmc, [cams[0]] * F, masks_t, world_t, normal_t, mind_t, maxd_t, sf)
    mdev = api.MapPointsDevice(None, *proj, t(scene["mp_desc"]), t(scene["mp_dmask"]))
    fm_t = torch.empty(F * cap, dtype=torch.int32, device=dev)
    outs = tuple(torch.zeros(k, dtype=torch.int32, device=dev) for k in (1, 1, 4))
    stream = torch.cuda.current_stream(dev)

    def device_chain():
        fm_t.fill_(-1)
        api.project_mappoints_device(mtmc_inv, mtmc, [cams[0]] * F, masks_t, world_t, normal_t, mind_t, maxd_t, sf, out=proj, stream=stream)
        return mt.SearchByProjectionDevice(packed, 1, F, 0, F, cap, [(W, H)] * F, sf, mdev, 3.0, fm_t, stream=stream, out=outs, diag=True)

    # warm-up and parity
    hn, hfmp, counts = host_chain()
    dn, dst, _, diag = device_chain()
    torch.cuda.synchronize()
    same = int(dn.item()) == hn and np.array_equal(api.slots_to_contiguous(fm_t.cpu().numpy(), counts, cap), hfmp)
    host_ms, dev_ms, dev_gpu_ms = [], [], []
    for _ in range(args.runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host_chain()
        host_ms.append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        device_chain()
        e1.record(stream)
        torch.cuda.synchronize()
        dev_ms.append((time.perf_counter() - t0) * 1e3)
        dev_gpu_ms.append(e0.elapsed_time(e1))
    # per-kernel split of one device chain
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        device_chain()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            hit = re.search(r"(\w+_kernel)(<[^>]*>)?", e.name)
            name = hit.group(0) if hit else e.name.strip()
            k = kern.setdefault(name, [0, 0.0])
            k[0] += 1
            k[1] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    d = diag.cpu().numpy().tolist()
    res = {"gpu": torch.cuda.get_device_name(dev), "frames_as_cameras": F, "image": f"{W}x{H}", "nfeatures": NF, "map_points": nmp,
           "keypoints": int(np.sum(counts)), "queries": d[2], "matches": hn, "identical_assignments": bool(same),
           "host_chain_ms": host_ms, "device_chain_wall_ms": dev_ms, "device_chain_gpu_ms": dev_gpu_ms,
           "fixpoint_rounds_run": d[0], "round_cap": api.lib().mcs_search_by_projection_max_rounds(), "walk_from_query": d[1],
           "rescans": d[3], "status": int(dst.item()),
           "kernels_ms": {k: {"launches": c, "ms": round(ms, 4)} for k, (c, ms) in sorted(kern.items(), key=lambda x: -x[1][1])}}
    try:
        import subprocess
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                                            text=True, timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        res["power_limit"] = f"unknown ({e})"
    print(json.dumps(res, indent=1))
    if args.out:
        pathlib.Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        pathlib.Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
