"""Measure TrackPreviousFrame's two searches on the device on a config-3-sized scene: WindowSearch(LastFrame, CurrentFrame, window,
., minOctave) (mcs_window_search_device) at (60, 4) -- as the tracker calls it with more than 5 key frames and 8 levels -- and at
(50, 0), its retry; and SearchByProjection(LastFrame, CurrentFrame, 40, .) (mcs_search_by_projection_frames_device) with the
current pose a few mm off and the (60, 4) window search's assignments on entry.  The scene is the one of
tools/motion_search_device.py: bench.py's 1280x720 cameras (4, searched as one frame), 2000 features, last and current frames from
consecutive images of bench.make_stream extracted into one packed buffer, map points on the bearing rays of 60 % of the last frame's
keypoints.  Per call: queries / matches / rounds / walk / rescans, the device call time (CUDA events and wall clock, runs alternated
with the host composition), whether the device call assigns what the host composition assigns, and a per-kernel split
(torch.profiler, a separate run).  The host compositions build queries (and, for the frames search, project) in Python: their times
are reported for reference and are not a C++ baseline.

    python tools/previous_frame_search_device.py [--runs 3] [--out /tmp/previous_frame_search_device.json]
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
INT_MAX = 2**31 - 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
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
    nc = len(cams)
    masks = np.stack([synth.mirror_mask(c) for c in cams])
    images = bench.make_stream(cams, list(range(nc)), 2, 1000)                  # [2 frames, nc, H, W]
    pitch = (W + 63) // 64 * 64
    dev_images = torch.zeros((2 * nc, H, pitch), dtype=torch.uint8, device=dev)
    dev_images[:, :, :W] = torch.from_numpy(images.reshape(2 * nc, H, W)).to(dev)
    ex = api.mdBRIEFextractorOct(nfeatures=NF, nlevels=bench.NLEVELS, do_dBrief=True, learnMasks=True)
    cap, ds = ex.capacity, 32
    packed = torch.zeros(rigmod.packed_layout(2 * nc, cap, ds)[1], dtype=torch.uint8, device=dev)
    v = ex.extract_batch_packed_device(dev_images, masks, cams, list(range(nc)) * 2, packed, width=W)
    torch.cuda.synchronize()
    counts = v["counts"].cpu().numpy()
    kps = v["kps"].cpu().numpy().view(api.KEYPOINT_DTYPE).reshape(2 * nc, cap)
    sf = [float(ex.info.scale_factor[l]) for l in range(bench.NLEVELS)]
    Fl, Fc = (api.Frame.from_cameras([(kps[i, :counts[i]], v["desc"][i, :counts[i]].cpu().numpy(), v["dmask"][i, :counts[i]].cpu().numpy())
                                      for i in range(t * nc, (t + 1) * nc)], [(W, H)] * nc, sf) for t in range(2))

    # a rig of nc cameras 360/nc degrees apart; map points on the rays of 60 % of the last frame's keypoints
    rng = np.random.default_rng(7)
    M_c = np.tile(np.eye(4), (nc, 1, 1))
    for c in range(nc):
        a = 2 * np.pi * c / nc
        M_c[c, :3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
        M_c[c, :3, 3] = [0.1 * np.sin(a), 0.0, 0.1 * np.cos(a)]
    M_t = np.eye(4)
    rig1 = api.Rig(cams, M_c, M_t)
    src = np.sort(rng.choice(len(Fl.keys), int(0.6 * len(Fl.keys)), replace=False))
    world = np.zeros((len(src), 3))
    for i, k in enumerate(src):
        c = int(Fl.key_cam[k])
        ray = np.array(api.img_to_world(cams[c], float(Fl.keys["x"][k]), float(Fl.keys["y"][k])))
        world[i] = (rig1.MtMc[c] @ np.append(ray * rng.uniform(2.0, 8.0), 1.0))[:3]
    mp_last = np.full(len(Fl.keys), -1, np.int32)
    mp_last[src] = np.arange(len(src))
    bad = np.zeros(len(src), np.uint8)
    M_t2 = M_t.copy()
    M_t2[:3, 3] += [0.004, -0.003, 0.002]
    rig2 = api.Rig(cams, M_c, M_t2)
    mt = api.cORBmatcher(0.8, False, ds, True)

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    masks_t, world_t, bad_t = t(masks), t(world), t(bad)
    last_mp_t = t(api.contiguous_to_slots(mp_last, counts[:nc], cap))
    cur_mp_t = torch.empty(nc * cap, dtype=torch.int32, device=dev)
    outs = tuple(torch.zeros(k, dtype=torch.int32, device=dev) for k in (1, 1, 4))
    stream = torch.cuda.current_stream(dev)
    cur, last = (packed, 1, 2 * nc, nc), (packed, 1, 2 * nc, 0)
    sizes = [(W, H)] * nc

    def host_ws(window, lo):
        n, v21 = mt.WindowSearch(Fl, Fc, window, mp_last >= 0, lo, INT_MAX)
        return n, np.where(v21 >= 0, mp_last[np.maximum(v21, 0)], -1).astype(np.int32)

    # the frames search starts from the (60, 4) window search's assignments, as TrackPreviousFrame does after PoseOptimization
    _, entry = host_ws(60, 4)
    entry_t = t(api.contiguous_to_slots(entry, counts[nc:], cap))

    cases = {
        "window_search_60_4": (lambda: mt.WindowSearchDevice(cur, last, cap, sizes, last_mp_t, 60, cur_mp_t, min_level=4, bad_t=bad_t,
                                                             stream=stream, out=outs, diag=True),
                               lambda: host_ws(60, 4)),
        "window_search_50_0": (lambda: mt.WindowSearchDevice(cur, last, cap, sizes, last_mp_t, 50, cur_mp_t, min_level=0, bad_t=bad_t,
                                                             stream=stream, out=outs, diag=True),
                               lambda: host_ws(50, 0)),
        "frames_search_40": (lambda: (cur_mp_t.copy_(entry_t),
                                      mt.SearchByProjectionFramesDevice(cur, last, cap, rig2, masks_t, last_mp_t, world_t, 40, cur_mp_t,
                                                                        bad_t=bad_t, stream=stream, out=outs, diag=True))[1],
                             lambda: mt.SearchByProjectionFramesRig(Fl, mp_last, Fc, rig2, entry, world, bad, 40)),
    }
    res = {"gpu": torch.cuda.get_device_name(dev), "cameras": nc, "image": f"{W}x{H}", "nfeatures": NF,
           "last_keypoints": int(counts[:nc].sum()), "current_keypoints": int(counts[nc:].sum()), "map_points": len(src),
           "round_cap": api.lib().mcs_search_by_projection_max_rounds(), "calls": {}}
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                                            text=True, timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        res["power_limit"] = f"unknown ({e})"
    from torch.profiler import ProfilerActivity, profile
    for name, (device_call, host_call) in cases.items():
        # warm-up and parity
        hn, hout = host_call()
        dn, dst, _, diag = device_call()
        torch.cuda.synchronize()
        same = int(dn.item()) == hn and np.array_equal(api.slots_to_contiguous(cur_mp_t.cpu().numpy(), counts[nc:], cap), hout)
        d = diag.cpu().numpy().tolist()
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
        torch.cuda.synchronize()
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
        res["calls"][name] = {
            "queries": d[2], "matches": hn, "identical_assignments": bool(same), "status": int(dst.item()),
            "host_composition_python_ms": host_ms, "device_call_wall_ms": dev_ms, "device_call_gpu_ms": dev_gpu_ms,
            "fixpoint_rounds_run": d[0], "walk_from_query": d[1], "rescans": d[3],
            "kernels_ms": {k: {"launches": c, "ms": round(ms, 4)} for k, (c, ms) in sorted(kern.items(), key=lambda x: -x[1][1])}}
    print(json.dumps(res, indent=1))
    if args.out:
        pathlib.Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        pathlib.Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
