"""m2_split.py -- where the time of the greedy stream matcher goes, on bench.py's config-2 workload.

Extracts the seeded config-2 stream (bench.make_stream, 128 frames x 3 cameras, mdBRIEF-256 with masks) once, then times with
torch.profiler, per kernel:
  greedy     match_stream_greedy_device(th_low = TH_LOW_, 0.9): the bounded K = 8 lists and the replay over them;
  floor      the same call with th_low = 0: the bound is 0, nothing is inserted, so its list kernel is the BMMA + epilogue
             floor on the same data;
  lists K=4 / K=8  match_stream_device, unbounded lists.
python tools/m2_split.py [--reps N] [--frames F]"""
import argparse
import json
import pathlib
import subprocess
import sys

import numpy as np
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
import multicol_slam_b200.api as api  # noqa: E402
from multicol_slam_b200 import rig, synth  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the timings stand without it
        return f"nvidia-smi unavailable ({e})"


def kernel_ms(fn, reps):
    """GPU time of every list and replay kernel fn launches (one launch of each per call), mean over the launches of reps calls
    (torch.profiler, CUDA activity), and the number of launches recorded"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and ("hamming_stream" in e.name or "replay" in e.name):
            name = e.name.split("(")[0].replace("void ", "").replace("mcs::", "")
            out.setdefault(name, []).append(e.time_range.elapsed_us() / 1e3)
    return {k: (float(np.mean(v)), len(v)) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--frames", type=int, default=bench.CONFIGS[2]["frames"])
    args = ap.parse_args()
    cfg = bench.CONFIGS[2]
    F, W, H, NC = args.frames, cfg["w"], cfg["h"], cfg["n_cams"]
    B = F * NC
    dev = torch.device("cuda", 0)
    cams = bench.rig_cams(cfg)
    masks = np.stack([synth.mirror_mask(c) for c in cams])
    images = bench.make_stream(cams, list(range(NC)), F, 1000)
    pitch = (W + 63) // 64 * 64
    dev_images = torch.zeros((B, H, pitch), dtype=torch.uint8, device=dev)
    dev_images[:, :, :W] = torch.from_numpy(images).to(dev).view(B, H, W)
    ex = api.mdBRIEFextractorOct(nfeatures=cfg["nfeatures"], nlevels=bench.NLEVELS, do_dBrief=True, learnMasks=True)
    cap, ds = ex.capacity, 32
    packed = torch.zeros(rig.packed_layout(B, cap, ds)[1], dtype=torch.uint8, device=dev)
    coi = np.tile(np.arange(NC, dtype=np.int32), F)
    v = ex.extract_batch_packed_device(dev_images, masks, cams, coi, packed, width=W)
    torch.cuda.synchronize()
    th = api.cORBmatcher(0.9, False, ds, True).TH_LOW_
    m12 = torch.empty((B, cap), dtype=torch.int32, device=dev)
    nmat = torch.empty(B, dtype=torch.int32, device=dev)
    lists = {K: (torch.empty((B, cap, K), dtype=torch.int32, device=dev), torch.empty((B, cap, K), dtype=torch.int32, device=dev))
             for K in (4, 8)}
    runs = {
        "greedy": lambda: api.match_stream_greedy_device(v["desc"], v["dmask"], v["counts"], F, NC, th, 0.9, out=(m12, nmat)),
        "floor (th_low = 0)": lambda: api.match_stream_greedy_device(v["desc"], v["dmask"], v["counts"], F, NC, 0, 0.9, out=(m12, nmat)),
        "lists K=4": lambda: api.match_stream_device(v["desc"], v["dmask"], v["counts"], F, NC, K=4, out=lists[4]),
        "lists K=8": lambda: api.match_stream_device(v["desc"], v["dmask"], v["counts"], F, NC, K=8, out=lists[8]),
    }
    res = {"gpu": gpu_info(), "images": B, "features": int(v["counts"].sum().item()), "reps": args.reps}
    for name, fn in runs.items():
        res[name] = kernel_ms(fn, args.reps)
    print(f"{res['gpu']}; {B} images, {res['features']} features; mean GPU time per launch, {args.reps} calls")
    for name in runs:
        for k, (ms, n) in res[name].items():
            print(f"  {name:20s} {k:40s} {ms:8.3f} ms  ({n} launches recorded)")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
