"""k3_split.py -- GPU time of the descriptor kernel (K3, describe_kernel) on bench.py's config-2 workload.

Extracts the seeded config-2 stream (bench.make_stream, 128 frames x 3 cameras, mdBRIEF-256 with masks) and times every
describe_kernel launch with torch.profiler, next to the card's name, power limit and the SM clock sampled while it ran, and the
K3 tier counts of one call (patterns decided by tier 1 / tier-1 repair / tier 2 / tier 3).  Run it on a build with a local edit
of the kernel (e.g. returning before the pattern loop) to split the time between set-up and staging and the pattern work.
python tools/k3_split.py [--reps N] [--frames F]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--frames", type=int, default=bench.CONFIGS[2]["frames"])
    args = ap.parse_args()
    from torch.profiler import ProfilerActivity, profile
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
    packed = torch.zeros(rig.packed_layout(B, ex.capacity, 32)[1], dtype=torch.uint8, device=dev)
    coi = np.tile(np.arange(NC, dtype=np.int32), F)

    def call():
        return ex.extract_batch_packed_device(dev_images, masks, cams, coi, packed, width=W)
    for _ in range(3):
        v = call()
    torch.cuda.synchronize()
    features = int(v["counts"].sum().item())
    ex.tier_stats(True)
    call()
    torch.cuda.synchronize()
    tiers = ex.tier_stats(False)

    clocks = bench.ClockSampler(0)
    clocks.start()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            call()
        torch.cuda.synchronize()
    clk = clocks.stop()
    ms = [e.time_range.elapsed_us() / 1e3 for e in prof.events()
          if e.device_type == torch.autograd.DeviceType.CUDA and "describe_kernel" in e.name]
    res = {"gpu": gpu_info(), "clock": clk, "images": B, "features": features, "describe_ms_mean": float(np.mean(ms)),
           "describe_ms_min": float(np.min(ms)), "launches": len(ms), "tiers": tiers.tolist()}
    print(f"{res['gpu']}; SM clock while timed {clk.get('sm_mhz')} MHz {clk.get('reasons')}; {B} images, {features} features")
    print(f"  describe_kernel {res['describe_ms_mean']:.3f} ms mean, {res['describe_ms_min']:.3f} min ({len(ms)} launches)")
    print(f"  tiers (1, 1 repaired, 2, 3): {tiers.tolist()}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
