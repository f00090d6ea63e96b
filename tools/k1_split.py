"""k1_split.py -- GPU time of the pyramid / FAST kernel (K1, pyr_fast_kernel) per pyramid level on bench.py's config-2 workload.

Extracts the seeded config-2 stream (bench.make_stream, 128 frames x 3 cameras, mdBRIEF-256 with masks) and times the 8
pyr_fast_kernel launches of every call with torch.profiler (launch i of a call is level i), next to the card's name, power limit
and the SM clock and throttle reasons sampled while it ran.
python tools/k1_split.py [--reps N] [--frames F]"""
import argparse
import json
import pathlib
import sys

import numpy as np
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import bench  # noqa: E402
import multicol_slam_b200.api as api  # noqa: E402
from k3_split import gpu_info  # noqa: E402
from multicol_slam_b200 import rig, synth  # noqa: E402


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
        call()
    torch.cuda.synchronize()

    clocks = bench.ClockSampler(0)
    clocks.start()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            call()
        torch.cuda.synchronize()
    clk = clocks.stop()
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "pyr_fast_kernel" in e.name),
                key=lambda e: e.time_range.start)
    L = bench.NLEVELS
    assert len(ev) == L * args.reps, f"{len(ev)} pyr_fast_kernel launches for {args.reps} calls of {L} levels"
    ms = np.array([e.time_range.elapsed_us() / 1e3 for e in ev]).reshape(args.reps, L)
    res = {"gpu": gpu_info(), "clock": clk, "images": B, "k1_ms_mean": float(ms.sum(1).mean()),
           "k1_ms_min": float(ms.sum(1).min()), "level_ms_mean": [round(float(v), 4) for v in ms.mean(0)]}
    print(f"{res['gpu']}; SM clock while timed {clk.get('sm_mhz')} MHz {clk.get('reasons')}; {B} images")
    print(f"  pyr_fast_kernel, 8 levels: {res['k1_ms_mean']:.3f} ms mean, {res['k1_ms_min']:.3f} min ({args.reps} calls)")
    print("  per level (ms): " + " ".join(f"{v:.3f}" for v in res["level_ms_mean"]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
