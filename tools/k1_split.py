"""k1_split.py -- GPU time of the pyramid / FAST kernel (K1, pyr_fast_kernel) per pyramid level on bench.py's config-2 workload.

Extracts the seeded config-2 stream (bench.make_stream, 128 frames x 3 cameras, mdBRIEF-256 with masks) and times the 8
pyr_fast_kernel launches of every call with torch.profiler (launch i of a call is level i), next to the card's name, power limit
and the SM clock and throttle reasons sampled while it ran.

--split times the kernel's phases: it builds three more libraries into a temporary directory, each with pyr_fast_kernel.cu compiled
with -DMCS_K1_SPLIT_EXIT=n (CTAs return after the staging and the tables, after the resize, after FAST) and linked with the other
objects of the in-tree build, then times them and the in-tree library in turn, --rounds times, one process per run.  The early
exits leave no corners for K2 and K3, so only the K1 times of those runs mean anything.
--lib times another build of libmcs_b200.so (for example the parent commit's) instead of the in-tree one.
python tools/k1_split.py [--reps N] [--frames F] [--lib PATH] [--split [--rounds R]]"""
import argparse
import json
import pathlib
import re
import shlex
import subprocess
import sys
import tempfile

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
CSRC = ROOT / "multicol_slam_b200" / "csrc"
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
SPLIT_EXITS = {1: "staging + tables", 2: "+ resize", 3: "+ stores, row sums, FAST"}


def nvcc_flags():
    """the compile flags of csrc/Makefile (ARCH and NVFLAGS), without -Xptxas -v"""
    mk = (CSRC / "Makefile").read_text()
    arch = re.search(r"^ARCH := (.*)$", mk, re.M).group(1)
    flags = re.search(r"^NVFLAGS := (.*)$", mk, re.M).group(1).replace("$(ARCH)", arch).replace("-Xptxas -v", "")
    return shlex.split(flags)


def build_split_libs(tmp):
    """one library per early exit: pyr_fast_kernel.cu with -DMCS_K1_SPLIT_EXIT=n and the other objects of the in-tree build"""
    nvcc = "/usr/local/cuda/bin/nvcc"
    others = sorted(str(o) for o in CSRC.glob("*.o") if o.name != "pyr_fast_kernel.o")
    assert others, "build the library first (__graft_entry__.build())"
    arch = shlex.split(re.search(r"^ARCH := (.*)$", (CSRC / "Makefile").read_text(), re.M).group(1))
    libs = {}
    for n in SPLIT_EXITS:
        d = pathlib.Path(tmp) / f"exit{n}"
        d.mkdir()
        obj = d / "pyr_fast_kernel.o"
        subprocess.check_call([nvcc, *nvcc_flags(), f"-DMCS_K1_SPLIT_EXIT={n}", "-c", str(CSRC / "pyr_fast_kernel.cu"), "-o", str(obj)])
        subprocess.check_call([nvcc, *arch, "-shared", "-o", str(d / "libmcs_b200.so"), str(obj), *others, "-cudart", "static", "-ldl"])
        libs[n] = d / "libmcs_b200.so"
    return libs


def split(args):
    with tempfile.TemporaryDirectory() as tmp:
        libs = build_split_libs(tmp)
        runs = {n: [] for n in [*SPLIT_EXITS, "full"]}
        for _ in range(args.rounds):
            for n in runs:
                cmd = [sys.executable, __file__, "--reps", str(args.reps), "--frames", str(args.frames)]
                if n != "full":
                    cmd += ["--lib", str(libs[n])]
                out = subprocess.run(cmd, check=True, capture_output=True, text=True).stdout
                runs[n].append(json.loads(out.strip().splitlines()[-1]))
    full = np.mean([r["k1_ms_mean"] for r in runs["full"]])
    print(runs["full"][0]["gpu"])
    print(f"  K1 phases, mean of {args.reps} calls per run, {args.rounds} runs each (ms, per level 0 .. 7 of the first run):")
    res = {"gpu": runs["full"][0]["gpu"], "clocks": [r["clock"] for v in runs.values() for r in v], "phases": {}}
    for n, v in runs.items():
        ms = [r["k1_ms_mean"] for r in v]
        name = SPLIT_EXITS.get(n, "full kernel")
        res["phases"][name] = {"k1_ms": ms, "level_ms": v[0]["level_ms_mean"]}
        print(f"  {name:28s} {' '.join(f'{m:.3f}' for m in ms)}  ({np.mean(ms) / full:.0%} of the full kernel)  "
              + " ".join(f"{m:.3f}" for m in v[0]["level_ms_mean"]))
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--frames", type=int)
    ap.add_argument("--lib", help="time this build of libmcs_b200.so instead of the in-tree one")
    ap.add_argument("--split", action="store_true", help="time the early-exit builds of the kernel next to the full one")
    ap.add_argument("--rounds", type=int, default=3, help="--split: runs of every build, alternated")
    args = ap.parse_args()
    import bench
    args.frames = args.frames or bench.CONFIGS[2]["frames"]
    if args.split:
        return split(args)
    import torch
    from torch.profiler import ProfilerActivity, profile
    import multicol_slam_b200.api as api
    if args.lib:
        api._LIB_PATH = pathlib.Path(args.lib).resolve()
    from k3_split import gpu_info
    from multicol_slam_b200 import rig, synth
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
