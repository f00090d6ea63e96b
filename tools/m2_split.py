"""m2_split.py -- where the time of the greedy stream matcher goes, on bench.py's config-2 workload.

Extracts the seeded config-2 stream (bench.make_stream, 128 frames x 3 cameras, mdBRIEF-256 with masks) once, then times with
torch.profiler, per kernel:
  greedy     match_stream_greedy_device(th_low = TH_LOW_, 0.9): the bounded K = 8 lists and the replay over them;
  floor      the same call with th_low = 0: the bound is 0, nothing is inserted, so its list kernel is the BMMA + epilogue
             floor on the same data;
  lists K=4 / K=8  match_stream_device, unbounded lists.
and counts what the greedy call's list upkeep (bmma_klists, K = 8, bound 35) does on the same data: keys appended per row,
folds per warp, and per fold the insertions of the busiest lane and of the mean lane (per-lane lists) or the rows merged
(quad lists).  The counts come from a replay of the upkeep in torch, for both rules -- one K-best list per lane and row with
the own and quad bounds, and one list per row held by the quad with the exact K-th key -- whose final lists are checked
against the kernel's.
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


KT, SHIFT, DEPTH = 8, 16, 7      # the greedy call's list length and key shift, kCandDepth (multicol_slam_b200/csrc/match_kernels.cu)
NONE = 1 << 40                   # an empty list entry or buffer slot, above every key


def masked_values(q, qm, d, dm):
    """[n, rows, cols] T = popc(x & qm) + popc(x & dm), x = q ^ d (masked distance T >> 1), for u8 descriptors [n, rows, dim]"""
    shifts = torch.arange(8, device=q.device, dtype=torch.uint8)
    bits = lambda x: ((x.unsqueeze(-1) >> shifts) & 1).flatten(-2).float()  # noqa: E731
    a, m1, b, m2 = bits(q), bits(qm), bits(d), bits(dm)
    lhs = torch.cat([m1, -2 * a * m1, a, -2 * a], -1)
    rhs = torch.cat([b, b, m2, b * m2], -1)
    t = (a * m1).sum(-1, keepdim=True) + (b * m2).sum(-1).unsqueeze(-2) + lhs @ rhs.transpose(-1, -2)
    return t.round().to(torch.int64)


def replay_upkeep(T, nq, nd, bound, quad):
    """Replays bmma_klists' list upkeep over values T [n, R, C] (R a multiple of 32, C of 8) of n image pairs with nq / nd
    valid rows / columns.  State [n, W, r, g, t]: lane (g, t) of warp w holds rows 32 w + 8 r + g and sees columns 8 s + 2 t + c.
    quad False: every lane keeps its own K-best lists, threshold the tighter of the own (strict) and the quad (inclusive) bound;
    quad True: one list per row, a pair is buffered iff its distance is below the row's K-th distance (strict: the columns still to
    come have larger indices than the K-th key's).  Returns (counters, [n, R, KT] keys)."""
    n, R, C = T.shape
    W, dev = R // 32, T.device
    col = torch.arange(C, device=dev)
    T = torch.where(col < nd[:, None, None], T, torch.full_like(T, 1 << 20))
    active = (torch.arange(R, device=dev).view(1, W, 4, 8) < nq.view(n, 1, 1, 1))
    thr = torch.where(active, 2 * bound, 0).unsqueeze(-1).repeat(1, 1, 1, 1, 4)
    cnt = torch.zeros_like(thr)
    buf = torch.full(thr.shape + (DEPTH,), NONE, device=dev, dtype=torch.int64)
    lst = torch.full((n, W, 4, 8) + (() if quad else (4,)) + (KT,), NONE, device=dev, dtype=torch.int64)
    slot = torch.arange(DEPTH, device=dev)
    c = {"appends": 0, "vote_steps": 0, "folds": 0, "fold_busiest": 0, "fold_mean": 0.0, "fold_rows": 0}

    def fold(mask):                                        # mask [n, W]: the warps that fold
        nonlocal lst, thr, buf, cnt
        m5 = mask.view(n, W, 1, 1, 1)
        c["folds"] += int(mask.sum())
        per_r = cnt * m5
        c["fold_busiest"] += int(per_r.amax(dim=(3, 4)).sum())          # the warp runs the busiest lane's insertions per row
        c["fold_mean"] += float(per_r.sum(dim=(2, 3, 4)).sum()) / 32    # insertions of the mean lane
        c["fold_rows"] += int((per_r.amax(dim=(3, 4)) > 0).sum())       # rows whose quad lists merge anything
        if quad:
            merged = torch.cat([lst, buf.flatten(-2)], -1).sort(-1).values[..., :KT]
            lst = torch.where(m5, merged, lst)
            kth = lst[..., KT - 1:KT]
            thr = torch.where(m5 & (kth < NONE), torch.minimum(thr, 2 * (kth >> SHIFT)), thr)
        else:
            merged = torch.cat([lst, buf], -1).sort(-1).values[..., :KT]
            lst = torch.where(m5.unsqueeze(-1), merged, lst)
            w = lst[..., KT - 1]
            own = torch.where(w < NONE, 2 * (w >> SHIFT), NONE)
            qb = torch.where(w < NONE, own + 2, NONE).amin(-1, keepdim=True)
            thr = torch.where(m5, torch.minimum(thr, torch.minimum(own, qb)), thr)
        buf = torch.where(m5.unsqueeze(-1), NONE, buf)
        cnt = torch.where(m5, 0, cnt)

    for s in range(C // 8):
        v = T[:, :, 8 * s:8 * s + 8].reshape(n, W, 4, 8, 4, 2)
        key = ((v >> 1) << SHIFT) | col[8 * s:8 * s + 8].view(4, 2)
        take = v < thr.unsqueeze(-1)
        for cc in range(2):
            put = take[..., cc]
            buf = torch.where((slot == cnt.unsqueeze(-1)) & put.unsqueeze(-1), key[..., cc].unsqueeze(-1), buf)
            cnt = cnt + put
        c["appends"] += int(take.sum())
        c["vote_steps"] += int(take.flatten(2).any(-1).sum())    # steps in which the warp appends: the vote passes
        full = (cnt > DEPTH - 2).flatten(2).any(-1)
        if bool(full.any()):
            fold(full)
    fold(active.flatten(2).any(-1))
    out = lst if quad else lst.flatten(-2).sort(-1).values[..., :KT]
    return c, out.reshape(n, R, KT)


def list_counts(v, n_frames, n_cams, bound, lists8, chunk=32):
    """the upkeep counters of both rules on the stream's image pairs (image i against i - n_cams), final lists checked against
    lists8 = match_stream_device's unbounded K = 8 lists"""
    desc, dmask, counts = v["desc"], v["dmask"], v["counts"].long()
    B, cap, _ = desc.shape
    R, C = (cap + 31) // 32 * 32, (cap + 7) // 8 * 8
    res = {}
    for quad in (False, True):
        tot = {"appends": 0, "vote_steps": 0, "folds": 0, "fold_busiest": 0, "fold_mean": 0.0, "fold_rows": 0}
        rows = warps = 0
        for i0 in range(n_cams, B, chunk):
            i1 = min(B, i0 + chunk)
            pad = lambda x, r: torch.nn.functional.pad(x, (0, 0, 0, r - cap))  # noqa: E731
            T = masked_values(pad(desc[i0:i1], R), pad(dmask[i0:i1], R), pad(desc[i0 - n_cams:i1 - n_cams], C),
                              pad(dmask[i0 - n_cams:i1 - n_cams], C))
            nq, nd = counts[i0:i1], counts[i0 - n_cams:i1 - n_cams]
            c, keys = replay_upkeep(T, nq, nd, bound, quad)
            for k in tot:
                tot[k] += c[k]
            rows += int(nq.sum())
            warps += int(((nq + 31) // 32).sum())
            idx = torch.where(keys < NONE, keys & 0xFFFF, -1)[:, :cap]
            dist = torch.where(keys < NONE, keys >> SHIFT, 0x7FFFFFFF)[:, :cap]
            li, ld = lists8[0][i0:i1].long(), lists8[1][i0:i1].long()
            cut = ld >= bound
            li, ld = torch.where(cut, -1, li), torch.where(cut, 0x7FFFFFFF, ld)
            ok = torch.arange(cap, device=desc.device)[None, :] < nq[:, None]
            assert bool(((idx == li) & (dist == ld)).all(-1)[ok].all()), "replayed lists differ from the kernel's"
        f = max(tot["folds"], 1)
        res["quad lists" if quad else "lane lists"] = {
            "appends_per_row": tot["appends"] / rows, "append_steps_per_warp": tot["vote_steps"] / warps,
            "folds_per_warp": tot["folds"] / warps,
            "insertions_per_fold_busiest_lane": tot["fold_busiest"] / f, "insertions_per_fold_mean_lane": tot["fold_mean"] / f,
            "rows_merged_per_fold": tot["fold_rows"] / f}
    return res


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
    bound = th                                           # greedy_dist_bound (multicol_slam_b200/csrc/kernels.h)
    while not th - 1 < 0.9 * bound:
        bound += 1
    runs["lists K=8"]()
    res["upkeep"] = list_counts(v, F, NC, bound, lists[8])
    print(f"{res['gpu']}; {B} images, {res['features']} features; mean GPU time per launch, {args.reps} calls")
    for name in runs:
        for k, (ms, n) in res[name].items():
            print(f"  {name:20s} {k:40s} {ms:8.3f} ms  ({n} launches recorded)")
    print(f"list upkeep of the greedy call (K = {KT}, bound {bound}), replayed:")
    for rule, c in res["upkeep"].items():
        print(f"  {rule:12s} " + ", ".join(f"{k} {x:.2f}" for k, x in c.items()))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
