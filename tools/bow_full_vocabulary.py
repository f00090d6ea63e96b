"""Time relocalisation's bag-of-words step on the device with a full-size vocabulary (tests/bow_scale.py: k = 10, L = 6, 1 064 066
nodes and 956 865 words, generated from its seed): ComputeBoW of the current frame (mcs_bow_vectors_device) and SearchByBoW(KF_i, F)
for 10 and 40 candidate key frames in one call (mcs_search_by_bow_device), at levelsup 4 and at levelsup 0, where n_kf * max_nodes
passes the search's grid and its warps stride.  The scene is config 3 of bench.py: four 1280x720 cameras, 2000 features, masks on;
the current frame and its 40 candidates are 41 consecutive frames of bench.make_stream extracted into one packed buffer; 70 % of
every key frame's keypoints carry a map point.  Per call: CUDA-event median and spread over --runs calls, whether the result equals
the host route (mcs_bow_vectors, mcs_search_by_bow per key frame), and, in a separate profiled call, the time per kernel and per
memset (ComputeBoW clears its per-node and per-word counters, 4 bytes per node and per word, on every call), and the sizes of the
(key frame, common node) groups the search met.

    python tools/bow_full_vocabulary.py [--runs 30] [--out /tmp/bow_full_vocabulary.json]
"""
import argparse
import json
import pathlib
import re
import subprocess
import sys

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
N_KF = 40


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    import bow_scale
    import multicol_slam_b200.api as api
    from multicol_slam_b200 import rig as rigmod
    from multicol_slam_b200 import synth

    dev = torch.device("cuda", 0)
    res = {"gpu": torch.cuda.get_device_name(dev)}
    res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                                        capture_output=True, text=True, timeout=30).stdout.strip()
    cfg = bench.CONFIGS[3]
    W, H, NF = cfg["w"], cfg["h"], cfg["nfeatures"]
    cams = bench.rig_cams(cfg)
    nc, nfr = len(cams), N_KF + 1
    images = bench.make_stream(cams, list(range(nc)), nfr, 1000)
    pitch = (W + 63) // 64 * 64
    dev_images = torch.zeros((nfr * nc, H, pitch), dtype=torch.uint8, device=dev)
    dev_images[:, :, :W] = torch.from_numpy(images.reshape(nfr * nc, H, W)).to(dev)
    ex = api.mdBRIEFextractorOct(nfeatures=NF, nlevels=bench.NLEVELS, do_dBrief=True, learnMasks=True)
    cap = ex.capacity
    packed = torch.zeros(rigmod.packed_layout(nfr * nc, cap, 32)[1], dtype=torch.uint8, device=dev)
    views = ex.extract_batch_packed_device(dev_images, np.stack([synth.mirror_mask(c) for c in cams]), cams, list(range(nc)) * nfr,
                                           packed, width=W)
    torch.cuda.synchronize()
    del dev_images
    counts = views["counts"].cpu().numpy().reshape(nfr, nc)
    tree = bow_scale.vocabulary()
    voc = api.ORBVocabulary(tree)
    stream = torch.cuda.current_stream(dev)
    CUR = N_KF // 2
    by_distance = sorted((f for f in range(nfr) if f != CUR), key=lambda f: (abs(f - CUR), f))
    frame = lambda f: (packed, 1, nfr * nc, f * nc)  # noqa: E731
    D = {f: np.concatenate([views["desc"][f * nc + c, :counts[f, c]].cpu().numpy() for c in range(nc)]) for f in range(nfr)}
    M = {f: np.concatenate([views["dmask"][f * nc + c, :counts[f, c]].cpu().numpy() for c in range(nc)]) for f in range(nfr)}
    rng = np.random.default_rng(7)
    mp = {f: np.where(rng.random(len(D[f])) < 0.7, np.arange(len(D[f])), -1).astype(np.int32) for f in range(nfr)}
    mp_t = {f: torch.from_numpy(api.contiguous_to_slots(mp[f], counts[f], cap)).to(dev) for f in range(nfr)}
    n_points = int(max(len(d) for d in D.values()))
    mt = api.cORBmatcher(0.75, False, 32, True)                                 # Relocalisation's matcher
    ns = nc * cap
    res.update({"cameras": nc, "image": f"{W}x{H}", "nfeatures": NF, "capacity": cap, "keypoints_current": int(counts[CUR].sum()),
                "vocabulary": {"nodes": len(tree["parent"]), "words": len(tree["word_node"]), "k": 10, "L": 6},
                "node_tiles": (len(tree["parent"]) + 2047) // 2048, "word_tiles": (len(tree["word_node"]) + 2047) // 2048, "cases": []})

    def slots_to_ids(slots, f):
        first = np.concatenate([[0], np.cumsum(counts[f])])
        slots = np.asarray(slots)
        return first[slots // cap] + slots % cap

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.runs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            fn()
            e1.record(stream)
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return {"gpu_ms_median": float(np.median(ms)), "gpu_ms_min_max": [float(min(ms)), float(max(ms))], "runs": args.runs}

    def split_of(fn):
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            fn()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            if e.device_type.name == "CUDA":
                hit = re.search(r"(\w+_kernel)(<[^>]*>)?", e.name)
                k = kern.setdefault(hit.group(0) if hit else e.name.strip(), [0, 0.0])
                k[0] += 1
                k[1] += (e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total) / 1e3
        return {k: {"launches": c, "ms": round(t, 4)} for k, (c, t) in sorted(kern.items(), key=lambda x: -x[1][1])}

    for levelsup in (4, 0):
        max_nodes = voc.level_nodes(levelsup)
        bows = {f: voc.transform_device(frame(f), nc, cap, levelsup, max_nodes, stream=stream) for f in range(nfr)}
        torch.cuda.synchronize()
        host = {f: voc.transform(D[f], levelsup) for f in range(nfr)}
        b = bows[CUR].host()
        h = host[CUR]
        same_bow = bool(np.array_equal(b[0], h[0]) and np.array_equal(b[1], h[1]) and np.array_equal(b[2][0], h[2][0]) and
                        np.array_equal(slots_to_ids(b[2][2], CUR), h[2][2]) and int(bows[CUR].status.item()) == 0)
        bow_call = lambda: voc.transform_device(frame(CUR), nc, cap, levelsup, max_nodes, stream=stream)  # noqa: E731
        case = {"levelsup": levelsup, "max_nodes": max_nodes, "n_bow_current": len(h[0]), "n_fv_current": len(h[2][0]),
                "cleared_bytes": 4 * (len(tree["parent"]) + len(tree["word_node"]) + min(max_nodes, ns)),
                "compute_bow": dict(timed(bow_call), identical_results=same_bow, kernels_ms=split_of(bow_call)), "search": {}}
        for n_kf in (10, N_KF):
            kfs = by_distance[:n_kf]
            outs = (torch.empty((n_kf, ns), dtype=torch.int32, device=dev), torch.empty((n_kf, ns), dtype=torch.int32, device=dev),
                    torch.zeros(n_kf, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))
            call = lambda kfs=kfs, outs=outs: mt.SearchByBoWDevice(  # noqa: E731
                [(bows[f], mp_t[f]) for f in kfs], bows[CUR], n_points, stream=stream, out=outs)
            call()
            torch.cuda.synchronize()
            msl, nm = outs[1].cpu().numpy(), outs[2].cpu().numpy()
            ok = int(outs[3].item()) == 0
            for k, f in enumerate(kfs):
                n_h, m_h = mt.SearchByBoWFrame(D[f], host[f][2], D[CUR], host[CUR][2], M[f], M[CUR], (mp[f] >= 0).astype(np.uint8))
                sl = api.slots_to_contiguous(msl[k], counts[CUR], cap)
                ok &= int(nm[k]) == n_h and np.array_equal(np.where(sl >= 0, slots_to_ids(np.maximum(sl, 0), f), -1), m_h)
            groups = []                 # (key-frame keypoints with a map point, frame keypoints) of every common node
            cn, co, _ = host[CUR][2]
            for f in kfs:
                kn, ko, kfeat = host[f][2]
                at = np.minimum(np.searchsorted(cn, kn), len(cn) - 1)
                for a in np.flatnonzero(cn[at] == kn):
                    groups.append((int((mp[f][kfeat[ko[a]:ko[a + 1]]] >= 0).sum()), int(co[at[a] + 1] - co[at[a]])))
            work = np.array([q * c for q, c in groups])
            case["search"][str(n_kf)] = dict(timed(call), identical_results=bool(ok), n_kf_x_max_nodes=n_kf * max_nodes,
                                             strided=n_kf * max_nodes > 16384 * 8, matches=nm.tolist(), groups=len(groups),
                                             largest_group=list(groups[int(work.argmax())]),
                                             median_group=[int(np.median([g[0] for g in groups])), int(np.median([g[1] for g in groups]))],
                                             kernels_ms=split_of(call))
        res["cases"].append(case)
        del bows
    print(json.dumps(res, indent=1))
    if args.out:
        pathlib.Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        pathlib.Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
