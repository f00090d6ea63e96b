"""Measure one SearchInNeighbors worth of Fuse calls on the device (mcs_fuse_device + the hit read-back + cORBmatcher.FuseReplay)
against the host route an integrator has without it, the mirror cORBmatcher.Fuse per key frame (projection on the host, one
mcs_search_windows call per key frame), and, where oracle/_ref is present, the reference's own Fuse on the CPU.

Scene: bench.py's config 3 (four 1280x720 cameras, 2000 features per camera, masks on).  A current key frame and up to 60 target
key frames are frames of bench.make_stream, extracted into one packed buffer; the targets' poses are the current one moved by a few
centimetres.  About 50 000 map points: one on the bearing ray of every keypoint of the current key frame (its row, the first
pass's queries), the rest on rays of the targets' keypoints, a third of which they hold.  Fuse(pKFi, curKF, .) (:1265, variant 0)
for every target: the device route makes ONE call for all targets, reads the hits back and replays them per target; the host
route calls Fuse per target; both on the same (unchanged) map state, so every target's ops must agree.  Runs alternate the
routes; medians and min-max are reported, with the card's name and power limit read in the same run.  The host routes are slow
(pure-Python projection), so each of their runs covers the first --host-kfs targets, alternated with the device route's runs
(the first --host-runs of them), and their per-target time is scaled to the batch; the ops check covers those targets.

    python tools/fuse_device.py [--runs 5] [--host-runs 5] [--host-kfs 2] [--out /tmp/fuse_device.json]
"""
import argparse
import json
import pathlib
import subprocess
import sys
import time

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))
N_TARGETS = (20, 60)
N_POINTS = 50000


def _stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--host-runs", type=int, default=5)
    ap.add_argument("--host-kfs", type=int, default=2)
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
    nc, nfr = len(cams), 1 + max(N_TARGETS)
    masks = np.stack([synth.mirror_mask(c) for c in cams])
    ex = api.mdBRIEFextractorOct(nfeatures=NF, nlevels=bench.NLEVELS, do_dBrief=True, learnMasks=True)
    cap, ds = ex.capacity, 32
    pitch = (W + 63) // 64 * 64
    counts = np.zeros(nfr * nc, np.int32)
    host = {}                                             # image -> (keypoints, descriptors, masks) as extracted
    for f0 in range(0, nfr, 16):                          # extraction in chunks of 16 frames, then one buffer for all frames
        nf = min(16, nfr - f0)
        images = bench.make_stream(cams, list(range(nc)), nf, 2000 + f0)
        dimg = torch.zeros((nf * nc, H, pitch), dtype=torch.uint8, device=dev)
        dimg[:, :, :W] = torch.from_numpy(images.reshape(nf * nc, H, W)).to(dev)
        part = torch.zeros(rigmod.packed_layout(nf * nc, cap, ds)[1], dtype=torch.uint8, device=dev)
        v = ex.extract_batch_packed_device(dimg, masks, cams, list(range(nc)) * nf, part, width=W)
        torch.cuda.synchronize()
        counts[f0 * nc:(f0 + nf) * nc] = v["counts"].cpu().numpy()
        kps, d, m = v["kps"].cpu().numpy(), v["desc"].cpu().numpy(), v["dmask"].cpu().numpy()
        for i in range(nf * nc):
            n = counts[f0 * nc + i]
            host[f0 * nc + i] = (kps[i].view(api.KEYPOINT_DTYPE).reshape(cap)[:n].copy(), d[i, :n].copy(), m[i, :n].copy())
    packed = torch.from_numpy(rigmod.pack([host[i] for i in range(nfr * nc)], cap, ds)).to(dev)
    sf = [float(ex.info.scale_factor[l]) for l in range(bench.NLEVELS)]
    sizes = [(W, H)] * nc
    frames = [api.Frame.from_cameras([host[t * nc + c] for c in range(nc)], sizes, sf) for t in range(nfr)]

    # the rig: cameras 90 degrees apart; targets moved by a few cm from the current key frame's pose
    rng = np.random.default_rng(1)
    M_c = np.tile(np.eye(4), (nc, 1, 1))
    for c in range(nc):
        a = 2 * np.pi * c / nc
        M_c[c, :3, :3] = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        M_c[c, :3, 3] = [0.1 * np.sin(a), 0.0, 0.1 * np.cos(a)]
    cur_rig = api.Rig(cams, M_c, np.eye(4))
    rigs = []
    for _ in range(max(N_TARGETS)):
        M_t = np.eye(4)
        M_t[:3, 3] = rng.normal(0, 0.03, 3)
        rigs.append(api.Rig(cams, M_c, M_t))

    def points_on_rays(F, rig, n):
        rays, _, _ = api.frame_prepare(F.keys, F.key_cam, cams)
        sel = rng.choice(len(F.keys), n, replace=False) if n < len(F.keys) else np.arange(len(F.keys))
        depth = rng.uniform(2.0, 6.0, len(sel))
        w = np.stack([(rig.MtMc[int(F.key_cam[k])] @ np.append(rays[k] * depth[i], 1.0))[:3] for i, k in enumerate(sel)])
        return sel, w, depth, rays

    Fc = frames[0]
    sel, w0, d0, cur_rays = points_on_rays(Fc, cur_rig, len(Fc.keys))
    world, desc, dmask, depth = [w0], [Fc.desc[sel]], [Fc.dmask[sel]], [d0]
    cur_row = np.full(len(Fc.keys), -1, np.int32)
    cur_row[sel] = np.arange(len(sel))
    n_pts = len(sel)
    rows = []
    per_t = (N_POINTS - n_pts) // max(N_TARGETS)
    for t in range(max(N_TARGETS)):
        F = frames[1 + t]
        s_t, w_t, d_t, _ = points_on_rays(F, rigs[t], per_t)
        row = np.full(len(F.keys), -1, np.int32)
        held = s_t[: len(s_t) // 3 * 3][::3]
        row[held] = n_pts + np.flatnonzero(np.isin(s_t, held))
        rows.append(row)
        world.append(w_t); desc.append(F.desc[s_t]); dmask.append(F.dmask[s_t]); depth.append(d_t)
        n_pts += len(s_t)
    world, desc, dmask, depth = np.concatenate(world), np.concatenate(desc), np.concatenate(dmask), np.concatenate(depth)
    min_d, max_d = depth * rng.uniform(0.5, 0.9, n_pts), depth * rng.uniform(1.2, 3.0, n_pts)
    bad = (rng.random(n_pts) < 0.02).astype(np.uint8)
    in_kf = [np.zeros(n_pts, bool) for _ in rigs]
    for t, r in enumerate(rows):
        in_kf[t][r[r >= 0]] = True
    kf_rays = [api.frame_prepare(frames[1 + t].keys, frames[1 + t].key_cam, cams)[0] for t in range(max(N_TARGETS))]

    mt = api.cORBmatcher(0.6, False, ds, True)
    tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    dm = dict(world=tt(world), lo=tt(min_d), hi=tt(max_d), desc=tt(desc), dmask=tt(dmask), bad=tt(bad))
    slot_rows = [tt(api.contiguous_to_slots(rows[t], counts[(1 + t) * nc:(2 + t) * nc], cap)) for t in range(max(N_TARGETS))]
    q_t = tt(api.contiguous_to_slots(cur_row, counts[:nc], cap))
    # curKF's slot order == its contiguous order once the -1 gaps are skipped; the replay indexes rays by query slot
    slot_rays = np.zeros((nc * cap, 3))
    o = 0
    for c in range(nc):
        slot_rays[c * cap:c * cap + counts[c]] = cur_rays[o:o + counts[c]]
        o += counts[c]
    q_ids = q_t.cpu().numpy()
    masks_t = tt(masks)
    stream = torch.cuda.current_stream(dev)

    res = {"gpu": torch.cuda.get_device_name(dev), "cameras": nc, "image": f"{W}x{H}", "nfeatures": NF, "capacity": cap, "map_points": n_pts,
           "queries": int((q_ids >= 0).sum()), "th": 3.0, "th_low": mt.TH_LOW_, "runs": args.runs, "host_runs": args.host_runs,
           "host_kfs": args.host_kfs}
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                                            text=True, timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        res["power_limit"] = f"unknown ({e})"

    def device_route(n_kf, n_replay):
        kfs = [((packed, 1, nfr * nc, (1 + t) * nc), slot_rows[t], rigs[t].MtMc_inv, rigs[t].M_t[:3, 3]) for t in range(n_kf)]
        hits, nh, st = mt.FuseDevice(kfs, q_t, cap, cams, masks_t, sf, dm["world"], dm["lo"], dm["hi"], dm["desc"], dm["dmask"], bad_t=dm["bad"],
                                     variant=0, th=3.0, max_hits=n_kf * 4 * cap, stream=stream)
        n = int(nh.item())                                    # the one device-to-host copy: the count, then the rows
        h = hits[:n].cpu().numpy()
        assert int(st.item()) == 0
        out = []
        for t in range(n_replay):
            r = h[h[:, 0] == t][:, 1:]
            out.append(mt.FuseReplay(frames[1 + t], rigs[t], rows[t], q_ids, r, cap, world, min_d, max_d, bad, in_kf[t], desc, dmask, th=3.0,
                                     variant=0, cur_rays=slot_rays, kf_rays=kf_rays[t], cur_rig=cur_rig))
        return n, out

    def host_route(t):
        return mt.Fuse(frames[1 + t], rigs[t], rows[t], q_ids, world, min_d, max_d, bad, in_kf[t], desc, dmask, th=3.0, variant=0,
                       cur_rays=slot_rays, kf_rays=kf_rays[t], cur_rig=cur_rig)

    rm = None
    try:
        import ref_match_api
        rm = ref_match_api if ref_match_api.available() else None
    except Exception:  # noqa: BLE001
        rm = None

    def reference_route(t):
        table = rm.MPTable(nc, desc, dmask=dmask, bad=bad, world_pos=world, min_dist=min_d, max_dist=max_d,
                           obs_kf=np.where(in_kf[t], 0, -1).astype(np.int32), obs_idx=np.zeros(n_pts, np.int32))
        K = rm.KF(frames[1 + t], cams, M_c=M_c, M_t=rigs[t].M_t, mp=rows[t], rays=kf_rays[t])
        Fq = api.Frame(Fc.keys, Fc.key_cam, Fc.desc, Fc.dmask, sizes, sf)
        Cq = rm.KF(Fq, cams, M_c=M_c, M_t=cur_rig.M_t, mp=cur_row, rays=cur_rays)
        return rm.fuse(0, K, table, cur_row, 3.0, 0.6, True, CurK=Cq)

    # warm-up and the identity check on the first host_kfs targets
    hk = args.host_kfs
    _, dev_out = device_route(max(N_TARGETS), hk)
    identical = True
    checks = []
    for t in range(hk):
        hn, hops, hmp = host_route(t)
        same = dev_out[t][0] == hn and np.array_equal(dev_out[t][1], hops) and np.array_equal(dev_out[t][2], hmp)
        rsame = None
        if rm is not None:
            rn, rops = reference_route(t)
            rsame = bool(rn == hn and np.array_equal(rops, hops))
            same = same and rsame
        identical &= bool(same)
        checks.append({"target": t, "ops": int(len(hops)), "fused": int(hn), "identical": bool(same), "reference_identical": rsame})
    res["checks"] = checks
    res["identical_ops"] = bool(identical)

    for n_kf in N_TARGETS:
        call_ms, route_ms, host_ms, ref_ms = [], [], [], []
        for r in range(args.runs):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record(stream)
            n_hits, _ = device_route(n_kf, 0)
            e1.record(stream)
            torch.cuda.synchronize()
            call_ms.append(e0.elapsed_time(e1))
            t1 = time.perf_counter()
            device_route(n_kf, n_kf)
            route_ms.append((time.perf_counter() - t1) * 1e3)
            if r < args.host_runs:                     # alternated with the device route
                t2 = time.perf_counter()
                for t in range(hk):
                    host_route(t)
                host_ms.append((time.perf_counter() - t2) * 1e3 / hk * n_kf)
                if rm is not None:
                    t3 = time.perf_counter()
                    for t in range(hk):
                        reference_route(t)
                    ref_ms.append((time.perf_counter() - t3) * 1e3 / hk * n_kf)
        res[f"targets_{n_kf}"] = {"hits": n_hits, "device_call_and_count_read_gpu_ms": _stats(call_ms),
                                  "device_route_with_replay_wall_ms": _stats(route_ms),
                                  "host_route_wall_ms_scaled_from_host_kfs": _stats(host_ms) if host_ms else "not measured",
                                  "reference_cpu_wall_ms_scaled_from_host_kfs": _stats(ref_ms) if ref_ms else "not measured"}
    print(json.dumps(res, indent=1))
    if args.out:
        pathlib.Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        pathlib.Path(args.out).write_text(json.dumps(res, indent=1))
    if not identical:
        sys.exit("the routes differ")


if __name__ == "__main__":
    main()
