"""Measure loop closing's two Sim3 searches on the device (cORBmatcher.SearchBySim3Device, SearchByProjectionKFScwDevice) against the
host mirror routes (cORBmatcher.SearchBySim3, SearchByProjectionKFScw: projection in Python, one mcs_search_windows call per
direction / call) and, where oracle/_ref is present, the reference's own SearchBySim3 on the CPU (its SearchByProjection(KF, Scw)
reads past a camera's descriptors on key frames of several cameras, so it is not run).  Every route must give the same
matches12 / vpMatched and counts.

Scene: bench.py's config 3 (four 1280x720 cameras, 2000 features per camera, masks on).  KF1 and KF2 are frames 0 and 1 of
bench.make_stream, extracted into one packed buffer, at rig poses a few centimetres apart.  Each key frame carries a map point on the
bearing ray of every keypoint; the Sim3 between them is their relative pose with s12 = 1.02, searched with th = 10 as at the call
site.  SearchByProjection(KF1, Scw) takes 3000 loop points (KF2's) with Scw = KF1's pose scaled by 1.02, and vpMatched = the
SearchBySim3 result.  Device times are CUDA-event medians around the Python wrapper call with its inputs resident: they include a
device copy of the input row (the call updates it in place) and the wrapper's host-side pose arithmetic and staging.  Host times are
wall-clock medians.  The card's name and power limit are read in the same run.

    python tools/sim3_searches_device.py [--runs 20] [--host-runs 3] [--out /tmp/sim3_searches_device.json]
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
N_LOOP = 3000
TH_SIM3 = 10.0             # the window factor the call site passes (ref src/cLoopClosing.cpp:343)


def _stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--host-runs", type=int, default=3)
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
    ex = api.mdBRIEFextractorOct(nfeatures=NF, nlevels=bench.NLEVELS, do_dBrief=True, learnMasks=True)
    cap, ds = ex.capacity, 32
    pitch = (W + 63) // 64 * 64
    images = bench.make_stream(cams, list(range(nc)), 2, 3000)
    dimg = torch.zeros((2 * nc, H, pitch), dtype=torch.uint8, device=dev)
    dimg[:, :, :W] = torch.from_numpy(images.reshape(2 * nc, H, W)).to(dev)
    packed = torch.zeros(rigmod.packed_layout(2 * nc, cap, ds)[1], dtype=torch.uint8, device=dev)
    v = ex.extract_batch_packed_device(dimg, masks, cams, list(range(nc)) * 2, packed, width=W)
    torch.cuda.synchronize()
    counts = v["counts"].cpu().numpy()
    kps, d, m = v["kps"].cpu().numpy(), v["desc"].cpu().numpy(), v["dmask"].cpu().numpy()
    host = [(kps[i].view(api.KEYPOINT_DTYPE).reshape(cap)[:counts[i]].copy(), d[i, :counts[i]].copy(), m[i, :counts[i]].copy())
            for i in range(2 * nc)]
    sf = [float(ex.info.scale_factor[l]) for l in range(bench.NLEVELS)]
    F1, F2 = (api.Frame.from_cameras(host[t * nc:(t + 1) * nc], [(W, H)] * nc, sf) for t in range(2))

    rng = np.random.default_rng(1)
    M_c = np.tile(np.eye(4), (nc, 1, 1))
    for c in range(nc):
        a = 2 * np.pi * c / nc
        M_c[c, :3, :3] = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        M_c[c, :3, 3] = [0.1 * np.sin(a), 0.0, 0.1 * np.cos(a)]
    rig1 = api.Rig(cams, M_c, np.eye(4))
    M_t2 = np.eye(4)
    M_t2[:3, 3] = [0.03, -0.01, 0.02]
    rig2 = api.Rig(cams, M_c, M_t2)

    def points_on_rays(F, rig):
        rays, _, _ = api.frame_prepare(F.keys, F.key_cam, cams)
        depth = rng.uniform(2.0, 6.0, len(F.keys))
        w = np.stack([(rig.MtMc[int(F.key_cam[k])] @ np.append(rays[k] * depth[k], 1.0))[:3] for k in range(len(F.keys))])
        return w, depth

    w1, d1 = points_on_rays(F1, rig1)
    w2, d2 = points_on_rays(F2, rig2)
    n1, n2 = len(F1.keys), len(F2.keys)
    world, depth = np.concatenate([w1, w2]), np.concatenate([d1, d2])
    desc, dmask = np.concatenate([F1.desc, F2.desc]), np.concatenate([F1.dmask, F2.dmask])
    min_d, max_d = depth * rng.uniform(0.5, 0.9, n1 + n2), depth * rng.uniform(1.2, 3.0, n1 + n2)
    bad = (rng.random(n1 + n2) < 0.02).astype(np.uint8)
    mp1, mp2 = np.arange(n1, dtype=np.int32), n1 + np.arange(n2, dtype=np.int32)
    T12 = api._mm(api.inv_rigid(rig1.M_t), rig2.M_t)
    s12, R12, t12 = 1.02, T12[:3, :3].copy(), T12[:3, 3].copy()
    Scw = api.inv_rigid(rig1.M_t)
    Scw[:3, :] *= 1.02
    loop = mp2[rng.choice(n2, min(N_LOOP, n1), replace=False)].astype(np.int32)

    mt = api.cORBmatcher(0.6, False, ds, True)
    tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    c1, c2 = counts[:nc], counts[nc:]
    dm = dict(world=tt(world), lo=tt(min_d), hi=tt(max_d), desc=tt(desc), dmask=tt(dmask), bad=tt(bad))
    mp1_t, mp2_t = tt(api.contiguous_to_slots(mp1, c1, cap)), tt(api.contiguous_to_slots(mp2, c2, cap))
    masks_t, loop_t = tt(masks), tt(loop)
    kf1, kf2 = (packed, 1, 2 * nc, 0), (packed, 1, 2 * nc, nc)
    pre = np.full(n1, -1, np.int32)
    stream = torch.cuda.current_stream(dev)

    res = {"gpu": torch.cuda.get_device_name(dev), "cameras": nc, "image": f"{W}x{H}", "nfeatures": NF, "capacity": cap,
           "keypoints": [int(n1), int(n2)], "map_points": int(n1 + n2), "loop_points": int(len(loop)), "s12": s12, "runs": args.runs,
           "host_runs": args.host_runs}
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                                            text=True, timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        res["power_limit"] = f"unknown ({e})"

    m12_0 = tt(api.contiguous_to_slots(pre, c1, cap))

    def dev_sim3():                                   # a device copy of the input row: the call updates it in place
        m12_t = m12_0.clone()
        return mt.SearchBySim3Device(kf1, kf2, cap, rig1, rig2, masks_t, sf, mp1_t, mp2_t, dm["world"], dm["lo"], dm["hi"], dm["desc"],
                                     dm["dmask"], s12, R12, t12, TH_SIM3, m12_t, bad_t=dm["bad"], stream=stream)

    def dev_scw(matched_t):
        mt_t = matched_t.clone()
        return mt.SearchByProjectionKFScwDevice(kf1, cap, rig1, Scw, masks_t, sf, loop_t, dm["world"], dm["lo"], dm["hi"], dm["desc"],
                                                dm["dmask"], 10, mt_t, bad_t=dm["bad"], stream=stream, diag=True)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        out = fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    for _ in range(3):                                                # warm-up: pool, module load
        dev_sim3(); torch.cuda.synchronize()
    ts, out = zip(*[timed(dev_sim3) for _ in range(args.runs)])
    dn = int(out[-1][0].item()); dst = int(out[-1][1].item())
    d12 = api.slots_to_contiguous(out[-1][2].cpu().numpy(), c1, cap)
    res["sim3_device_ms"] = _stats(ts)
    hs = []
    for _ in range(args.host_runs):
        t0 = time.perf_counter()
        hn, h12 = mt.SearchBySim3(F1, rig1, mp1, F2, rig2, mp2, world, min_d, max_d, bad, desc, dmask, s12, R12, t12, TH_SIM3, matches12=pre)
        hs.append((time.perf_counter() - t0) * 1e3)
    res["sim3_host_mirror_ms"] = _stats(hs)
    res["sim3_found"] = dn
    res["sim3_identical"] = bool(dst == 0 and dn == hn and np.array_equal(d12, h12))

    h12_t = tt(api.contiguous_to_slots(h12, c1, cap))
    for _ in range(3):
        dev_scw(h12_t); torch.cuda.synchronize()
    ts, out = zip(*[timed(lambda: dev_scw(h12_t)) for _ in range(args.runs)])
    sn, sst = int(out[-1][0].item()), int(out[-1][1].item())
    smatched = api.slots_to_contiguous(out[-1][2].cpu().numpy(), c1, cap)
    res["scw_device_ms"] = _stats(ts)
    res["scw_diag"] = out[-1][3].cpu().numpy().tolist()
    hs = []
    for _ in range(args.host_runs):
        t0 = time.perf_counter()
        hsn, hsm = mt.SearchByProjectionKFScw(F1, rig1, Scw, loop, h12, world, min_d, max_d, bad, desc, dmask, th=10)
        hs.append((time.perf_counter() - t0) * 1e3)
    res["scw_host_mirror_ms"] = _stats(hs)
    res["scw_matches"] = sn
    res["scw_identical"] = bool(sst == 0 and sn == hsn and np.array_equal(smatched, hsm))

    try:
        import ref_match_api as rm
        available = rm.available()
    except Exception:  # noqa: BLE001
        available = False
    if available:
        obs_kf = np.concatenate([np.zeros(n1, np.int32), np.ones(n2, np.int32)])
        obs_idx = np.concatenate([np.arange(n1), np.arange(n2)]).astype(np.int32)
        table = rm.MPTable(nc, desc, dmask=dmask, bad=bad, world_pos=world, min_dist=min_d, max_dist=max_d, obs_kf=obs_kf, obs_idx=obs_idx)
        k1 = rm.KF(F1, cams, M_c=M_c, M_t=rig1.M_t, mp=mp1)
        k2 = rm.KF(F2, cams, M_c=M_c, M_t=rig2.M_t, mp=mp2)
        rs = []
        for _ in range(args.host_runs):
            t0 = time.perf_counter()
            rn, r12 = rm.search_by_sim3(k1, k2, table, s12, R12, t12, TH_SIM3, pre, 0.6, True)
            rs.append((time.perf_counter() - t0) * 1e3)
        res["sim3_reference_ms"] = _stats(rs)
        res["sim3_reference_identical"] = bool(rn == dn and np.array_equal(r12, d12))
        # the reference's SearchByProjection(KF, Scw) reads past camera c's descriptor matrix for cameras > 0 (undefined), so it is
        # not run on this four-camera key frame
        res["scw_reference_ms"] = "not measured: undefined behaviour on multi-camera key frames"
    else:
        res["reference"] = "not measured: oracle/_ref not built"
    print(json.dumps(res))
    if args.out:
        pathlib.Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
