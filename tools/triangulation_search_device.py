"""Time local mapping's SearchForTriangulationRaw(KF1, KF_i) along CreateNewMapPoints' loop over the neighbours: the device call
(mcs_search_for_triangulation_device, one per neighbour), the host entry point a caller has without it (mcs_search_for_triangulation
on contiguous host arrays) and, where the reference library travelled (oracle/_ref), the reference's own SearchForTriangulationRaw.
Config-3 scene: 4 cameras of 1280x720, 2000 features per camera, masks on; KF1 and its 5 best covisible neighbours (noisy views of
KF1 a few centimetres away), about half of every frame's keypoints free.  After each neighbour a seeded stand-in for the
triangulation checks writes new map-point ids into KF1's and the neighbour's rows on the device, so the next search has fewer queries.
Checks that every route gives the same pairs, and prints the card's name and power limit from the same run.

    python tools/triangulation_search_device.py [--reps 50]
"""
import argparse
import pathlib
import statistics
import subprocess
import sys

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))

N_CAMS, W, H, FEATS, DIM, N_NB = 4, 1280, 720, 2000, 32, 5


def rig_pose(api, shift):
    """4 cameras 90 degrees apart, 10 cm off the rig centre, the rig at `shift`"""
    M_c = np.tile(np.eye(4), (N_CAMS, 1, 1))
    for c in range(N_CAMS):
        a = 2 * np.pi * c / N_CAMS
        M_c[c, :3, :3] = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        M_c[c, :3, 3] = [0.1 * np.sin(a), 0.0, 0.1 * np.cos(a)]
    M_t = np.eye(4)
    M_t[:3, 3] = shift
    return M_c, M_t


def scene(api, seed=0):
    """KF1 and N_NB neighbours as api.Frame (same keypoints, descriptors with 1-5 % of the bits flipped and a tenth of the rows
    shuffled), their contiguous map-point ids (about half free) and their poses"""
    rng = np.random.default_rng(seed)
    n = N_CAMS * FEATS
    keys = np.zeros(n, api.KEYPOINT_DTYPE)
    keys["x"], keys["y"] = rng.uniform(0, W, n), rng.uniform(0, H, n)
    keys["octave"] = rng.integers(0, 8, n)
    cam = np.repeat(np.arange(N_CAMS, dtype=np.int32), FEATS)
    desc = rng.integers(0, 256, (n, DIM), dtype=np.uint8)
    dmask = np.packbits((rng.random((n, DIM * 8)) < 0.9).astype(np.uint8), axis=1, bitorder="little")
    sf = [1.2 ** i for i in range(8)]
    KF1 = api.Frame(keys, cam, desc, dmask, [(W, H)] * N_CAMS, sf)
    mp1 = np.where(rng.random(n) < 0.5, -1, np.arange(n)).astype(np.int32)
    nbs, mps, poses = [], [], []
    for k in range(N_NB):
        flip = np.packbits((rng.random((n, DIM * 8)) < 0.01 + 0.01 * k).astype(np.uint8), axis=1, bitorder="little")
        d = desc ^ flip
        perm = rng.permutation(n // 10)
        d[:n // 10] = d[perm]
        nbs.append(api.Frame(keys, cam, d, dmask, [(W, H)] * N_CAMS, sf))
        mps.append(np.where(rng.random(n) < 0.5, -1, (k + 1) * n + np.arange(n)).astype(np.int32))
        poses.append(rig_pose(api, rng.uniform(-0.05, 0.05, 3)))
    return KF1, mp1, nbs, mps, rig_pose(api, np.zeros(3)), poses, (N_NB + 1) * n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    import multicol_slam_b200.api as api
    from multicol_slam_b200 import rig, settings, synth
    if api.device_count() < 1:
        raise SystemExit("needs an sm_90 (H100) device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"device: {q}")
    try:
        import ref_match_api
        rm = ref_match_api if ref_match_api.available() else None
    except Exception:                                              # noqa: BLE001 - the reference is optional here
        rm = None
    cams = [dict(synth.lafida_cams()[0], width=W, height=H)] * N_CAMS
    m = api.cORBmatcher(0.8, False, DIM, True)                   # the matcher CreateNewMapPoints builds (ref src/cLocalMapping.cpp:228)
    KF1, mp1, nbs, mps, pose1, poses, next_id = scene(api)
    cap, counts = FEATS, [FEATS] * N_CAMS
    frames = [KF1] + nbs
    per = [[(F.keys[F.key_cam == c], F.desc[F.key_cam == c], F.dmask[F.key_cam == c]) for c in range(N_CAMS)] for F in frames]
    buf = torch.from_numpy(np.concatenate([rig.pack([c], cap, DIM) for p in per for c in p])).cuda()
    packs = [(buf, N_CAMS * len(frames), 1, N_CAMS * i) for i in range(len(frames))]
    slot = lambda mp: torch.from_numpy(api.contiguous_to_slots(mp, counts, cap)).cuda()  # noqa: E731
    mp1_t = slot(mp1)
    rays = np.array([api.img_to_world(cams[int(KF1.key_cam[i])], float(k["x"]), float(k["y"])) for i, k in enumerate(KF1.keys)])
    cam = KF1.key_cam
    gen = torch.Generator(device="cuda").manual_seed(1)
    rig1 = api.Rig(cams, *pose1)

    def event_ms(fn, reps):
        out = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn()
            e1.record()
            e1.synchronize()
            out.append(e0.elapsed_time(e1))
        return statistics.median(out), r

    all_same = True
    for k in range(N_NB):
        mp2_t = slot(mps[k])
        E = settings.essential_matrices(rig1.MtMc_inv, api.Rig(cams, *poses[k]).MtMc)
        call = lambda: m.SearchForTriangulationRawDevice(packs[0], mp1_t, packs[1 + k], mp2_t, cams, cap, E, diag=True)  # noqa: E731
        for _ in range(5):
            call()
        torch.cuda.synchronize()
        t_dev, (n_t, m12_t, diag_t) = event_ms(call, args.reps)
        m12 = m12_t.cpu().numpy()
        n_dev, diag = int(n_t.item()), diag_t.cpu().numpy()
        dev_pairs = np.array([(i, b) for i, b in enumerate(api.slots_to_contiguous(m12, counts, cap)) if b >= 0], np.int32).reshape(-1, 2)
        # the host entry point on the same state, contiguous order (slot == contiguous index here: every camera is full)
        free1 = (api.slots_to_contiguous(mp1_t.cpu().numpy(), counts, cap) == -1).astype(np.uint8)
        free2 = (mps[k] == -1).astype(np.uint8)
        F2 = nbs[k]
        host = lambda: m.SearchForTriangulationRaw(KF1.desc, KF1.dmask, cam, free1, rays, F2.desc, F2.dmask, cam, free2, rays, E)  # noqa: E731
        t_host, (n_host, hm12) = event_ms(host, 3)
        host_pairs = np.array([(i, b) for i, b in enumerate(hm12) if b >= 0], np.int32).reshape(-1, 2)
        same = n_host == n_dev and np.array_equal(host_pairs, dev_pairs)
        line = (f"neighbour {k}: queries {diag[0]}, rescans {diag[1]}, matches {n_dev}; device {t_dev:.3f} ms (CUDA-event median of "
                f"{args.reps}), host entry {t_host:.1f} ms (median of 3), identical {same}")
        if rm is not None:
            k1 = rm.KF(KF1, cams, M_c=pose1[0], M_t=pose1[1], mp=np.where(free1 == 1, -1, 0).astype(np.int32), rays=rays)
            k2 = rm.KF(F2, cams, M_c=poses[k][0], M_t=poses[k][1], mp=np.where(free2 == 1, -1, 0).astype(np.int32), rays=rays)
            table = rm.MPTable(N_CAMS, np.zeros((1, 32), np.uint8))
            t_ref, (rn, rpairs) = event_ms(lambda: rm.search_for_triangulation_raw(k1, k2, table, 0.6, True), 1)
            rsame = rn == n_dev and np.array_equal(rpairs, dev_pairs)
            line += f", reference {t_ref:.1f} ms (one pass), identical {rsame}"
            same = same and rsame
        else:
            line += ", reference: not run (oracle/_ref absent)"
        print(line, flush=True)
        all_same = all_same and same
        # the stand-in for the triangulation checks, on the device: about 70 % of the pairs become new points
        keep = (m12_t >= 0) & (torch.rand(m12_t.shape, generator=gen, device="cuda") < 0.7)
        ids = next_id + torch.cumsum(keep.to(torch.int32), 0, dtype=torch.int32) - 1
        mp1_t[keep] = ids[keep]
        mp2_t[m12_t[keep].long()] = ids[keep]
        next_id += int(keep.sum().item())
    if not all_same:
        raise SystemExit("the routes differ")


if __name__ == "__main__":
    main()
