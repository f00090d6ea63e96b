"""Time loop closing's SearchByBoW(KF1, KF_k) over the loop candidates: the device call (mcs_search_by_bow_keyframes_device) against
the host route a caller has without it (read back, slots_to_contiguous, one brute-force SearchByBoW per candidate) and, where the
reference library travelled (oracle/_ref), the reference's own SearchByBoW(KF1, KF2) per candidate.  Config-3 scene: 4 cameras of
1280x720, 2000 features per camera, masks on, about half of the keypoints carrying map points; candidates are noisy views of KF1.
Checks that every route gives the same matches, and prints the card's name and power limit from the same run.

    python tools/loop_bow_search_device.py [--candidates 1 4 16] [--reps 50]
"""
import argparse
import pathlib
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))

N_CAMS, W, H, FEATS, DIM = 4, 1280, 720, 2000, 32


def scene(api, n_kf, seed=0):
    """KF1 and n_kf candidates as api.Frame, their contiguous map-point ids and the bad flags"""
    rng = np.random.default_rng(seed)
    n = N_CAMS * FEATS
    keys = np.zeros(n, api.KEYPOINT_DTYPE)
    keys["x"], keys["y"] = rng.uniform(0, W, n), rng.uniform(0, H, n)
    keys["octave"] = rng.integers(0, 8, n)
    cam = np.repeat(np.arange(N_CAMS, dtype=np.int32), FEATS)
    desc = rng.integers(0, 256, (n, DIM), dtype=np.uint8)
    dmask = (rng.random((n, DIM * 8)) < 0.9).astype(np.uint8)
    dmask = np.packbits(dmask, axis=1, bitorder="little")
    sf = [1.2 ** i for i in range(8)]
    KF1 = api.Frame(keys, cam, desc, dmask, [(W, H)] * N_CAMS, sf)
    mp1 = np.where(rng.random(n) < 0.5, np.arange(n), -1).astype(np.int32)
    cands, mps = [], []
    for k in range(n_kf):
        flip = np.packbits((rng.random((n, DIM * 8)) < 0.01 + 0.004 * (k % 8)).astype(np.uint8), axis=1, bitorder="little")
        perm = rng.permutation(n // 10)                            # a tenth of each candidate's rows shuffled within the block
        d = desc ^ flip
        d[:n // 10] = d[perm]
        cands.append(api.Frame(keys, cam, d, dmask, [(W, H)] * N_CAMS, sf))
        mps.append(np.where(rng.random(n) < 0.5, (k + 1) * n + np.arange(n), -1).astype(np.int32))
    bad = (rng.random((n_kf + 1) * n) < 0.02).astype(np.uint8)
    return KF1, mp1, cands, mps, bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--candidates", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    import multicol_slam_b200.api as api
    from multicol_slam_b200 import rig
    if api.device_count() < 1:
        raise SystemExit("needs an sm_90 (H100) device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"device: {q}")
    try:
        import ref_match_api
        rm = ref_match_api if ref_match_api.available() else None
    except Exception:                                              # noqa: BLE001 - the reference is optional here
        rm = None
    m = api.cORBmatcher(0.9, False, DIM, True)                   # the matcher ComputeSim3 builds (ref src/cLoopClosing.cpp:254)
    cap = FEATS
    for n_kf in args.candidates:
        KF1, mp1, cands, mps, bad = scene(api, n_kf)
        frames = [KF1] + cands
        per = [[(F.keys[F.key_cam == c], F.desc[F.key_cam == c], F.dmask[F.key_cam == c]) for c in range(N_CAMS)] for F in frames]
        buf = torch.from_numpy(np.concatenate([rig.pack([c], cap, DIM) for p in per for c in p])).cuda()
        packs = [(buf, N_CAMS * len(frames), 1, N_CAMS * i) for i in range(len(frames))]
        counts = [FEATS] * N_CAMS
        slot = lambda mp: torch.from_numpy(api.contiguous_to_slots(mp, counts, cap)).cuda()  # noqa: E731
        mp1_t, kfs = slot(mp1), [(packs[1 + k], slot(mps[k])) for k in range(n_kf)]
        bad_t, n_points = torch.from_numpy(bad).cuda(), len(bad)
        out = m.SearchByBoWKeyFramesDevice(packs[0], mp1_t, kfs, N_CAMS, cap, n_points, bad_t)
        for _ in range(5):
            m.SearchByBoWKeyFramesDevice(packs[0], mp1_t, kfs, N_CAMS, cap, n_points, bad_t, out=out)
        torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            m.SearchByBoWKeyFramesDevice(packs[0], mp1_t, kfs, N_CAMS, cap, n_points, bad_t, out=out)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        d = [t.cpu().numpy() for t in out]
        hts = []
        for _ in range(3):
            t0 = time.perf_counter()
            h = m.SearchByBoWKeyFramesHost(packs[0], mp1_t, kfs, N_CAMS, cap, n_points, bad_t)
            hts.append((time.perf_counter() - t0) * 1e3)
        same = all(np.array_equal(a, b) for a, b in zip(d, h))
        line = (f"candidates {n_kf:3d}: device {statistics.median(times):.3f} ms (CUDA-event median of {args.reps}), host route "
                f"{statistics.median(hts):.1f} ms (wall, median of 3), matches per candidate {int(np.median(d[2]))}, identical {same}")
        if rm is not None:
            table = rm.MPTable(3, np.zeros((n_points, 32), np.uint8), bad=bad)
            from multicol_slam_b200 import synth
            cams = [dict(synth.lafida_cams()[0], width=W, height=H)] * N_CAMS
            k1 = rm.KF(KF1, cams, mp=mp1)
            t0 = time.perf_counter()
            ref = [rm.search_by_bow_kfkf(k1, rm.KF(cands[k], cams, mp=mps[k]), table, 0.9, True) for k in range(n_kf)]
            rt = (time.perf_counter() - t0) * 1e3
            rsame = all(r[0] == d[2][k] and np.array_equal(r[1], api.slots_to_contiguous(d[0][k], counts, cap)) for k, r in enumerate(ref))
            line += f", reference {rt:.1f} ms (wall, one pass, key-frame set-up included), identical {rsame}"
        else:
            line += ", reference: not run (oracle/_ref absent)"
        print(line, flush=True)
        if not same:
            raise SystemExit("the device call and the host route differ")


if __name__ == "__main__":
    main()
