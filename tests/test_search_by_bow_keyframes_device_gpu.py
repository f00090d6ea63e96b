"""GPU: loop closing's device SearchByBoW(KF1, KF_k) for many candidates, cORBmatcher.SearchByBoWKeyFramesDevice
(mcs_search_by_bow_keyframes_device), against the host route (SearchByBoWKeyFramesHost on the library's brute-force matcher), the
same route on the oracle's matcher and the reference's own SearchByBoW(KF1, KF2) (oracle/_ref where it travelled).  Everything compared
is integer: bit for bit, matches12, match_slot, nmatches and status."""
import numpy as np
import pytest

from device_frames import BIG_ID, GUARD, SIZES, counts, frames, from_slots, on_device, pack_frames, rm, to_slots  # noqa: F401  (frames, rm: fixtures)
from search_scenes import bow_kf_scene, host_bow_kf, host_sim3, max_count, reference_bow_kf, sim3_scene

pytestmark = pytest.mark.gpu


def device_route(api, m, s, cap, layout="single", cands=None, stream=None, bad=True, mp1=None, mps=None, guard=True):
    """SearchByBoWKeyFramesDevice on the scene -> (matches12, match_slot, nmatches, status) as numpy, after checking that no slot at
    or beyond a KF1 camera's count was written"""
    import torch
    idx = list(range(len(s["cands"]))) if cands is None else cands
    mps = s["mps"] if mps is None else mps
    packs = pack_frames([s["KF1"]] + [s["cands"][k] for k in idx], cap, layout=layout)
    kfs = [(packs[1 + i], to_slots(api, s["cands"][k], mps[k], cap, BIG_ID)) for i, k in enumerate(idx)]
    nc, ns = len(s["KF1"].cam_w), len(s["KF1"].cam_w) * cap
    out = None
    if guard:
        out = (torch.full((len(idx), ns), GUARD, dtype=torch.int32, device="cuda"), torch.full((len(idx), ns), GUARD, dtype=torch.int32, device="cuda"),
               torch.full((len(idx),), GUARD, dtype=torch.int32, device="cuda"), torch.full((1,), GUARD, dtype=torch.int32, device="cuda"))
    bad_t = on_device(s["bad"]) if bad else None
    r = m.SearchByBoWKeyFramesDevice(packs[0], to_slots(api, s["KF1"], s["mp1"] if mp1 is None else mp1, cap, BIG_ID), kfs, nc, cap,
                                     s["n_points"], bad_t, stream=stream, out=out)
    torch.cuda.synchronize()
    m12, sl, nm, st = (t.cpu().numpy() for t in r)
    cc = counts(s["KF1"])

    def live(rows):
        """-1 at and beyond each count, after checking those slots still hold GUARD"""
        back = [from_slots(api, row, cc, cap, GUARD) if guard else api.slots_to_contiguous(row, cc, cap) for row in rows]
        return np.array([api.contiguous_to_slots(b, cc, cap) for b in back], np.int32).reshape(rows.shape)
    return live(m12), live(sl), nm, st


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("layout", ["single", "parts", "joint"])
@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masks", [False, True])
def test_parity(api, oa, rm, frames, cams, masks, dim, layout):
    """device == host route == oracle route (== the reference at 32 bytes); KF1 is also one of its own candidates"""
    s = bow_kf_scene(api, frames, 4, dim=dim)
    s["cands"].append(s["KF1"]); s["mps"].append(s["mp1"])
    m = api.cORBmatcher(0.75, False, dim, masks)
    cap = max_count(s) + 3
    d = device_route(api, m, s, cap, layout)
    h = host_bow_kf(api, m, s, cap, layout, "cuda")
    o = host_bow_kf(api, m, s, cap, _bf=oa.match_bruteforce)
    assert _same(d, h) and _same(d, o) and d[3][0] == api.MCS_OK and (d[2] > 20).all()
    # match_slot names a candidate slot holding the id in matches12
    for k, F in enumerate(s["cands"]):
        row = to_slots(api, F, s["mps"][k], cap, BIG_ID, "cpu").numpy()
        hit = d[1][k] >= 0
        assert np.array_equal(row[d[1][k][hit]], d[0][k][hit])
    if rm and dim == 32:
        for k in range(len(s["cands"])):
            rn, rout = reference_bow_kf(rm, cams, s, k, 0.75, masks)
            assert rn == d[2][k] and np.array_equal(rout, api.slots_to_contiguous(d[0][k], counts(s["KF1"]), cap))


def test_batch_equals_single_calls(api, frames):
    """16 candidates in one call == 16 calls with one candidate each"""
    s = bow_kf_scene(api, frames, 16, seed=9)
    m = api.cORBmatcher(0.75, False, 32, True)
    cap = max_count(s) + 1
    d = device_route(api, m, s, cap, "parts")
    for k in range(16):
        one = device_route(api, m, s, cap, "single", cands=[k])
        assert all(np.array_equal(a[k], b[0]) for a, b in zip(d[:3], one[:3])), k
    assert _same(d, host_bow_kf(api, m, s, cap, "parts", "cuda"))


def _frame(api, per_cam_desc, dim):
    """a Frame from per-camera descriptor rows: keypoints on a diagonal, masks all ones"""
    keys, cam, desc = [], [], []
    for c, d in enumerate(per_cam_desc):
        k = np.zeros(len(d), api.KEYPOINT_DTYPE)
        k["x"] = np.arange(len(d)) % 700 + 10; k["y"] = np.arange(len(d)) // 700 + 10
        keys.append(k); cam += [c] * len(d); desc.append(np.asarray(d, np.uint8).reshape(-1, dim))
    D = np.concatenate(desc)
    return api.Frame(np.concatenate(keys), np.asarray(cam, np.int32), D, np.full_like(D, 0xFF), SIZES, [1.2 ** i for i in range(8)])


def _flip(base, bits):
    d = base.copy()
    for b in bits:
        d[b // 8] ^= 1 << (b % 8)
    return d


def _contention_scene(api, n_kf, rng):
    """KF1: 20 identical queries A per camera 0 among random rows; candidate k: 12 entries A with 1, 2, .., 12 bits flipped (camera
    1), random rows elsewhere.  With nnratio 0.9 the first eight queries take the entries at distances 1 .. 8 (k < 0.9 (k + 1) for
    k <= 8); their K = 8 lists hold exactly those eight entries, so from the eighth query on every list is used up (at most one
    unmatched entry, and its distance dK < th_low): each of those queries is decided by an exact rescan, and query 8's acceptance of
    the entry at distance 8 rests on the rescan finding the one at distance 9 as its second."""
    A = rng.integers(0, 256, 32, dtype=np.uint8)
    q = [np.concatenate([rng.integers(0, 256, (15, 32), dtype=np.uint8), np.tile(A, (20, 1)), rng.integers(0, 256, (10, 32), dtype=np.uint8)]),
         rng.integers(0, 256, (30, 32), dtype=np.uint8), rng.integers(0, 256, (25, 32), dtype=np.uint8)]
    KF1 = _frame(api, q, 32)
    cands, mps, off = [], [], len(KF1.keys)
    for k in range(n_kf):
        bits = rng.permutation(256)
        cl = np.stack([_flip(A, bits[:i + 1]) for i in range(12)])[rng.permutation(12)]        # cluster order shuffled
        F = _frame(api, [rng.integers(0, 256, (20, 32), dtype=np.uint8), np.concatenate([rng.integers(0, 256, (7, 32), dtype=np.uint8), cl]),
                         rng.integers(0, 256, (18, 32), dtype=np.uint8)], 32)
        cands.append(F)
        mps.append((off + np.arange(len(F.keys))).astype(np.int32))
        off += len(F.keys)
    mp1 = np.arange(len(KF1.keys), dtype=np.int32)
    return dict(KF1=KF1, mp1=mp1, cands=cands, mps=mps, bad=np.zeros(off, np.uint8), n_points=off), A


def test_contention_rescans(api, oa):
    """clusters of near-identical descriptors across candidates, where the lists run out and the walk rescans (proof in
    _contention_scene): device == host route == oracle route, and the match that needs the rescan is there"""
    rng = np.random.default_rng(17)
    s, A = _contention_scene(api, 5, rng)
    m = api.cORBmatcher(0.9, False, 32, False)
    cap = 48
    d = device_route(api, m, s, cap)
    assert _same(d, host_bow_kf(api, m, s, cap, "single", "cuda")) and _same(d, host_bow_kf(api, m, s, cap, _bf=oa.match_bruteforce))
    for k, F in enumerate(s["cands"]):
        row = api.slots_to_contiguous(d[1][k], counts(s["KF1"]), cap)[15:35]      # KF1's cluster queries (camera 0): candidate slots
        desc_of = dict(zip(api.slots_to_contiguous(np.arange(3 * cap, dtype=np.int32), counts(F), cap).tolist(), F.desc))
        assert [int(np.unpackbits(desc_of[int(j)] ^ A).sum()) for j in row if j >= 0] == list(range(1, 9)), k
        assert (row[:8] >= 0).all() and (row[8:] < 0).all()


@pytest.mark.parametrize("nnratio", [0.75, 1.5])
def test_decision_edges(api, oa, nnratio):
    """best == th_low - 1 (accepted) vs th_low (rejected), best == second, best exactly at nnratio * second (rejected) and just below
    (accepted), at nnratio 0.75.  Equal best distances split across camera boundaries: with nnratio <= 1 such a query is rejected
    whatever the order, so nnratio 1.5 (the reference takes any ratio) shows the tie-break: the first in slot order is the best, for
    the first query in camera 0's last slot, for the second, identical one in camera 1's slot 2."""
    rng = np.random.default_rng(3)
    m = api.cORBmatcher(nnratio, False, 32, False)
    th = m.TH_LOW_
    Q = [rng.integers(0, 256, 32, dtype=np.uint8) for _ in range(6)]
    far = lambda a: _flip(a, rng.permutation(256)[:2 * th])  # noqa: E731
    at = lambda a, n: _flip(a, rng.permutation(256)[:n])  # noqa: E731
    # candidate rows per camera: (query, distance) pairs, the far rows keep every test's second at or beyond 2 th_low
    c0 = [at(Q[0], th - 1), far(Q[0]), at(Q[1], th), far(Q[1]), at(Q[2], 5), at(Q[2], 5), at(Q[3], 6), at(Q[3], 8), at(Q[5], 3)]
    c1 = [at(Q[4], 5), at(Q[4], 8), at(Q[5], 3)]
    c2 = [at(Q[5], 3), at(Q[5], 7)]
    KF1 = _frame(api, [np.stack(Q[:3]), np.stack(Q[3:5]), np.stack([Q[5], Q[5]])], 32)
    K2 = _frame(api, [np.stack(c0), np.stack(c1), np.stack(c2)], 32)
    s = dict(KF1=KF1, mp1=np.arange(7, dtype=np.int32), cands=[K2, K2], mps=[np.arange(7, 21, dtype=np.int32)] * 2,
             bad=np.zeros(21, np.uint8), n_points=21)
    cap = 9                                                                       # camera 0 of the candidate at capacity
    d = device_route(api, m, s, cap)
    assert _same(d, host_bow_kf(api, m, s, cap, "single", "cuda")) and _same(d, host_bow_kf(api, m, s, cap, _bf=oa.match_bruteforce))
    row = api.slots_to_contiguous(d[1][0], counts(KF1), cap)
    if nnratio < 1:
        assert row.tolist() == [0, -1, -1, -1, cap, -1, -1] and d[2][0] == 2
    else:
        assert row.tolist() == [0, -1, 4, 6, cap, 8, cap + 2] and d[2][0] == 6
    assert d[3][0] == api.MCS_OK


def test_invalid_ids_bad_and_empty_camera(api, frames):
    """an id >= n_points in KF1's or a candidate's row drops that slot and raises MCS_ERR_INVALID, the rest equals the host route
    without it; bad points on both sides; bad_dev NULL; a candidate with an empty camera; counts at capacity; a busy stream"""
    import torch
    s = bow_kf_scene(api, frames, 3, seed=21)
    m = api.cORBmatcher(0.75, False, 32, True)
    cap = max_count(s)                                                       # the fullest camera at capacity
    assert s["bad"][s["mp1"][s["mp1"] >= 0]].any() and s["bad"][s["mps"][1][s["mps"][1] >= 0]].any()
    mp1, mps = s["mp1"].copy(), [r.copy() for r in s["mps"]]
    i1, i2 = int(np.flatnonzero(mp1 >= 0)[4]), int(np.flatnonzero(mps[1] >= 0)[9])
    mp1[i1], mps[1][i2] = s["n_points"] + 4, s["n_points"] + 7
    d = device_route(api, m, s, cap, mp1=mp1, mps=mps)
    h = host_bow_kf(api, m, dict(s, mp1=mp1, mps=mps), cap, "single", "cuda")
    assert d[3][0] == h[3][0] == api.MCS_ERR_INVALID and _same(d[:3], h[:3])
    clean1, cleans = mp1.copy(), [r.copy() for r in mps]
    clean1[i1], cleans[1][i2] = -1, -1
    assert _same(d[:3], host_bow_kf(api, m, dict(s, mp1=clean1, mps=cleans), cap, "single", "cuda")[:3])
    # bad_dev NULL is "no point is bad"
    d = device_route(api, m, s, cap, bad=False)
    assert d[3][0] == api.MCS_OK and _same(d, host_bow_kf(api, m, dict(s, bad=np.zeros_like(s["bad"])), cap, "single", "cuda"))
    # a candidate whose camera 1 holds no keypoint
    F = s["cands"][0]
    keep = F.key_cam != 1
    s2 = dict(s, cands=[api.Frame(F.keys[keep], F.key_cam[keep], F.desc[keep], F.dmask[keep], SIZES, F.scale_factors)] + s["cands"][1:],
              mps=[s["mps"][0][keep]] + s["mps"][1:])
    assert _same(device_route(api, m, s2, cap, "joint"), host_bow_kf(api, m, s2, cap, "joint", "cuda"))
    # a busy stream: the call waits for the work queued before it
    st_ = torch.cuda.Stream()
    with torch.cuda.stream(st_):
        big = torch.randn(4096, 4096, device="cuda")
        for _ in range(8):
            big = big @ big
            big /= big.norm()
        d = device_route(api, m, s, cap, "parts", stream=st_)
    assert _same(d, host_bow_kf(api, m, s, cap, "parts", "cuda"))


def test_feeds_search_by_sim3(api, oa, frames, cams):
    """ComputeSim3's first two steps on the device: a candidate's matches12_dev row goes as it is into mcs_search_by_sim3_device
    (every match an inlier), and gives what the host composition gives"""
    import torch
    s3 = sim3_scene(api, oa, cams, frames[0])
    m = api.cORBmatcher(0.75, False, 32, True)
    s = dict(KF1=s3["KF1"], mp1=s3["mp1"], cands=[s3["KF2"]], mps=[s3["mp2"]], bad=s3["bad"], n_points=len(s3["world"]))
    cap = max(counts(s3["KF1"])) + 2
    packs = pack_frames([s3["KF1"], s3["KF2"]], cap, layout="parts")
    mp1_t, mp2_t = to_slots(api, s3["KF1"], s3["mp1"], cap, BIG_ID), to_slots(api, s3["KF2"], s3["mp2"], cap, BIG_ID)
    bad_t = on_device(s3["bad"])
    m12_t, slot_t, nm_t, st_t = m.SearchByBoWKeyFramesDevice(packs[0], mp1_t, [(packs[1], mp2_t)], 3, cap, s["n_points"], bad_t)
    hm12, hslot, hnm, _ = host_bow_kf(api, m, s, cap, "parts", "cuda")
    assert np.array_equal(m12_t.cpu().numpy()[0], hm12[0]) and int(nm_t[0]) == hnm[0] > 30 and int(st_t[0]) == api.MCS_OK
    pre = api.slots_to_contiguous(hm12[0], counts(s3["KF1"]), cap)
    a2 = np.zeros(cap * 3, np.uint8)                                # vbAlreadyMatched2: the KF2 slots the BoW matches hold
    a2[hslot[0][hslot[0] >= 0]] = 1
    row = m12_t[0].clone()
    dn, dst, out = m.SearchBySim3Device(packs[0], packs[1], cap, s3["rig1"], s3["rig2"], on_device(np.stack(s3["rig1"].masks)),
                                        s3["KF1"].scale_factors, mp1_t, mp2_t, on_device(np.asarray(s3["world"], np.float64)),
                                        on_device(np.asarray(s3["min_d"], np.float64)), on_device(np.asarray(s3["max_d"], np.float64)),
                                        on_device(s3["desc"]), on_device(s3["dmask"]), s3["s12"], s3["R12"], s3["t12"], 10.0, row,
                                        already2_t=on_device(a2), bad_t=bad_t)
    torch.cuda.synchronize()
    hn, h12 = host_sim3(m, s3, 10.0, pre=pre)
    assert int(dst[0]) == api.MCS_OK and int(dn[0]) == hn and np.array_equal(api.slots_to_contiguous(out.cpu().numpy(), counts(s3["KF1"]), cap), h12)
