"""GPU: loop closing's device Sim3 searches, cORBmatcher.SearchBySim3Device (mcs_search_by_sim3_device) and
cORBmatcher.SearchByProjectionKFScwDevice (mcs_search_by_projection_scw_device), against the host mirrors on the CUDA window search,
the mirrors on the oracle's window search and the reference's own methods (oracle/_ref, where it travelled).  Key frames come from
packed feature buffers, alone in a buffer with decoys around or as one-image parts of an allgather-style buffer.  Everything compared
is integer: bit for bit."""
import numpy as np
import pytest

from device_frames import BIG_ID, GUARD, SIZES, counts, flip_bits, frames, from_slots, on_device, pack_frames, rm, to_slots, widen, widener  # noqa: F401
from device_searches import dev_map, device_scw
from search_scenes import host_scw, host_sim3, make_scene, reference_scw, reference_sim3, scw_scene, sim3_scene

pytestmark = pytest.mark.gpu


def _sim3_at(api, s, dim):
    if dim == 32:
        return s
    w = widener(dim)
    return dict(s, KF1=widen(api, s["KF1"], dim), KF2=widen(api, s["KF2"], dim), desc=w(s["desc"]), dmask=w(s["dmask"]))


def _scw_at(api, s, dim):
    if dim == 32:
        return s
    w = widener(dim)
    return dict(s, KF=widen(api, s["KF"], dim), desc=w(s["desc"]), dmask=w(s["dmask"]))


def device_sim3(api, m, s, cap, layout, th=7.5, already2=True, pre=None, mp1=None, mp2=None, stream=None):
    """SearchBySim3Device on the scene -> (nfound, status, matches12 in KF1's contiguous order)"""
    import torch
    KF1, KF2 = s["KF1"], s["KF2"]
    if KF1 is KF2 and layout == "same":
        kf1 = kf2 = pack_frames([KF1], cap, layout="single")[0]
    else:
        kf1, kf2 = pack_frames([KF1, KF2], cap, layout="parts" if layout == "same" else layout)
    pre = s["pre"] if pre is None else pre
    a2 = np.zeros(len(KF2.keys), np.uint8)
    for i in np.flatnonzero(pre >= 0):
        j = int(s["obs_idx"][pre[i]]) if pre[i] < len(s["obs_idx"]) else -1
        if 0 <= j < len(KF2.keys):
            a2[j] = 1
    dm = dev_map(s, bad=s["bad"])
    m12_t = to_slots(api, KF1, pre, cap, GUARD)
    masks_t = on_device(np.stack(s["rig1"].masks))
    n, st, out = m.SearchBySim3Device(kf1, kf2, cap, s["rig1"], s["rig2"], masks_t, KF1.scale_factors,
                                      to_slots(api, KF1, s["mp1"] if mp1 is None else mp1, cap, BIG_ID),
                                      to_slots(api, KF2, s["mp2"] if mp2 is None else mp2, cap, BIG_ID), dm["world_t"], dm["min_t"], dm["max_t"],
                                      dm["desc_t"], dm["dmask_t"], s["s12"], s["R12"], s["t12"], th, m12_t,
                                      already2_t=to_slots(api, KF2, a2, cap, 1, dtype=np.uint8) if already2 else None,
                                      bad_t=dm["bad_t"], stream=stream)
    torch.cuda.synchronize()
    return int(n.item()), int(st.item()), from_slots(api, out, counts(KF1), cap, GUARD)


# ---- SearchBySim3 ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["single", "parts"])
@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masks", [False, True])
def test_sim3_parity(api, oa, rm, frames, cams, masks, dim, layout):
    """device == mirror on the CUDA window search == the reference (or the mirror on the oracle's window search)"""
    s = _sim3_at(api, sim3_scene(api, oa, cams, frames[0]), dim)
    m = api.cORBmatcher(0.6, False, dim, masks)
    hn, h12 = host_sim3(m, s, 7.5)
    cap = max(counts(s["KF1"])) + 5
    dn, st, d12 = device_sim3(api, m, s, cap, layout)
    assert st == api.MCS_OK and dn == hn and np.array_equal(d12, h12) and dn > 30
    if rm and dim == 32:
        rn, r12 = reference_sim3(rm, cams, s, 7.5, masks)
    else:
        rn, r12 = host_sim3(m, s, 7.5, _sw=oa.search_windows)
    assert rn == dn and np.array_equal(r12, d12)
    if dim == 32 and layout == "single":                               # th = 10, as loop closing calls it (ref src/cLoopClosing.cpp:343)
        hn, h12 = host_sim3(m, s, 10.0)
        dn10, st, d12_10 = device_sim3(api, m, s, cap, layout, th=10.0)
        rn, r12 = reference_sim3(rm, cams, s, 10.0, masks) if rm else host_sim3(m, s, 10.0, _sw=oa.search_windows)
        assert st == api.MCS_OK and dn10 == hn == rn and np.array_equal(d12_10, h12) and np.array_equal(r12, h12)
    # vbAlreadyMatched2 matters: without it the device finds other agreements
    an, _, a12 = device_sim3(api, m, s, cap, layout, already2=False)
    hn2, h2 = m.SearchBySim3(s["KF1"], s["rig1"], s["mp1"], s["KF2"], s["rig2"], s["mp2"], s["world"], s["min_d"], s["max_d"], s["bad"],
                             s["desc"], s["dmask"], s["s12"], s["R12"], s["t12"], 7.5, matches12=s["pre"], obs_idx2=None)
    assert an == hn2 and np.array_equal(a12, h2) and not np.array_equal(a12, d12)


def test_sim3_same_key_frame_in_one_buffer(api, oa, frames, cams):
    """KF1 == KF2, one packed frame for both"""
    s = sim3_scene(api, oa, cams, frames[0])
    s = dict(s, KF2=s["KF1"])
    m = api.cORBmatcher(0.6, False, 32, True)
    hn, h12 = host_sim3(m, s, 7.5)
    dn, st, d12 = device_sim3(api, m, s, max(counts(s["KF1"])) + 1, "same")
    assert st == api.MCS_OK and dn == hn > 30 and np.array_equal(d12, h12)


def test_sim3_invalid_ids_and_edges(api, oa, frames, cams):
    """an id >= n_points in mp1, mp2 or matches12 drops that slot and raises MCS_ERR_INVALID; the rest equals the mirror without
    those slots.  Counts at capacity, and a busy stream."""
    import torch
    s = sim3_scene(api, oa, cams, frames[0])
    m = api.cORBmatcher(0.6, False, 32, False)
    n_pts = len(s["world"])
    cap = max(counts(s["KF1"]))                                        # the fullest camera exactly at capacity
    for which in ("mp1", "mp2", "pre"):
        row = (s["pre"] if which == "pre" else s[which]).copy()
        k = int(np.flatnonzero(s["mp1"] >= 0)[3]) if which != "mp2" else int(np.flatnonzero(s["mp2"] >= 0)[5])
        row[k] = n_pts + 4
        kw = {which: row}
        dn, st, d12 = device_sim3(api, m, s, cap, "single", **kw)
        assert st == api.MCS_ERR_INVALID, which
        clean = row.copy()
        clean[k] = -1
        if which == "pre":                # a dropped matches12 entry is no query and is left as it was
            hn, h12 = host_sim3(m, dict(s, mp1=np.where(np.arange(len(row)) == k, -1, s["mp1"])), 7.5, pre=clean)
            h12[k] = row[k]
        else:
            hn, h12 = host_sim3(m, dict(s, **{which: clean}), 7.5)
        assert dn == hn and np.array_equal(d12, h12), which
    # an invalid matches12 entry at a slot that carries no map point raises status too, and is left as it was
    row = s["pre"].copy()
    k = int(np.flatnonzero(s["mp1"] < 0)[2])
    row[k] = n_pts + 4
    dn, st, d12 = device_sim3(api, m, s, cap, "single", pre=row)
    hn, h12 = host_sim3(m, s, 7.5)
    h12[k] = row[k]
    assert st == api.MCS_ERR_INVALID and dn == hn and np.array_equal(d12, h12)
    # a busy stream: the call waits for the work queued before it
    st_ = torch.cuda.Stream()
    with torch.cuda.stream(st_):
        big = torch.randn(4096, 4096, device="cuda")
        for _ in range(8):
            big = big @ big
            big /= big.norm()
        dn, st, d12 = device_sim3(api, m, s, cap, "parts", stream=st_)
    hn, h12 = host_sim3(m, s, 7.5)
    assert st == api.MCS_OK and dn == hn and np.array_equal(d12, h12)


def _dist1(api, s, i1):
    """|p4| of KF1 keypoint i1's point in direction 1, in the mirror's (and the reference's) arithmetic"""
    p, cam = int(s["mp1"][i1]), int(s["KF1"].key_cam[i1])
    T1 = api.inv_rigid(s["rig1"].M_t)
    sR21 = (1.0 / s["s12"]) * s["R12"].T.copy()
    t21 = api._mm(-sR21, s["t12"])
    pa = api._mm(T1[:3, :3], s["world"][p]) + T1[:3, 3]
    pb = api._mm(sR21, pa) + t21
    p4 = api._mm(api.inv_rigid(s["rig2"].M_c[cam]), np.append(pb, 1.0))
    return float(np.sqrt(p4[0] * p4[0] + p4[1] * p4[1] + p4[2] * p4[2]))


def distance_edge_scenes(api, s, n=12, _sw=None):
    """(kept, {kind: flipped}, {kind: edited KF1 keypoints}) for the direction-1 range and level edges of agreeing pairs: |p4| equal
    to min (flipped: min one ulp above it), equal to max (flipped: max one ulp below it), and d / min equal to scale factor
    octave + 1 (flipped: min one ulp lower, so the level is octave + 2 and the window's levels miss the keypoint)"""
    m = api.cORBmatcher(0.6, False, 32, False)
    _, h12 = host_sim3(m, s, 7.5, _sw=_sw)
    agree = [int(i) for i in np.flatnonzero((s["mp1"] >= 0) & (h12 == s["mp2"]) & (s["pre"] < 0))]
    sf = np.asarray(s["KF1"].scale_factors, np.float64)
    octs = s["KF2"].keys["octave"]
    lo, hi = s["min_d"].copy(), s["max_d"].copy()
    flips = {k: (s["min_d"].copy(), s["max_d"].copy()) for k in ("min", "max", "ratio")}
    edited = {k: [] for k in flips}
    for i1 in agree:
        p, d, o = int(s["mp1"][i1]), _dist1(api, s, i1), int(octs[i1])
        if o == 0 and len(edited["min"]) < n:                          # ratio 1: level 0, the window keeps octave 0
            lo[p] = d
            flips["min"][0][p] = np.nextafter(d, np.inf)
            kind = "min"
        elif len(edited["max"]) < n:
            hi[p] = d
            flips["max"][1][p] = np.nextafter(d, -np.inf)
            kind = "max"
        elif o <= 5 and len(edited["ratio"]) < n:
            mn = d / sf[o + 1]
            below = np.nextafter(mn, 0.0)
            if d / mn != sf[o + 1] or not d / below > sf[o + 1]:
                continue
            lo[p], hi[p] = mn, d * 2.0
            flips["ratio"][0][p], flips["ratio"][1][p] = below, d * 2.0
            kind = "ratio"
        else:
            continue
        edited[kind].append(i1)
    for k, (a, b) in flips.items():                                  # each flipped scene carries the other kinds' kept edits
        for other in flips:
            if other != k:
                for i1 in edited[other]:
                    p = int(s["mp1"][i1])
                    a[p], b[p] = lo[p], hi[p]
    return dict(s, min_d=lo, max_d=hi), {k: dict(s, min_d=a, max_d=b) for k, (a, b) in flips.items()}, edited


def z_edge_scene(api, oa, cams, F):
    """rig-frame z of direction 1 at 0 and one ulp either side.  Identity poses, R12 = I, t12 = 0, s12 = 2 (all exact), so
    p3Dc2 = X / 2.  Camera 0 has the rig's orientation and sits 10 cm behind its centre, so its frame's z is the rig's plus 0.1:
    every probe lies at camera-frame z = 0.1, in front of the camera, where a test of the camera frame's z would keep the -ulp probes
    too.  KF1 keypoint i of camera 0 gets X on its bearing ray with X.z set to the edge value; KF2 (the same keypoints) gets a point
    that projects back onto keypoint i at rig z 0.1, so a kept probe agrees.  Returns the scene and the probes' z class per keypoint
    (0: zero, 1: +ulp, 2: -ulp, -1: no probe)."""
    rays, _, _ = oa.frame_prepare(F.keys, F.key_cam, cams)
    M_c = make_scene(api, oa, cams, F, 61, npts=10)["M_c"].copy()
    M_c[0] = np.eye(4)
    M_c[0, 2, 3] = -0.1
    rig = api.Rig(cams, M_c, np.eye(4))
    rng = np.random.default_rng(62)
    n = len(F.keys)
    cam0 = np.flatnonzero((F.key_cam == 0) & (rays[:, 2] > 0.05))
    tiny = np.nextafter(0.0, 1.0)
    back = np.array([0.0, 0.0, 0.1])
    world, desc, depth = np.zeros((2 * n, 3)), np.zeros((2 * n, F.desc.shape[1]), np.uint8), np.ones(2 * n)
    mp1, mp2, zcls = np.full(n, -1, np.int32), np.full(n, -1, np.int32), np.full(n, -1)
    for k, i in enumerate(cam0):
        r = rays[i]
        lam, lam2 = 0.1 / r[2], 0.2 / r[2]
        x = 2.0 * (lam * r - back)
        x[2] = (0.0, 2 * tiny, -2 * tiny)[k % 3]                     # p3Dc2.z = X.z / 2: 0, +ulp, -ulp
        world[i], world[n + i] = x, (lam2 * r - back) / 2.0
        depth[i], depth[n + i] = lam, lam2
        desc[i], desc[n + i] = flip_bits(rng, F.desc[[i, i]], 4)
        mp1[i], mp2[i], zcls[i] = i, n + i, k % 3
    oct_ = np.concatenate([F.keys["octave"], F.keys["octave"]])
    min_d = depth / (1.1 * np.asarray(F.scale_factors)[oct_])
    s = dict(KF1=F, KF2=F, rig1=rig, rig2=rig, M_c=M_c, world=world, desc=desc, dmask=np.concatenate([F.dmask, F.dmask]),
             bad=np.zeros(2 * n, np.uint8), min_d=min_d, max_d=min_d * 12, mp1=mp1, mp2=mp2, s12=2.0, R12=np.eye(3), t12=np.zeros(3),
             pre=np.full(n, -1, np.int32), obs_idx=np.concatenate([np.arange(n), np.arange(n)]).astype(np.int32))
    return s, zcls


def test_sim3_distance_and_level_edges(api, oa, frames, cams):
    """|p4| on min and on max, and d / min equal to a scale factor, each kept; one ulp the other way drops every edited pair's
    agreement.  The device equals the mirror on the kept scene and on each flipped one."""
    s = sim3_scene(api, oa, cams, frames[0])
    m = api.cORBmatcher(0.6, False, 32, False)
    cap = max(counts(s["KF1"])) + 2
    kept, flipped, edited = distance_edge_scenes(api, s)
    assert all(len(v) >= 8 for v in edited.values()), {k: len(v) for k, v in edited.items()}
    hn, h12 = host_sim3(m, kept, 7.5)
    dn, st, d12 = device_sim3(api, m, kept, cap, "single")
    assert st == api.MCS_OK and dn == hn and np.array_equal(d12, h12)
    for kind, i1s in edited.items():
        assert all(d12[i] == s["mp2"][i] for i in i1s), kind           # kept: the edited pairs still agree
        fn, f12 = host_sim3(m, flipped[kind], 7.5)
        gn, st, g12 = device_sim3(api, m, flipped[kind], cap, "parts")
        assert st == api.MCS_OK and gn == fn and np.array_equal(g12, f12), kind
        assert all(g12[i] != s["mp2"][i] for i in i1s), kind           # flipped: every edited pair lost its agreement


def test_sim3_rig_frame_z_edge(api, oa, frames, cams):
    """p3Dc2.z = 0 and +ulp keep the probe and -ulp drops it, although every probe's camera-frame z is 0.1 (in front)"""
    s, zcls = z_edge_scene(api, oa, cams, frames[0])
    m = api.cORBmatcher(0.6, False, 32, False)
    for i in np.flatnonzero(zcls >= 0):                               # the camera frame's z, as the reference computes p4
        p4 = api._mm(api.inv_rigid(s["M_c"][0]), np.append(s["world"][i] / 2.0, 1.0))
        assert 0.1 - 1e-12 < p4[2] < 0.1 + 1e-12
    hn, h12 = host_sim3(m, s, 7.5)
    dn, st, d12 = device_sim3(api, m, s, max(counts(s["KF1"])) + 1, "single")
    assert st == api.MCS_OK and dn == hn and np.array_equal(d12, h12)
    agree = d12 == s["mp2"]
    assert (agree & (zcls == 0)).sum() >= 10 and (agree & (zcls == 1)).sum() >= 10
    assert not (agree & (zcls == 2)).any()


# ---- SearchByProjection(KF, Scw) ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["single", "parts"])
@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masks", [False, True])
def test_scw_parity(api, oa, rm, frames, cams, masks, dim, layout):
    """the scene of the CPU tape (camera 0 alone, where the reference's reads are defined): device == mirror == reference"""
    s = _scw_at(api, scw_scene(api, oa, cams, frames[0]), dim)
    m = api.cORBmatcher(0.6, False, dim, masks)
    hn, hm = host_scw(m, s)
    cap = max(counts(s["KF"])) + 3
    dn, st, dmatched, diag = device_scw(api, m, s, cap, layout)
    assert st == api.MCS_OK and dn == hn > 50 and np.array_equal(dmatched, hm)
    if rm and dim == 32:
        rn, rmatched = reference_scw(rm, cams, s, masks)
    else:
        rn, rmatched = host_scw(m, s, _sw=oa.search_windows)
    assert rn == dn and np.array_equal(rmatched, dmatched)


def scw_model(api, oa, m, s, rows=True, drop=True, zero="contiguous", points=None, matched=None, th=10):
    """a plain-Python SearchByProjection(KF, Scw) with each quirk switchable: rows (descriptor row first(c) + contiguous id), drop
    (candidates whose row is missing are left out; otherwise they are compared through their own descriptor), zero ("contiguous":
    contiguous keypoint 0 is never accepted, "slot0": the first keypoint of camera 0 instead, None: no such rule)"""
    KF = s["KF"]
    pts = s["points"] if points is None else points
    out = (s["matched"] if matched is None else matched).copy()
    found = set(int(x) for x in out if x >= 0)
    n_cam = counts(KF)
    first = np.concatenate([[0], np.cumsum(n_cam)])
    rig = api._sim3_rig(s["rig"], s["Scw"])
    sf = np.asarray(KF.scale_factors)
    dist = (lambda a, b, ma, mb: api.DescriptorDistance64Masked(a, b, ma, mb, KF.desc.shape[1])) if m.havingMasks else \
        (lambda a, b, ma, mb: api.DescriptorDistance64(a, b, KF.desc.shape[1]))
    ents, qs = [], []
    for i, p in enumerate(pts):
        p = int(p)
        if p < 0 or s["bad"][p] or p in found or i >= len(KF.keys):
            continue
        c = int(KF.key_cam[i])
        uv, ok, lvl = api._project(rig, sf, s["world"], s["min_d"], s["max_d"], [p], np.array([[c]]), False)
        if ok[0, 0]:
            l = int(lvl[0, 0])
            ents.append((p, c))
            qs.append(api._queries(np.array([c]), uv[:, 0, 0], uv[:, 0, 1], float(th) * sf[l], l - 1, l, np.array([p])))
    if not qs:
        return 0, out
    cand, _, cnt, _ = oa.window_search(KF, np.concatenate(qs), s["desc"], s["dmask"], max_cand=4096)
    n = 0
    for k, (p, c) in enumerate(ents):
        best, bi = 2**31 - 1, -1
        for idx in cand[k, :cnt[k]]:
            idx = int(idx)
            if out[idx] >= 0:
                continue
            r = first[c] + idx if rows else idx
            if rows and r >= first[c + 1]:
                if drop:
                    continue
                r = idx
            d = dist(s["desc"][p], KF.desc[r], s["dmask"][p], KF.dmask[r])
            if d < best:
                best, bi = d, idx
        z = {"contiguous": 0, "slot0": 0 if n_cam[0] else -1, None: -1}[zero]
        if best <= m.TH_LOW_ and bi >= 0 and bi != z:
            out[bi] = p
            n += 1
    return n, out


def quirk_scene(api, oa, cams, F, empty_cam0=False, seed=71):
    """all three cameras; entry i of vpPoints is a point on keypoint i's own ray (so that the camera the reference looks up with the
    entry's position is the point's camera), with keypoint i's descriptor a few bits off; entry 0 sits on keypoint 0 exactly"""
    if empty_cam0:
        sel = np.flatnonzero(F.key_cam != 0)
        F = api.Frame(F.keys[sel], F.key_cam[sel], F.desc[sel], F.dmask[sel], SIZES, F.scale_factors)
    s = scw_scene(api, oa, cams, F, seed=seed, cam0_only=False, scale=1.0)
    KF, sc = s["KF"], s["sc"]
    rays, _, _ = oa.frame_prepare(KF.keys, KF.key_cam, cams)
    n = len(KF.keys)
    rng = np.random.default_rng(seed)
    depth = rng.uniform(2.0, 5.0, n)
    world = np.stack([api._mm(sc["rig"].MtMc[int(KF.key_cam[k])], np.append(rays[k] * depth[k], 1.0))[:3] for k in range(n)])
    desc = flip_bits(rng, KF.desc, 6)
    desc[0] = KF.desc[0]
    oct_ = KF.keys["octave"]
    min_d = depth / (1.1 * np.asarray(KF.scale_factors)[oct_])        # level octave + 1: the window keeps the octave
    pts = np.where(rng.random(n) < 0.9, np.arange(n), -1).astype(np.int32)
    pts[0] = 0
    matched = np.full(n, -1, np.int32)
    return dict(s, world=world, desc=desc, dmask=KF.dmask.copy(), bad=np.zeros(n, np.uint8), min_d=min_d, max_d=min_d * 10, points=pts,
                matched=matched)


@pytest.mark.parametrize("masks", [False, True])
def test_scw_quirks_each_matter(api, oa, frames, cams, masks):
    """on all three cameras: contiguous keypoint 0 is entry 0's best and is refused; candidates of cameras > 0 are compared through
    row first(c) + id and dropped where that row is missing; with camera 0 empty, contiguous 0 lies in camera 1.  The device equals
    the mirror and the model with every quirk; the model with any one quirk ignored gives another result"""
    m = api.cORBmatcher(0.6, False, 32, masks)
    for empty in (False, True):
        s = quirk_scene(api, oa, cams, frames[0], empty_cam0=empty)
        cap = max(counts(s["KF"])) + 2
        hn, hm = host_scw(m, s)
        mn, mm = scw_model(api, oa, m, s)
        dn, st, dmatched, _ = device_scw(api, m, s, cap, "single")
        assert st == api.MCS_OK and dn == hn == mn and np.array_equal(dmatched, hm) and np.array_equal(mm, hm) and dn > 20, empty
        assert hm[0] == -1
        for kw in (dict(rows=False), dict(drop=False), dict(zero=None)) + ((dict(zero="slot0"),) if empty else ()):
            _, alt = scw_model(api, oa, m, s, **kw)
            assert not np.array_equal(alt, hm), (empty, kw)


def test_scw_entries_past_the_keypoints(api, oa, frames, cams):
    """entries at or beyond the key frame's keypoint count raise MCS_ERR_INVALID and are dropped; the rest equals the mirror on the
    truncated list"""
    s = scw_scene(api, oa, cams, frames[0])
    m = api.cORBmatcher(0.6, False, 32, True)
    n_keys = len(s["KF"].keys)
    extra = np.concatenate([s["points"], np.full(n_keys - len(s["points"]), -1, np.int32), np.arange(20, dtype=np.int32)])
    dn, st, dmatched, diag = device_scw(api, m, s, max(counts(s["KF"])) + 1, "parts", points=extra)
    hn, hm = host_scw(m, s)
    assert st == api.MCS_ERR_INVALID and dn == hn and np.array_equal(dmatched, hm)
    # NULL, bad or already found entries past the count never reach the camera look-up: no status
    tail = np.concatenate([s["points"], np.full(n_keys - len(s["points"]) + 5, -1, np.int32)])
    dn, st, dmatched, _ = device_scw(api, m, s, max(counts(s["KF"])) + 1, "parts", points=tail)
    assert st == api.MCS_OK and dn == hn and np.array_equal(dmatched, hm)


def contention_scene(api, oa, cams, F, L=40):
    """camera 0's keypoints 1 .. L moved into one 6-pixel cluster at octave 0 with descriptors on a chain (keypoint k = a base with
    its first 3k bits flipped); entry i wants keypoint i (distance 1) and, once entry i - 1 took it, keypoint i + 1 (distance 2), so
    the fixpoint rounds settle one entry per round and the walk has to finish"""
    s = scw_scene(api, oa, cams, F, seed=91, cam0_only=True, scale=1.0)
    KF = s["KF"]
    keys, desc, dmask = KF.keys.copy(), KF.desc.copy(), np.full_like(KF.dmask, 0xFF)
    rng = np.random.default_rng(5)
    centre = (300.0, 200.0)
    base = desc[0].copy()
    bits = np.unpackbits(base)
    for k in range(1, L + 1):
        keys["x"][k], keys["y"][k] = centre[0] + rng.uniform(-3, 3), centre[1] + rng.uniform(-3, 3)
        keys["octave"][k] = 0
        b = bits.copy(); b[:3 * k] ^= 1
        desc[k] = np.packbits(b)
    KF = api.Frame(keys, KF.key_cam, desc, dmask, SIZES, KF.scale_factors)
    rays, _, _ = oa.frame_prepare(keys, KF.key_cam, cams)
    n = len(keys)
    world = np.zeros((n, 3)); qdesc = np.zeros_like(desc); min_d = np.ones(n); pts = np.full(n, -1, np.int32)
    for i in range(L):
        d = 3.0
        world[i] = api._mm(s["rig"].MtMc[0], np.append(rays[1] * d, 1.0))[:3]
        b = bits.copy(); b[:3 * i + 1] ^= 1                             # keypoint i (the base for i = 0) and one bit of the next step
        qdesc[i] = np.packbits(b)
        min_d[i] = d / 1.1                                               # ratio 1.1: level 1, candidates on levels {0, 1}
        pts[i] = i
    return dict(s, KF=KF, world=world, desc=qdesc, dmask=np.full_like(qdesc, 0xFF), bad=np.zeros(n, np.uint8), min_d=min_d,
                max_d=min_d * 10, points=pts, matched=np.full(n, -1, np.int32))


@pytest.mark.parametrize("masks", [False, True])
def test_scw_dense_contention(api, oa, frames, cams, masks):
    """many loop points on few keypoints: the rounds run to their cap, the walk finishes, and the result equals the sequential mirror"""
    s = contention_scene(api, oa, cams, frames[0])
    m = api.cORBmatcher(0.6, False, 32, masks)
    hn, hm = host_scw(m, s)
    dn, st, dmatched, diag = device_scw(api, m, s, max(counts(s["KF"])) + 1, "single")
    assert st == api.MCS_OK and dn == hn and np.array_equal(dmatched, hm) and hn >= 30
    assert diag[0] == api.lib().mcs_search_by_projection_max_rounds() and diag[1] >= 0 and diag[2] >= 30, diag


def test_scw_edges(api, oa, frames, cams):
    """invalid ids in vpPoints and vpMatched, an empty list, counts at capacity, a busy stream"""
    import torch
    s = scw_scene(api, oa, cams, frames[0])
    m = api.cORBmatcher(0.6, False, 32, False)
    n_pts = len(s["world"])
    cap = max(counts(s["KF"]))
    pts = s["points"].copy()
    pts[7] = n_pts + 3
    dn, st, dm_, _ = device_scw(api, m, s, cap, "single", points=pts)
    clean = pts.copy(); clean[7] = -1
    hn, hm = host_scw(m, s, points=clean)
    assert st == api.MCS_ERR_INVALID and dn == hn and np.array_equal(dm_, hm)
    # an id >= n_points in vpMatched: its keypoint is taken, no point is found, no status
    mt = s["matched"].copy()
    k = int(np.flatnonzero(mt < 0)[10])
    mt[k] = n_pts + 9
    dn, st, dm_, _ = device_scw(api, m, s, cap, "single", matched=mt)
    hn, hm = host_scw(m, s, matched=mt)
    assert st == api.MCS_OK and dn == hn and np.array_equal(dm_, hm) and dm_[k] == n_pts + 9
    dn, st, dm_, diag = device_scw(api, m, s, cap, "parts", points=np.zeros(0, np.int32))
    assert st == api.MCS_OK and dn == 0 and np.array_equal(dm_, s["matched"]) and diag[2] == 0
    st_ = torch.cuda.Stream()
    with torch.cuda.stream(st_):
        big = torch.randn(4096, 4096, device="cuda")
        for _ in range(8):
            big = big @ big
            big /= big.norm()
        dn, st, dm_, _ = device_scw(api, m, s, cap, "parts", stream=st_)
    hn, hm = host_scw(m, s)
    assert st == api.MCS_OK and dn == hn and np.array_equal(dm_, hm)
