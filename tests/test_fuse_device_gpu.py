"""GPU: the device Fuse (mcs_fuse_device, cORBmatcher.FuseDevice) with its hits replayed by cORBmatcher.FuseReplay, against the
host Fuse on the same state and the reference's own Fuse (oracle/_ref, where it travelled; the oracle's window search otherwise).
Key frames come from packed feature buffers, alone in a buffer with decoys around or as one-image parts of an allgather-style
buffer.  Everything compared is integer: bit for bit."""
import numpy as np
import pytest

from device_frames import BIG_ID, GUARD, SIZES, counts, keep_cameras, on_device, pack_frames, to_slots, widen, widener
from device_frames import frames, rm  # noqa: F401  (fixtures)
from device_searches import dev_map, fuse_device, fuse_pose, fuse_replay, fuse_targets
from search_scenes import fuse_scene, host_fuse, reference_ops

pytestmark = pytest.mark.gpu


def _with_dim(api, KF, s, dim):
    """the key frame and scene at descriptor width dim: 16 = the first half of every row, 64 = the row and its complement"""
    if dim == 32:
        return KF, s
    w = widener(dim)
    return widen(api, KF, dim), dict(s, desc=w(s["desc"]), dmask=w(s["dmask"]))


@pytest.mark.parametrize("layout", ["single", "parts"])
@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("variant", [0, 1, 2])
def test_per_key_frame_parity(api, oa, rm, frames, cams, variant, masks, dim, layout, monkeypatch):
    """device hits + the shared replay == the host Fuse, and == the reference's own Fuse (the oracle's window search where the
    reference did not travel), at every width; variant 0's scene has occupied hits on which the epipolar check passes and fails"""
    KF0 = frames[0]
    s0 = fuse_scene(api, oa, cams, KF0, variant)
    KF, s = _with_dim(api, KF0, s0, dim)
    m = api.cORBmatcher(0.6, False, dim, masks)
    hn, hops, hmp = host_fuse(api, m, KF, s, variant)
    cap = max(counts(KF)) + 7
    hits, n, status, _ = fuse_device(api, m, [KF], [s["sc"]["rig"]], [None], s["points"], dev_map(s), cap, layout, variant, Scw=s["Scw"])
    assert status == api.MCS_OK and n == len(hits) > 50
    dn, dops, dmp = fuse_replay(m, KF, s, variant, hits, cap)
    assert dn == hn and np.array_equal(dops, hops) and np.array_equal(dmp, hmp)
    assert (hops[:, 0] == 0).sum() > 10 and (hops[:, 0] == 1).sum() > 10
    if rm:
        rn, rops = reference_ops(api, rm, cams, KF, s, variant, masks)
    else:
        rn, rops, _ = host_fuse(api, m, KF, s, variant, _sw=oa.search_windows)
    assert rn == dn and np.array_equal(rops, dops)
    if variant == 0:
        # the device route's replay rejected occupied hits on the epipolar check: with a check that always holds it fuses more
        monkeypatch.setattr(api, "check_epipolar", lambda *a: True)
        an, _, _ = fuse_replay(m, KF, s, variant, hits, cap)
        assert 10 < dn < an


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_batch_equals_separate_calls(api, oa, frames, cams, variant):
    """one call over 22 key frames, all one-image parts of one buffer, a third with their row as pre-filter == 22 single-key-frame
    calls on buffers of their own"""
    KF = frames[0]
    s = fuse_scene(api, oa, cams, KF, variant)
    m = api.cORBmatcher(0.6, False, 32, True)
    rigs = fuse_targets(api, cams, s["sc"], 22, 3)
    cap = max(counts(KF)) + 3
    dm = dev_map(s)
    mps = [None if k % 3 else to_slots(api, KF, s["kf_mp"], cap, BIG_ID) for k in range(22)]
    batch, n, status, _ = fuse_device(api, m, [KF] * 22, rigs, mps, s["points"], dm, cap, "parts", variant, Scw=s["Scw"])
    assert status == api.MCS_OK
    sep = []
    for k in range(22):
        h, _, st, _ = fuse_device(api, m, [KF], [rigs[k]], [mps[k]], s["points"], dm, cap, "single", variant, Scw=s["Scw"])
        assert st == api.MCS_OK
        h = h.copy()
        h[:, 0] = k
        sep.append(h)
    sep = np.concatenate(sep)
    assert n == len(sep) > 500 and np.array_equal(batch, sep)


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_prefilter_is_exact(api, oa, frames, cams, variant):
    """with the key frame's row and the bad flags on the device, the hits are a subset of those without, and replay to the same ops"""
    KF = frames[0]
    s = fuse_scene(api, oa, cams, KF, variant)
    # in_kf must follow the row (the caller's guarantee): every point a slot holds is in the key frame
    s["in_kf"] = s["in_kf"].copy()
    s["in_kf"][s["kf_mp"][s["kf_mp"] >= 0]] = True
    m = api.cORBmatcher(0.6, False, 32, False)
    cap = max(counts(KF)) + 3
    # map points held by the key frame among the queries too, so that the row filters some queries out
    extra = np.flatnonzero(s["kf_mp"] >= 0)[:40]
    s["points"] = np.concatenate([s["points"], s["kf_mp"][extra]]).astype(np.int32)
    full, _, st0, _ = fuse_device(api, m, [KF], [s["sc"]["rig"]], [None], s["points"], dev_map(s), cap, "single", variant, Scw=s["Scw"])
    filt, _, st1, _ = fuse_device(api, m, [KF], [s["sc"]["rig"]], [to_slots(api, KF, s["kf_mp"], cap, BIG_ID)], s["points"], dev_map(s, bad=s["bad"]),
                              cap, "single", variant, Scw=s["Scw"])
    assert st0 == st1 == api.MCS_OK and len(filt) < len(full)
    fs = set(map(tuple, full.tolist()))
    assert all(tuple(r) in fs for r in filt.tolist())
    a, b = fuse_replay(m, KF, s, variant, full, cap), fuse_replay(m, KF, s, variant, filt, cap)
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]) and len(a[1]) > 50


class _Map:
    """a small map model between Fuse calls: per target key frame its row and observed points; a Replace marks the point bad,
    moves its slots to the survivor (erasing a slot where the survivor is already present) and rewrites the survivor's
    descriptor (here: its complement, a deterministic stand-in for ComputeDistinctiveDescriptors that surely changes decisions)"""

    def __init__(self, bad, desc, rows):
        self.bad, self.desc = bad.copy(), desc.copy()
        self.rows = [r.copy() for r in rows]
        self.obs = [set(int(i) for i in r if i >= 0) for r in rows]
        self.rewritten = set()

    def in_kf(self, k):
        f = np.zeros(len(self.bad), bool)
        f[list(self.obs[k])] = True
        return f

    def apply(self, k, ops):
        for kind, i, x in ops.tolist():
            if kind == 0:
                self.rows[k][x] = i
                self.obs[k].add(i)
            else:
                self.bad[i] = 1
                for t, row in enumerate(self.rows):
                    held = np.flatnonzero(row == i)
                    if len(held):
                        row[held] = -1 if x in self.obs[t] else x
                        self.obs[t].discard(i)
                        self.obs[t].add(x)
                self.desc[x] = 255 - self.desc[x]
                self.rewritten.add(x)


def test_search_in_neighbors_sequence(api, oa, frames, cams):
    """SearchInNeighbors on a small map: the first pass Fuse(pKFi, curKF, .) over 6 target key frames from ONE device call,
    replayed key frame by key frame over the live map, then the candidate pass Fuse(curKF, candidates) -- the same mutations as
    the host route run key frame by key frame on the live state.  Queries become Replace survivors before later key frames: the
    replay searches them again, and without that the mutations would differ."""
    import torch
    KF = frames[0]
    s = fuse_scene(api, oa, cams, KF, 0)
    sc, n = s["sc"], s["n"]
    m = api.cORBmatcher(0.6, False, 32, True)
    cap = max(counts(KF)) + 3
    n_kf = 6
    rigs = [sc["rig"]] + fuse_targets(api, cams, sc, n_kf - 1, 8)
    # target 0's occupied slots hold query points (points it observes), so its Replace survivors are queries of the later targets
    rng = np.random.default_rng(4)
    rows0 = s["kf_mp"].copy()
    occ = np.flatnonzero(rows0 >= 0)
    rows0[occ[: len(occ) // 2]] = rng.choice(n, len(occ) // 2, replace=False)
    rows = [rows0] + [np.where(rng.random(len(KF.keys)) < 0.2, n + rng.integers(0, len(s["occupied"]), len(KF.keys)), -1).astype(np.int32)
                      for _ in range(n_kf - 1)]
    base = _Map(s["bad"], s["desc"], rows)

    def run(device, use_stale=True):
        mp = _Map(base.bad, base.desc, base.rows)
        ops_all, researched = [], 0
        if device:
            dm = dev_map(s, bad=mp.bad, desc=mp.desc)
            mps = [to_slots(api, KF, mp.rows[k], cap, BIG_ID) for k in range(n_kf)]
            hits, _, st, _ = fuse_device(api, m, [KF] * n_kf, rigs, mps, s["points"], dm, cap, "parts", 0)
            assert st == api.MCS_OK
        for k in range(n_kf):
            args = (KF, rigs[k], mp.rows[k], s["points"])
            tail = (s["world"], s["min_d"], s["max_d"], mp.bad, mp.in_kf(k), mp.desc, s["dmask"])
            kw = dict(th=2.5, variant=0, cur_rays=s["cur"]["rays"], kf_rays=sc["rays"], cur_rig=s["cur"]["rig"])
            if device:
                _, ops, _ = m.FuseReplay(*args, hits[hits[:, 0] == k][:, 1:], cap, *tail, stale=mp.rewritten if use_stale else (), **kw)
                researched += m.fuse_researched
            else:
                _, ops, _ = m.Fuse(*args, *tail, **kw)
            mp.apply(k, ops)
            ops_all.append(ops)
        # the candidate pass: the targets' non-bad points against the current key frame, after the first pass's bookkeeping
        cand = sorted(set(int(i) for r in mp.rows for i in r if i >= 0 and not mp.bad[i]))
        cand = np.asarray(cand, np.int32)
        # curKF as a frame: its keypoints in camera-major order (cMultiFrame's), keypoint j carrying point order[j]
        order = np.argsort(s["cur"]["key_cam"], kind="stable")
        src = sc["src"][order]
        Fc = api.Frame(KF.keys[src], KF.key_cam[src], KF.desc[src], KF.dmask[src], SIZES, KF.scale_factors)
        cur_row = s["points"][order].copy()
        cur_row[1::2] = -1                          # half of curKF's keypoints free: the candidates both replace and add
        cur_in = np.zeros(len(mp.bad), bool)
        cur_in[cur_row[cur_row >= 0]] = True
        if device:
            cc = max(counts(Fc)) + 3
            dm = dev_map(s, bad=mp.bad, desc=mp.desc)
            h2, _, st, _ = fuse_device(api, m, [Fc], [s["cur"]["rig"]], [to_slots(api, Fc, cur_row, cc, BIG_ID)], cand, dm, cc, "single", 1)
            assert st == api.MCS_OK
            _, ops, _ = m.FuseReplay(Fc, s["cur"]["rig"], cur_row, cand, h2[:, 1:], cc, s["world"], s["min_d"], s["max_d"], mp.bad, cur_in,
                                     mp.desc, s["dmask"], th=2.5, variant=1)
        else:
            _, ops, _ = m.Fuse(Fc, s["cur"]["rig"], cur_row, cand, s["world"], s["min_d"], s["max_d"], mp.bad, cur_in, mp.desc, s["dmask"],
                               th=2.5, variant=1)
        ops_all.append(ops)
        torch.cuda.synchronize()
        return ops_all, researched

    host, _ = run(False)
    dev, researched = run(True)
    assert len(host) == len(dev) and all(np.array_equal(a, b) for a, b in zip(host, dev))
    assert sum(len(o) for o in host) > 200 and len(host[-1]) > 0
    assert researched > 0
    stale_off, _ = run(True, use_stale=False)
    assert not all(np.array_equal(a, b) for a, b in zip(host, stale_off))


def test_capacity_and_edges(api, oa, frames, cams):
    import torch
    KF = frames[0]
    s = fuse_scene(api, oa, cams, KF, 2)
    m = api.cORBmatcher(0.6, False, 32, False)
    cap = max(counts(KF)) + 3
    dm = dev_map(s)
    rig = s["sc"]["rig"]
    full, n, st, _ = fuse_device(api, m, [KF], [rig], [None], s["points"], dm, cap, "single", 2, Scw=s["Scw"])
    assert st == api.MCS_OK and n > 100
    # max_hits below the total: the true total, the first rows, and nothing written past max_hits
    k = n // 3
    packed = pack_frames([KF], cap, layout="single")
    mi, ow = fuse_pose(rig, 2, s["Scw"])
    q_t = on_device(s["points"])
    masks_t = on_device(np.stack(rig.masks))
    out = (torch.full((k + 5, 3), GUARD, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"),
           torch.zeros(1, dtype=torch.int32, device="cuda"))
    m.FuseDevice([(packed[0], None, mi, ow)], q_t, cap, rig.cams, masks_t, KF.scale_factors, dm["world_t"], dm["min_t"], dm["max_t"], dm["desc_t"],
                 variant=2, th=2.5, max_hits=k, out=(out[0][:k], out[1], out[2]))
    torch.cuda.synchronize()
    h = out[0].cpu().numpy()
    assert int(out[2].item()) == api.MCS_ERR_CAPACITY and int(out[1].item()) == n
    assert np.array_equal(h[:k], full[:k]) and np.all(h[k:] == GUARD)
    # n_q = 0, every query NULL
    for pts in (np.zeros(0, np.int32), np.full(50, -1, np.int32)):
        h, n0, st0, _ = fuse_device(api, m, [KF], [rig], [None], pts, dm, cap, "single", 2, Scw=s["Scw"])
        assert st0 == api.MCS_OK and n0 == 0
    # ids >= n_points: MCS_ERR_INVALID, those queries dropped, the others' hits unchanged
    bad_ids = s["points"].copy()
    bad_ids[::50] = len(s["world"]) + 7
    h, nb, stb, _ = fuse_device(api, m, [KF], [rig], [None], bad_ids, dm, cap, "single", 2, Scw=s["Scw"])
    keep = full[full[:, 1] % 50 != 0]
    assert stb == api.MCS_ERR_INVALID and np.array_equal(h, keep)
    # counts at capacity: the key frame's fullest camera fills its slots exactly
    h, nc_, stc, _ = fuse_device(api, m, [KF], [rig], [None], s["points"], dm, max(counts(KF)), "parts", 2, Scw=s["Scw"])
    c_full = full.copy()
    c_full[:, 2] = (full[:, 2] // cap) * max(counts(KF)) + full[:, 2] % cap
    assert stc == api.MCS_OK and np.array_equal(h, c_full)
    # a camera without keypoints: its hits vanish, the other cameras' stay
    K2, _ = keep_cameras(api, KF, [0, 2])
    h, _, ste, _ = fuse_device(api, m, [K2], [rig], [None], s["points"], dm, cap, "single", 2, Scw=s["Scw"])
    assert ste == api.MCS_OK and np.array_equal(h, full[full[:, 2] // cap != 1])
    # a busy stream: the call queues behind the stream's work and returns the same hits
    st_ = torch.cuda.Stream()
    with torch.cuda.stream(st_):
        a = torch.randn(4096, 4096, device="cuda")
        for _ in range(20):
            a = a @ a
            a = a / a.norm()
        hb, nbz, stz, _ = fuse_device(api, m, [KF], [rig], [None], s["points"], dm, cap, "single", 2, Scw=s["Scw"], stream=st_)
    assert stz == api.MCS_OK and np.array_equal(hb, full)


# ---- projection edges: dist3D on and one ulp around the distance bounds, ratios on scale-factor ties ------------------------------
def _edge_scene(api, oa, cams, KF, variant):
    """fuse_scene with the distance bounds of its live points (not bad, not in the key frame) replaced by edge values.  dist3D is
    computed as the reference does (double norm, rounded to float for :1265 / :1420).  Per point, by its keypoint's octave o:
      o == 0:  min = dist3D (passes), min = the next value above it (fails: one float ulp for :1265 / :1420, one double ulp for
               :1570), min = dist3D in the OTHER precision (passes or fails by the rounding direction: a wrong precision flips it),
               or a ratio tie with scale factor 1 (level 1);
      o >= 1:  max = dist3D, max = the next value below it, max = dist3D in the other precision (min puts the level on o), or
               dist3D / min == scale_factors[o + 1] exactly: lower_bound gives o + 1, whose levels {o, o + 1} hold the keypoint,
               while an upper bound would give o + 2 and lose it.
    Returns the scene and the kinds."""
    s = fuse_scene(api, oa, cams, KF, variant)
    sc = s["sc"]
    rig = sc["rig"] if variant != 2 else api._sim3_rig(sc["rig"], s["Scw"])
    Ow = rig.M_t[:3, 3].copy()
    sf = np.asarray(KF.scale_factors, np.float64)
    min_d, max_d = s["min_d"].copy(), s["max_d"].copy()
    kinds = {}
    f32 = variant != 2
    for i in range(s["n"]):
        if s["bad"][i] or s["in_kf"][i]:
            continue
        po = s["world"][i] - Ow
        d = float(np.sqrt(po[0] * po[0] + po[1] * po[1] + po[2] * po[2]))
        dd = float(np.float32(d)) if f32 else d
        other = d if f32 else float(np.float32(d))
        up = float(np.nextafter(np.float32(dd), np.float32(np.inf))) if f32 else float(np.nextafter(d, np.inf))
        dn = float(np.nextafter(np.float32(dd), np.float32(-np.inf))) if f32 else float(np.nextafter(d, -np.inf))
        o = int(KF.keys["octave"][sc["src"][i]])
        kind = ("min_on", "min_up", "min_other", "tie")[i % 4] if o == 0 else ("max_on", "max_dn", "max_other", "tie", "tie")[i % 5]
        if kind == "tie" and o + 1 >= len(sf):
            kind = "max_on"
        if kind.startswith("min"):
            min_d[i], max_d[i] = {"min_on": dd, "min_up": up, "min_other": other}[kind], 2 * dd
        elif kind.startswith("max"):
            max_d[i] = {"max_on": dd, "max_dn": dn, "max_other": other}[kind]
            min_d[i] = dd / sf[o] * (1 + 1e-9) if o > 0 else dd
        else:
            lv = o + 1
            mn = dd / sf[lv]
            for _ in range(8):                           # the bound whose ratio is the scale factor exactly
                if dd / mn == sf[lv]:
                    break
                mn = float(np.nextafter(mn, np.inf if dd / mn > sf[lv] else -np.inf))
            if dd / mn != sf[lv]:
                continue
            min_d[i], max_d[i] = mn, 4 * dd
        kinds[i] = kind
    s["min_d"], s["max_d"] = min_d, max_d
    return s, kinds


def _host_hits(api, m, KF, s, variant, float_dist=None):
    """the host route's hits (q, camera, keypoint) of Fuse's queries: _project + FuseCandidates, after Fuse's skip tests"""
    sc = s["sc"]
    rig = sc["rig"] if variant != 2 else api._sim3_rig(sc["rig"], s["Scw"])
    pts = s["points"]
    if variant == 2:
        already = set(int(x) for x in s["kf_mp"] if x >= 0 and not s["bad"][x])
        qs = [q for q, i in enumerate(pts) if not s["bad"][i] and int(i) not in already]
    else:
        qs = [q for q, i in enumerate(pts) if i >= 0 and not s["bad"][i] and not s["in_kf"][i]]
    ids = pts[qs]
    nc = len(rig.cams)
    uv, ok, lvl = api._project(rig, KF.scale_factors, s["world"], s["min_d"], s["max_d"], ids, np.tile(np.arange(nc), (len(ids), 1)),
                               float_dist=(variant != 2) if float_dist is None else float_dist)
    best = m.FuseCandidates(KF, uv, ok, lvl, 2.5, s["desc"], None, first_wins=(variant == 1), points=ids)
    hits = [(qs[kk], c, int(best[kk, c])) for kk in range(len(qs)) for c in range(nc) if best[kk, c] >= 0]
    return hits, dict(zip(ids.tolist(), ok)), dict(zip(ids.tolist(), lvl)), set(qs)


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_projection_edges(api, oa, rm, frames, cams, variant, monkeypatch):
    """dist3D on and one ulp around min / max, in float for :1265 / :1420 and in double for :1570, and ratios on scale-factor ties:
    the device hits equal the host projection's (api._project) hit for hit, the replayed ops equal the host Fuse's and the
    reference's.  The scene decides both ways at every edge, and a projection in the other precision or an upper-bound level
    changes the host's hits, so either mistake on the device would show.  (The points lie on keypoint rays, not on constructed .5
    pixel ties, so DESIGN section 2's atan exception does not arise.)"""
    KF = frames[0]
    s, kinds = _edge_scene(api, oa, cams, KF, variant)
    m = api.cORBmatcher(0.6, False, 32, False)
    hh, ok, lvl, live = _host_hits(api, m, KF, s, variant)
    cam_of = {i: int(KF.key_cam[s["sc"]["src"][i]]) for i in kinds}
    passed = {k: [bool(ok[i][cam_of[i]]) for i, kk in kinds.items() if kk == k] for k in set(kinds.values())}
    assert all(passed["min_on"]) and all(passed["max_on"]) and all(passed["tie"]) and len(passed["tie"]) > 20
    assert not any(passed["min_up"]) and not any(passed["max_dn"]) and len(passed["min_up"]) > 5 and len(passed["max_dn"]) > 20
    assert 0 < sum(passed["min_other"] + passed["max_other"]) < len(passed["min_other"] + passed["max_other"])
    ties = [i for i, kk in kinds.items() if kk == "tie"]
    assert all(lvl[i][cam_of[i]] == KF.keys["octave"][s["sc"]["src"][i]] + 1 for i in ties)
    # the device, hit for hit on the queries Fuse does not skip (without the key frame's row on the device, the call also searches
    # the points already in the key frame; the replay skips them)
    cap = max(counts(KF)) + 5
    dhits, n, status, _ = fuse_device(api, m, [KF], [s["sc"]["rig"]], [None], s["points"], dev_map(s), cap, "single", variant, Scw=s["Scw"])
    first = np.concatenate([[0], np.cumsum(counts(KF))])
    dh = [(int(q), int(sl) // cap, int(first[sl // cap] + sl % cap)) for _, q, sl in dhits if int(q) in live]
    assert status == api.MCS_OK and dh == hh and len(hh) > 100
    # and the replayed ops
    hn, hops, _ = host_fuse(api, m, KF, s, variant)
    dn, dops, _ = fuse_replay(m, KF, s, variant, dhits, cap)
    assert dn == hn and np.array_equal(dops, hops)
    if rm:
        rn, rops = reference_ops(api, rm, cams, KF, s, variant, False)
        assert rn == dn and np.array_equal(rops, dops)
    # the edges discriminate: the other precision, or lower_bound replaced by an upper bound, gives other hits
    assert _host_hits(api, m, KF, s, variant, float_dist=(variant == 2))[0] != hh
    monkeypatch.setattr(api, "_predict_level", lambda sfs, r: min(int(np.searchsorted(sfs, r, side="right")), len(sfs) - 1))
    assert _host_hits(api, m, KF, s, variant)[0] != hh
