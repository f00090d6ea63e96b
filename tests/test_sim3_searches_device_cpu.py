"""CPU: argument validation of loop closing's device Sim3 searches (mcs_search_by_sim3_device, mcs_search_by_projection_scw_device)
happens on the host before any launch, and without a device the accepted shapes fail with MCS_ERR_NO_DEVICE.  The host mirrors the
device calls are compared with, cORBmatcher.SearchBySim3 and cORBmatcher.SearchByProjectionKFScw, reproduce the reference's own
methods (recorded in tests/golden/ref_tape_sim3_searches_device_cpu.*) on the scenes the GPU tests use."""
import numpy as np
import pytest

import test_ref_match_cpu as T

FAKE = 0x10000      # stands for a device pointer: never dereferenced by the host
frames = T.frames


@pytest.fixture(scope="module")
def rm():
    """the reference's own matcher, live while recording and replayed from tests/golden/ref_tape_sim3_searches_device_cpu.* otherwise"""
    import ref_tape
    return ref_tape.module("ref_match_api", "sim3_searches_device_cpu", T.TAPE_LIMIT)


def _frame(fr):
    from multicol_slam_b200.ctypes_defs import PackedFrame
    return PackedFrame(*fr) if fr is not None else None


def _sim3(api, cams, n_cams=3, capacity=2000, dim=32, kf1=(FAKE, 1, 6, 0), kf2=(FAKE, 1, 6, 3), cams_ok=True, masks_dev=FAKE, n_levels=8,
          sf=True, t1w=True, t2w=True, mc_inv=True, s12=1.1, r12=True, t12=True, mp1=FAKE, mp2=FAKE, n_points=500, world=FAKE, dmin=FAKE,
          dmax=FAKE, desc=FAKE, dmask=FAKE, bad=None, already2=None, masks=1, m12=FAKE, nfound=FAKE, status=FAKE):
    e4 = np.eye(4).reshape(-1).copy()
    mi = np.tile(np.eye(4), (max(n_cams, 1), 1, 1)).reshape(-1).copy()
    r, t = np.eye(3).reshape(-1).copy(), np.zeros(3)
    s = np.ascontiguousarray([1.2 ** i for i in range(max(n_levels, 1))], np.float64)
    oc = api._ocams(cams[:n_cams] if len(cams) >= n_cams else list(cams) * n_cams) if cams_ok else None
    return api.lib().mcs_search_by_sim3_device(_frame(kf1), _frame(kf2), n_cams, capacity, dim, oc, masks_dev, n_levels,
                                               api._p(s) if sf else None, api._p(e4) if t1w else None, api._p(e4) if t2w else None,
                                               api._p(mi) if mc_inv else None, s12, api._p(r) if r12 else None, api._p(t) if t12 else None,
                                               7.5, mp1, mp2, n_points, world, dmin, dmax, desc, dmask, bad, already2, 48, masks, m12, nfound,
                                               status, None)


def _scw(api, cams, n_cams=3, capacity=2000, dim=32, kf=(FAKE, 1, 3, 0), cams_ok=True, masks_dev=FAKE, n_levels=8, sf=True, mtmc=True,
         ow=True, points=FAKE, n_q=300, n_points=500, world=FAKE, dmin=FAKE, dmax=FAKE, desc=FAKE, dmask=FAKE, bad=None, masks=1,
         matched=FAKE, nmatches=FAKE, status=FAKE, diag=None):
    mi = np.tile(np.eye(4), (max(n_cams, 1), 1, 1)).reshape(-1).copy()
    o = np.zeros(3)
    s = np.ascontiguousarray([1.2 ** i for i in range(max(n_levels, 1))], np.float64)
    oc = api._ocams(cams[:n_cams] if len(cams) >= n_cams else list(cams) * n_cams) if cams_ok else None
    return api.lib().mcs_search_by_projection_scw_device(_frame(kf), n_cams, capacity, dim, oc, masks_dev, n_levels, api._p(s) if sf else None,
                                                         api._p(mi) if mtmc else None, api._p(o) if ow else None, points, n_q, n_points, world,
                                                         dmin, dmax, desc, dmask, bad, 10, 32, masks, matched, nmatches, status, diag, None)


FRAMES_BAD = [(None, 1, 6, 0), (FAKE, 0, 6, 0), (FAKE, 1, 0, 0), (FAKE, 1, 6, -1), (FAKE, 1, 6, 4), (FAKE, 2, 1, 0)]


def test_sim3_validation(api, cams):
    three = [dict(c) for c in cams[:3]]
    nulls = [dict(kf1=None), dict(kf2=None), dict(cams_ok=False), dict(masks_dev=None), dict(sf=False), dict(t1w=False), dict(t2w=False),
             dict(mc_inv=False), dict(r12=False), dict(t12=False), dict(mp1=None), dict(mp2=None), dict(world=None), dict(dmin=None),
             dict(dmax=None), dict(desc=None), dict(dmask=None), dict(m12=None), dict(nfound=None), dict(status=None)]
    sizes = [dict(n_levels=0), dict(n_levels=17), dict(n_points=-1), dict(s12=0.0), dict(dim=24), dict(dim=0), dict(dim=128),
             dict(capacity=0), dict(capacity=65536), dict(n_cams=0)]
    frames_bad = [dict(kf1=f) for f in FRAMES_BAD] + [dict(kf2=f) for f in FRAMES_BAD]
    for kw in nulls + sizes + frames_bad:
        assert _sim3(api, three, **kw) == api.MCS_ERR_INVALID, kw
    neg = [dict(c) for c in three]
    neg[1]["height"] = 0
    assert _sim3(api, neg) == api.MCS_ERR_INVALID
    mixed = [dict(c) for c in three]
    mixed[2]["width"] = mixed[2]["width"] + 2
    assert _sim3(api, mixed) == api.MCS_ERR_UNSUPPORTED
    # one query per slot: n_cams * capacity below 2^24
    assert _sim3(api, three, n_cams=257, capacity=65535, kf1=(FAKE, 1, 257, 0), kf2=(FAKE, 1, 257, 0)) == api.MCS_ERR_UNSUPPORTED
    ok = [dict(), dict(bad=FAKE), dict(already2=FAKE), dict(masks=0, dmask=None), dict(dim=16), dict(dim=64), dict(n_points=0),
          dict(capacity=65535), dict(kf2=(FAKE, 1, 6, 0)), dict(kf1=(FAKE, 3, 1, 0), kf2=(FAKE, 3, 2, 3)), dict(s12=0.5),
          dict(n_cams=256, capacity=65535, kf1=(FAKE, 1, 256, 0), kf2=(FAKE, 1, 256, 0))]
    if api.device_count() == 0:
        for kw in ok:
            assert _sim3(api, three, **kw) == api.MCS_ERR_NO_DEVICE, kw


def test_scw_validation(api, cams):
    three = [dict(c) for c in cams[:3]]
    nulls = [dict(kf=None), dict(cams_ok=False), dict(masks_dev=None), dict(sf=False), dict(mtmc=False), dict(ow=False), dict(points=None),
             dict(world=None), dict(dmin=None), dict(dmax=None), dict(desc=None), dict(dmask=None), dict(matched=None), dict(nmatches=None),
             dict(status=None)]
    sizes = [dict(n_levels=0), dict(n_levels=17), dict(n_points=-1), dict(n_q=-1), dict(dim=24), dict(dim=0), dict(dim=128),
             dict(capacity=0), dict(capacity=65536), dict(n_cams=0)]
    for kw in nulls + sizes + [dict(kf=f) for f in FRAMES_BAD]:
        assert _scw(api, three, **kw) == api.MCS_ERR_INVALID, kw
    neg = [dict(c) for c in three]
    neg[0]["width"] = 0
    assert _scw(api, neg) == api.MCS_ERR_INVALID
    mixed = [dict(c) for c in three]
    mixed[1]["height"] = mixed[1]["height"] + 1
    assert _scw(api, mixed) == api.MCS_ERR_UNSUPPORTED
    assert _scw(api, three, n_q=1 << 24) == api.MCS_ERR_UNSUPPORTED
    assert _scw(api, three, n_cams=257, capacity=65535, kf=(FAKE, 1, 257, 0)) == api.MCS_ERR_UNSUPPORTED
    ok = [dict(), dict(n_q=0), dict(points=None, n_q=0), dict(n_q=(1 << 24) - 1), dict(bad=FAKE), dict(diag=FAKE), dict(masks=0, dmask=None),
          dict(dim=16), dict(dim=64), dict(n_points=0), dict(capacity=65535), dict(kf=(FAKE, 3, 1, 0)),
          dict(n_cams=256, capacity=65535, kf=(FAKE, 1, 256, 0))]
    if api.device_count() == 0:
        for kw in ok:
            assert _scw(api, three, **kw) == api.MCS_ERR_NO_DEVICE, kw


def test_symbols_are_declared_and_exported(api):
    import pathlib
    hdr = (pathlib.Path(api.__file__).resolve().parents[1] / "include" / "mcs_b200.h").read_text()
    for name in ("mcs_search_by_sim3_device", "mcs_search_by_projection_scw_device"):
        assert f"int  {name}(" in hdr and hasattr(api.lib(), name)
    assert callable(api.cORBmatcher.SearchBySim3Device) and callable(api.cORBmatcher.SearchByProjectionKFScwDevice)


# ---- the scenes ------------------------------------------------------------------------------------------------------------------
def second_view(api, KF, seed):
    """another key frame over the same keypoints: positions jittered by up to half a pixel, a few descriptor bits flipped"""
    rng = np.random.default_rng(seed)
    keys = KF.keys.copy()
    keys["x"] += rng.uniform(-0.5, 0.5, len(keys)).astype(np.float32)
    keys["y"] += rng.uniform(-0.5, 0.5, len(keys)).astype(np.float32)
    return api.Frame(keys, KF.key_cam.copy(), T.flip_bits(rng, KF.desc, 3), KF.dmask.copy(), list(zip(KF.cam_w, KF.cam_h)), KF.scale_factors)


def sim3_scene(api, oa, cams, KF1, seed=51, s12=1.01):
    """SearchBySim3 between KF1 and a second view KF2 of its keypoints from a rig pose a few centimetres away.  KF1 carries map points
    0..299 on its keypoints' rays, KF2 points 300..599 a few millimetres from them with descriptor variants of their own; a few
    bad points; the Sim3 is the true relative pose with s12 != 1.  Ten KF1 keypoints are matched beforehand to KF2 points whose
    keypoint in KF2 (obs_idx) is then vbAlreadyMatched2."""
    sc1 = T.make_scene(api, oa, cams, KF1, seed, npts=300)
    KF2 = second_view(api, KF1, seed + 1)
    rng = np.random.default_rng(seed + 2)
    M_t2 = sc1["M_t"].copy()
    M_t2[:3, 3] += [0.012, -0.008, 0.006]
    a = 0.002
    Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1.0]])
    M_t2[:3, :3] = api._mm(Rz, M_t2[:3, :3])
    rig2 = api.Rig(cams, sc1["M_c"], M_t2)
    world2 = sc1["world"] + rng.normal(0, 0.003, sc1["world"].shape)
    world = np.concatenate([sc1["world"], world2])
    desc = np.concatenate([sc1["desc"], T.flip_bits(rng, KF2.desc[sc1["src"]], 30)])
    dmask = np.concatenate([sc1["dmask"], KF2.dmask[sc1["src"]]])
    bad = np.concatenate([sc1["bad"], np.roll(sc1["bad"], 7)])
    # distance ranges whose predicted level is the point's keypoint octave + 1 (ratio 1.1 * scale factor): the window's levels
    # {l - 1, l} keep the keypoint, so that most queries find it
    cam = KF1.key_cam[sc1["src"]]
    depth = np.array([np.linalg.norm(api._mm(sc1["rig"].MtMc_inv[int(c)], np.append(x, 1.0))[:3]) for c, x in zip(cam, sc1["world"])])
    min1 = depth / (1.1 * np.asarray(KF1.scale_factors)[KF1.keys["octave"][sc1["src"]]])
    min_d = np.concatenate([min1, min1])
    max_d = min_d * 12.0
    mp1 = np.full(len(KF1.keys), -1, np.int32); mp1[sc1["src"]] = np.arange(300)
    mp2 = np.full(len(KF2.keys), -1, np.int32); mp2[sc1["src"]] = 300 + np.arange(300)
    T12 = api._mm(api.inv_rigid(sc1["M_t"]), M_t2)                 # KF2's rig frame -> KF1's: T1w * Tw2
    pre = np.full(len(KF1.keys), -1, np.int32)
    some = rng.choice(sc1["src"], 10, replace=False)
    pre[some] = 300 + rng.choice(300, 10, replace=False)
    obs_idx = np.concatenate([sc1["src"], sc1["src"]]).astype(np.int32)
    return dict(KF1=KF1, KF2=KF2, rig1=sc1["rig"], rig2=rig2, M_c=sc1["M_c"], M_t1=sc1["M_t"], M_t2=M_t2, world=world, desc=desc,
                dmask=dmask, bad=bad, min_d=min_d, max_d=max_d, mp1=mp1, mp2=mp2, s12=s12, R12=T12[:3, :3].copy(), t12=T12[:3, 3].copy(),
                pre=pre, obs_idx=obs_idx)


def reference_sim3(rm, cams, s, th, masks):
    obs_kf = np.concatenate([np.zeros(300, np.int32), np.ones(300, np.int32)])
    table = rm.MPTable(3, s["desc"], dmask=s["dmask"], bad=s["bad"], world_pos=s["world"], min_dist=s["min_d"], max_dist=s["max_d"],
                       obs_kf=obs_kf, obs_idx=s["obs_idx"])
    k1 = rm.KF(s["KF1"], cams, M_c=s["M_c"], M_t=s["M_t1"], mp=s["mp1"])
    k2 = rm.KF(s["KF2"], cams, M_c=s["M_c"], M_t=s["M_t2"], mp=s["mp2"])
    return rm.search_by_sim3(k1, k2, table, s["s12"], s["R12"], s["t12"], th, s["pre"], 0.6, masks)


def host_sim3(m, s, th, _sw=None, **kw):
    return m.SearchBySim3(s["KF1"], s["rig1"], s["mp1"], s["KF2"], s["rig2"], s["mp2"], s["world"], s["min_d"], s["max_d"], s["bad"],
                          s["desc"], s["dmask"], s["s12"], s["R12"], s["t12"], th, matches12=kw.get("pre", s["pre"]),
                          obs_idx2=s["obs_idx"], _sw=_sw)


def scw_scene(api, oa, cams, F, seed=33, cam0_only=True, scale=1.25):
    """SearchByProjection(pKF, Scw, vpPoints, vpMatched, th): loop points on the key frame's rays (entry i of vpPoints projects near
    keypoint src[i]), some NULL and some bad; vpMatched holds taken keypoints, some of them holding points of the list (already found).
    cam0_only: the key frame keeps camera 0's keypoints alone, where the reference's descriptor reads stay defined (contiguous id ==
    row)."""
    if cam0_only:
        sel = np.flatnonzero(F.key_cam == 0)
        KF = api.Frame(F.keys[sel], F.key_cam[sel], F.desc[sel], F.dmask[sel], T.SIZES, F.scale_factors)
    else:
        KF = F
    n_keys = len(KF.keys)
    sc = T.make_scene(api, oa, cams, KF, seed, npts=min(n_keys - 5, 400))
    n = len(sc["world"])
    rng = np.random.default_rng(seed + 1)
    points = np.arange(n, dtype=np.int32)
    points[rng.random(n) < 0.05] = -1
    matched = np.full(n_keys, -1, np.int32)
    taken = rng.choice(n_keys, 40, replace=False)
    matched[taken] = rng.choice(n, 40, replace=False)                # points of the list, now already found
    Scw = api.inv_rigid(sc["M_t"]).copy()
    Scw[:3, :3] *= scale
    Scw[:3, 3] *= scale
    return dict(KF=KF, sc=sc, rig=sc["rig"], M_c=sc["M_c"], M_t=sc["M_t"], world=sc["world"], desc=sc["desc"], dmask=sc["dmask"], bad=sc["bad"],
                min_d=sc["min_d"], max_d=sc["max_d"], points=points, matched=matched, Scw=Scw)


def reference_scw(rm, cams, s, masks):
    table = rm.MPTable(3, s["desc"], dmask=s["dmask"], bad=s["bad"], world_pos=s["world"], min_dist=s["min_d"], max_dist=s["max_d"])
    return rm.search_by_projection_scw(rm.KF(s["KF"], cams, M_c=s["M_c"], M_t=s["M_t"]), table, s["Scw"], s["points"], s["matched"], 10,
                                       0.6, masks)


def host_scw(m, s, _sw=None, **kw):
    return m.SearchByProjectionKFScw(s["KF"], s["rig"], s["Scw"], kw.get("points", s["points"]), kw.get("matched", s["matched"]), s["world"],
                                     s["min_d"], s["max_d"], kw.get("bad", s["bad"]), s["desc"], s["dmask"], th=kw.get("th", 10), _sw=_sw)


@pytest.mark.parametrize("th", [7.5, 10.0])
@pytest.mark.parametrize("masks", [False, True])
def test_host_sim3_equals_reference(oa, rm, api, frames, cams, masks, th):
    """two different key frames at different poses, s12 != 1, pre-matched entries with their vbAlreadyMatched2, bad points; th = 10
    is what loop closing passes (ref src/cLoopClosing.cpp:343)"""
    s = sim3_scene(api, oa, cams, frames[0])
    rn, r12 = reference_sim3(rm, cams, s, th, masks)
    m = api.cORBmatcher(0.6, False, 32, masks)
    on, o12 = host_sim3(m, s, th, _sw=oa.search_windows)
    assert rn == on and np.array_equal(r12, o12)
    assert rn > 50
    # the pre-matched entries are kept, and the bad points of both key frames occur among the carried points
    assert np.array_equal(o12[s["pre"] >= 0], s["pre"][s["pre"] >= 0])
    assert s["bad"][s["mp1"][s["mp1"] >= 0]].any() and s["bad"][s["mp2"][s["mp2"] >= 0]].any()


@pytest.mark.parametrize("masks", [False, True])
def test_host_scw_equals_reference(oa, rm, api, frames, cams, masks):
    """vpMatched holds taken keypoints and already found points; NULL and bad entries; keypoint 0 is some entry's best"""
    s = scw_scene(api, oa, cams, frames[0])
    rn, rmatched = reference_scw(rm, cams, s, masks)
    m = api.cORBmatcher(0.6, False, 32, masks)
    on, omatched = host_scw(m, s, _sw=oa.search_windows)
    assert rn == on and np.array_equal(rmatched, omatched) and rn > 50
    assert omatched[0] == s["matched"][0]                            # keypoint 0 is never assigned (:2385)
