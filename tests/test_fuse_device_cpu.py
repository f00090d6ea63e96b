"""CPU: argument validation of the device Fuse (mcs_fuse_device) happens on the host before any launch, and without a device the
accepted shapes fail with MCS_ERR_NO_DEVICE.  The host Fuse, whose bookkeeping now runs through the replay it shares with the
device route, still reproduces the reference's recorded map mutations, for all three overloads."""
import numpy as np
import pytest

import test_ref_match_cpu as T

FAKE = 0x10000      # stands for a device pointer: never dereferenced by the host
frames = T.frames


@pytest.fixture(scope="module")
def rm():
    """the reference's own matcher, live while recording and replayed from tests/golden/ref_tape_fuse_device_cpu.* otherwise"""
    import ref_tape
    return ref_tape.module("ref_match_api", "fuse_device_cpu", T.TAPE_LIMIT)


def _fuse(api, cams, n_kf=2, n_cams=3, capacity=2000, dim=32, frame=None, frames_=None, mtmc=True, n_levels=8, sf="ok", variant=0, q=FAKE,
          n_q=100, n_points=500, world=FAKE, dmin=FAKE, dmax=FAKE, desc=FAKE, dmask=FAKE, bad=None, masks=1, hits=FAKE, max_hits=64,
          n_hits=FAKE, status=FAKE, masks_dev=FAKE, cams_ok=True, kfs_ok=True, mp=FAKE):
    from multicol_slam_b200.ctypes_defs import FuseTarget, PackedFrame
    mi = np.tile(np.eye(4), (max(n_cams, 1), 1, 1)).reshape(-1).copy()
    tg = (FuseTarget * max(n_kf, 1))()
    for k in range(max(n_kf, 1)):
        fr = frames_[k] if frames_ is not None else (frame if frame is not None else (FAKE, 1, n_cams * max(n_kf, 1), k * n_cams))
        tg[k].frame = PackedFrame(*fr)
        tg[k].mp_dev = mp if k == 0 else None
        tg[k].mtmc_inv = mi.ctypes.data if (mtmc or k == 0) else None
    oc = api._ocams(cams[:n_cams] if len(cams) >= n_cams else list(cams) * n_cams) if cams_ok else None
    s = np.ascontiguousarray([1.2 ** i for i in range(max(n_levels, 1))], np.float64)
    return api.lib().mcs_fuse_device(tg if kfs_ok else None, n_kf, n_cams, capacity, dim, oc, masks_dev, n_levels, api._p(s) if sf else None,
                                     variant, q, n_q, n_points, world, dmin, dmax, desc, dmask, bad, 3.0, 64, masks, hits, max_hits, n_hits,
                                     status, None)


def test_validation(api, cams):
    three = [dict(c) for c in cams[:3]]
    nulls = [dict(kfs_ok=False), dict(cams_ok=False), dict(masks_dev=None), dict(sf=None), dict(q=None), dict(world=None), dict(dmin=None),
             dict(dmax=None), dict(desc=None), dict(hits=None), dict(n_hits=None), dict(status=None), dict(dmask=None), dict(mtmc=False)]
    sizes = [dict(n_kf=0), dict(n_kf=-1), dict(n_q=-1), dict(max_hits=-1), dict(n_points=-1), dict(n_levels=0), dict(n_levels=17),
             dict(variant=-1), dict(variant=3), dict(dim=24), dict(dim=0), dict(dim=128), dict(capacity=0), dict(capacity=65536), dict(n_cams=0)]
    frames_bad = [dict(frame=f) for f in [(None, 1, 6, 0), (FAKE, 0, 6, 0), (FAKE, 1, 0, 0), (FAKE, 1, 6, -1), (FAKE, 1, 6, 4), (FAKE, 2, 1, 0)]]
    frames_bad.append(dict(frames_=[(FAKE, 1, 6, 0), (FAKE, 1, 6, 5)]))              # the second key frame's cameras run past its buffer
    for kw in nulls + sizes + frames_bad:
        assert _fuse(api, three, **kw) == api.MCS_ERR_INVALID, kw
    neg = [dict(c) for c in three]
    neg[1]["width"] = 0
    assert _fuse(api, neg) == api.MCS_ERR_INVALID
    # one [n_cams][h][w] mask array: cameras of different sizes are refused as in the motion-model search
    mixed = [dict(c) for c in three]
    mixed[2]["width"] = mixed[2]["width"] + 2
    assert _fuse(api, mixed) == api.MCS_ERR_UNSUPPORTED
    # the front end's 24-bit slot and query indices
    assert _fuse(api, three, n_kf=86, capacity=65535, n_q=1, frame=(FAKE, 1, 258, 0)) == api.MCS_ERR_UNSUPPORTED     # 258 * 65535 >= 2^24
    assert _fuse(api, three, n_kf=2, n_q=(1 << 24) // 6 + 1) == api.MCS_ERR_UNSUPPORTED
    ok = [dict(), dict(n_q=0), dict(max_hits=0), dict(n_points=0), dict(bad=FAKE), dict(mp=None), dict(masks=0, dmask=None), dict(dim=16),
          dict(dim=64), dict(variant=1), dict(variant=2), dict(capacity=65535), dict(frames_=[(FAKE, 3, 1, 0), (FAKE, 3, 1, 0)]),
          dict(n_kf=85, capacity=65535, n_q=1, frame=(FAKE, 1, 255, 0)), dict(n_kf=2, n_q=(1 << 24) // 6),
          dict(q=None, n_q=0), dict(hits=None, max_hits=0)]
    if api.device_count() == 0:
        for kw in ok:
            assert _fuse(api, three, **kw) == api.MCS_ERR_NO_DEVICE, kw


def test_symbol_is_declared_and_exported(api):
    import pathlib
    hdr = (pathlib.Path(api.__file__).resolve().parents[1] / "include" / "mcs_b200.h").read_text()
    assert "int  mcs_fuse_device(" in hdr and "typedef struct mcs_fuse_target" in hdr
    assert hasattr(api.lib(), "mcs_fuse_device")
    assert callable(api.cORBmatcher.FuseDevice) and callable(api.cORBmatcher.FuseReplay)


def fuse_scene(api, oa, cams, KF, variant, seed=5):
    """the scene of test_ref_match_cpu.py::test_fuse_equals_reference; variant 0 adds a current key frame: a second rig pose a few
    centimetres away whose keypoints carry the query points (their rays are the bearing rays of the points seen from it)"""
    sc = T.make_scene(api, oa, cams, KF, 11 + variant)
    rng = np.random.default_rng(seed)
    n = len(sc["world"])
    kf_mp = np.full(len(KF.keys), -1, np.int32)
    occupied = rng.choice(len(KF.keys), len(KF.keys) // 3, replace=False)
    extra_bad = (rng.random(len(occupied)) < 0.1).astype(np.uint8)
    kf_mp[occupied] = n + np.arange(len(occupied))
    bad = np.concatenate([sc["bad"], extra_bad])
    in_kf = np.concatenate([(rng.random(n) < 0.1), np.ones(len(occupied), bool)])
    pad = lambda a, fill=0.0: np.concatenate([a, np.full((len(occupied),) + a.shape[1:], fill, a.dtype)])  # noqa: E731
    s = dict(sc=sc, n=n, kf_mp=kf_mp, occupied=occupied, bad=bad, in_kf=in_kf, points=np.arange(n, dtype=np.int32),
             world=pad(sc["world"]), min_d=pad(sc["min_d"], 1.0), max_d=pad(sc["max_d"], 2.0), desc=pad(sc["desc"]), dmask=pad(sc["dmask"]),
             Scw=None, cur=None)
    if variant == 2:
        Scw = api.inv_rigid(sc["M_t"]).copy()
        Scw[:3, :3] *= 1.3
        Scw[:3, 3] *= 1.3
        s["Scw"] = Scw
    if variant == 0:
        # curKF: the same keypoints on a rig moved by a few cm; keypoint j of curKF carries points[j] (one key frame of map points
        # per keypoint, as vpMapPointMatches of curKF).  Rays: the point's bearing from the moved rig, jittered so that the
        # epipolar check both passes and fails among the occupied hits.
        M_t2 = sc["M_t"].copy()
        M_t2[:3, 3] += [0.03, -0.01, 0.02]
        cur_rig = api.Rig(cams, sc["M_c"], M_t2)
        rays = np.zeros((n, 3))
        for j in range(n):
            c = int(KF.key_cam[sc["src"][j]])
            pc = api._mm(cur_rig.MtMc_inv[c], np.append(sc["world"][j], 1.0))[:3]
            r = pc / np.linalg.norm(pc) + rng.normal(0, 0.08 if j % 2 else 0.0005, 3)
            rays[j] = r / np.linalg.norm(r)
        key_cam = np.asarray(KF.key_cam[sc["src"]], np.int32)
        s["cur"] = dict(rig=cur_rig, M_t=M_t2, rays=rays, key_cam=key_cam)
    return s


def reference_ops(api, rm, cams, KF, s, variant, masks):
    sc = s["sc"]
    table = rm.MPTable(3, s["desc"], dmask=s["dmask"], bad=s["bad"], world_pos=s["world"], min_dist=s["min_d"], max_dist=s["max_d"],
                       obs_kf=np.where(s["in_kf"], 0, -1).astype(np.int32), obs_idx=np.zeros(len(s["bad"]), np.int32))
    kfr = rm.KF(KF, cams, M_c=sc["M_c"], M_t=sc["M_t"], mp=s["kf_mp"], rays=sc["rays"])
    cur = None
    if variant == 0:
        Fc = api.Frame(KF.keys[sc["src"]], s["cur"]["key_cam"], KF.desc[sc["src"]], KF.dmask[sc["src"]], T.SIZES, KF.scale_factors)
        cur = rm.KF(Fc, cams, M_c=sc["M_c"], M_t=s["cur"]["M_t"], mp=s["points"], rays=s["cur"]["rays"])
    return rm.fuse(variant, kfr, table, s["points"], 2.5, 0.6, masks, CurK=cur, Scw=s["Scw"])


def host_fuse(api, m, KF, s, variant, _sw=None, **kw):
    sc = s["sc"]
    cur = s["cur"] or {}
    return m.Fuse(KF, sc["rig"], s["kf_mp"], s["points"], s["world"], s["min_d"], s["max_d"], s["bad"], s["in_kf"], s["desc"], s["dmask"],
                  th=2.5, variant=variant, Scw=s["Scw"], cur_rays=cur.get("rays"), kf_rays=sc["rays"], cur_rig=cur.get("rig"), _sw=_sw, **kw)


@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("variant", [0, 1, 2])
def test_host_fuse_through_the_shared_replay_equals_reference(oa, rm, api, frames, cams, masks, variant, monkeypatch):
    """Fuse(pKF, curKF, ., th) with its epipolar check, Fuse(pKF, ., th) and Fuse(pKF, Scw, ., th): the host composition over the
    oracle's window search, its bookkeeping in the replay the device route shares, gives the reference's mutations in order"""
    KF = frames[0]
    s = fuse_scene(api, oa, cams, KF, variant)
    rn, rops = reference_ops(api, rm, cams, KF, s, variant, masks)
    m = api.cORBmatcher(0.6, False, 32, masks)
    on, oops, _ = host_fuse(api, m, KF, s, variant, _sw=oa.search_windows)
    assert rn == on and np.array_equal(rops, oops)
    assert len(rops) > 100 and (rops[:, 0] == 0).sum() > 10 and (rops[:, 0] == 1).sum() > 10
    if variant == 0:
        # the epipolar check decided occupied hits both ways: with a check that always holds, more of them are fused
        monkeypatch.setattr(api, "check_epipolar", lambda *a: True)
        an, _, _ = host_fuse(api, m, KF, s, variant, _sw=oa.search_windows)
        assert 10 < on < an
