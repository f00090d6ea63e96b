"""CPU: argument validation of the device Fuse (mcs_fuse_device) happens on the host before any launch, and without a device the
accepted shapes fail with MCS_ERR_NO_DEVICE.  The host Fuse, whose bookkeeping now runs through the replay it shares with the
device route, still reproduces the reference's recorded map mutations, for all three overloads."""
import numpy as np
import pytest

from device_frames import FAKE, frames, taped_rm  # noqa: F401  (frames: a fixture)
from search_scenes import fuse_scene, host_fuse, reference_ops

rm = taped_rm("fuse_device_cpu")


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
