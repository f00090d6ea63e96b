"""CPU: argument validation of loop closing's device Sim3 searches (mcs_search_by_sim3_device, mcs_search_by_projection_scw_device)
happens on the host before any launch, and without a device the accepted shapes fail with MCS_ERR_NO_DEVICE.  The host mirrors the
device calls are compared with, cORBmatcher.SearchBySim3 and cORBmatcher.SearchByProjectionKFScw, reproduce the reference's own
methods (recorded in tests/golden/ref_tape_sim3_searches_device_cpu.*) on the scenes the GPU tests use."""
import numpy as np
import pytest

from device_frames import FAKE, frames, taped_rm  # noqa: F401  (frames: a fixture)
from search_scenes import host_scw, host_sim3, reference_scw, reference_sim3, scw_scene, sim3_scene

rm = taped_rm("sim3_searches_device_cpu")


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
