"""CPU: argument validation of loop closing's device SearchByBoW(KF1, KF_k) (mcs_search_by_bow_keyframes_device) happens on the host
before any launch, and without a device the accepted shapes fail with MCS_ERR_NO_DEVICE.  The host route the device call is compared
with (cORBmatcher.SearchByBoWKeyFramesHost: read back, slots_to_contiguous, one brute-force SearchByBoW per candidate), run here on
the oracle's brute-force matcher, reproduces the reference's own SearchByBoW(KF1, KF2) (recorded in
tests/golden/ref_tape_search_by_bow_keyframes_device_cpu.*) on the scenes the GPU tests use."""
import ctypes as C

import numpy as np
import pytest

from device_frames import FAKE, counts, declared_symbols, frames, taped_rm  # noqa: F401  (frames: a fixture)
from search_scenes import bow_kf_scene, host_bow_kf, max_count, reference_bow_kf

rm = taped_rm("search_by_bow_keyframes_device_cpu")


def _call(api, kf1=(FAKE, 1, 4, 0), mp1=FAKE, kfs=((FAKE, 1, 4, 0),), mps=None, n_kf=None, n_cams=4, capacity=2000, dim=32, n_points=500,
          bad=None, masks=1, m12=FAKE, slot=FAKE, nm=FAKE, status=FAKE):
    from multicol_slam_b200.ctypes_defs import PackedFrame
    arr = None if kfs is None else (PackedFrame * max(len(kfs), 1))(*[PackedFrame(*f) for f in kfs])
    if mps is None and kfs is not None:
        mps = [FAKE] * len(kfs)
    mp_arr = None if mps is None else (C.c_void_p * max(len(mps), 1))(*mps)
    n_kf = (0 if kfs is None else len(kfs)) if n_kf is None else n_kf
    return api.lib().mcs_search_by_bow_keyframes_device(C.byref(PackedFrame(*kf1)) if kf1 is not None else None, mp1, arr, mp_arr, n_kf,
                                                        n_cams, capacity, dim, n_points, bad, 64, 0.75, masks, m12, slot, nm, status, None)


FRAMES_BAD = [(None, 1, 4, 0), (FAKE, 0, 4, 0), (FAKE, 1, 0, 0), (FAKE, 1, 4, -1), (FAKE, 1, 4, 1), (FAKE, 3, 1, 0)]


def test_validation(api):
    two = ((FAKE, 1, 4, 0), (FAKE, 2, 4, 4))
    bad = [dict(n_kf=-1), dict(kf1=None), dict(mp1=None), dict(kfs=None, n_kf=1), dict(kfs=two, mps=[FAKE, None]), dict(m12=None),
           dict(nm=None), dict(status=None), dict(n_points=-1), dict(n_cams=0), dict(capacity=0), dict(capacity=65536), dict(dim=24),
           dict(dim=0), dict(dim=128)]
    bad += [dict(kf1=f) for f in FRAMES_BAD] + [dict(kfs=((FAKE, 1, 4, 0), f)) for f in FRAMES_BAD]
    for kw in bad:
        assert _call(api, **kw) == api.MCS_ERR_INVALID, kw
    _call(api, kfs=((FAKE, 1, 4, 0), (FAKE, 1, 4, 1)))
    assert b"candidate 1" in api.lib().mcs_last_error()
    # the "taken" bits of one candidate's database in one CTA's shared memory: n_cams * capacity <= 1 622 016
    assert _call(api, n_cams=25, capacity=65535, kf1=(FAKE, 1, 25, 0), kfs=((FAKE, 1, 25, 0),)) == api.MCS_ERR_UNSUPPORTED
    assert _call(api, n_cams=31, capacity=52324, kf1=(FAKE, 1, 31, 0), kfs=((FAKE, 1, 31, 0),)) == api.MCS_ERR_UNSUPPORTED
    # n_kf * n_cams * capacity below 2^31
    many = ((FAKE, 1, 24, 0),) * 1400
    assert _call(api, n_cams=24, capacity=65535, kf1=(FAKE, 1, 24, 0), kfs=many) == api.MCS_ERR_UNSUPPORTED
    assert b"2^31" in api.lib().mcs_last_error()
    # no candidates: a successful no-op, whatever else is passed
    assert _call(api, kfs=(), n_kf=0) == api.MCS_OK and _call(api, kfs=None, n_kf=0, kf1=None, mp1=None, m12=None) == api.MCS_OK
    ok = [dict(), dict(kfs=two), dict(kfs=((FAKE, 4, 1, 0),) * 8), dict(kf1=(FAKE, 2, 4, 4), kfs=((FAKE, 2, 4, 0), (FAKE, 2, 4, 4))),
          dict(slot=None), dict(bad=FAKE), dict(masks=0), dict(dim=16), dict(dim=64), dict(n_points=0), dict(capacity=65535),
          dict(n_cams=32, capacity=50688, kf1=(FAKE, 1, 32, 0), kfs=((FAKE, 1, 32, 0),)),
          dict(n_cams=2, capacity=65535, kf1=(FAKE, 1, 2, 0), kfs=((FAKE, 1, 2, 0),) * 16000)]
    if api.device_count() == 0:
        for kw in ok:
            assert _call(api, **kw) == api.MCS_ERR_NO_DEVICE, kw


def test_symbol_is_declared_and_exported(api):
    assert "mcs_search_by_bow_keyframes_device" in declared_symbols() and hasattr(api.lib(), "mcs_search_by_bow_keyframes_device")
    assert callable(api.cORBmatcher.SearchByBoWKeyFramesDevice) and callable(api.cORBmatcher.SearchByBoWKeyFramesHost)


@pytest.mark.parametrize("masks", [False, True])
def test_host_route_equals_reference(oa, rm, api, frames, cams, masks):
    """the oracle-backed host route == the reference's SearchByBoW(KF1, KF_k), map-point id for map-point id, candidate by
    candidate; one of the candidates is KF1 itself"""
    s = bow_kf_scene(api, frames, 5)
    s["cands"].append(s["KF1"]); s["mps"].append(s["mp1"])
    m = api.cORBmatcher(0.75, False, 32, masks)
    cap = max_count(s) + 3
    m12, slot12, nm, st = host_bow_kf(api, m, s, cap, _bf=oa.match_bruteforce)
    assert st[0] == api.MCS_OK
    for k in range(len(s["cands"])):
        rn, rout = reference_bow_kf(rm, cams, s, k, 0.75, masks)
        assert rn == nm[k] > 20, k
        assert np.array_equal(rout, api.slots_to_contiguous(m12[k], counts(s["KF1"]), cap)), k
    # KF1 against itself: every valid keypoint whose own descriptor is not ambiguous matches itself
    self_row = api.slots_to_contiguous(m12[-1], counts(s["KF1"]), cap)
    assert (self_row[self_row >= 0] == s["mp1"][self_row >= 0]).mean() > 0.9
