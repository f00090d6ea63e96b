"""CPU: argument validation of the device-resident SearchByProjection entry points (mcs_project_mappoints_device,
mcs_search_by_projection_device) happens on the host before any launch, and without a device both fail with MCS_ERR_NO_DEVICE."""
import ctypes as C

import numpy as np
import pytest

from device_frames import FAKE

PTR = C.c_void_p(FAKE)      # FAKE as a pointer argument


def _mps(n_points=10, **null):
    from multicol_slam_b200.ctypes_defs import MapPointDevView
    v = MapPointDevView()
    v.n_points = n_points
    for k in ("bad", "in_view", "level", "proj_x", "proj_y", "view_cos", "desc", "dmask"):
        setattr(v, k, None if null.get(k) else FAKE)
    return v


def _search(api, mps=None, packed=PTR, n_parts=1, part_images=4, first_image=0, n_cams=4, capacity=2016, dim=32, masks=1,
            frame_mp=PTR, cam_w=None, n_levels=8):
    cw = np.full(max(n_cams, 1), 1280, np.int32) if cam_w is None else np.ascontiguousarray(cam_w, np.int32)
    ch = np.full(max(n_cams, 1), 720, np.int32)
    sf = np.ones(max(n_levels, 1))
    mv = _mps() if mps is None else mps
    return api.lib().mcs_search_by_projection_device(packed, n_parts, part_images, first_image, n_cams, capacity, dim, api._p(cw), api._p(ch),
                                                     n_levels, api._p(sf), C.byref(mv), C.c_double(3.0), C.c_double(0.8), 48, masks,
                                                     frame_mp, PTR, PTR, None, None)


def test_search_by_projection_device_validation(api):
    bad = [dict(packed=None), dict(frame_mp=None), dict(n_cams=0), dict(dim=24), dict(capacity=0), dict(capacity=70000),
           dict(n_parts=0), dict(part_images=0), dict(first_image=-1), dict(first_image=1),            # 1 + 4 cameras > 1 x 4 images
           dict(n_parts=3, part_images=1), dict(n_levels=0), dict(n_levels=17), dict(cam_w=[1280, 0, 1280, 1280]),
           dict(mps=_mps(dmask=True)), dict(mps=_mps(in_view=True)), dict(mps=_mps(desc=True)), dict(mps=_mps(n_points=-1))]
    for kw in bad:
        assert _search(api, **kw) == api.MCS_ERR_INVALID, kw
    # masks not requested: no mask array needed; an allgather layout (4 parts of 1 image) at first_image 0 is accepted
    ok = [dict(mps=_mps(dmask=True), masks=0), dict(n_parts=4, part_images=1), dict(n_parts=2, part_images=4, first_image=3),
          dict(mps=_mps(bad=True))]
    if api.device_count() == 0:
        for kw in ok:
            assert _search(api, **kw) == api.MCS_ERR_NO_DEVICE, kw
    assert _search(api, mps=_mps(n_points=1 << 22)) == api.MCS_ERR_UNSUPPORTED          # 2^24 (point, camera) entries
    assert api.lib().mcs_search_by_projection_max_rounds() >= 1


def test_project_mappoints_device_validation(api, cams):
    from multicol_slam_b200.ctypes_defs import Ocam
    lib = api.lib()
    poses = np.tile(np.eye(4), (3, 1, 1))
    sf = np.ones(8)
    ocs = (Ocam * 3)(*[api.as_ocam(c) for c in cams])

    def call(n_cams=3, mi=poses, masks=PTR, n_points=100, n_levels=8, cams_=ocs, out=PTR):
        return lib.mcs_project_mappoints_device(n_cams, api._p(mi) if mi is not None else None, api._p(poses), cams_, masks, n_points, PTR,
                                                PTR, PTR, PTR, api._p(sf), n_levels, None, out, PTR, PTR, PTR, PTR, None)
    for kw in (dict(mi=None), dict(masks=None), dict(out=None), dict(n_cams=0), dict(n_points=-1), dict(n_levels=0)):
        assert call(**kw) == api.MCS_ERR_INVALID, kw
    big = api.as_ocam(cams[0])
    big.width, big.height = 1280, 720
    mixed = (Ocam * 3)(big, api.as_ocam(cams[1]), api.as_ocam(cams[2]))
    assert call(cams_=mixed) == api.MCS_ERR_UNSUPPORTED
    if api.device_count() == 0:
        assert call() == api.MCS_ERR_NO_DEVICE
        assert call(n_points=0) == api.MCS_ERR_NO_DEVICE


def test_slot_conversion_round_trip(api):
    counts = [3, 0, 2]
    slots = np.array([5, 6, 7, -1, -9, -9, -9, -9, 8, 9, -9, -9], np.int32)
    c = api.slots_to_contiguous(slots, counts, 4)
    assert c.tolist() == [5, 6, 7, 8, 9]
    back = api.contiguous_to_slots(c, counts, 4)
    assert back.tolist() == [5, 6, 7, -1, -1, -1, -1, -1, 8, 9, -1, -1]
    with pytest.raises(ValueError):
        api.slots_to_contiguous(np.zeros(7, np.int32), counts, 4)
