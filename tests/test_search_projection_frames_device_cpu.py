"""CPU: argument validation of the device-resident SearchByProjection(F1, F2, window) (mcs_search_by_projection_frames_device)
happens on the host before any launch, and without a device the call fails with MCS_ERR_NO_DEVICE."""
import ctypes as C

import numpy as np

from device_frames import FAKE, declared_symbols


def _search(api, cams, cur=(FAKE, 1, 4, 0), last=(FAKE, 1, 4, 0), n_cams=4, capacity=2016, dim=32, models=None, masks=FAKE, mi="ok",
            last_mp=FAKE, n_points=1000, world=FAKE, cur_mp=FAKE, nm=FAKE, status=FAKE):
    from multicol_slam_b200.ctypes_defs import Ocam, PackedFrame
    if models is None:
        models = [_sized(api, cams[c % 3], 1280, 720) for c in range(max(n_cams, 1))]
    ocs = (Ocam * len(models))(*models)
    fc = None if cur is None else PackedFrame(*cur)
    fl = None if last is None else PackedFrame(*last)
    mia = np.tile(np.eye(4), (max(n_cams, 1), 1, 1))
    return api.lib().mcs_search_by_projection_frames_device(
        C.byref(fc) if fc is not None else None, C.byref(fl) if fl is not None else None, n_cams, capacity, dim, ocs, masks,
        api._p(mia) if mi else None, last_mp, n_points, world, None, 40, 0.8, 48, 1, cur_mp, nm, status, None, None)


def _sized(api, cam, w, h):
    o = api.as_ocam(cam)
    o.width, o.height = w, h
    return o


def test_search_by_projection_frames_device_validation(api, cams):
    bad = [dict(cur=None), dict(last=None), dict(masks=None), dict(mi=None), dict(last_mp=None), dict(world=None), dict(cur_mp=None),
           dict(nm=None), dict(status=None), dict(cur=(None, 1, 4, 0)), dict(last=(None, 1, 4, 0)),
           dict(n_cams=0), dict(dim=24), dict(dim=0), dict(capacity=0), dict(capacity=65536), dict(n_points=-1),
           dict(cur=(FAKE, 0, 4, 0)), dict(last=(FAKE, 1, 0, 0)), dict(cur=(FAKE, 1, 4, -1)),
           dict(cur=(FAKE, 1, 4, 1)), dict(last=(FAKE, 1, 4, 1)), dict(last=(FAKE, 3, 1, 0))]     # first_image + n_cams > images
    for kw in bad:
        assert _search(api, cams, **kw) == api.MCS_ERR_INVALID, kw
    assert _search(api, cams, n_cams=1, models=[_sized(api, cams[0], 0, 720)]) == api.MCS_ERR_INVALID
    # cameras of different sizes: the mirror masks are one [n_cams][h][w] array
    assert _search(api, cams, n_cams=3, models=[api.as_ocam(c) for c in cams[:2]] + [_sized(api, cams[2], 1280, 720)]) == \
        api.MCS_ERR_UNSUPPORTED
    # one query per (last-frame slot, camera): n_cams * n_cams * capacity must stay below the 24-bit query index
    # (17 * 17 * 58053 = 2^24 + 101, 17 * 17 * 58052 = 2^24 - 188)
    rig17 = dict(n_cams=17, cur=(FAKE, 1, 17, 0), last=(FAKE, 17, 1, 0))
    assert _search(api, cams, capacity=58053, **rig17) == api.MCS_ERR_UNSUPPORTED
    # accepted shapes: the allgather layout, a non-zero first image, both frames in one buffer, no map points, the largest
    # capacity of a 17-camera rig
    ok = [dict(cur=(FAKE, 4, 1, 0), last=(FAKE, 4, 1, 0)), dict(cur=(FAKE, 2, 4, 4), last=(FAKE, 2, 4, 0)), dict(n_points=0),
          dict(dim=16), dict(dim=64), dict(capacity=65535), dict(capacity=58052, **rig17)]
    if api.device_count() == 0:
        for kw in ok:
            assert _search(api, cams, **kw) == api.MCS_ERR_NO_DEVICE, kw


def test_symbol_is_declared_and_exported(api):
    assert "mcs_search_by_projection_frames_device" in declared_symbols()
    assert hasattr(api.lib(), "mcs_search_by_projection_frames_device")
    assert hasattr(api.cORBmatcher, "SearchByProjectionFramesDevice")
