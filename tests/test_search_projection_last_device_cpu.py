"""CPU: argument validation of the device-resident motion-model search (mcs_search_by_projection_last_device) happens on the host
before any launch, and without a device the call fails with MCS_ERR_NO_DEVICE."""
import ctypes as C

import numpy as np

from device_frames import FAKE, declared_symbols


def _search(api, cams, cur=(FAKE, 1, 4, 0), last=(FAKE, 1, 4, 0), n_cams=4, capacity=2016, dim=32, models=None, masks=FAKE, n_levels=8,
            last_mp=FAKE, world=FAKE, cur_mp=FAKE, nm=FAKE, status=FAKE, n_points=1000, sf="ok", mi="ok"):
    from multicol_slam_b200.ctypes_defs import Ocam, PackedFrame
    if models is None:
        models = []
        for c in range(max(n_cams, 1)):
            o = api.as_ocam(cams[c % 3])
            o.width, o.height = 1280, 720
            models.append(o)
    ocs = (Ocam * len(models))(*models)
    fc = None if cur is None else PackedFrame(*cur)
    fl = None if last is None else PackedFrame(*last)
    sfa = np.ones(max(n_levels, 1))
    mia = np.tile(np.eye(4), (max(n_cams, 1), 1, 1))
    return api.lib().mcs_search_by_projection_last_device(
        C.byref(fc) if fc is not None else None, C.byref(fl) if fl is not None else None, n_cams, capacity, dim, ocs, masks, n_levels,
        api._p(sfa) if sf else None, api._p(mia) if mi else None, last_mp, None, n_points, world, None, 50.0, 48, 1, cur_mp, nm, status,
        None, None)


def test_search_by_projection_last_device_validation(api, cams):
    bad = [dict(cur=None), dict(last=None), dict(masks=None), dict(sf=None), dict(mi=None), dict(last_mp=None), dict(world=None),
           dict(cur_mp=None), dict(nm=None), dict(status=None), dict(cur=(None, 1, 4, 0)), dict(last=(None, 1, 4, 0)),
           dict(n_cams=0), dict(dim=24), dict(dim=0), dict(capacity=0), dict(capacity=65536), dict(n_levels=0), dict(n_levels=17),
           dict(n_points=-1),
           dict(cur=(FAKE, 0, 4, 0)), dict(last=(FAKE, 1, 0, 0)), dict(cur=(FAKE, 1, 4, -1)),
           dict(cur=(FAKE, 1, 4, 1)), dict(last=(FAKE, 1, 4, 1)), dict(last=(FAKE, 3, 1, 0))]     # first_image + n_cams > images
    for kw in bad:
        assert _search(api, cams, **kw) == api.MCS_ERR_INVALID, kw
    zero = api.as_ocam(cams[0])
    zero.width = 0
    assert _search(api, cams, n_cams=1, models=[zero]) == api.MCS_ERR_INVALID
    # cameras of different sizes: the mirror masks are one [n_cams][h][w] array
    assert _search(api, cams, n_cams=3, models=[api.as_ocam(c) for c in cams[:2]] + [_sized(api, cams[2], 1280, 720)]) == \
        api.MCS_ERR_UNSUPPORTED
    # the owner words of the acceptance hold a 24-bit query (= slot) index
    assert _search(api, cams, n_cams=257, capacity=65535, cur=(FAKE, 1, 257, 0), last=(FAKE, 257, 1, 0)) == api.MCS_ERR_UNSUPPORTED
    # accepted shapes: the allgather layout, a non-zero first image, both frames in one buffer, no map points
    ok = [dict(cur=(FAKE, 4, 1, 0), last=(FAKE, 4, 1, 0)), dict(cur=(FAKE, 2, 4, 4), last=(FAKE, 2, 4, 0)), dict(n_points=0),
          dict(dim=16), dict(dim=64), dict(capacity=65535)]
    if api.device_count() == 0:
        for kw in ok:
            assert _search(api, cams, **kw) == api.MCS_ERR_NO_DEVICE, kw


def _sized(api, cam, w, h):
    o = api.as_ocam(cam)
    o.width, o.height = w, h
    return o


def test_symbol_is_declared_and_exported(api):
    assert "mcs_search_by_projection_last_device" in declared_symbols()
    assert hasattr(api.lib(), "mcs_search_by_projection_last_device")
    assert hasattr(api.cORBmatcher, "SearchByProjectionLastDevice")
