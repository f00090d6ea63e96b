"""CPU: argument validation of the device-resident WindowSearch (mcs_window_search_device) happens on the host before any launch,
and without a device the call fails with MCS_ERR_NO_DEVICE."""
import numpy as np

from device_frames import FAKE, declared_symbols


def _search(api, cur=(FAKE, 1, 4, 0), last=(FAKE, 1, 4, 0), n_cams=4, capacity=2016, dim=32, sizes=None, last_mp=FAKE, n_points=1000,
            cur_mp=FAKE, nm=FAKE, status=FAKE, window=60, min_level=4, max_level=2**31 - 1, cw="ok", ch="ok"):
    import ctypes as C
    from multicol_slam_b200.ctypes_defs import PackedFrame
    if sizes is None:
        sizes = [(1280, 720)] * max(n_cams, 1)
    w = np.ascontiguousarray([s[0] for s in sizes], np.int32)
    h = np.ascontiguousarray([s[1] for s in sizes], np.int32)
    fc = None if cur is None else PackedFrame(*cur)
    fl = None if last is None else PackedFrame(*last)
    return api.lib().mcs_window_search_device(
        C.byref(fc) if fc is not None else None, C.byref(fl) if fl is not None else None, n_cams, capacity, dim,
        api._p(w) if cw else None, api._p(h) if ch else None, last_mp, n_points, None, window, min_level, max_level, 0.8, 48, 1, cur_mp,
        nm, status, None, None)


def test_window_search_device_validation(api):
    bad = [dict(cur=None), dict(last=None), dict(cw=None), dict(ch=None), dict(last_mp=None), dict(cur_mp=None), dict(nm=None),
           dict(status=None), dict(cur=(None, 1, 4, 0)), dict(last=(None, 1, 4, 0)),
           dict(n_cams=0), dict(dim=24), dict(dim=0), dict(capacity=0), dict(capacity=65536), dict(n_points=-1),
           dict(cur=(FAKE, 0, 4, 0)), dict(last=(FAKE, 1, 0, 0)), dict(cur=(FAKE, 1, 4, -1)),
           dict(cur=(FAKE, 1, 4, 1)), dict(last=(FAKE, 1, 4, 1)), dict(last=(FAKE, 3, 1, 0)),     # first_image + n_cams > images
           dict(n_cams=2, sizes=[(1280, 720), (0, 720)]), dict(n_cams=1, sizes=[(1280, -1)])]
    for kw in bad:
        assert _search(api, **kw) == api.MCS_ERR_INVALID, kw
    # the owner words of the acceptance hold a 24-bit query (= slot) index
    assert _search(api, n_cams=257, capacity=65535, cur=(FAKE, 1, 257, 0), last=(FAKE, 257, 1, 0)) == api.MCS_ERR_UNSUPPORTED
    # accepted shapes: the allgather layout, a non-zero first image, both frames in one buffer, no map points, cameras of different
    # sizes (no masks are read), every level filter
    ok = [dict(cur=(FAKE, 4, 1, 0), last=(FAKE, 4, 1, 0)), dict(cur=(FAKE, 2, 4, 4), last=(FAKE, 2, 4, 0)), dict(n_points=0),
          dict(dim=16), dict(dim=64), dict(capacity=65535), dict(sizes=[(1280, 720), (640, 480), (754, 480), (1920, 1080)]),
          dict(min_level=0, max_level=3), dict(window=50, min_level=0), dict(n_cams=256, capacity=65535, cur=(FAKE, 1, 256, 0),
                                                                             last=(FAKE, 256, 1, 0))]
    if api.device_count() == 0:
        for kw in ok:
            assert _search(api, **kw) == api.MCS_ERR_NO_DEVICE, kw


def test_symbol_is_declared_and_exported(api):
    assert "mcs_window_search_device" in declared_symbols()
    assert hasattr(api.lib(), "mcs_window_search_device")
    assert hasattr(api.cORBmatcher, "WindowSearchDevice")
