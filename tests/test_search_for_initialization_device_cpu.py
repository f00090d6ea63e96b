"""CPU: argument validation of map initialisation's device search (mcs_search_for_initialization_device) and of its seed call
(mcs_search_for_initialization_seed_device) happens on the host before any launch, and without a device the accepted shapes fail
with MCS_ERR_NO_DEVICE."""
import numpy as np

from device_frames import FAKE, declared_symbols


def _search(api, f1=(FAKE, 1, 4, 0), f2=(FAKE, 1, 4, 0), n_cams=4, capacity=4000, dim=32, sizes=None, prev=FAKE, m12=FAKE, nm=FAKE,
            diag=None, window=50, cw="ok", ch="ok"):
    import ctypes as C
    from multicol_slam_b200.ctypes_defs import PackedFrame
    if sizes is None:
        sizes = [(1280, 720)] * max(n_cams, 1)
    w = np.ascontiguousarray([s[0] for s in sizes], np.int32)
    h = np.ascontiguousarray([s[1] for s in sizes], np.int32)
    a = None if f1 is None else PackedFrame(*f1)
    b = None if f2 is None else PackedFrame(*f2)
    return api.lib().mcs_search_for_initialization_device(
        C.byref(a) if a is not None else None, C.byref(b) if b is not None else None, n_cams, capacity, dim, api._p(w) if cw else None,
        api._p(h) if ch else None, prev, window, 0.9, 32, 1, m12, nm, diag, None)


def _seed(api, f1=(FAKE, 1, 4, 0), n_cams=4, capacity=4000, dim=32, prev=FAKE):
    import ctypes as C
    from multicol_slam_b200.ctypes_defs import PackedFrame
    a = None if f1 is None else PackedFrame(*f1)
    return api.lib().mcs_search_for_initialization_seed_device(C.byref(a) if a is not None else None, n_cams, capacity, dim, prev, None)


BAD_FRAMES = [(None, 1, 4, 0), (FAKE, 0, 4, 0), (FAKE, 1, 0, 0), (FAKE, 1, 4, -1), (FAKE, 1, 4, 1), (FAKE, 3, 1, 0)]


def test_search_validation(api):
    bad = [dict(f1=None), dict(f2=None), dict(cw=None), dict(ch=None), dict(prev=None), dict(m12=None), dict(nm=None),
           dict(n_cams=0), dict(dim=24), dict(dim=0), dict(dim=128), dict(capacity=0), dict(capacity=65536),
           dict(n_cams=2, sizes=[(1280, 720), (0, 720)]), dict(n_cams=1, sizes=[(1280, -1)])]
    bad += [dict(f1=f) for f in BAD_FRAMES] + [dict(f2=f) for f in BAD_FRAMES]
    for kw in bad:
        assert _search(api, **kw) == api.MCS_ERR_INVALID, kw
    # the front end keeps query and slot indices below 2^24
    assert _search(api, n_cams=257, capacity=65535, f1=(FAKE, 1, 257, 0), f2=(FAKE, 257, 1, 0)) == api.MCS_ERR_UNSUPPORTED
    ok = [dict(), dict(f1=(FAKE, 4, 1, 0), f2=(FAKE, 4, 1, 0)), dict(f1=(FAKE, 2, 4, 4), f2=(FAKE, 2, 4, 0)), dict(dim=16), dict(dim=64),
          dict(capacity=65535), dict(diag=FAKE), dict(window=0), dict(window=-3), dict(sizes=[(1280, 720), (640, 480), (754, 480), (1920, 1080)]),
          dict(n_cams=256, capacity=65535, f1=(FAKE, 1, 256, 0), f2=(FAKE, 256, 1, 0))]
    if api.device_count() == 0:
        for kw in ok:
            assert _search(api, **kw) == api.MCS_ERR_NO_DEVICE, kw


def test_seed_validation(api):
    bad = [dict(f1=None), dict(prev=None), dict(n_cams=0), dict(dim=24), dict(capacity=0), dict(capacity=65536)]
    bad += [dict(f1=f) for f in BAD_FRAMES]
    for kw in bad:
        assert _seed(api, **kw) == api.MCS_ERR_INVALID, kw
    assert _seed(api, n_cams=257, capacity=65535, f1=(FAKE, 257, 1, 0)) == api.MCS_ERR_UNSUPPORTED
    ok = [dict(), dict(f1=(FAKE, 4, 1, 0)), dict(f1=(FAKE, 2, 4, 4)), dict(dim=16), dict(dim=64), dict(capacity=65535)]
    if api.device_count() == 0:
        for kw in ok:
            assert _seed(api, **kw) == api.MCS_ERR_NO_DEVICE, kw


def test_symbols_are_declared_and_exported(api):
    for name in ("mcs_search_for_initialization_device", "mcs_search_for_initialization_seed_device"):
        assert name in declared_symbols()
        assert hasattr(api.lib(), name)
    assert hasattr(api.cORBmatcher, "SearchForInitializationDevice")
    assert hasattr(api.cORBmatcher, "SearchForInitializationSeedDevice")
