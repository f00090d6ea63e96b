"""CPU: argument validation of the device bag-of-words calls (mcs_bow_vectors_device, mcs_search_by_bow_device) happens on the host
before any launch, and without a device the calls fail with MCS_ERR_NO_DEVICE.  The vocabulary object lives on a device, so what
needs one (mcs_vocabulary_level_nodes' counts, the other-device refusal) is in tests/test_bow_vectors_device_gpu.py."""
import ctypes as C

from device_frames import FAKE, declared_symbols    # FAKE also stands for a vocabulary that is never looked into


def _vectors(api, voc=FAKE, frame=(FAKE, 1, 4, 0), n_cams=4, capacity=2016, dim=32, levelsup=4, max_nodes=81, null=()):
    from multicol_slam_b200.ctypes_defs import PackedFrame
    fr = None if frame is None else PackedFrame(*frame)
    names = ["word", "weight", "node", "fv_nodes", "fv_offsets", "n_fv", "fv_features", "bow_words", "bow_values", "n_bow", "status"]
    outs = [None if n in null else FAKE for n in names]
    return api.lib().mcs_bow_vectors_device(voc, C.byref(fr) if fr is not None else None, n_cams, capacity, dim, levelsup, max_nodes, *outs,
                                            None)


def test_bow_vectors_device_validation(api):
    bad = [dict(voc=None), dict(frame=None), dict(frame=(None, 1, 4, 0)), dict(n_cams=0), dict(capacity=0), dict(capacity=65536),
           dict(dim=24), dict(dim=0), dict(max_nodes=0), dict(max_nodes=-3), dict(frame=(FAKE, 0, 4, 0)), dict(frame=(FAKE, 1, 0, 0)),
           dict(frame=(FAKE, 1, 4, -1)), dict(frame=(FAKE, 1, 4, 1)), dict(frame=(FAKE, 3, 1, 0))]
    bad += [dict(null=(n,)) for n in ("fv_nodes", "fv_offsets", "n_fv", "fv_features", "bow_words", "bow_values", "n_bow", "status")]
    for kw in bad:
        assert _vectors(api, **kw) == api.MCS_ERR_INVALID, kw
    # the vocabulary's descriptors are FORB's 32 bytes; the slot index must stay below 2^24
    assert _vectors(api, dim=16) == api.MCS_ERR_UNSUPPORTED and _vectors(api, dim=64) == api.MCS_ERR_UNSUPPORTED
    assert _vectors(api, n_cams=257, capacity=65535, frame=(FAKE, 1, 257, 0)) == api.MCS_ERR_UNSUPPORTED
    # accepted shapes: the per-slot outputs are optional, every buffer layout, any levelsup
    ok = [dict(), dict(null=("word", "weight", "node")), dict(frame=(FAKE, 4, 1, 0)), dict(frame=(FAKE, 2, 4, 4)), dict(levelsup=0, max_nodes=6999),
          dict(levelsup=9, max_nodes=1), dict(capacity=65535), dict(n_cams=1, frame=(FAKE, 1, 1, 0))]
    if api.device_count() == 0:
        for kw in ok:
            assert _vectors(api, **kw) == api.MCS_ERR_NO_DEVICE, kw


def _search(api, kfs=((FAKE, 1, 4, 0),), cur=(FAKE, 1, 4, 0), n_kf=None, n_cams=4, capacity=2016, dim=32, max_nodes=81, n_points=1000,
            kf_null=(), cur_null=(), match_mp=FAKE, match_slot=FAKE, nm=FAKE, status=FAKE):
    from multicol_slam_b200.ctypes_defs import BowFrame, PackedFrame

    def bow(frame, null, mp):
        b = BowFrame()
        b.frame = PackedFrame(*frame)
        for f in ("fv_nodes_dev", "fv_offsets_dev", "n_fv_dev", "fv_features_dev"):
            setattr(b, f, None if f in null else FAKE)
        b.mp_dev = None if (mp is None or "mp_dev" in null) else mp
        return b
    arr = None if kfs is None else (BowFrame * max(len(kfs), 1))(*[bow(f, kf_null if i == len(kfs) - 1 else (), FAKE) for i, f in enumerate(kfs)])
    fc = None if cur is None else bow(cur, cur_null, None)
    n_kf = (0 if kfs is None else len(kfs)) if n_kf is None else n_kf
    return api.lib().mcs_search_by_bow_device(arr, n_kf, C.byref(fc) if fc is not None else None, n_cams, capacity, dim, max_nodes, n_points,
                                              None, 64, 0.9, 1, match_mp, match_slot, nm, status, None)


def test_search_by_bow_device_validation(api):
    two = ((FAKE, 1, 4, 0), (FAKE, 2, 4, 4))
    bad = [dict(n_kf=-1), dict(kfs=None, n_kf=1), dict(cur=None), dict(match_mp=None), dict(nm=None), dict(status=None),
           dict(cur=(None, 1, 4, 0)), dict(kfs=((None, 1, 4, 0),)), dict(n_cams=0), dict(dim=24), dict(dim=0), dict(capacity=0),
           dict(capacity=65536), dict(max_nodes=0), dict(n_points=-1), dict(cur=(FAKE, 1, 4, 1)), dict(cur=(FAKE, 3, 1, 0)),
           dict(kfs=((FAKE, 1, 4, 0), (FAKE, 1, 4, 1))), dict(kfs=((FAKE, 1, 4, 0), (FAKE, 0, 4, 0))), dict(kfs=two, kf_null=("mp_dev",))]
    bad += [dict(cur_null=(f,)) for f in ("fv_nodes_dev", "fv_offsets_dev", "n_fv_dev", "fv_features_dev")]
    bad += [dict(kfs=two, kf_null=(f,)) for f in ("fv_nodes_dev", "fv_offsets_dev", "n_fv_dev", "fv_features_dev")]
    for kw in bad:
        assert _search(api, **kw) == api.MCS_ERR_INVALID, kw
    assert b"key frame 1" in api.lib().mcs_last_error()
    assert _search(api, n_cams=257, capacity=65535, cur=(FAKE, 1, 257, 0), kfs=((FAKE, 257, 1, 0),)) == api.MCS_ERR_UNSUPPORTED
    # no key frames: a successful no-op, whatever else is passed
    assert _search(api, kfs=(), n_kf=0) == api.MCS_OK and _search(api, kfs=None, n_kf=0, cur=None, match_mp=None) == api.MCS_OK
    # accepted shapes: key frames in their own buffers of either layout or in the current frame's, no match_slot, every width
    ok = [dict(), dict(kfs=two), dict(kfs=((FAKE, 4, 1, 0),) * 8), dict(kfs=((FAKE, 2, 4, 0),), cur=(FAKE, 2, 4, 4)), dict(match_slot=None),
          dict(dim=16), dict(dim=64), dict(capacity=65535), dict(n_points=0), dict(max_nodes=6999)]
    if api.device_count() == 0:
        for kw in ok:
            assert _search(api, **kw) == api.MCS_ERR_NO_DEVICE, kw


def test_level_nodes_refuses_null(api):
    n = C.c_int32(0)
    assert api.lib().mcs_vocabulary_level_nodes(None, 4, C.byref(n)) == api.MCS_ERR_INVALID
    assert api.lib().mcs_vocabulary_level_nodes(FAKE, 4, None) == api.MCS_ERR_INVALID


def test_symbols_are_declared_exported_and_mirrored(api):
    from multicol_slam_b200 import ctypes_defs
    for s in ("mcs_vocabulary_level_nodes", "mcs_bow_vectors_device", "mcs_search_by_bow_device"):
        assert s in declared_symbols() and hasattr(api.lib(), s)
    assert hasattr(api.ORBVocabulary, "transform_device") and hasattr(api.ORBVocabulary, "level_nodes")
    assert hasattr(api.cORBmatcher, "SearchByBoWDevice") and hasattr(api, "DeviceBoW")
    # mcs_bow_frame: the packed frame (pointer + 3 ints, padded) and five pointers
    assert C.sizeof(ctypes_defs.BowFrame) == C.sizeof(ctypes_defs.PackedFrame) + 5 * 8 == 64
