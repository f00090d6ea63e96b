"""CPU: libmcs_b200.so loads, exports every function include/mcs_b200.h declares, validates arguments,
and refuses to compute without a GPU (no CPU fallback)."""
import ctypes as C

import numpy as np
import pytest

from device_frames import declared_symbols


def test_exports_every_declared_symbol(api):
    syms = declared_symbols()
    assert len(syms) >= 20
    lib = api.lib()
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/mcs_b200.h but not exported"


def test_struct_layouts(api):
    from multicol_slam_b200.ctypes_defs import ExtractorParams, KEYPOINT_DTYPE, Ocam, WindowQuery
    assert C.sizeof(Ocam) == 8 * 22 + 16 and C.sizeof(ExtractorParams) == 52
    assert KEYPOINT_DTYPE.itemsize == 28 and C.sizeof(WindowQuery) == 40
    from multicol_slam_b200 import rig
    assert api.lib().mcs_slot_bytes(2016, 32) == rig.slot_bytes(2016, 32) == 256 + (2016 * 28 + 255) // 256 * 256 + 2 * 2016 * 32


def test_host_helpers_match_oracle(api, oa, cams):
    # camera model + mirror mask + scalar Hamming distances are host-side helpers of the C ABI
    rng = np.random.default_rng(1)
    for cam in cams:
        assert np.array_equal(api.mirror_mask(cam), __import__("multicol_slam_b200.synth", fromlist=["x"]).mirror_mask(cam))
        oc = api.as_ocam(cam)
        for _ in range(50):
            u, v = rng.uniform(100, 600), rng.uniform(50, 400)
            x, y, z = api.img_to_world(cam, u, v)
            ox, oy, oz = C.c_double(), C.c_double(), C.c_double()
            oa.lib().mcso_cam_img_to_world(C.byref(oc), C.c_double(u), C.c_double(v), C.byref(ox), C.byref(oy), C.byref(oz))
            assert (x, y, z) == (ox.value, oy.value, oz.value)
            uu, vv = api.world_to_img(cam, x, y, z)
            assert abs(uu - u) < 0.05 and abs(vv - v) < 0.05   # the inverse polynomial is a fit, not exact
    a, b, ma, mb = (rng.integers(0, 256, 32).astype(np.uint8) for _ in range(4))
    assert api.DescriptorDistance64(a, b) == oa.distance64(a, b)
    assert api.DescriptorDistance64Masked(a, b, ma, mb) == oa.distance64_masked(a, b, ma, mb)


def test_argument_validation(api):
    from multicol_slam_b200.ctypes_defs import make_params
    lib = api.lib()
    h = C.c_void_p()
    assert lib.mcs_extractor_create(None, C.byref(h)) == api.MCS_ERR_INVALID
    assert lib.mcs_extractor_check_status(None, None) == api.MCS_ERR_INVALID
    p = make_params(use_agast=True)
    assert lib.mcs_extractor_create(C.byref(p), C.byref(h)) == api.MCS_ERR_UNSUPPORTED
    p = make_params(desc_size=24)
    assert lib.mcs_extractor_create(C.byref(p), C.byref(h)) == api.MCS_ERR_INVALID
    assert b"desc_size" in lib.mcs_last_error()


def test_no_cpu_fallback(api):
    if api.device_count() > 0:
        pytest.skip("GPU present")
    with pytest.raises(api.McsError) as e:
        api.mdBRIEFextractorOct()
    assert e.value.code == api.MCS_ERR_NO_DEVICE
    q = np.zeros((4, 32), np.uint8)
    with pytest.raises(api.McsError):
        api.hamming_topk(q, q, 2)


def test_bow_validation_and_no_cpu_fallback(api):
    """Vocabulary arguments are validated on the host before any device work; without a device the bag-of-words entry
    points fail with MCS_ERR_NO_DEVICE like the rest of the library (no CPU path)."""
    import pathlib
    voc = np.load(pathlib.Path(__file__).resolve().parent / "golden" / "voc_small_9_6.npz")
    bad = {k: voc[k].copy() for k in voc.files}
    bad["parent"][7] = 7                                   # a node that is its own parent
    with pytest.raises(api.McsError) as e:
        api.ORBVocabulary(bad)
    assert e.value.code == api.MCS_ERR_INVALID
    bad = {k: voc[k].copy() for k in voc.files}
    bad["word_node"][3] = 1                                # word id attached to an inner node
    with pytest.raises(api.McsError) as e:
        api.ORBVocabulary(bad)
    assert e.value.code == api.MCS_ERR_INVALID
    with pytest.raises(api.McsError) as e:
        api.ORBVocabulary(voc, scoring=9)
    assert e.value.code == api.MCS_ERR_INVALID
    if api.device_count() > 0:
        return
    with pytest.raises(api.McsError) as e:
        api.ORBVocabulary(voc)
    assert e.value.code == api.MCS_ERR_NO_DEVICE
    d = np.zeros((8, 32), np.uint8)
    fv = (np.array([1], np.int32), np.array([0, 8], np.int32), np.arange(8, dtype=np.int32))
    with pytest.raises(api.McsError) as e:
        api.cORBmatcher(0.9, False, 32, False).SearchByBoWFrame(d, fv, d, fv)
    assert e.value.code == api.MCS_ERR_NO_DEVICE


def test_search_by_bow_argument_validation(api):
    """malformed feature vectors are refused on the host (before any device work); a well-formed call gets past the validation
    (and, without a device, ends in MCS_ERR_NO_DEVICE)"""
    d = np.zeros((8, 32), np.uint8)
    m = api.cORBmatcher(0.9, False, 32, False)
    good = (np.array([1, 5], np.int32), np.array([0, 3, 8], np.int32), np.arange(8, dtype=np.int32))
    for bad in ((np.array([5, 1], np.int32), good[1], good[2]),                       # node ids not ascending
                (good[0], np.array([0, 9, 8], np.int32), good[2]),                    # offsets decreasing
                (good[0], good[1], np.array([0, 1, 2, 3, 4, 5, 6, 99], np.int32))):   # feature index out of range
        with pytest.raises(api.McsError) as e:
            m.SearchByBoWFrame(d, bad, d, good)
        assert e.value.code == api.MCS_ERR_INVALID
        with pytest.raises(api.McsError) as e:
            m.SearchByBoWFrame(d, good, d, bad)
        assert e.value.code == api.MCS_ERR_INVALID
    if api.device_count() == 0:
        with pytest.raises(api.McsError) as e:
            m.SearchByBoWFrame(d, good, d, good)
        assert e.value.code == api.MCS_ERR_NO_DEVICE
    else:
        n, out = m.SearchByBoWFrame(d, good, d, good)
        assert len(out) == 8
