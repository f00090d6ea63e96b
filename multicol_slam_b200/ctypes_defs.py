"""ctypes mirrors of the POD types in include/mcs_b200.h (shared by the product wrapper and by the
test-only oracle wrapper)."""
import ctypes as C

MAX_LEVELS = 16


class Ocam(C.Structure):
    _fields_ = [("c", C.c_double), ("d", C.c_double), ("e", C.c_double), ("u0", C.c_double), ("v0", C.c_double),
                ("pol", C.c_double * 5), ("inv_pol", C.c_double * 12),
                ("width", C.c_int32), ("height", C.c_int32), ("mirror_mask", C.c_int32), ("_pad", C.c_int32)]


class ExtractorParams(C.Structure):
    _fields_ = [("nfeatures", C.c_int32), ("scale_factor", C.c_float), ("nlevels", C.c_int32),
                ("edge_threshold", C.c_int32), ("first_level", C.c_int32), ("score_type", C.c_int32),
                ("patch_size", C.c_int32), ("fast_threshold", C.c_int32), ("use_agast", C.c_int32),
                ("fast_agast_type", C.c_int32), ("do_dbrief", C.c_int32), ("learn_masks", C.c_int32),
                ("desc_size", C.c_int32)]


class ExtractorInfo(C.Structure):
    _fields_ = [("nlevels", C.c_int32), ("capacity", C.c_int32), ("desc_size", C.c_int32),
                ("features_per_level", C.c_int32 * MAX_LEVELS),
                ("scale_factor", C.c_double * MAX_LEVELS), ("inv_scale_factor", C.c_double * MAX_LEVELS)]


class FrameView(C.Structure):
    _fields_ = [("n_cams", C.c_int32), ("n_keys", C.c_int32), ("keys", C.c_void_p), ("key_cam", C.c_void_p),
                ("desc", C.c_void_p), ("dmask", C.c_void_p), ("cam_width", C.c_void_p), ("cam_height", C.c_void_p),
                ("dim", C.c_int32), ("n_levels", C.c_int32), ("scale_factors", C.c_void_p)]


class WindowQuery(C.Structure):
    _fields_ = [("cam", C.c_int32), ("min_level", C.c_int32), ("max_level", C.c_int32), ("desc_index", C.c_int32),
                ("x", C.c_double), ("y", C.c_double), ("r", C.c_double)]


class MapPointView(C.Structure):
    _fields_ = [("n_points", C.c_int32), ("bad", C.c_void_p), ("in_view", C.c_void_p), ("level", C.c_void_p),
                ("proj_x", C.c_void_p), ("proj_y", C.c_void_p), ("view_cos", C.c_void_p), ("desc", C.c_void_p),
                ("dmask", C.c_void_p)]


class MapPointDevView(C.Structure):
    """mcs_mappoint_dev_view: the same fields as MapPointView, every pointer in device memory"""
    _fields_ = MapPointView._fields_


class PackedFrame(C.Structure):
    """mcs_packed_frame: camera c = global image first_image + c of n_parts consecutive packed layouts of part_images images"""
    _fields_ = [("packed_dev", C.c_void_p), ("n_parts", C.c_int32), ("part_images", C.c_int32), ("first_image", C.c_int32)]


class BowFrame(C.Structure):
    """mcs_bow_frame: a frame in packed feature buffers with its FeatureVector (CSR, slots) and, for a key frame, its slot-indexed
    map-point ids, all device pointers"""
    _fields_ = [("frame", PackedFrame), ("fv_nodes_dev", C.c_void_p), ("fv_offsets_dev", C.c_void_p), ("n_fv_dev", C.c_void_p),
                ("fv_features_dev", C.c_void_p), ("mp_dev", C.c_void_p)]


class FuseTarget(C.Structure):
    """mcs_fuse_target: a Fuse target key frame in packed feature buffers, its slot-indexed map-point ids (device, or NULL), the
    MtMc_inv of the pose to project with (host [n_cams * 16]) and the centre of the depth test"""
    _fields_ = [("frame", PackedFrame), ("mp_dev", C.c_void_p), ("mtmc_inv", C.c_void_p), ("ow", C.c_double * 3)]


class MpKeyFrame(C.Structure):
    """mcs_mp_keyframe: a key frame in packed feature buffers, its GetCameraCenter() and isBad()"""
    _fields_ = [("frame", PackedFrame), ("ow", C.c_double * 3), ("bad", C.c_int32)]


def set_prototypes(lib):
    """argument types of the entry points whose many arguments are easiest to get wrong from Python"""
    P, I, D = C.c_void_p, C.c_int32, C.c_double
    f = lib.mcs_search_by_projection_last_device
    f.argtypes = [C.POINTER(PackedFrame), C.POINTER(PackedFrame), I, I, I, P, P, I, P, P, P, P, I, P, P, D, I, I, P, P, P, P, P]
    f.restype = C.c_int
    f = lib.mcs_window_search_device
    f.argtypes = [C.POINTER(PackedFrame), C.POINTER(PackedFrame), I, I, I, P, P, P, I, P, I, I, I, D, I, I, P, P, P, P, P]
    f.restype = C.c_int
    f = lib.mcs_search_by_projection_frames_device
    f.argtypes = [C.POINTER(PackedFrame), C.POINTER(PackedFrame), I, I, I, P, P, P, P, I, P, P, I, D, I, I, P, P, P, P, P]
    f.restype = C.c_int
    f = lib.mcs_search_for_initialization_device
    f.argtypes = [C.POINTER(PackedFrame), C.POINTER(PackedFrame), I, I, I, P, P, P, I, D, I, I, P, P, P, P]
    f.restype = C.c_int
    f = lib.mcs_search_for_initialization_seed_device
    f.argtypes = [C.POINTER(PackedFrame), I, I, I, P, P]
    f.restype = C.c_int
    f = lib.mcs_fuse_device
    f.argtypes = [C.POINTER(FuseTarget), I, I, I, I, P, P, I, P, I, P, I, I, P, P, P, P, P, P, D, I, I, P, I, P, P, P]
    f.restype = C.c_int
    f = lib.mcs_search_by_sim3_device
    f.argtypes = [C.POINTER(PackedFrame), C.POINTER(PackedFrame), I, I, I, P, P, I, P, P, P, P, D, P, P, D, P, P, I, P, P, P, P, P, P, P, I, I,
                  P, P, P, P]
    f.restype = C.c_int
    f = lib.mcs_search_by_bow_keyframes_device
    f.argtypes = [C.POINTER(PackedFrame), P, C.POINTER(PackedFrame), P, I, I, I, I, I, P, I, D, I, P, P, P, P, P]
    f.restype = C.c_int
    f = lib.mcs_search_for_triangulation_device
    f.argtypes = [C.POINTER(PackedFrame), P, C.POINTER(PackedFrame), P, I, I, I, P, P, D, I, I, P, P, P, P]
    f.restype = C.c_int
    f = lib.mcs_search_by_projection_scw_device
    f.argtypes = [C.POINTER(PackedFrame), I, I, I, P, P, I, P, P, P, P, I, I, P, P, P, P, P, P, I, I, I, P, P, P, P, P]
    f.restype = C.c_int
    f = lib.mcs_update_mappoints_device
    f.argtypes = [C.POINTER(MpKeyFrame), I, I, I, I, I, P, I, I, P, I, I, P, P, P, P, P, P, P, P, P, P, P, P, P]
    f.restype = C.c_int
    f = lib.mcs_vocabulary_level_nodes
    f.argtypes = [P, I, C.POINTER(I)]
    f.restype = C.c_int
    f = lib.mcs_bow_vectors_device
    f.argtypes = [P, C.POINTER(PackedFrame), I, I, I, I, I, P, P, P, P, P, P, P, P, P, P, P, P]
    f.restype = C.c_int
    f = lib.mcs_search_by_bow_device
    f.argtypes = [C.POINTER(BowFrame), I, C.POINTER(BowFrame), I, I, I, I, I, P, I, D, I, P, P, P, P, P]
    f.restype = C.c_int


import numpy as np

# numpy dtype binary-compatible with mcs_keypoint / cv::KeyPoint (28 bytes)
KEYPOINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                           ("octave", "<i4"), ("class_id", "<i4")])
WINDOW_QUERY_DTYPE = np.dtype([("cam", "<i4"), ("min_level", "<i4"), ("max_level", "<i4"), ("desc_index", "<i4"),
                               ("x", "<f8"), ("y", "<f8"), ("r", "<f8")])
assert KEYPOINT_DTYPE.itemsize == 28 and WINDOW_QUERY_DTYPE.itemsize == 40


def make_params(nfeatures=1000, scale_factor=1.2, nlevels=8, fast_threshold=20, do_dbrief=False, learn_masks=False,
                desc_size=32, use_agast=False, fast_agast_type=2):
    """Same defaults as the reference constructor (include/mdBRIEFextractorOct.h:340-352)."""
    return ExtractorParams(nfeatures, scale_factor, nlevels, 25, 0, 0, 32, fast_threshold, int(use_agast),
                           fast_agast_type, int(do_dbrief), int(learn_masks), desc_size)


def make_ocam(d):
    o = Ocam()
    o.c, o.d, o.e, o.u0, o.v0 = d["c"], d["d"], d["e"], d["u0"], d["v0"]
    for i in range(5):
        o.pol[i] = d["pol"][i] if i < len(d["pol"]) else 0.0
    for i in range(12):
        o.inv_pol[i] = d["inv_pol"][i] if i < len(d["inv_pol"]) else 0.0
    o.width, o.height, o.mirror_mask = d["width"], d["height"], d.get("mirror_mask", 1)
    return o
