"""ctypes wrapper of oracle/_ref/libmcs_ref.so: the REFERENCE's own extractor, camera model and misc helpers
(src/mdBRIEFextractorOct.cpp, src/cam_model_omni.cpp, src/misc.cpp) compiled where they lie by `make -C oracle ref`
against the stand-in OpenCV header oracle/ref_mcs/stub.  TEST INFRASTRUCTURE: pins oracle/mcs_oracle.cpp's extractor
restatement and generates tests/golden/ref_extract_*.npz (tests/golden/make_ref_extract_golden.py)."""
import ctypes as C
import os
import pathlib
import sys

import numpy as np

_HERE = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(_HERE.parent))
from multicol_slam_b200.ctypes_defs import KEYPOINT_DTYPE, Ocam, make_ocam, make_params  # noqa: E402

SO = _HERE / "_ref" / "libmcs_ref.so"
# the reference checkout `make -C oracle ref` compiles from (same default as oracle/Makefile)
REFERENCE_DIR = pathlib.Path(os.environ.get("MCS_REFERENCE_DIR", "/root/reference"))


def reference_present():
    """a readable reference checkout (os.path.isdir is False, not an error, where the path cannot be reached)"""
    return os.path.isdir(REFERENCE_DIR / "include") and os.access(REFERENCE_DIR / "include", os.R_OK | os.X_OK)
_lib = None


def available():
    return SO.exists()


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(SO))
        _lib.mcsref_extractor_create.restype = C.c_void_p
        _lib.mcsref_cv_fast_atan2.restype = C.c_float
        _lib.mcsref_cv_fast_atan2.argtypes = [C.c_float, C.c_float]
        _lib.mcsref_const.restype = C.c_double
        _lib.mcsref_cv_round.argtypes = [C.c_double]
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def set_deterministic(on):
    """True (default): monotonic heap during a call (reproducible pointer tie-break, one call at a time); False: stock allocator,
    re-entrant -- for timing the reference on many threads (bench.py --impl reference)"""
    lib().mcsref_set_deterministic(int(bool(on)))


def _oc(cam):
    return cam if isinstance(cam, Ocam) else make_ocam(cam)


class RefExtractor:
    """MultiColSLAM::mdBRIEFextractorOct of the reference; keyword arguments as multicol_slam_b200.ctypes_defs.make_params."""

    def __init__(self, **kw):
        self.params = make_params(**kw)
        self.h = C.c_void_p(lib().mcsref_extractor_create(C.byref(self.params)))
        self.nlevels, self.ds = self.params.nlevels, self.params.desc_size

    def capacity(self, width, height):
        """most keypoints DistributeOctTree can return for a width x height image: per level max(4 nIni, N + 2).  Its first pass
        divides each of the nIni = cvRound((maxX - minX) / (maxY - minY)) roots into at most 4 nodes, whatever the quota N; every
        later division adds at most 3 nodes and starts below N (src/mdBRIEFextractorOct.cpp:640, :693-854)."""
        q, _, isf, _ = self.tables()
        cap = 0
        for l in range(self.nlevels):
            w, h = lib().mcsref_cv_round(C.c_double(width * isf[l])), lib().mcsref_cv_round(C.c_double(height * isf[l]))
            n_ini = lib().mcsref_cv_round(C.c_double((w - 44) / (h - 44)))       # maxX - minX = w - 2 * (EDGE_THRESHOLD - 3)
            cap += max(4 * n_ini, int(q[l]) + 2)
        return cap

    def __del__(self):
        if getattr(self, "h", None):
            lib().mcsref_extractor_destroy(self.h)
            self.h = None

    def tables(self):
        L = self.nlevels
        q, sf, isf, um = np.zeros(L, np.int32), np.zeros(L), np.zeros(L), np.zeros(17, np.int32)
        lib().mcsref_extractor_tables(self.h, _p(q), _p(sf), _p(isf), _p(um))
        return q, sf, isf, um

    def extract(self, image, mask, cam):
        """operator() -> (kps structured array, desc [n,ds] u8, dmask [n,ds] u8)"""
        image = np.ascontiguousarray(image, np.uint8)
        mask = np.ascontiguousarray(mask, np.uint8)
        h, w = image.shape
        cap, ds = self.capacity(w, h), self.ds
        kps = np.zeros(cap, KEYPOINT_DTYPE)
        desc = np.zeros((cap, ds), np.uint8)
        dmask = np.zeros((cap, ds), np.uint8)
        n = C.c_int(0)
        oc = _oc(cam)
        st = lib().mcsref_extract(self.h, _p(image), w, h, image.strides[0], _p(mask), mask.strides[0], C.byref(oc),
                                  _p(kps), _p(desc), _p(dmask), cap, C.byref(n))
        assert st != -4, f"the reference returned {n.value} keypoints, above the bound {cap}"   # MCS_ERR_CAPACITY: nothing copied
        if st != 0:
            raise RuntimeError(f"reference extract failed {st}")
        return kps[:n.value].copy(), desc[:n.value].copy(), dmask[:n.value].copy()

    def debug_read(self, level, what):
        """what: 0 image level as the last call left it (blurred when the level had keypoints), 1 mask level, 2 level incl. ring"""
        w, h = C.c_int(0), C.c_int(0)
        buf = np.zeros(1 << 23, np.uint8)
        st = lib().mcsref_debug_read(self.h, level, what, _p(buf), buf.nbytes, C.byref(w), C.byref(h))
        if st != 0:
            raise RuntimeError(f"debug_read {st}")
        return buf[:w.value * h.value].reshape(h.value, w.value).copy()

    def octree(self, xyr, minX, maxX, minY, maxY, N):
        xyr = np.ascontiguousarray(xyr, np.float32)
        out = np.zeros((max(len(xyr), 1), 3), np.float32)
        n = lib().mcsref_octree(self.h, _p(xyr), len(xyr), minX, maxX, minY, maxY, N, _p(out), out.shape[0])
        return out[:n].copy()


def world_to_img(cam, x, y, z):
    u, v = C.c_double(), C.c_double()
    lib().mcsref_cam_world_to_img(C.byref(_oc(cam)), C.c_double(x), C.c_double(y), C.c_double(z), C.byref(u), C.byref(v))
    return u.value, v.value


def world_to_img_many(cam, xyz):
    """world_to_img of each row of xyz [n,3] -> [n,2]"""
    return np.array([world_to_img(cam, float(p[0]), float(p[1]), float(p[2])) for p in np.asarray(xyz, np.float64)]).reshape(-1, 2)


def img_to_world(cam, u, v):
    x, y, z = C.c_double(), C.c_double(), C.c_double()
    lib().mcsref_cam_img_to_world(C.byref(_oc(cam)), C.c_double(u), C.c_double(v), C.byref(x), C.byref(y), C.byref(z))
    return x.value, y.value, z.value


def undistort(cam, px, py):
    x, y = C.c_double(), C.c_double()
    lib().mcsref_cam_undistort(C.byref(_oc(cam)), C.c_double(px), C.c_double(py), C.byref(x), C.byref(y))
    return x.value, y.value


def mirror_mask(cam):
    oc = _oc(cam)
    out = np.zeros((oc.height, oc.width), np.uint8)
    lib().mcsref_cam_mirror_mask(C.byref(oc), _p(out))
    return out


def points_in_mask(cam, uv):
    uv = np.ascontiguousarray(uv, np.float64)
    out = np.zeros(len(uv), np.uint8)
    lib().mcsref_cam_points_in_mask(C.byref(_oc(cam)), _p(uv), len(uv), _p(out))
    return out


def check_epipolar(ray1, ray2, E, thresh):
    r1, r2, e = (np.ascontiguousarray(a, np.float64) for a in (ray1, ray2, E))
    return bool(lib().mcsref_check_epipolar(_p(r1), _p(r2), _p(e), C.c_double(thresh)))


def compute_E(T1, T2):
    a, b = np.ascontiguousarray(T1, np.float64), np.ascontiguousarray(T2, np.float64)
    e = np.zeros((3, 3))
    lib().mcsref_compute_E(_p(a), _p(b), _p(e))
    return e


# ---- the stand-in's OpenCV primitives (pinned against the real cv2 by oracle/pin_ref.py) ----
def cv_resize(src, dw, dh, interpolation):
    src = np.ascontiguousarray(src, np.uint8)
    dst = np.zeros((dh, dw), np.uint8)
    lib().mcsref_cv_resize(_p(src), src.shape[1], src.shape[0], _p(dst), dw, dh, interpolation)
    return dst


def cv_make_border(src, b, reflect=True):
    src = np.ascontiguousarray(src, np.uint8)
    dst = np.zeros((src.shape[0] + 2 * b, src.shape[1] + 2 * b), np.uint8)
    lib().mcsref_cv_make_border(_p(src), src.shape[1], src.shape[0], b, int(reflect), _p(dst))
    return dst


def cv_box5_roi(buf, x0, y0, w, h):
    """5x5 normalized box filter in place on the ROI of a copy of buf; returns the whole buffer"""
    buf = np.ascontiguousarray(buf, np.uint8).copy()
    lib().mcsref_cv_box5(_p(buf), buf.shape[1], buf.shape[0], x0, y0, w, h)
    return buf


def cv_fast_atan2(y, x):
    return lib().mcsref_cv_fast_atan2(C.c_float(y), C.c_float(x))


def cv_fast(img, mask, threshold):
    """FAST-9/16 + NMS + mask filter on a (possibly strided) 2-D view; -> [n,3] float32 (x, y, response)"""
    assert img.strides[1] == 1
    out = np.zeros((img.shape[0] * img.shape[1] + 1, 3), np.float32)
    n = lib().mcsref_cv_fast(_p(img), img.shape[1], img.shape[0], img.strides[0], _p(mask), mask.strides[0] if mask is not None else 0,
                             threshold, _p(out), out.shape[0])
    return out[:n].copy()
