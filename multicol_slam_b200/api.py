"""ctypes binding of libmcs_b200.so (include/mcs_b200.h) plus thin Python mirrors of the reference's
operator/matcher interface for this path:

    mdBRIEFextractorOct(...)(image, mask, camModel) -> keypoints, descriptors, descriptorMasks
        (ref include/mdBRIEFextractorOct.h:333-368, src/mdBRIEFextractorOct.cpp:1244-1337)
    cORBmatcher(nnratio, checkOri, featDim, havingMasks).SearchByProjection / SearchForInitialization /
        SearchByBoW(KF1, KF2)   (ref include/cORBmatcher.h:58-158, src/cORBmatcher.cpp:46-166, 579-726, 885-966)

There is no CPU fallback: the shared library must be present (build it with `python __graft_entry__.py`)
and every compute call needs an sm_90 (H100) device, otherwise it raises.
"""
import ctypes as C
import math
import pathlib

import numpy as np

from .ctypes_defs import (MAX_LEVELS, BowFrame, ExtractorInfo, ExtractorParams, FrameView, FuseTarget, KEYPOINT_DTYPE, MapPointDevView,
                          MapPointView, MpKeyFrame, Ocam, PackedFrame, WINDOW_QUERY_DTYPE, make_ocam, make_params, set_prototypes)

_PKG = pathlib.Path(__file__).resolve().parent
_LIB_PATH = _PKG / "libmcs_b200.so"
_lib = None

MCS_OK, MCS_ERR_INVALID, MCS_ERR_UNSUPPORTED, MCS_ERR_CUDA, MCS_ERR_CAPACITY, MCS_ERR_NO_DEVICE = 0, -1, -2, -3, -4, -5


class McsError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libmcs_b200 error {code}: {msg}")
        self.code = code


def lib():
    """Load libmcs_b200.so; fails loudly when the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise ImportError(f"{_LIB_PATH} is missing: the CUDA extension is mandatory (run __graft_entry__.build())")
        _lib = C.CDLL(str(_LIB_PATH))
        _lib.mcs_last_error.restype = C.c_char_p
        _lib.mcs_slot_bytes.restype = C.c_size_t
        set_prototypes(_lib)
    return _lib


def _check(rc):
    if rc != 0:
        raise McsError(rc, lib().mcs_last_error().decode())


def _p(a):
    if a is None:
        return None
    return a.ctypes.data_as(C.c_void_p)


def _dptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _contig(a, dtype):
    """np.ascontiguousarray(a, dtype), None passed through (an optional host array)"""
    return None if a is None else np.ascontiguousarray(a, dtype)


def _stream_handle(stream, dev):
    import torch
    return C.c_void_p(stream.cuda_stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream)


def _on_stream(stream, dev):
    """the context that puts the fills of a call's new output tensors on the stream the call runs on: `stream`, or dev's current one"""
    import torch
    return torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream(dev))


def _ocams(cams):
    """the camera models as an mcs_ocam array"""
    return (Ocam * len(cams))(*[as_ocam(c) for c in cams])


def _cam_wh(cam_sizes):
    """[(w, h)] per camera -> (widths, heights) int32 arrays"""
    return np.ascontiguousarray([s[0] for s in cam_sizes], np.int32), np.ascontiguousarray([s[1] for s in cam_sizes], np.int32)


def _extract_inputs(masks, cams, cam_of_image=None):
    """the host inputs of an extraction call: masks [n_cams,H,W] u8, the camera models as an mcs_ocam array, cam_of_image i32"""
    return np.ascontiguousarray(masks, np.uint8), _ocams(cams), _contig(cam_of_image, np.int32)


def device_count():
    return lib().mcs_device_count()


def as_ocam(cam):
    return cam if isinstance(cam, Ocam) else make_ocam(cam)


def mirror_mask(cam):
    oc = as_ocam(cam)
    out = np.zeros((oc.height, oc.width), np.uint8)
    _check(lib().mcs_cam_mirror_mask(C.byref(oc), _p(out)))
    return out


def distort_table(cam):
    """mcs_cam_distort_table: the per-radius table of the descriptor kernel's tiers 1 and 2 for one camera -> float64 [n, row]"""
    oc = as_ocam(cam)
    n, row = C.c_int32(0), C.c_int32(0)
    _check(lib().mcs_cam_distort_table(C.byref(oc), None, 0, C.byref(n), C.byref(row)))
    out = np.zeros((n.value, row.value), np.float64)
    _check(lib().mcs_cam_distort_table(C.byref(oc), _p(out), n.value, C.byref(n), C.byref(row)))
    return out


def octree_plan(width, height, **params):
    """mcs_extractor_octree_plan (host only): -> (return code, node_table, nodes_ini [nlevels], sel_cap [nlevels], capacity) of
    width x height images for an extractor made with make_params(**params)"""
    p = make_params(**params)
    nt, cap = C.c_int32(0), C.c_int32(0)
    ni, sc = np.zeros(MAX_LEVELS, np.int32), np.zeros(MAX_LEVELS, np.int32)
    rc = lib().mcs_extractor_octree_plan(C.byref(p), width, height, C.byref(nt), _p(ni), _p(sc), C.byref(cap))
    return rc, nt.value, ni[:p.nlevels], sc[:p.nlevels], cap.value


def world_to_img(cam, x, y, z):
    oc = as_ocam(cam)
    u, v = C.c_double(), C.c_double()
    lib().mcs_cam_world_to_img(C.byref(oc), C.c_double(x), C.c_double(y), C.c_double(z), C.byref(u), C.byref(v))
    return u.value, v.value


def img_to_world(cam, u, v):
    oc = as_ocam(cam)
    x, y, z = C.c_double(), C.c_double(), C.c_double()
    lib().mcs_cam_img_to_world(C.byref(oc), C.c_double(u), C.c_double(v), C.byref(x), C.byref(y), C.byref(z))
    return x.value, y.value, z.value


class mdBRIEFextractorOct:
    """Same constructor arguments, order and defaults as the reference class."""
    HARRIS_SCORE, FAST_SCORE = 0, 1

    def __init__(self, nfeatures=1000, scaleFactor=1.2, nlevels=8, edgeThreshold=25, firstLevel=0, scoreType=0,
                 patchSize=32, fastThreshold=20, useAgast=False, fastAgastType=2, do_dBrief=False, learnMasks=False,
                 descSize=32):
        self.params = ExtractorParams(nfeatures, scaleFactor, nlevels, edgeThreshold, firstLevel, scoreType, patchSize,
                                      fastThreshold, int(useAgast), fastAgastType, int(do_dBrief), int(learnMasks), descSize)
        self._h = C.c_void_p()
        _check(lib().mcs_extractor_create(C.byref(self.params), C.byref(self._h)))
        self.info = ExtractorInfo()
        _check(lib().mcs_extractor_get_info(self._h, C.byref(self.info)))

    def __del__(self):
        if getattr(self, "_h", None):
            lib().mcs_extractor_destroy(self._h)
            self._h = None

    # reference getters
    def GetLevels(self):
        return self.info.nlevels

    def GetScaleFactor(self):
        return float(np.float32(self.params.scale_factor))

    def GetMasksLearned(self):
        return bool(self.params.learn_masks)

    def GetDescriptorSize(self):
        return self.info.desc_size

    @property
    def capacity(self):
        return self.info.capacity

    def __call__(self, image, mask, camModel):
        """operator(): -> (keypoints structured array [n], descriptors [n,descSize] u8, descriptorMasks [n,descSize] u8).
        An empty image returns None (the reference returns without touching its outputs)."""
        if image is None or image.size == 0:
            return None
        image = np.ascontiguousarray(image, np.uint8)
        mask = np.ascontiguousarray(mask, np.uint8)
        cap, ds = self.info.capacity, self.info.desc_size
        kps = np.zeros(cap, KEYPOINT_DTYPE)
        desc = np.zeros((cap, ds), np.uint8)
        dmask = np.zeros((cap, ds), np.uint8)
        n = C.c_int32(0)
        oc = as_ocam(camModel)
        h, w = image.shape
        _check(lib().mcs_extract(self._h, _p(image), w, h, image.strides[0], _p(mask), mask.strides[0], C.byref(oc),
                                 _p(kps), _p(desc), _p(dmask), cap, C.byref(n)))
        return kps[:n.value].copy(), desc[:n.value].copy(), dmask[:n.value].copy()

    def extract_batch(self, images, masks, cams, cam_of_image):
        """images [B,H,W] u8 host; masks [n_cams,H,W]; cams list; -> (kps [B,cap], desc [B,cap,ds], dmask, counts [B])"""
        images = np.ascontiguousarray(images, np.uint8)
        masks, ocs, coi = _extract_inputs(masks, cams, cam_of_image)
        B, H, W = images.shape
        cap, ds = self.info.capacity, self.info.desc_size
        kps = np.zeros((B, cap), KEYPOINT_DTYPE)
        desc = np.zeros((B, cap, ds), np.uint8)
        dmask = np.zeros((B, cap, ds), np.uint8)
        counts = np.zeros(B, np.int32)
        _check(lib().mcs_extract_batch(self._h, B, _p(images), W, H, W, _p(masks), ocs, len(cams), _p(coi), _p(kps),
                                       _p(desc), _p(dmask), _p(counts), cap))
        return kps, desc, dmask, counts

    def extract_batch_device(self, images_t, masks, cams, cam_of_image, out=None, stream=None, width=None):
        """torch CUDA tensors in/out (plumbing only): images_t [B,H,P] uint8 cuda, P = row pitch >= width (a 16-byte
        aligned pitch lets K1 use 128-bit loads).  Returns dict of cuda tensors {kps [B,cap,7] int32-view,
        desc [B,cap,ds], dmask, counts [B]}; asynchronous on `stream` when given."""
        import torch
        assert images_t.is_cuda and images_t.dtype == torch.uint8 and images_t.is_contiguous()
        B, H, P = images_t.shape
        W = P if width is None else width
        cap, ds = self.info.capacity, self.info.desc_size
        dev = images_t.device
        if out is None:
            out = dict(kps=torch.empty((B, cap, 7), dtype=torch.int32, device=dev),
                       desc=torch.empty((B, cap, ds), dtype=torch.uint8, device=dev),
                       dmask=torch.empty((B, cap, ds), dtype=torch.uint8, device=dev),
                       counts=torch.empty((B,), dtype=torch.int32, device=dev))
        masks, ocs, coi = _extract_inputs(masks, cams, cam_of_image)
        _check(lib().mcs_extract_batch_device(self._h, B, _dptr(images_t), W, H, P, _p(masks), ocs, len(cams), _p(coi), _dptr(out["kps"]),
                                              _dptr(out["desc"]), _dptr(out["dmask"]), _dptr(out["counts"]), cap,
                                              _stream_handle(stream, dev)))
        return out

    def packed_views(self, packed_t, n_images):
        """views of a packed feature buffer (mcs_packed_layout) as the four output tensors"""
        import torch
        from . import rig
        cap, ds = self.info.capacity, self.info.desc_size
        offs, total = rig.packed_layout(n_images, cap, ds)
        assert packed_t.numel() >= total
        return dict(counts=packed_t[offs[0]:offs[0] + 4 * n_images].view(torch.int32),
                    kps=packed_t[offs[1]:offs[1] + n_images * cap * 28].view(torch.int32).view(n_images, cap, 7),
                    desc=packed_t[offs[2]:offs[2] + n_images * cap * ds].view(n_images, cap, ds),
                    dmask=packed_t[offs[3]:offs[3] + n_images * cap * ds].view(n_images, cap, ds))

    def extract_batch_packed_device(self, images_t, masks, cams, cam_of_image, packed_t, stream=None, width=None):
        """mcs_extract_batch_packed_device: K3 writes counts | keypoints | descriptors | masks straight into packed_t (uint8
        cuda tensor of rig.packed_layout(B, capacity, descSize)[1] bytes) -- the buffer mcs_allgather_features exchanges."""
        B, H, P = images_t.shape
        W = P if width is None else width
        masks, ocs, coi = _extract_inputs(masks, cams, cam_of_image)
        _check(lib().mcs_extract_batch_packed_device(self._h, B, _dptr(images_t), W, H, P, _p(masks), ocs, len(cams), _p(coi),
                                                     _dptr(packed_t), self.info.capacity, _stream_handle(stream, images_t.device)))
        return self.packed_views(packed_t, B)

    def extract_match_stream(self, images, masks, cams, K=2, out=None, packed_t=None, greedy=None):
        """images [F,C,H,W] u8 host (frame-major).  Extract every image and brute-force match each (frame,cam)
        against (frame-1,cam).  Returns dict(kps [F*C,cap], desc, dmask, counts, match_idx [F*C,cap,K], match_dist).
        `out` may hold preallocated (e.g. pinned) numpy arrays with the same keys."""
        images = np.ascontiguousarray(images, np.uint8)
        masks, ocs, _ = _extract_inputs(masks, cams)
        F, Cn, H, W = images.shape
        cap, ds, B = self.info.capacity, self.info.desc_size, F * Cn
        if out is None:
            out = dict(kps=np.zeros((B, cap), KEYPOINT_DTYPE), desc=np.zeros((B, cap, ds), np.uint8),
                       dmask=np.zeros((B, cap, ds), np.uint8), counts=np.zeros(B, np.int32),
                       match_idx=np.zeros((B, cap, K), np.int32), match_dist=np.zeros((B, cap, K), np.int32))
        if packed_t is not None or greedy is not None:
            # packed_t: features also stay in the caller's packed exchange buffer on the GPU; greedy = (th_low, nnratio): the greedy
            # acceptance of SearchByBoW(KF1, KF2) on the device -> out["matches12"] [B,cap], out["nmatches"] [B], out["redo"] [B]
            th, ratio = greedy if greedy is not None else (0, 0.0)
            if greedy is not None:
                for k, shp in (("matches12", (B, cap)), ("nmatches", (B,)), ("redo", (B,))):
                    if k not in out:
                        out[k] = np.zeros(shp, np.int32)
            _check(lib().mcs_extract_match_stream_packed(self._h, F, Cn, _p(images), W, H, W, _p(masks), ocs, _p(out["kps"]),
                                                         _p(out["desc"]), _p(out["dmask"]), _p(out["counts"]), cap, K,
                                                         _p(out["match_idx"]), _p(out["match_dist"]),
                                                         _dptr(packed_t), int(th),
                                                         C.c_double(ratio), _p(out.get("matches12")) if greedy is not None else None,
                                                         _p(out.get("nmatches")) if greedy is not None else None,
                                                         _p(out.get("redo")) if greedy is not None else None))
            return out
        _check(lib().mcs_extract_match_stream(self._h, F, Cn, _p(images), W, H, W, _p(masks), ocs, _p(out["kps"]),
                                              _p(out["desc"]), _p(out["dmask"]), _p(out["counts"]), cap, K,
                                              _p(out["match_idx"]), _p(out["match_dist"])))
        return out

    def set_profiling(self, enable=True):
        _check(lib().mcs_extractor_set_profiling(self._h, int(enable)))

    def tier_stats(self, enable=True):
        """K3 diagnostics: (tier 1, tier 1 repaired, tier 2, tier 3) pattern counts since counting was switched on; enable/disable counting"""
        out = np.zeros(4, np.int64)
        _check(lib().mcs_extractor_tier_stats(self._h, int(enable), _p(out)))
        return out

    def check_status(self, stream=None):
        """mcs_extractor_check_status: overflow report of the last asynchronous extract call (raises MCS_ERR_CAPACITY); synchronises the stream"""
        st = C.c_void_p(stream.cuda_stream) if stream is not None else None
        _check(lib().mcs_extractor_check_status(self._h, st))

    def graph_replays(self):
        """calls served by replaying the cached CUDA graph of the per-frame sequence (mcs_extractor_graph_replays)"""
        n = C.c_int64(0)
        _check(lib().mcs_extractor_graph_replays(self._h, C.byref(n)))
        return n.value

    def get_timings(self):
        """(K1 pyramid+blur+FAST all levels, K2 octree, K3 describe) of the last extract call, milliseconds."""
        ms = (C.c_float * 3)()
        _check(lib().mcs_extractor_get_timings(self._h, ms))
        return tuple(ms)

    def debug_read(self, level, what, image_index=0):
        w, h = C.c_int32(0), C.c_int32(0)
        buf = np.zeros(1 << 24, np.uint8)
        _check(lib().mcs_extractor_debug_read(self._h, image_index, level, what, _p(buf), C.c_size_t(buf.nbytes), C.byref(w), C.byref(h)))
        if what == 3:
            return buf[:w.value * 12].view(np.int32).reshape(-1, 3).copy()
        return buf[:w.value * h.value].reshape(h.value, w.value).copy()


# ---- matcher --------------------------------------------------------------------------------------
def DescriptorDistance64(a, b, dim=32):
    a = np.ascontiguousarray(a, np.uint8)
    b = np.ascontiguousarray(b, np.uint8)
    return lib().mcs_descriptor_distance64(_p(a), _p(b), dim)


def DescriptorDistance64Masked(a, b, ma, mb, dim=32):
    a, b, ma, mb = (np.ascontiguousarray(v, np.uint8) for v in (a, b, ma, mb))
    return lib().mcs_descriptor_distance64_masked(_p(a), _p(b), _p(ma), _p(mb), dim)


def hamming_topk(q, d, K=2, qmask=None, dmask=None, db_skip=None):
    q = np.ascontiguousarray(q, np.uint8)
    d = np.ascontiguousarray(d, np.uint8)
    qmask, dmask, db_skip = (_contig(a, np.uint8) for a in (qmask, dmask, db_skip))
    nq, dim = q.shape
    idx = np.zeros((nq, K), np.int32)
    dist = np.zeros((nq, K), np.int32)
    _check(lib().mcs_hamming_topk(_p(q), _p(qmask), nq, _p(d), _p(dmask), d.shape[0], _p(db_skip), dim, K, _p(idx), _p(dist)))
    return idx, dist


def hamming_topk_device(q_t, d_t, K=2, qmask_t=None, dmask_t=None, skip_t=None, out=None, stream=None):
    """torch CUDA uint8 tensors [nq,dim] / [nd,dim] -> (idx [nq,K] int32, dist [nq,K] int32) cuda tensors."""
    import torch
    nq, dim = q_t.shape
    dev = q_t.device
    if out is None:
        out = (torch.empty((nq, K), dtype=torch.int32, device=dev), torch.empty((nq, K), dtype=torch.int32, device=dev))
    st = _stream_handle(stream, dev)
    _check(lib().mcs_hamming_topk_device(_dptr(q_t), _dptr(qmask_t), nq, _dptr(d_t), _dptr(dmask_t), d_t.shape[0], _dptr(skip_t), dim, K,
                                         _dptr(out[0]), _dptr(out[1]), st))
    return out


def match_stream_device(desc_t, dmask_t, counts_t, n_frames, n_cams, K=2, out=None, stream=None):
    """torch CUDA tensors: desc [F*C,cap,dim] u8, dmask same or None, counts [F*C] i32 -> (idx, dist) [F*C,cap,K] i32."""
    import torch
    B, cap, dim = desc_t.shape
    dev = desc_t.device
    if out is None:
        out = (torch.empty((B, cap, K), dtype=torch.int32, device=dev), torch.empty((B, cap, K), dtype=torch.int32, device=dev))
    st = _stream_handle(stream, dev)
    _check(lib().mcs_match_stream_device(_dptr(desc_t), _dptr(dmask_t), _dptr(counts_t), n_frames, n_cams, cap, dim, K, _dptr(out[0]),
                                         _dptr(out[1]), st))
    return out


def match_stream_replay_device(idx_t, dist_t, counts_t, desc_t, dmask_t, n_frames, n_cams, th_low, nnratio, out=None, stream=None):
    """mcs_match_stream_replay_device: greedy SearchByBoW acceptance over the K-best lists, on the device.
    -> (matches12 [F*C,cap] i32, nmatches [F*C] i32, redo [F*C] i32) cuda tensors"""
    import torch
    B, cap, K = idx_t.shape
    dev = idx_t.device
    if out is None:
        out = (torch.empty((B, cap), dtype=torch.int32, device=dev), torch.empty(B, dtype=torch.int32, device=dev),
               torch.empty(B, dtype=torch.int32, device=dev))
    st = _stream_handle(stream, dev)
    _check(lib().mcs_match_stream_replay_device(_dptr(idx_t), _dptr(dist_t), _dptr(counts_t), _dptr(desc_t), _dptr(dmask_t), n_frames, n_cams, cap,
                                                desc_t.shape[-1], K, int(th_low), C.c_double(nnratio), _dptr(out[0]), _dptr(out[1]), _dptr(out[2]), st))
    return out


def match_bruteforce_batch_device(q_t, qmask_t, valid1, seg_start, d_t, dmask_t, valid2, th_low, nnratio, stream=None):
    """mcs_match_bruteforce_batch_device: the query sets q_t[seg_start[s]:seg_start[s+1]] each matched against the database as a separate
    SearchByBoW(KF1, KF2) would, K-best lists of all sets from one launch.  Returns (nmatches [n_seg] numpy, matches12 numpy)."""
    nq, dim = q_t.shape
    nd = d_t.shape[0]
    seg = np.ascontiguousarray(seg_start, np.int32)
    assert seg[-1] == nq
    v1, v2 = _contig(valid1, np.uint8), _contig(valid2, np.uint8)
    m12 = np.zeros(nq, np.int32)
    nm = np.zeros(len(seg) - 1, np.int32)
    st = _stream_handle(stream, q_t.device)
    _check(lib().mcs_match_bruteforce_batch_device(_dptr(q_t), _dptr(qmask_t), _p(v1), _p(seg), len(seg) - 1, _dptr(d_t), _dptr(dmask_t), _p(v2), nd, dim,
                                                   int(th_low), C.c_double(nnratio), _p(m12), _p(nm), st))
    return nm, m12


def match_stream_greedy_device(desc_t, dmask_t, counts_t, n_frames, n_cams, th_low, nnratio, out=None, stream=None):
    """mcs_match_stream_greedy_device: every image against the same camera's image one frame earlier with SearchByBoW(KF1, KF2)'s
    acceptance rule, lists + replay in one call.  desc_t/dmask_t [F*C,cap,dim] u8 cuda, counts_t [F*C] i32 cuda.
    -> (matches12 [F*C,cap] i32, nmatches [F*C] i32) cuda tensors"""
    import torch
    B, cap, dim = desc_t.shape
    dev = desc_t.device
    if out is None:
        out = (torch.empty((B, cap), dtype=torch.int32, device=dev), torch.empty(B, dtype=torch.int32, device=dev))
    st = _stream_handle(stream, dev)
    _check(lib().mcs_match_stream_greedy_device(_dptr(desc_t), _dptr(dmask_t), _dptr(counts_t), n_frames, n_cams, cap, dim, int(th_low),
                                                C.c_double(nnratio), _dptr(out[0]), _dptr(out[1]), st))
    return out


def match_bruteforce_device(q_t, qmask_t, valid1, d_t, dmask_t, valid2, th_low, nnratio, stream=None):
    """mcs_match_bruteforce_device: SearchByBoW(KF1, KF2) with descriptors resident on the GPU (torch uint8 [n, dim]);
    valid1 / valid2 host uint8 arrays or None.  Returns (nmatches, matches12 numpy)."""
    nq, dim = q_t.shape
    nd = d_t.shape[0]
    v1, v2 = _contig(valid1, np.uint8), _contig(valid2, np.uint8)
    m12 = np.zeros(nq, np.int32)
    n = C.c_int32(0)
    st = _stream_handle(stream, q_t.device)
    _check(lib().mcs_match_bruteforce_device(_dptr(q_t), _dptr(qmask_t), _p(v1), nq, _dptr(d_t), _dptr(dmask_t), _p(v2), nd, dim, int(th_low),
                                             C.c_double(nnratio), _p(m12), C.byref(n), st))
    return n.value, m12


class Frame:
    """Flat stand-in for the fields of cMultiFrame / cMultiKeyFrame the matchers read
    (ref include/cMultiFrame.h:90-175): contiguous keypoints in camera-major order."""

    def __init__(self, keys, key_cam, desc, dmask, cam_sizes, scale_factors):
        self.keys = np.ascontiguousarray(keys, KEYPOINT_DTYPE)
        self.key_cam = np.ascontiguousarray(key_cam, np.int32)
        self.desc = np.ascontiguousarray(desc, np.uint8)
        self.dmask = _contig(dmask, np.uint8)
        self.cam_w, self.cam_h = _cam_wh(cam_sizes)
        self.scale_factors = np.ascontiguousarray(scale_factors, np.float64)

    @staticmethod
    def from_cameras(per_cam, cam_sizes, scale_factors):
        """per_cam: list of (kps, desc, dmask) as returned by the extractor, in camera order (ref :168-184)."""
        keys = np.concatenate([p[0] for p in per_cam])
        key_cam = np.concatenate([np.full(len(p[0]), c, np.int32) for c, p in enumerate(per_cam)])
        desc = np.concatenate([p[1] for p in per_cam])
        dmask = np.concatenate([p[2] for p in per_cam]) if per_cam[0][2] is not None else None
        return Frame(keys, key_cam, desc, dmask, cam_sizes, scale_factors)

    def view(self):
        v = FrameView()
        v.n_cams, v.n_keys = len(self.cam_w), len(self.keys)
        v.keys, v.key_cam, v.desc = _p(self.keys).value, _p(self.key_cam).value, _p(self.desc).value
        v.dmask = _p(self.dmask).value if self.dmask is not None else None
        v.cam_width, v.cam_height = _p(self.cam_w).value, _p(self.cam_h).value
        v.dim, v.n_levels = self.desc.shape[1], len(self.scale_factors)
        v.scale_factors = _p(self.scale_factors).value
        return v


class MapPoints:
    """Parallel arrays of the cMapPoint tracking fields (ref include/cMapPoint.h: mbTrackInView, mnTrackScaleLevel,
    mTrackProjX/Y, mTrackViewCos; GetDescriptorPtr / GetDescriptorMaskPtr)."""

    def __init__(self, bad, in_view, level, proj_x, proj_y, view_cos, desc, dmask=None):
        self.bad = np.ascontiguousarray(bad, np.uint8)
        self.in_view = np.ascontiguousarray(in_view, np.uint8)
        self.level = np.ascontiguousarray(level, np.int32)
        self.proj_x = np.ascontiguousarray(proj_x, np.float64)
        self.proj_y = np.ascontiguousarray(proj_y, np.float64)
        self.view_cos = np.ascontiguousarray(view_cos, np.float64)
        self.desc = np.ascontiguousarray(desc, np.uint8)
        self.dmask = _contig(dmask, np.uint8)

    def view(self):
        v = MapPointView()
        v.n_points = len(self.bad)
        v.bad, v.in_view, v.level = _p(self.bad).value, _p(self.in_view).value, _p(self.level).value
        v.proj_x, v.proj_y, v.view_cos = _p(self.proj_x).value, _p(self.proj_y).value, _p(self.view_cos).value
        v.desc = _p(self.desc).value
        v.dmask = _p(self.dmask).value if self.dmask is not None else None
        return v


def window_search(frame, queries, qdesc, qmask=None, max_cand=64):
    queries = np.ascontiguousarray(queries, WINDOW_QUERY_DTYPE)
    qdesc = np.ascontiguousarray(qdesc, np.uint8)
    qmask = _contig(qmask, np.uint8)
    nq = len(queries)
    idx = np.zeros((nq, max_cand), np.int32)
    dist = np.zeros((nq, max_cand), np.int32)
    cnt = np.zeros(nq, np.int32)
    fv = frame.view()
    rc = lib().mcs_window_search(C.byref(fv), _p(queries), nq, _p(qdesc), _p(qmask), max_cand, _p(idx), _p(dist), _p(cnt))
    if rc not in (MCS_OK, MCS_ERR_CAPACITY):
        _check(rc)
    return idx, dist, cnt, rc


def frame_prepare(keys, key_cam, cams):
    """GPU epilogue of the cMultiFrame constructor (ref src/cMultiFrame.cpp:143-184): bearing rays [n,3] and the 64x48 grid as
    CSR (cell_start [n_cams*64*48+1], cell_items [n_in_grid])."""
    keys = np.ascontiguousarray(keys, KEYPOINT_DTYPE)
    key_cam = np.ascontiguousarray(key_cam, np.int32)
    nc, n = len(cams), len(keys)
    rays = np.zeros((n, 3))
    start = np.zeros(nc * 64 * 48 + 1, np.int32)
    items = np.zeros(max(n, 1), np.int32)
    ning = C.c_int32(0)
    _check(lib().mcs_frame_prepare(_p(keys), _p(key_cam), n, _ocams(cams), nc, _p(rays), _p(start), _p(items), C.byref(ning)))
    return rays, start, items[:ning.value].copy()


def project_mappoints(mtmc_inv, mtmc, cams, masks, world_pos, normal, min_dist, max_dist, scale_factors):
    """Batched cMultiFrame::isInFrustum (ref src/cMultiFrame.cpp:218-270): mtmc_inv / mtmc [n_cams,4,4], masks [n_cams,H,W],
    world_pos / normal [n,3].  Returns (in_view [n,n_cams] u8, level i32, proj_x, proj_y, view_cos f64) -- the MapPoints fields."""
    mi = np.ascontiguousarray(mtmc_inv, np.float64)
    mm = np.ascontiguousarray(mtmc, np.float64)
    masks = np.ascontiguousarray(masks, np.uint8)
    pos = np.ascontiguousarray(world_pos, np.float64)
    nrm = np.ascontiguousarray(normal, np.float64)
    dmin = np.ascontiguousarray(min_dist, np.float64)
    dmax = np.ascontiguousarray(max_dist, np.float64)
    sf = np.ascontiguousarray(scale_factors, np.float64)
    nc, n = len(cams), len(pos)
    in_view = np.zeros((n, nc), np.uint8)
    level = np.zeros((n, nc), np.int32)
    px, py, vc = np.zeros((n, nc)), np.zeros((n, nc)), np.zeros((n, nc))
    _check(lib().mcs_project_mappoints(nc, _p(mi), _p(mm), _ocams(cams), _p(masks), n, _p(pos), _p(nrm), _p(dmin), _p(dmax), _p(sf),
                                       len(sf), _p(in_view), _p(level), _p(px), _p(py), _p(vc)))
    return in_view, level, px, py, vc


def project_mappoints_device(mtmc_inv, mtmc, cams, masks_t, world_t, normal_t, min_dist_t, max_dist_t, scale_factors, skip_t=None,
                             out=None, stream=None):
    """mcs_project_mappoints_device: project_mappoints with the map points resident on the GPU.  mtmc_inv / mtmc [n_cams,4,4] and
    scale_factors on the host; masks_t [n_cams,H,W] u8, world_t / normal_t [n,3] f64, min/max_dist_t [n] f64 cuda tensors;
    skip_t [n] u8 cuda or None (flagged points keep their previous entries in `out`).  Returns `out` = (in_view [n,n_cams] u8,
    level i32, proj_x, proj_y, view_cos f64) cuda tensors, written asynchronously on `stream`."""
    import torch
    mi = np.ascontiguousarray(mtmc_inv, np.float64)
    mm = np.ascontiguousarray(mtmc, np.float64)
    sf = np.ascontiguousarray(scale_factors, np.float64)
    nc, n, dev = len(cams), world_t.shape[0], world_t.device
    if out is None:
        out = (torch.zeros((n, nc), dtype=torch.uint8, device=dev), torch.zeros((n, nc), dtype=torch.int32, device=dev),
               *(torch.zeros((n, nc), dtype=torch.float64, device=dev) for _ in range(3)))
    _check(lib().mcs_project_mappoints_device(nc, _p(mi), _p(mm), _ocams(cams), _dptr(masks_t), n, _dptr(world_t), _dptr(normal_t),
                                              _dptr(min_dist_t), _dptr(max_dist_t), _p(sf), len(sf), _dptr(skip_t),
                                              *(_dptr(t) for t in out), _stream_handle(stream, dev)))
    return out


class MapPointsDevice:
    """MapPoints with every array a torch CUDA tensor (bad may be None); in_view / level / proj_x / proj_y / view_cos [n, n_cams]
    as project_mappoints_device fills them, desc / dmask [n, dim] u8."""

    def __init__(self, bad, in_view, level, proj_x, proj_y, view_cos, desc, dmask=None):
        self.bad, self.in_view, self.level = bad, in_view, level
        self.proj_x, self.proj_y, self.view_cos, self.desc, self.dmask = proj_x, proj_y, view_cos, desc, dmask

    @staticmethod
    def from_host(mps, device):
        """MapPoints (host arrays) -> the same fields on `device`"""
        import torch
        t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(device)  # noqa: E731
        return MapPointsDevice(t(mps.bad), t(mps.in_view), t(mps.level), t(mps.proj_x), t(mps.proj_y), t(mps.view_cos), t(mps.desc),
                               t(mps.dmask))

    def view(self):
        v = MapPointDevView()
        v.n_points = self.desc.shape[0]
        for k in ("bad", "in_view", "level", "proj_x", "proj_y", "view_cos", "desc", "dmask"):
            t = getattr(self, k)
            setattr(v, k, t.data_ptr() if t is not None else None)
        return v


def slots_to_contiguous(frame_mp_slots, counts, capacity):
    """slot-indexed frame_mp [n_cams * capacity] (slot c * capacity + j) -> the contiguous keypoint order of Frame / cMultiFrame
    (camera-major, ref src/cMultiFrame.cpp:168-184)"""
    a = np.asarray(frame_mp_slots).reshape(-1, capacity)
    return np.concatenate([a[c, :int(n)] for c, n in enumerate(counts)]).astype(np.int32)


def contiguous_to_slots(frame_mp, counts, capacity, fill=-1):
    """inverse of slots_to_contiguous; slots beyond a camera's count get `fill`"""
    out = np.full((len(counts), capacity), fill, np.int32)
    o = 0
    for c, n in enumerate(counts):
        out[c, :int(n)] = frame_mp[o:o + int(n)]
        o += int(n)
    return out.reshape(-1)


RULE_RATIO, RULE_BEST, RULE_LEVEL_RATIO, RULE_BEST_FREE, RULE_FIRST_FREE, RULE_SCW = 0, 1, 2, 3, 4, 5


def search_windows(frame, queries, qdesc, qmask, query_tag, rule, nnratio, threshold, assigned):
    """mcs_search_windows: generic projection-window search + greedy acceptance (see include/mcs_b200.h)."""
    queries = np.ascontiguousarray(queries, WINDOW_QUERY_DTYPE)
    qdesc = np.ascontiguousarray(qdesc, np.uint8)
    qmask = _contig(qmask, np.uint8)
    tags = np.ascontiguousarray(query_tag, np.int32)
    assigned = np.ascontiguousarray(assigned, np.int32)
    n = C.c_int32(0)
    fv = frame.view()
    if qmask is None:
        fv.dmask = None
    _check(lib().mcs_search_windows(C.byref(fv), _p(queries), len(queries), _p(qdesc), _p(qmask), _p(tags), rule,
                                    C.c_double(nnratio), threshold, _p(assigned), C.byref(n)))
    return n.value, assigned


MCS_MP_DESCRIPTOR, MCS_MP_NORMAL_DEPTH = 1, 2


def _dist64(a, b, ma=None, mb=None):
    """DescriptorDistance64 (ma is None) or DescriptorDistance64Masked over two descriptor rows"""
    x = np.bitwise_xor(a, b)
    if ma is None:
        return int(np.unpackbits(x).sum())
    return (int(np.unpackbits(x & ma).sum()) + int(np.unpackbits(x & mb).sum())) // 2


def ComputeDistinctiveDescriptors(obs, kf_desc, kf_bad, having_masks=False, kf_dmask=None, bad=False):
    """cMapPoint::ComputeDistinctiveDescriptors(havingMasks) (ref src/cMapPoint.cpp:294-388) on one point.  obs: its observations
    as (k, slot) pairs in mObservations order (each key frame's slots adjacent, in AddObservation order); kf_desc[k] / kf_dmask[k]:
    key frame k's descriptor rows [n_cams * capacity, dim] u8 by slot (c * capacity + j); kf_bad[k]: isBad().  Returns the
    position in obs of the row that becomes mDescriptor (and, with having_masks, mDescriptorMask), or None when nothing changes
    (a bad point, or no row of a non-bad key frame)."""
    if bad:
        return None
    rows = [i for i, (k, _) in enumerate(obs) if not kf_bad[k]]
    if not rows:
        return None
    N = len(rows)
    if N <= 2:
        return rows[0]

    def row(i):
        k, s = obs[rows[i]]
        return kf_desc[k][s], (kf_dmask[k][s] if having_masks else None)
    best_median, best = 2**31 - 1, 0
    for i in range(N - 1):
        di, mi = row(i)
        d = sorted(_dist64(di, dj, mi, mj) for dj, mj in (row(j) for j in range(i + 1, N)))
        median = d[len(d) // 2]                           # misc.h:96-104: nth_element at size / 2
        if median < best_median:
            best_median, best = median, i
    return rows[best]


def UpdateNormalAndDepth(obs, kf_ow, ref_kf, world_pos, kf_octave, scale_factors, bad=False):
    """cMapPoint::UpdateNormalAndDepth() (ref src/cMapPoint.cpp:449-492) followed by GetMin/MaxDistanceInvariance (:494-504) on one
    point.  obs as for ComputeDistinctiveDescriptors; kf_ow[k]: GetCameraCenter() of key frame k; ref_kf: mpRefKF as an index of
    the key frames; kf_octave[k][slot]: the keypoint octaves by slot.  Returns (normal [3], 0.8 * mfMinDistance, 1.2 *
    mfMaxDistance), or None for a bad point.  The arithmetic is the reference's in its order, with OpenCV's Vec / scalar being
    Vec * (1. / scalar) (core/matx.hpp, Matx_ScaleOp); a point without observations gets the NaN normal 0 * (1. / 0)."""
    if bad:
        return None
    X = [float(v) for v in world_pos]
    normal, n, prev = [0.0, 0.0, 0.0], 0, None
    for k, _ in obs:                                      # one term per key frame, bad ones included
        if k == prev:
            continue
        prev = k
        d = [X[i] - float(kf_ow[k][i]) for i in range(3)]
        nr = math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
        inv = 1.0 / nr if nr else math.inf
        normal = [normal[i] + d[i] * inv for i in range(3)]
        n += 1
    p = [X[i] - float(kf_ow[ref_kf][i]) for i in range(3)]
    dist = math.sqrt((p[0] * p[0] + p[1] * p[1]) + p[2] * p[2])
    level = next((int(kf_octave[k][s]) for k, s in obs if k == ref_kf), 1)
    sf, nl = [float(v) for v in scale_factors], len(scale_factors)
    s = sf[level]
    mn = ((1.0 / s) * dist) / s
    mx = (s * dist) * sf[nl - 1 - level]
    inv_n = 1.0 / n if n else math.inf
    return np.array([v * inv_n for v in normal]), 0.8 * mn, 1.2 * mx


def mappoint_obs_csr(obs_lists):
    """the observation CSR of update_mappoints_device from per-point lists of (k, slot): (offsets [n + 1], obs_kf, obs_slot) int32"""
    off = np.zeros(len(obs_lists) + 1, np.int32)
    off[1:] = np.cumsum([len(o) for o in obs_lists])
    flat = [e for o in obs_lists for e in o]
    kf = np.array([k for k, _ in flat], np.int32)
    slot = np.array([s for _, s in flat], np.int32)
    return off, kf, slot


def update_mappoints_host(kf_desc, kf_dmask, kf_octave, kf_ow, kf_bad, n_cams, capacity, kf_counts, scale_factors, point_ids, obs_offsets,
                          obs_kf, obs_slot, ref_kf, bad, world_pos, desc, dmask, normal, min_dist, max_dist, what=3, having_masks=False):
    """update_mappoints_device on the host, through ComputeDistinctiveDescriptors / UpdateNormalAndDepth: the same checks, and the
    same rows of the same numpy arrays written in place.  kf_desc / kf_dmask / kf_octave / kf_ow / kf_bad / kf_counts [n_kf]:
    each key frame's slot-indexed descriptor rows, masks and octaves, its centre, isBad() and per-camera keypoint counts.
    Returns the status (MCS_OK or MCS_ERR_INVALID)."""
    status, n_kf, n_points, nl = MCS_OK, len(kf_ow), len(obs_offsets) - 1, len(scale_factors)
    for pid in (int(i) for i in point_ids):
        if not 0 <= pid < n_points:
            status = MCS_ERR_INVALID
            continue
        if bad is not None and bad[pid]:
            continue
        o0, o1 = int(obs_offsets[pid]), int(obs_offsets[pid + 1])
        obs = [(int(obs_kf[e]), int(obs_slot[e])) for e in range(o0, o1)] if 0 <= o0 <= o1 else None
        ok = obs is not None
        for e, (k, s) in enumerate(obs or []):
            ok = ok and 0 <= k < n_kf and 0 <= s < n_cams * capacity and s % capacity < kf_counts[k][s // capacity]
            ok = ok and not (e > 0 and obs[e - 1][0] != k and any(kk == k for kk, _ in obs[:e - 1]))
        if ok and what & MCS_MP_NORMAL_DEPTH:
            ok = 0 <= int(ref_kf[pid]) < n_kf
            if ok:
                lv = next((int(kf_octave[k][s]) for k, s in obs if k == int(ref_kf[pid])), 1)
                ok = 0 <= lv < nl
        if not ok:
            status = MCS_ERR_INVALID
            continue
        if what & MCS_MP_DESCRIPTOR:
            b = ComputeDistinctiveDescriptors(obs, kf_desc, kf_bad, having_masks, kf_dmask)
            if b is not None:
                k, s = obs[b]
                desc[pid] = kf_desc[k][s]
                if having_masks:
                    dmask[pid] = kf_dmask[k][s]
        if what & MCS_MP_NORMAL_DEPTH:
            normal[pid], min_dist[pid], max_dist[pid] = UpdateNormalAndDepth(obs, kf_ow, int(ref_kf[pid]), world_pos[pid], kf_octave,
                                                                             scale_factors)
    return status


def update_mappoints_device(kfs, n_cams, capacity, scale_factors, point_ids_t, obs_offsets_t, obs_kf_t, obs_slot_t, what=3,
                            having_masks=False, desc_t=None, dmask_t=None, normal_t=None, min_dist_t=None, max_dist_t=None, ref_kf_t=None,
                            world_t=None, bad_t=None, dim=None, status=None, stream=None):
    """mcs_update_mappoints_device: ComputeDistinctiveDescriptors (what & 1) and UpdateNormalAndDepth (what & 2) for the map points
    point_ids_t lists, writing their rows of the device tables the searches read (see include/mcs_b200.h).  kfs: per key frame
    (frame, ow, bad) with frame = (packed uint8 cuda tensor, n_parts, part_images, first_image), ow its GetCameraCenter() and bad
    its isBad().  Cuda tensors: point_ids_t int32 [n_upd]; the observation CSR obs_offsets_t [n_points + 1], obs_kf_t, obs_slot_t
    int32 (mappoint_obs_csr); desc_t / dmask_t [n_points, dim] u8, normal_t [n_points, 3], min_dist_t / max_dist_t [n_points],
    world_t [n_points, 3] f64, ref_kf_t int32 and bad_t u8 [n_points] (bad_t may be None).  Asynchronous on `stream`.  Returns the
    status tensor [1] int32."""
    import torch
    dev = point_ids_t.device
    if status is None:
        with _on_stream(stream, dev):
            status = torch.zeros(1, dtype=torch.int32, device=dev)
    if dim is None:
        dim = int((desc_t if desc_t is not None else dmask_t).shape[1])
    # the observation arrays must have an address even when no point has an observation
    obs_kf_t = obs_kf_t if obs_kf_t.numel() else torch.zeros(1, dtype=torch.int32, device=dev)
    obs_slot_t = obs_slot_t if obs_slot_t.numel() else torch.zeros(1, dtype=torch.int32, device=dev)
    ks = (MpKeyFrame * len(kfs))()
    for t, (frame, ow, bad) in zip(ks, kfs):
        t.frame = PackedFrame(frame[0].data_ptr(), *frame[1:4])
        t.ow[:] = [float(x) for x in ow]
        t.bad = int(bool(bad))
    sf = np.ascontiguousarray(scale_factors, np.float64)
    _check(lib().mcs_update_mappoints_device(ks, len(kfs), n_cams, capacity, dim, len(sf), _p(sf), int(what), int(bool(having_masks)),
                                             _dptr(point_ids_t) if point_ids_t.numel() else None, int(point_ids_t.numel()),
                                             int(obs_offsets_t.numel()) - 1, _dptr(obs_offsets_t), _dptr(obs_kf_t), _dptr(obs_slot_t),
                                             _dptr(ref_kf_t), _dptr(bad_t), _dptr(world_t), _dptr(desc_t), _dptr(dmask_t), _dptr(normal_t),
                                             _dptr(min_dist_t), _dptr(max_dist_t), _dptr(status), _stream_handle(stream, dev)))
    return status


def _queries(cam, x, y, r, min_level, max_level, desc_index):
    q = np.zeros(len(cam), WINDOW_QUERY_DTYPE)
    q["cam"], q["x"], q["y"], q["r"] = cam, x, y, r
    q["min_level"], q["max_level"], q["desc_index"] = min_level, max_level, desc_index
    return q


def _mm(A, B):
    """cv::Matx product: s = 0; s += a(i,k) * b(k,j) in index order, plain doubles (no FMA, no BLAS reordering)"""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    B2 = B.reshape(B.shape[0], -1)
    out = np.zeros((A.shape[0], B2.shape[1]))
    for i in range(A.shape[0]):
        for j in range(B2.shape[1]):
            acc = 0.0
            for k in range(A.shape[1]):
                acc += float(A[i, k]) * float(B2[k, j])
            out[i, j] = acc
    return out.reshape((A.shape[0],) + B.shape[1:])


def inv_rigid(M):
    """cConverter::invMat (ref src/cConverter.cpp:31-44): [R^T | -R^T t]"""
    M = np.asarray(M, np.float64)
    Rt = M[:3, :3].T.copy()
    t = _mm(-Rt, M[:3, 3])
    out = np.eye(4)
    out[:3, :3], out[:3, 3] = Rt, t
    return out


class Rig:
    """cMultiCamSys_ as the matchers use it (ref include/cam_system_omni.h:53-206): MCS pose M_t, camera offsets M_c[c], interior
    orientations; MtMc = M_t * M_c[c] and its rigid inverse kept like the reference does (flagMcMt)."""

    def __init__(self, cams, M_c=None, M_t=None):
        self.cams = list(cams)
        n = len(self.cams)
        self.M_c = np.ascontiguousarray(np.tile(np.eye(4), (n, 1, 1)) if M_c is None else M_c, np.float64)
        self.masks = [mirror_mask(c) for c in self.cams]
        self.set_pose(np.eye(4) if M_t is None else M_t)

    def set_pose(self, M_t):
        self.M_t = np.ascontiguousarray(M_t, np.float64)
        self.MtMc = np.stack([_mm(self.M_t, self.M_c[c]) for c in range(len(self.cams))])
        self.MtMc_inv = np.stack([inv_rigid(m) for m in self.MtMc])

    def world_to_cam(self, c, p3):
        """WorldToCamHom_fast (ref src/cam_system_omni.cpp:92-133) -> (u, v, camera-frame point)"""
        pc = _mm(self.MtMc_inv[c], np.array([p3[0], p3[1], p3[2], 1.0]))
        u, v = world_to_img(self.cams[c], float(pc[0]), float(pc[1]), float(pc[2]))
        return u, v, pc

    def in_mirror_mask(self, c, u, v):
        """isPointInMirrorMask(u, v, 0) (ref src/cam_model_omni.cpp:163-178)"""
        if not (np.isfinite(u) and np.isfinite(v)):
            return False
        ur, vr = int(np.rint(u)), int(np.rint(v))
        m = self.masks[c]
        if ur >= m.shape[1] or ur <= 0 or vr >= m.shape[0] or vr <= 0:
            return False
        return bool(m[vr, ur] > 0)


def compute_E_rel(Trel):
    """inline ComputeE(const cv::Matx44d& Trel) (ref include/misc.h:232-241): [t/|t|]_x * R"""
    Trel = np.asarray(Trel, np.float64)
    R = Trel[:3, :3]
    t = Trel[:3, 3].copy()
    n = float(np.sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]))
    t = t / n
    tx = np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])
    return _mm(tx, R)


def check_epipolar(ray1, ray2, E, thresh):
    """CheckDistEpipolarLine (ref src/misc.cpp:53-69), cv::Matx accumulation order"""
    r1, r2, E = (np.asarray(a, np.float64) for a in (ray1, ray2, E))
    nom = float(_mm(_mm(r2.reshape(1, 3), E), r1.reshape(3, 1))[0, 0])
    ex1 = _mm(E, r1.reshape(3, 1)).ravel()
    etx2 = _mm(E.T.copy(), r2.reshape(3, 1)).ravel()
    den = float(ex1[0] * ex1[0] + ex1[1] * ex1[1] + ex1[2] * ex1[2] + etx2[0] * etx2[0] + etx2[1] * etx2[1] + etx2[2] * etx2[2])
    if den == 0.0:
        return False
    return (nom * nom) / den < thresh


def _predict_level(scale_factors, ratio):
    """lower_bound over the scale factors, clamped to the last level (ref src/cORBmatcher.cpp:1313-1317)"""
    return min(int(np.searchsorted(scale_factors, ratio, side="left")), len(scale_factors) - 1)


def _sim3_rig(rig, Scw):
    """the rig with its pose replaced by the rigid part of the similarity Scw: camSys.Set_M_t(invMat(Rt2Hom(Rcw, tcw)))
    (ref :1576-1584, :2279-2287)"""
    S = np.asarray(Scw, np.float64)
    sR = S[:3, :3]
    inv_s = 1.0 / float(np.sqrt(sR[0, 0] * sR[0, 0] + sR[0, 1] * sR[0, 1] + sR[0, 2] * sR[0, 2]))
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = inv_s * sR, inv_s * S[:3, 3]
    return Rig(rig.cams, rig.M_c, inv_rigid(T))


def _project(rig, scale_factors, world_pos, min_dist, max_dist, ids, cams, float_dist):
    """projection front end of the Fuse overloads and SearchByProjection(KF, Scw) for map point ids[k] in camera cams[k, j] of rig:
    WorldToCamHom_fast -> isPointInMirrorMask -> distance range -> predicted level (ref :1288-1318).
    Returns uv [n, m, 2], ok [n, m] u8 (inside the mirror mask and the distance range), level [n, m] i32."""
    world_pos = np.asarray(world_pos, np.float64)
    Ow = rig.M_t[:3, 3].copy()
    uv, ok, lvl = np.zeros(cams.shape + (2,)), np.zeros(cams.shape, np.uint8), np.zeros(cams.shape, np.int32)
    for (k, j), c in np.ndenumerate(cams):
        i, c = int(ids[k]), int(c)
        p = world_pos[i]
        u, v, _ = rig.world_to_cam(c, p)
        if not rig.in_mirror_mask(c, u, v):
            continue
        po = p - Ow
        d = float(np.sqrt(po[0] * po[0] + po[1] * po[1] + po[2] * po[2]))
        if float_dist:
            d = float(np.float32(d))                      # `const float dist3D = cv::norm(PO);` (ref :1301, :1472)
        if d < min_dist[i] or d > max_dist[i]:
            continue
        uv[k, j] = (u, v); ok[k, j] = 1
        lvl[k, j] = _predict_level(scale_factors, d / min_dist[i])
    return uv, ok, lvl


def _packed_pair(cur, last):
    """the mcs_packed_frame records, by reference, of cur / last = (packed uint8 cuda tensor, n_parts, part_images, first_image)"""
    return [C.byref(PackedFrame(f[0].data_ptr(), *f[1:4])) for f in (cur, last)]


def _unpack_frame(f, n_cams, capacity, dim):
    """the (keypoints, descriptors, masks) of each camera of packed frame f = (packed uint8 tensor, n_parts, part_images,
    first_image), read back to the host"""
    from . import rig
    buf = f[0].cpu().numpy()
    part = rig.packed_layout(f[2], capacity, dim)[1]
    out = []
    for c in range(n_cams):
        g = f[3] + c
        out.append(rig.unpack(buf[(g // f[2]) * part:(g // f[2] + 1) * part], f[2], capacity, dim)[g % f[2]])
    return out


def _contiguous_frame(f, mp_t, n_cams, capacity, dim):
    """packed frame f (see _unpack_frame) read back in the contiguous keypoint order of Frame / cMultiFrame: (keys, descriptors,
    masks, the camera of each keypoint, the counts per camera, the slot-indexed int32 tensor mp_t in contiguous order, the slot of
    each contiguous index)"""
    per = _unpack_frame(f, n_cams, capacity, dim)
    counts = [len(k) for k, _, _ in per]
    cam = np.concatenate([np.full(n, c, np.int32) for c, n in enumerate(counts)])
    return (np.concatenate([k for k, _, _ in per]), np.concatenate([d for _, d, _ in per]), np.concatenate([m for _, _, m in per]), cam,
            counts, slots_to_contiguous(mp_t.cpu().numpy(), counts, capacity),
            slots_to_contiguous(np.arange(n_cams * capacity, dtype=np.int32), counts, capacity))


def _search_outputs(out, diag, stream, dev):
    """(nmatches [1], status [1], diag [4]) int32 cuda tensors, `out` or new, and the call's last four arguments (diag NULL unless asked)"""
    if out is None:
        import torch
        out = tuple(torch.zeros(k, dtype=torch.int32, device=dev) for k in (1, 1, 4))
    return out, (_dptr(out[0]), _dptr(out[1]), _dptr(out[2]) if diag else None, _stream_handle(stream, dev))


def _search_result(out, frame_mp_t, diag):
    """(nmatches, status, frame_mp_t), plus diag when it is asked for"""
    return (out[0], out[1], frame_mp_t) + ((out[2],) if diag else ())


def _init_search_outputs(out, diag, stream, dev):
    """_search_outputs for mcs_search_for_initialization_device, which has no status (none of its inputs can be invalid in a
    data-dependent way) and a two-entry diag: (nmatches [1], diag [2]), `out` or new, and the call's last three arguments"""
    if out is None:
        import torch
        out = tuple(torch.zeros(k, dtype=torch.int32, device=dev) for k in (1, 2))
    return out, (_dptr(out[0]), _dptr(out[1]) if diag else None, _stream_handle(stream, dev))


def _fuse_replay(variant, rows, kf_mp, bad, rig, cur_rig=None, cur_rays=None, kf_rays=None):
    """The map bookkeeping of the three Fuse overloads (ref :1377-1416, :1540-1565, :1692-1716) over their hits, in the
    reference's order.  rows: (map point i, its keypoint in curKF for variant 0's ray, the hit keypoint of pKF per camera or -1),
    query by query.  A hit on a keypoint with a non-bad occupant is a Replace (variant 0: only when CheckDistEpipolarLine holds,
    with camera c's MtMc_inv of curKF and MtMc of pKF), a free keypoint gets AddObservation + AddMapPoint and kf_mp is updated in
    place.  Returns (nFused, ops [k, 3]): rows (0, mp, keypoint) and (1, mp, other)."""
    ops, fused = [], 0
    for i, ray, hit in rows:
        for cam, b in enumerate(hit):
            b = int(b)
            if b < 0:
                continue
            other = int(kf_mp[b])
            if other >= 0:
                good = not bad[other]
                if variant == 0 and good:
                    T1 = inv_rigid(cur_rig.MtMc[cam]) if cur_rig is not None else np.eye(4)
                    E = compute_E_rel(_mm(T1, rig.MtMc[cam]))
                    good = check_epipolar(cur_rays[ray], kf_rays[b], E, 1e-2)
                if good:
                    ops.append((1, i, other)); fused += 1
            else:
                ops.append((0, i, b)); kf_mp[b] = i
    return fused, np.asarray(ops, np.int32).reshape(-1, 3)


class cORBmatcher:
    """ref include/cORBmatcher.h:55-178; thresholds as in src/cORBmatcher.cpp:46-64."""

    def __init__(self, nnratio=0.6, checkOri=True, featDim=32, havingMasks=False):
        self.mfNNratio, self.mbCheckOrientation, self.mbFeatDim, self.havingMasks = nnratio, checkOri, featDim, havingMasks
        if havingMasks:
            self.TH_HIGH_, self.TH_LOW_ = int(math.floor(1.5 * featDim)), int(math.floor(featDim))
        else:
            self.TH_HIGH_, self.TH_LOW_ = 3 * featDim, 2 * featDim

    def SearchByProjection(self, F, mapPoints, th, frame_mp=None):
        """SearchByProjection(cMultiFrame&, vector<cMapPoint*>&, th) (ref :67-166).
        frame_mp: F.mvpMapPoints as int32 indices (-1 = none), updated in place.  Returns (nmatches, frame_mp)."""
        if frame_mp is None:
            frame_mp = np.full(len(F.keys), -1, np.int32)
        frame_mp = np.ascontiguousarray(frame_mp, np.int32)
        n = C.c_int32(0)
        fv, mv = F.view(), mapPoints.view()
        _check(lib().mcs_search_by_projection(C.byref(fv), C.byref(mv), C.c_double(th), C.c_double(self.mfNNratio), self.TH_HIGH_,
                                              int(self.havingMasks), _p(frame_mp), C.byref(n)))
        return n.value, frame_mp

    def SearchByProjectionDevice(self, packed_t, n_parts, part_images, first_image, n_cams, capacity, cam_sizes, scale_factors, mps_dev,
                                 th, frame_mp_t, stream=None, out=None, diag=False):
        """mcs_search_by_projection_device: SearchByProjection with the frame in packed feature buffers (packed_t: uint8 cuda tensor of
        n_parts layouts of part_images images; camera c = image first_image + c) and the map points in a MapPointsDevice.  frame_mp_t:
        int32 cuda tensor [n_cams * capacity] indexed by slot, updated in place.  Asynchronous on `stream`.  Returns (nmatches [1],
        status [1], frame_mp_t), plus diag [4] when diag is set, as cuda tensors."""
        dim = mps_dev.desc.shape[1]
        cw, ch = _cam_wh(cam_sizes)
        sf = np.ascontiguousarray(scale_factors, np.float64)
        out, tail = _search_outputs(out, diag, stream, packed_t.device)
        mv = mps_dev.view()
        _check(lib().mcs_search_by_projection_device(_dptr(packed_t), n_parts, part_images, first_image, n_cams, capacity, dim, _p(cw), _p(ch),
                                                     len(sf), _p(sf), C.byref(mv), C.c_double(th), C.c_double(self.mfNNratio), self.TH_HIGH_,
                                                     int(self.havingMasks), _dptr(frame_mp_t), *tail))
        return _search_result(out, frame_mp_t, diag)

    def SearchByProjectionLastDevice(self, cur, last, capacity, rig_cur, masks_t, scale_factors, last_mp_t, world_t, th, cur_mp_t,
                                     bad_t=None, last_outlier_t=None, stream=None, out=None, diag=False):
        """mcs_search_by_projection_last_device: SearchByProjection(CurrentFrame, LastFrame, th) (ref :1990-2118, motion model) with
        both frames in packed feature buffers.  cur / last: (packed uint8 cuda tensor, n_parts, part_images, first_image); camera c =
        image first_image + c.  rig_cur: a Rig at the current pose (its MtMc_inv and camera models); masks_t [n_cams,H,W] u8 cuda,
        their mirror masks; scale_factors: CurrentFrame's.  last_mp_t / cur_mp_t: int32 cuda [n_cams * capacity] map-point ids by
        slot (-1 none), cur_mp_t updated in place; world_t [n_points,3] f64 cuda; bad_t [n_points] / last_outlier_t [n_cams *
        capacity] u8 cuda or None.  Asynchronous on `stream`.  Returns (nmatches [1], status [1], cur_mp_t), plus diag [4] when
        diag is set, as cuda tensors."""
        nc = len(rig_cur.cams)
        sf = np.ascontiguousarray(scale_factors, np.float64)
        mi = np.ascontiguousarray(rig_cur.MtMc_inv, np.float64)
        out, tail = _search_outputs(out, diag, stream, cur[0].device)
        _check(lib().mcs_search_by_projection_last_device(*_packed_pair(cur, last), nc, capacity, self.mbFeatDim, _ocams(rig_cur.cams),
                                                          _dptr(masks_t), len(sf), _p(sf), _p(mi), _dptr(last_mp_t), _dptr(last_outlier_t),
                                                          world_t.shape[0], _dptr(world_t), _dptr(bad_t), th, self.TH_HIGH_,
                                                          int(self.havingMasks), _dptr(cur_mp_t), *tail))
        return _search_result(out, cur_mp_t, diag)

    def WindowSearchDevice(self, cur, last, capacity, cam_sizes, last_mp_t, window, cur_mp_t, min_level=0, max_level=2**31 - 1, bad_t=None,
                           stream=None, out=None, diag=False):
        """mcs_window_search_device: WindowSearch(F1 = last, F2 = cur, window, ., min_level, max_level) (ref :326-473) with both
        frames in packed feature buffers.  cur / last: (packed uint8 cuda tensor, n_parts, part_images, first_image); cam_sizes
        [(w, h)] per camera.  last_mp_t: int32 cuda [n_cams * capacity] map-point ids by slot (-1 none); cur_mp_t: same shape,
        overwritten (every slot below a camera's count starts at -1); bad_t [n_points] u8 cuda or None, n_points = len(bad_t) or
        every id when None.  Asynchronous on `stream`.  Returns (nmatches [1], status [1], cur_mp_t), plus diag [4] when diag is set,
        as cuda tensors."""
        nc = len(cam_sizes)
        cw, ch = _cam_wh(cam_sizes)
        n_points = bad_t.shape[0] if bad_t is not None else 2**31 - 1
        out, tail = _search_outputs(out, diag, stream, cur[0].device)
        _check(lib().mcs_window_search_device(*_packed_pair(cur, last), nc, capacity, self.mbFeatDim, _p(cw), _p(ch), _dptr(last_mp_t),
                                              n_points, _dptr(bad_t), int(window), int(min_level), int(max_level), self.mfNNratio,
                                              self.TH_HIGH_, int(self.havingMasks), _dptr(cur_mp_t), *tail))
        return _search_result(out, cur_mp_t, diag)

    def SearchByProjectionFramesDevice(self, cur, last, capacity, rig_cur, masks_t, last_mp_t, world_t, window, cur_mp_t, bad_t=None,
                                       stream=None, out=None, diag=False):
        """mcs_search_by_projection_frames_device: SearchByProjection(F1 = last, F2 = cur, window, .) (ref :476-577) with both frames
        in packed feature buffers.  cur / last as for WindowSearchDevice; rig_cur: a Rig at the current pose (after
        PoseOptimization); masks_t [n_cams,H,W] u8 cuda, its mirror masks.  last_mp_t / cur_mp_t: int32 cuda [n_cams * capacity]
        map-point ids by slot (-1 none), cur_mp_t updated in place (its entries are "already found"); world_t [n_points,3] f64 cuda;
        bad_t [n_points] u8 cuda or None.  Asynchronous on `stream`.  Returns (nmatches [1], status [1], cur_mp_t), plus diag [4]
        when diag is set, as cuda tensors."""
        nc = len(rig_cur.cams)
        mi = np.ascontiguousarray(rig_cur.MtMc_inv, np.float64)
        out, tail = _search_outputs(out, diag, stream, cur[0].device)
        _check(lib().mcs_search_by_projection_frames_device(*_packed_pair(cur, last), nc, capacity, self.mbFeatDim, _ocams(rig_cur.cams),
                                                            _dptr(masks_t), _p(mi), _dptr(last_mp_t), world_t.shape[0], _dptr(world_t),
                                                            _dptr(bad_t), int(window), self.mfNNratio, self.TH_HIGH_,
                                                            int(self.havingMasks), _dptr(cur_mp_t), *tail))
        return _search_result(out, cur_mp_t, diag)

    def SearchForInitialization(self, F1, F2, vbPrevMatched, windowSize=10):
        """ref :579-726.  vbPrevMatched [n1,2] float64 updated in place.  Returns (nmatches, vnMatches12)."""
        prev = np.ascontiguousarray(vbPrevMatched, np.float64)
        m12 = np.zeros(len(F1.keys), np.int32)
        n = C.c_int32(0)
        f1, f2 = F1.view(), F2.view()
        _check(lib().mcs_search_for_initialization(C.byref(f1), C.byref(f2), _p(prev), windowSize, C.c_double(self.mfNNratio),
                                                   self.TH_LOW_, int(self.havingMasks), _p(m12), C.byref(n)))
        if prev is not vbPrevMatched:
            vbPrevMatched[...] = prev
        return n.value, m12

    def SearchForInitializationDevice(self, f1, f2, capacity, cam_sizes, prev_t, window, m12_t, stream=None, out=None, diag=False):
        """mcs_search_for_initialization_device: SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, window) (ref :579-726)
        with both frames in packed feature buffers.  f1 / f2: (packed uint8 cuda tensor, n_parts, part_images, first_image); cam_sizes
        [(w, h)] per camera.  prev_t: float64 cuda [n_cams * capacity * 2] window centres by F1 slot, updated in place; m12_t: int32
        cuda [n_cams * capacity], overwritten below each camera's count with the F2 slot matched or -1.  Asynchronous on `stream`.
        Returns (nmatches [1], m12_t), plus diag [2] (queries, rescans) when diag is set, as cuda tensors."""
        nc = len(cam_sizes)
        cw, ch = _cam_wh(cam_sizes)
        out, tail = _init_search_outputs(out, diag, stream, f1[0].device)
        _check(lib().mcs_search_for_initialization_device(*_packed_pair(f1, f2), nc, capacity, self.mbFeatDim, _p(cw), _p(ch), _dptr(prev_t),
                                                          int(window), self.mfNNratio, self.TH_LOW_, int(self.havingMasks), _dptr(m12_t),
                                                          *tail))
        return (out[0], m12_t) + ((out[1],) if diag else ())

    def SearchForInitializationSeedDevice(self, f1, n_cams, capacity, prev_t, stream=None):
        """mcs_search_for_initialization_seed_device: FirstInitialization's vbPrevMatched (ref src/cTracking.cpp:383-386) on the
        device: prev_t [n_cams * capacity * 2] float64 cuda gets every F1 keypoint's position, by slot.  Returns prev_t."""
        _check(lib().mcs_search_for_initialization_seed_device(C.byref(PackedFrame(f1[0].data_ptr(), *f1[1:4])), n_cams, capacity,
                                                               self.mbFeatDim, _dptr(prev_t), _stream_handle(stream, f1[0].device)))
        return prev_t

    def _masks(self, *masks):
        """the descriptor masks a search reads: each of `masks` as u8 when havingMasks and none of them is None, else None for
        each; one mask in, one out"""
        use = self.havingMasks and all(m is not None for m in masks)
        masks = tuple(np.ascontiguousarray(m, np.uint8) if use else None for m in masks)
        return masks if len(masks) > 1 else masks[0]

    def _best_free(self, KF, q, qdesc, qmask, rule, threshold, _sw=None):
        """RULE_BEST_FREE / RULE_FIRST_FREE on the queries q against KF -> the best keypoint of KF per query (-1 none).  These rules
        ignore the tags and write each query's answer to assigned[query], so `assigned` has max(n_queries, n_keys) entries."""
        _, res = (search_windows if _sw is None else _sw)(KF, q, qdesc, self._masks(qmask), np.zeros(len(q), np.int32), rule,
                                                           self.mfNNratio, threshold, np.full(max(len(q), len(KF.keys)), -1, np.int32))
        return res[:len(q)]

    def WindowSearch(self, F1, F2, windowSize, valid1, minScaleLevel=0, maxScaleLevel=2**31 - 1, _sw=None):
        """WindowSearch(F1, F2, windowSize, vpMapPointMatches2, minScaleLevel, maxScaleLevel) (ref :326-474).
        valid1[i1]: F1 keypoint i1 carries a non-bad map point.  Returns (nmatches, vnMatches21: F1 index per F2 keypoint)."""
        lv = F1.keys["octave"]
        sel = np.flatnonzero((np.asarray(valid1) != 0) & ((minScaleLevel <= 0) | (lv >= minScaleLevel)) &
                             ((maxScaleLevel >= 2**31 - 1) | (lv <= maxScaleLevel)))
        q = _queries(F1.key_cam[sel], F1.keys["x"][sel].astype(np.float64), F1.keys["y"][sel].astype(np.float64),
                     float(windowSize), -1, -1, sel)
        return (search_windows if _sw is None else _sw)(F2, q, F1.desc, self._masks(F1.dmask), sel, RULE_RATIO, self.mfNNratio,
                                                        self.TH_HIGH_, np.full(len(F2.keys), -1, np.int32))

    def SearchByProjectionFrames(self, F1, F2, windowSize, valid1, uv, in_mask, assigned2=None, mp1=None, _sw=None):
        """SearchByProjection(F1, F2, windowSize, vpMapPointMatches2) (ref :476-573).  valid1[i1]: keypoint i1 of F1 carries a
        map point that is not bad, not already found in F2 and not seen before in F1 (the caller's bookkeeping, :490-499);
        uv[i1, c] = projection of that map point into camera c of F2 (WorldToCamHom_fast), in_mask[i1, c] = isPointInMirrorMask.
        assigned2 = F2.mvpMapPoints as indices (-1 = NULL); mp1: map point id per F1 keypoint, when given a new match writes mp1[i1]
        instead of i1.  Returns (nmatches, assigned2 with F1 indices (or mp1 ids) for new matches)."""
        if assigned2 is None:
            assigned2 = np.full(len(F2.keys), -1, np.int32)
        i1, c = np.nonzero((np.asarray(valid1) != 0)[:, None] & (np.asarray(in_mask) != 0))      # i1 outer, camera inner
        lv = F1.keys["octave"][i1]
        q = _queries(c, np.asarray(uv)[i1, c, 0], np.asarray(uv)[i1, c, 1], float(windowSize), lv, lv, i1)
        return (search_windows if _sw is None else _sw)(F2, q, F1.desc, self._masks(F1.dmask), i1 if mp1 is None else np.asarray(mp1)[i1],
                                                        RULE_RATIO, self.mfNNratio, self.TH_HIGH_, assigned2)

    def SearchByProjectionLast(self, CurrentFrame, LastFrame, th, valid_last, uv, in_mask, assigned_cur=None, last_mp=None, _sw=None):
        """SearchByProjection(CurrentFrame, LastFrame, th) (ref :1990-2118, motion model).  valid_last[i]: LastFrame keypoint i has a
        non-bad, non-outlier map point; uv[i] = its projection into its own camera of CurrentFrame, in_mask[i] = mirror-mask test.
        last_mp: map point id per LastFrame keypoint, when given a new match writes last_mp[i] instead of i.
        Returns (nmatches, CurrentFrame.mvpMapPoints as LastFrame indices (or last_mp ids))."""
        if assigned_cur is None:
            assigned_cur = np.full(len(CurrentFrame.keys), -1, np.int32)
        sel = np.flatnonzero((np.asarray(valid_last) != 0) & (np.asarray(in_mask) != 0))
        lv = LastFrame.keys["octave"][sel]
        r = th * CurrentFrame.scale_factors[lv]
        q = _queries(LastFrame.key_cam[sel], np.asarray(uv)[sel, 0], np.asarray(uv)[sel, 1], r, lv - 1, lv + 1, sel)
        return (search_windows if _sw is None else _sw)(CurrentFrame, q, LastFrame.desc, self._masks(LastFrame.dmask),
                                                        sel if last_mp is None else np.asarray(last_mp)[sel], RULE_BEST, self.mfNNratio,
                                                        self.TH_HIGH_, assigned_cur)

    def FuseCandidates(self, KF, uv, in_mask, level, th, mp_desc, mp_dmask=None, first_wins=False, points=None, _sw=None):
        """Matching core of Fuse(pKF, curKF, vpMapPoints, th) (ref :1265-1418) and Fuse(pKF, Scw, vpPoints, th) (:1570-1719): for map
        point i and camera c (in_mask[i,c]) the best keypoint of KF within th*scale[level] of uv[i,c] on levels {level-1, level},
        accepted when its distance <= TH_LOW_.  first_wins=True is Fuse(pKF, vpMapPoints, th) (:1420-1568) as the reference behaves:
        the distance is discarded there, the first in-level candidate of the window wins (MCS_RULE_FIRST_FREE).  points: map point
        id per row i of uv, when given its queries read mp_desc[points[i]] instead of mp_desc[i].
        Returns best [n, n_cams] (keypoint index or -1); replacing / adding observations stays with the caller (host map bookkeeping)."""
        in_mask = np.asarray(in_mask) != 0
        i, c = np.nonzero(in_mask)
        lv = np.asarray(level)[i, c]
        q = _queries(c, np.asarray(uv)[i, c, 0], np.asarray(uv)[i, c, 1], th * KF.scale_factors[lv], lv - 1, lv,
                     i if points is None else np.asarray(points, np.int64)[i])
        best = np.full(in_mask.shape, -1, np.int32)
        best[i, c] = self._best_free(KF, q, mp_desc, mp_dmask, RULE_FIRST_FREE if first_wins else RULE_BEST_FREE, self.TH_LOW_, _sw)
        return best

    def SearchByProjectionScw(self, KF, query_cam, uv, level, th, valid, mp_desc, mp_dmask=None, matched=None, points=None, _sw=None):
        """Matching part of SearchByProjection(pKF, Scw, vpPoints, vpMatched, th) (ref :2265-2392) as written there.  Entry i of
        vpPoints: valid[i] (not NULL / bad / already found, projected inside the mirror mask, distance in range), query_cam[i] =
        keypoint_to_cam[i] -- the reference looks the camera up with the POINT's list position (:2326) --, uv[i], level[i] the
        predicted level.  matched = vpMatched as map point ids per keypoint (-1 = NULL), updated.  points: map point id per
        entry i, when given its query reads mp_desc[points[i]] and a match writes points[i], instead of mp_desc[i] and i.  Candidate
        descriptors are read the way the reference does (contiguous id as per-camera row; MCS_RULE_SCW) and keypoint 0 can never be
        matched (:2385)."""
        if matched is None:
            matched = np.full(len(KF.keys), -1, np.int32)
        sel = np.flatnonzero(np.asarray(valid) != 0)
        lv = np.asarray(level)[sel]
        ids = sel if points is None else np.asarray(points, np.int64)[sel]
        q = _queries(np.asarray(query_cam)[sel], np.asarray(uv)[sel, 0], np.asarray(uv)[sel, 1], th * KF.scale_factors[lv], lv - 1, lv, ids)
        return (search_windows if _sw is None else _sw)(KF, q, mp_desc, self._masks(mp_dmask), ids, RULE_SCW, self.mfNNratio, self.TH_LOW_,
                                                        matched)

    def Fuse(self, KF, rig, kf_mp, points, world_pos, min_dist, max_dist, bad, in_kf, mp_desc, mp_dmask=None, th=2.5, variant=1,
             Scw=None, cur_rays=None, kf_rays=None, cur_rig=None, _sw=None):
        """The three Fuse overloads of the reference as whole entry points (projection on the host with the reference's double
        arithmetic, window search + distances on the GPU, map bookkeeping replayed in order):
          variant 0  Fuse(pKF, curKF, vpMapPoints, th)  (ref :1265-1418): points[i] is the map point of keypoint i of curKF; a hit
                     on an occupied keypoint needs the epipolar check of the two bearing rays (cur_rays, kf_rays, cur_rig)
          variant 1  Fuse(pKF, vpMapPoints, th)         (ref :1420-1568): distance discarded, first in-level candidate wins
          variant 2  Fuse(pKF, Scw, vpPoints, th)       (ref :1570-1719): the rig pose is replaced by the Sim3's rigid part
        kf_mp [n_keys] map point id per keypoint (-1 none), updated like pKF->AddMapPoint does; points: candidate map point ids
        (-1 = NULL); bad / in_kf (IsInKeyFrame(pKF)) per map point.  Returns (nFused, ops) with ops rows (0, mp, keypoint) =
        AddObservation + AddMapPoint and (1, mp, other) = Replace(other), in the reference's call order."""
        kf_mp = np.ascontiguousarray(kf_mp, np.int32).copy()
        if variant == 2:
            rig = _sim3_rig(rig, Scw)
            already = set(int(m) for m in kf_mp if m >= 0 and not bad[m])
            idx = [int(i) for i in points if not bad[i] and int(i) not in already]
        else:
            idx = [int(i) for i in points if i >= 0 and not bad[i] and not in_kf[i]]
        nc = len(rig.cams)
        uv, ok, lvl = _project(rig, KF.scale_factors, world_pos, min_dist, max_dist, idx, np.tile(np.arange(nc), (len(idx), 1)),
                               float_dist=(variant != 2))
        best = self.FuseCandidates(KF, uv, ok, lvl, th, mp_desc, mp_dmask, first_wins=(variant == 1), points=idx, _sw=_sw)
        pos_of = {}
        if variant == 0:
            pos_of = {int(i): j for j, i in enumerate(points) if i >= 0}     # keypoint of curKF that carries map point i
        rows = ((i, pos_of.get(i), best[kk]) for kk, i in enumerate(idx))
        fused, ops = _fuse_replay(variant, rows, kf_mp, bad, rig, cur_rig, cur_rays, kf_rays)
        return fused, ops, kf_mp

    def FuseDevice(self, kfs, queries_t, capacity, cams, masks_t, scale_factors, world_t, min_dist_t, max_dist_t, desc_t, dmask_t=None,
                   bad_t=None, variant=0, th=3.0, max_hits=None, stream=None, out=None):
        """mcs_fuse_device: the matching part of the Fuse overloads for many key frames in one call (see include/mcs_b200.h).
        kfs: per target key frame (frame, mp_t, MtMc_inv, ow) with frame = (packed uint8 cuda tensor, n_parts, part_images,
        first_image), mp_t its int32 cuda [n_cams * capacity] map-point ids by slot or None, MtMc_inv [n_cams, 4, 4] of the pose
        to project with and ow [3] the centre of the depth test.  queries_t: int32 cuda [n_q] map-point ids (-1 = NULL).  cams:
        the rig's camera models, masks_t [n_cams,H,W] u8 cuda their mirror masks.  world_t [n_points,3] f64, min_dist_t /
        max_dist_t [n_points] f64, desc_t / dmask_t [n_points, dim] u8, bad_t [n_points] u8 (or None): cuda tensors.  variant 0 =
        Fuse(pKF, curKF, ., th) (:1265), 1 = Fuse(pKF, ., th) (:1420), 2 = Fuse(pKF, Scw, ., th) (:1570).  max_hits defaults to
        n_kf * n_q * n_cams (every entry).  Asynchronous on `stream`.  Returns (hits [max_hits, 3] (k, q, slot) rows, n_hits [1],
        status [1]) as cuda tensors."""
        import torch
        dev = queries_t.device
        nc, n_q, n_kf = len(cams), int(queries_t.shape[0]), len(kfs)
        if max_hits is None:
            max_hits = max(n_kf * n_q * nc, 1)
        if out is None:
            out = (torch.zeros((max_hits, 3), dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev),
                   torch.zeros(1, dtype=torch.int32, device=dev))
        mi = [np.ascontiguousarray(k[2], np.float64).reshape(-1) for k in kfs]          # kept alive through the call
        tg = (FuseTarget * n_kf)()
        for t, (frame, mp_t, _, ow), m in zip(tg, kfs, mi):
            t.frame = PackedFrame(frame[0].data_ptr(), *frame[1:4])
            t.mp_dev, t.mtmc_inv = _dptr(mp_t), m.ctypes.data
            t.ow[:] = [float(x) for x in ow]
        sf = np.ascontiguousarray(scale_factors, np.float64)
        _check(lib().mcs_fuse_device(tg, n_kf, nc, capacity, int(desc_t.shape[1]), _ocams(cams), _dptr(masks_t), len(sf), _p(sf), int(variant),
                                     _dptr(queries_t), n_q, int(world_t.shape[0]), _dptr(world_t), _dptr(min_dist_t), _dptr(max_dist_t),
                                     _dptr(desc_t), _dptr(dmask_t), _dptr(bad_t), float(th), self.TH_LOW_, int(self.havingMasks),
                                     _dptr(out[0]), int(out[0].shape[0]), _dptr(out[1]), _dptr(out[2]), _stream_handle(stream, dev)))
        return out

    def FuseReplay(self, KF, rig, kf_mp, points, hits, capacity, world_pos, min_dist, max_dist, bad, in_kf, mp_desc, mp_dmask=None, th=2.5,
                   variant=1, Scw=None, cur_rays=None, kf_rays=None, cur_rig=None, stale=(), _sw=None):
        """Fuse on one target key frame from the hits FuseDevice computed for it: the same arguments and results as Fuse, plus
        hits = that key frame's (q, slot) rows (q indexes `points`, slot = c * capacity + j) and `stale`, the map points whose
        descriptor was rewritten since the device call (a Replace survivor's ComputeDistinctiveDescriptors).  The skip tests read
        the live bad / in_kf / kf_mp given here; a stale query is searched again on the host (FuseCandidates) for variants 0 and 2,
        whose decisions read the descriptor, and self.fuse_researched counts those queries.  KF's keypoints are in camera-major
        order (cMultiFrame's, as Frame.from_cameras builds it), so that slot c * capacity + j is keypoint first[c] + j.  Variant
        0 reads curKF's ray of query q at cur_rays[q] (the reference's GetKeyPointRay(i)).  Returns (nFused, ops, kf_mp), what
        Fuse returns on the same state."""
        kf_mp = np.ascontiguousarray(kf_mp, np.int32).copy()
        nc = len(rig.cams)
        if variant == 2:
            rig = _sim3_rig(rig, Scw)
            already = set(int(m) for m in kf_mp if m >= 0 and not bad[m])
            live = [q for q, i in enumerate(points) if i >= 0 and not bad[i] and int(i) not in already]
        else:
            live = [q for q, i in enumerate(points) if i >= 0 and not bad[i] and not in_kf[i]]
        counts = np.bincount(np.asarray(KF.key_cam, np.int64), minlength=nc)
        first = np.concatenate([[0], np.cumsum(counts)])
        best = {q: np.full(nc, -1, np.int32) for q in live}
        for q, slot in np.asarray(hits, np.int64).reshape(-1, 2):
            if int(q) in best:
                c = int(slot) // capacity
                best[int(q)][c] = first[c] + int(slot) - c * capacity
        stale = set(int(i) for i in stale) if variant != 1 else set()
        redo = [q for q in live if int(points[q]) in stale]
        if redo:
            ids = [int(points[q]) for q in redo]
            uv, ok, lvl = _project(rig, KF.scale_factors, world_pos, min_dist, max_dist, ids, np.tile(np.arange(nc), (len(ids), 1)),
                                   float_dist=(variant != 2))
            again = self.FuseCandidates(KF, uv, ok, lvl, th, mp_desc, mp_dmask, first_wins=False, points=ids, _sw=_sw)
            for q, row in zip(redo, again):
                best[q] = row
        self.fuse_researched = len(redo)
        rows = ((int(points[q]), q, best[q]) for q in live)
        fused, ops = _fuse_replay(variant, rows, kf_mp, bad, rig, cur_rig, cur_rays, kf_rays)
        return fused, ops, kf_mp

    def SearchByProjectionKFScw(self, KF, rig, Scw, points, matched, world_pos, min_dist, max_dist, bad, mp_desc, mp_dmask=None, th=10,
                                _sw=None):
        """SearchByProjection(pKF, Scw, vpPoints, vpMatched, th) (ref :2265-2392) as a whole entry point, quirks included: the
        camera of entry iMP of vpPoints is keypoint_to_cam[iMP] (:2326), candidate descriptors are read with the contiguous id as
        per-camera row (:2367, :2372) and keypoint 0 is never matched (:2385).  points: map point ids (-1 = NULL), len <= n_keys;
        matched: vpMatched as map point ids per keypoint (-1 = NULL).  Returns (nmatches, vpMatched)."""
        matched = np.ascontiguousarray(matched, np.int32).copy()
        found = set(int(m) for m in matched if m >= 0)
        entries = np.asarray([iMP for iMP, i in enumerate(points) if i >= 0 and not bad[i] and int(i) not in found], np.int64)
        ids, cams = np.asarray(points, np.int64)[entries], KF.key_cam[entries]
        uv, ok, lvl = _project(_sim3_rig(rig, Scw), KF.scale_factors, world_pos, min_dist, max_dist, ids, cams[:, None], float_dist=False)
        if not ok.any():
            return 0, matched
        return self.SearchByProjectionScw(KF, cams, uv[:, 0], lvl[:, 0], float(int(th)), ok[:, 0], mp_desc, mp_dmask, matched, ids, _sw)

    def SearchByProjectionFramesRig(self, F1, mp1, F2, rig2, mp2, world_pos, bad, windowSize, _sw=None):
        """SearchByProjection(F1, F2, windowSize, vpMapPointMatches2) (ref :476-577) as a whole entry point: every map point of F1
        (first occurrence only, not bad, not already in F2) is projected into EVERY camera of F2's rig and searched there on the level
        of its F1 keypoint; ratio test + TH_HIGH_, greedy.  mp1 / mp2: map point id per keypoint (-1 none).
        Returns (nmatches, vpMapPointMatches2 as map point ids)."""
        out = np.ascontiguousarray(mp2, np.int32).copy()
        already = set(int(x) for x in out)                   # spMapPointsAlreadyFound holds NULL as well: harmless
        world_pos = np.asarray(world_pos, np.float64)
        n1, nc = len(F1.keys), len(rig2.cams)
        valid1, uv, in_mask = np.zeros(n1, bool), np.zeros((n1, nc, 2)), np.zeros((n1, nc), bool)
        seen = set()
        for i1 in range(n1):
            p = int(mp1[i1])
            if p < 0 or bad[p] or p in already or p in seen:
                continue
            seen.add(p)
            valid1[i1] = True
            for c in range(nc):
                u, v, _ = rig2.world_to_cam(c, world_pos[p])
                uv[i1, c], in_mask[i1, c] = (u, v), rig2.in_mirror_mask(c, u, v)
        if not in_mask.any():
            return 0, out
        return self.SearchByProjectionFrames(F1, F2, int(windowSize), valid1, uv, in_mask, out, mp1, _sw)

    def SearchByProjectionLastRig(self, CurrentFrame, rig_cur, cur_mp, LastFrame, last_mp, last_outlier, world_pos, bad, th, _sw=None):
        """SearchByProjection(CurrentFrame, LastFrame, th) (ref :1990-2118, motion model) as a whole entry point: the map point of
        every LastFrame keypoint (not bad, not an outlier) is projected into the SAME camera of the current rig pose and searched
        on levels octave-1 .. octave+1 within th*scale[octave]; best distance <= TH_HIGH_, greedy on CurrentFrame.mvpMapPoints.
        Returns (nmatches, CurrentFrame.mvpMapPoints as map point ids)."""
        out = np.ascontiguousarray(cur_mp, np.int32).copy()
        world_pos = np.asarray(world_pos, np.float64)
        n = len(LastFrame.keys)
        valid, uv, in_mask = np.zeros(n, bool), np.zeros((n, 2)), np.zeros(n, bool)
        for i in range(n):
            p = int(last_mp[i])
            if p < 0 or bad[p] or (last_outlier is not None and last_outlier[i]):
                continue
            cam = int(LastFrame.key_cam[i])
            u, v, _ = rig_cur.world_to_cam(cam, world_pos[p])
            valid[i], uv[i], in_mask[i] = True, (u, v), rig_cur.in_mirror_mask(cam, u, v)
        if not in_mask.any():
            return 0, out
        return self.SearchByProjectionLast(CurrentFrame, LastFrame, th, valid, uv, in_mask, out, last_mp, _sw)

    def SearchBySim3(self, KF1, rig1, mp1, KF2, rig2, mp2, world_pos, min_dist, max_dist, bad, mp_desc, mp_dmask, s12, R12, t12, th,
                     matches12=None, obs_idx2=None, _sw=None):
        """SearchBySim3(pKF1, pKF2, vpMatches12, s12, R12, t12, th) (ref :1721-1988) as a whole entry point: the map points of each
        key frame are carried into the other one by the similarity, searched in a th*scale[level] window on levels {l-1, l}
        (best distance <= TH_HIGH_), and only mutual agreements are kept.  mp1 / mp2: map point id per keypoint (-1 none);
        matches12 [n1]: already matched map point ids (-1 none) -- their keypoints are excluded, obs_idx2[id] = keypoint of KF2 that
        observes map point id (GetIndexInKeyFrame(pKF2)[0]).  Returns (nFound, vpMatches12 as map point ids)."""
        n1, n2 = len(KF1.keys), len(KF2.keys)
        m12 = np.full(n1, -1, np.int32) if matches12 is None else np.ascontiguousarray(matches12, np.int32).copy()
        world_pos = np.asarray(world_pos, np.float64)
        R12, t12 = np.asarray(R12, np.float64), np.asarray(t12, np.float64)
        T1, T2 = inv_rigid(rig1.M_t), inv_rigid(rig2.M_t)                       # GetPoseInverse()
        sR12 = s12 * R12
        sR21 = (1.0 / s12) * R12.T.copy()
        t21 = _mm(-sR21, t12)
        done1, done2 = np.zeros(n1, bool), np.zeros(n2, bool)
        for i in range(n1):
            if m12[i] >= 0:
                done1[i] = True
                j = int(obs_idx2[m12[i]]) if obs_idx2 is not None else -1
                if 0 <= j < n2:
                    done2[j] = True

        def one_way(KFa, mpa, Ta, sR, tt, KFb, rigb, skip_a):
            """points of a -> frame b; returns best keypoint of b per keypoint of a (-1 none)"""
            qc, quv, qlv, qi, qd = [], [], [], [], []
            for i in range(len(KFa.keys)):
                p = int(mpa[i])
                if p < 0 or skip_a[i] or bad[p]:
                    continue
                cam = int(KFa.key_cam[i])
                pa = _mm(Ta[:3, :3], world_pos[p]) + Ta[:3, 3]                  # point in the MCS frame of a
                pb = _mm(sR, pa) + tt                                           # ... of b
                p4 = _mm(inv_rigid(rigb.M_c[cam]), np.array([pb[0], pb[1], pb[2], 1.0]))
                if pb[2] < 0.0:
                    continue
                u, v = world_to_img(rigb.cams[cam], float(p4[0]), float(p4[1]), float(p4[2]))
                if not rigb.in_mirror_mask(cam, u, v):
                    continue
                d = float(np.sqrt(p4[0] * p4[0] + p4[1] * p4[1] + p4[2] * p4[2]))
                if d < min_dist[p] or d > max_dist[p]:
                    continue
                qc.append(cam); quv.append((u, v)); qlv.append(_predict_level(KFb.scale_factors, d / min_dist[p])); qi.append(i); qd.append(p)
            best = np.full(len(KFa.keys), -1, np.int32)
            if qi:
                lv, quv2 = np.asarray(qlv), np.asarray(quv)
                q = _queries(np.asarray(qc), quv2[:, 0], quv2[:, 1], th * KFb.scale_factors[lv], lv - 1, lv, np.asarray(qd))
                best[np.asarray(qi)] = self._best_free(KFb, q, mp_desc, mp_dmask, RULE_BEST_FREE, self.TH_HIGH_, _sw)
            return best
        b1 = one_way(KF1, mp1, T1, sR21, t21, KF2, rig2, done1)
        b2 = one_way(KF2, mp2, T2, sR12, t12, KF1, rig1, done2)
        found = 0
        for i1 in range(n1):
            i2 = int(b1[i1])
            if i2 >= 0 and int(b2[i2]) == i1:
                m12[i1] = mp2[i2]
                found += 1
        return found, m12

    def SearchBySim3Device(self, kf1, kf2, capacity, rig1, rig2, masks_t, scale_factors, mp1_t, mp2_t, world_t, min_dist_t, max_dist_t,
                           desc_t, dmask_t, s12, R12, t12, th, matches12_t, already2_t=None, bad_t=None, stream=None, out=None):
        """mcs_search_by_sim3_device: SearchBySim3 (ref :1721-1988) with both key frames in packed feature buffers (see
        include/mcs_b200.h).  kf1 / kf2: (packed uint8 cuda tensor, n_parts, part_images, first_image); rig1 / rig2: Rigs at the key
        frames' poses (GetPoseInverse is inv_rigid(M_t); the camera offsets and models are rig2's, the rig both share).  mp1_t / mp2_t
        int32 cuda [n_cams * capacity] map-point ids by slot; matches12_t likewise for KF1, updated in place (-1 = not matched yet);
        already2_t u8 cuda by KF2 slot or None.  The map points as cuda tensors, as for FuseDevice.  Asynchronous on `stream`.
        Returns (nfound [1], status [1], matches12_t) as cuda tensors."""
        out, tail = _search_outputs(out, False, stream, mp1_t.device)
        sf = np.ascontiguousarray(scale_factors, np.float64)
        t1w, t2w = inv_rigid(rig1.M_t), inv_rigid(rig2.M_t)
        mc_inv = np.ascontiguousarray(np.stack([inv_rigid(m) for m in rig2.M_c]), np.float64)
        r12, v12 = np.ascontiguousarray(R12, np.float64), np.ascontiguousarray(t12, np.float64)
        _check(lib().mcs_search_by_sim3_device(*_packed_pair(kf1, kf2), len(rig2.cams), capacity, int(desc_t.shape[1]), _ocams(rig2.cams),
                                               _dptr(masks_t), len(sf), _p(sf), _p(t1w), _p(t2w), _p(mc_inv), float(s12), _p(r12), _p(v12),
                                               float(th), _dptr(mp1_t), _dptr(mp2_t), int(world_t.shape[0]), _dptr(world_t), _dptr(min_dist_t),
                                               _dptr(max_dist_t), _dptr(desc_t), _dptr(dmask_t), _dptr(bad_t), _dptr(already2_t), self.TH_HIGH_,
                                               int(self.havingMasks), _dptr(matches12_t), tail[0], tail[1], tail[3]))
        return out[0], out[1], matches12_t

    def SearchByProjectionKFScwDevice(self, kf, capacity, rig, Scw, masks_t, scale_factors, points_t, world_t, min_dist_t, max_dist_t,
                                      desc_t, dmask_t, th, matched_t, bad_t=None, stream=None, out=None, diag=False):
        """mcs_search_by_projection_scw_device: SearchByProjection(pKF, Scw, vpPoints, vpMatched, th) (ref :2265-2392) with the key
        frame in packed feature buffers, quirks included (see include/mcs_b200.h).  kf: (packed uint8 cuda tensor, n_parts,
        part_images, first_image); rig: the key frame's Rig, whose pose Scw's rigid part replaces (_sim3_rig).  points_t int32 cuda
        [n_q] map-point ids (-1 = NULL); matched_t int32 cuda [n_cams * capacity], vpMatched by slot, updated in place.  Asynchronous
        on `stream`.  Returns (nmatches [1], status [1], matched_t), plus diag [4] when diag is set, as cuda tensors."""
        out, tail = _search_outputs(out, diag, stream, matched_t.device)
        sf = np.ascontiguousarray(scale_factors, np.float64)
        r = _sim3_rig(rig, Scw)
        mi, ow = np.ascontiguousarray(r.MtMc_inv, np.float64), np.ascontiguousarray(r.M_t[:3, 3], np.float64)
        _check(lib().mcs_search_by_projection_scw_device(C.byref(PackedFrame(kf[0].data_ptr(), *kf[1:4])), len(rig.cams), capacity,
                                                         int(desc_t.shape[1]), _ocams(rig.cams), _dptr(masks_t), len(sf), _p(sf), _p(mi), _p(ow),
                                                         _dptr(points_t), int(points_t.shape[0]), int(world_t.shape[0]), _dptr(world_t),
                                                         _dptr(min_dist_t), _dptr(max_dist_t), _dptr(desc_t), _dptr(dmask_t), _dptr(bad_t),
                                                         int(th), self.TH_LOW_, int(self.havingMasks), _dptr(matched_t), *tail))
        return _search_result(out, matched_t, diag)

    def SearchForTriangulationBetweenCameras(self, KF, rig, kf_mp, rays, cam1, cam2, _sw=None):
        """SearchForTriangulationBetweenCameras(pKF1, cam1, cam2, ...) (ref :1158-1263): every keypoint of camera cam1 without a
        map point is carried along its bearing ray into camera cam2 of the same rig (relative orientation of the two cameras),
        searched in a 40 px window (all levels, nothing skipped), and accepted when the best distance is <= 100 and the two rays
        satisfy the epipolar constraint.  Returns (nmatches, pairs [n,2] of contiguous keypoint ids)."""
        rel = _mm(inv_rigid(rig.M_c[cam1]), rig.M_c[cam2])
        E12 = compute_E_rel(rel)
        Rrel = rel[:3, :3].T.copy()
        trel = _mm(-Rrel, rel[:3, 3])
        qi, quv = [], []
        for i in range(len(KF.keys)):
            if kf_mp[i] >= 0 or int(KF.key_cam[i]) != cam1:
                continue
            rp = _mm(Rrel, rays[i]) + trel
            rp = rp / float(np.sqrt(rp[0] * rp[0] + rp[1] * rp[1] + rp[2] * rp[2]))
            u, v = world_to_img(rig.cams[cam2], float(rp[0]), float(rp[1]), float(rp[2]))
            if not rig.in_mirror_mask(cam2, u, v):
                continue
            qi.append(i); quv.append((u, v))
        pairs = []
        if qi:
            quv = np.asarray(quv)
            q = _queries(np.full(len(qi), cam2), quv[:, 0], quv[:, 1], 40.0, -1, -1, np.asarray(qi))
            res = self._best_free(KF, q, KF.desc, KF.dmask, RULE_BEST_FREE, 100, _sw)
            for k, i in enumerate(qi):
                b = int(res[k])
                # the reference evaluates the epipolar test with the best candidate even when its distance fails (:1247-1249);
                # RULE_BEST_FREE already applied bestDist <= 100
                if b >= 0 and check_epipolar(rays[i], rays[b], E12, 1e-2):
                    pairs.append((i, b))
        return len(pairs), np.asarray(pairs, np.int32).reshape(-1, 2)

    def SearchForTriangulationRaw(self, desc1, mask1, cam1, free1, rays1, desc2, mask2, cam2, free2, rays2, E, epi_thresh=1e-2):
        """SearchForTriangulationRaw(KF1, KF2, ...) (ref :968-1156): free1/free2 flag keypoints WITHOUT a map point, rays = bearing
        vectors [n,3], E [n_cams,n_cams,3,3] from ComputeE.  Returns (nmatches, vMatches12)."""
        d1, d2 = np.ascontiguousarray(desc1, np.uint8), np.ascontiguousarray(desc2, np.uint8)
        m1, m2 = self._masks(mask1, mask2)
        c1, c2 = np.ascontiguousarray(cam1, np.int32), np.ascontiguousarray(cam2, np.int32)
        f1, f2 = np.ascontiguousarray(free1, np.uint8), np.ascontiguousarray(free2, np.uint8)
        r1, r2 = np.ascontiguousarray(rays1, np.float64), np.ascontiguousarray(rays2, np.float64)
        Em = np.ascontiguousarray(E, np.float64)
        m12 = np.zeros(len(d1), np.int32)
        n = C.c_int32(0)
        _check(lib().mcs_search_for_triangulation(_p(d1), _p(m1), _p(c1), _p(f1), _p(r1), len(d1), _p(d2), _p(m2), _p(c2), _p(f2), _p(r2),
                                                  len(d2), d1.shape[1], self.TH_LOW_, _p(Em), Em.shape[0], C.c_double(epi_thresh), _p(m12), C.byref(n)))
        return n.value, m12

    def SearchForTriangulationRawDevice(self, kf1, mp1_t, kf2, mp2_t, cams, capacity, E, epi_thresh=1e-2, stream=None, out=None,
                                        diag=False):
        """mcs_search_for_triangulation_device: SearchForTriangulationRaw(KF1, KF2, ...) (ref :968-1107) for one neighbour key frame,
        both frames in packed feature buffers (see include/mcs_b200.h).  kf1 / kf2: (packed uint8 cuda tensor, n_parts, part_images,
        first_image); mp1_t / mp2_t: int32 cuda [n_cams * capacity] map-point ids by slot, -1 = free; cams: the camera models; E
        [n_cams, n_cams, 3, 3] host (ComputeE, or the settings' essential matrices).  Asynchronous on `stream`.  Returns (nmatches
        [1], matches12 [n_cams * capacity]: per KF1 slot the KF2 slot matched or -1, slots at or beyond a count not written), plus
        diag [2] (queries, rescans) when diag is set, as int32 cuda tensors."""
        import torch
        dev = mp1_t.device
        nc = len(cams)
        Em = np.ascontiguousarray(E, np.float64)
        if Em.shape != (nc, nc, 3, 3):
            raise ValueError(f"E must be [{nc}, {nc}, 3, 3], not {list(Em.shape)}")
        if out is None:
            with _on_stream(stream, dev):
                out = (torch.zeros(1, dtype=torch.int32, device=dev), torch.full((nc * capacity,), -1, dtype=torch.int32, device=dev),
                       torch.zeros(2, dtype=torch.int32, device=dev))
        p1, p2 = _packed_pair(kf1, kf2)
        _check(lib().mcs_search_for_triangulation_device(p1, _dptr(mp1_t), p2, _dptr(mp2_t), nc, capacity, self.mbFeatDim, _ocams(cams),
                                                         _p(Em), C.c_double(epi_thresh), self.TH_LOW_, int(self.havingMasks),
                                                         _dptr(out[1]), _dptr(out[0]), _dptr(out[2]) if diag else None,
                                                         _stream_handle(stream, dev)))
        return (out[0], out[1]) + ((out[2],) if diag else ())

    def SearchForTriangulationRawHost(self, kf1, mp1_t, kf2, mp2_t, cams, capacity, E, epi_thresh=1e-2, _st=None):
        """The host route of SearchForTriangulationRawDevice, what a caller does without it: read both frames and map-point rows
        back, put them in contiguous order (slots_to_contiguous), compute the rays on the host (img_to_world of each keypoint) and
        call SearchForTriangulationRaw (mcs_search_for_triangulation).  Same arguments; returns (nmatches, matches12) with matches12
        int32 [n_cams * capacity] as the device call's: the KF2 slot or -1, and -1 at every slot at or beyond a camera's count.
        _st: another search with oracle_api.search_for_triangulation's arguments (the tests' oracle route); the frames may then be
        CPU tensors."""
        nc = len(cams)

        def frame(f, mp_t):
            keys, d, m, cam, _, mp, slots = _contiguous_frame(f, mp_t, nc, capacity, self.mbFeatDim)
            rays = np.array([img_to_world(cams[cam[i]], float(k["x"]), float(k["y"])) for i, k in enumerate(keys)], np.float64).reshape(-1, 3)
            return (d, m, cam, (mp == -1).astype(np.uint8), rays), slots

        a1, s1 = frame(kf1, mp1_t)
        a2, s2 = frame(kf2, mp2_t)
        if _st is None:
            n, b = self.SearchForTriangulationRaw(*a1, *a2, E, epi_thresh)
        else:
            masks = (lambda m: m) if self.havingMasks else (lambda m: None)
            n, b = _st(a1[0], masks(a1[1]), *a1[2:], a2[0], masks(a2[1]), *a2[2:], E, self.TH_LOW_, epi_thresh)
        m12 = np.full(nc * capacity, -1, np.int32)
        hit = b >= 0
        m12[s1[hit]] = s2[b[hit]]
        return int(n), m12

    def SearchByBoW(self, desc1, desc2, mask1=None, mask2=None, valid1=None, valid2=None):
        """SearchByBoW(cMultiKeyFrame*, cMultiKeyFrame*, vpMatches12) (ref :885-966): all-pairs scan over the
        map-point-bearing keypoints of two keyframes.  Returns (nmatches, matches12 indices into desc2)."""
        d1 = np.ascontiguousarray(desc1, np.uint8)
        d2 = np.ascontiguousarray(desc2, np.uint8)
        m1, m2 = self._masks(mask1, mask2)
        v1, v2 = _contig(valid1, np.uint8), _contig(valid2, np.uint8)
        m12 = np.zeros(len(d1), np.int32)
        n = C.c_int32(0)
        _check(lib().mcs_match_bruteforce(_p(d1), _p(m1), _p(v1), len(d1), _p(d2), _p(m2), _p(v2), len(d2), d1.shape[1],
                                          self.TH_LOW_, C.c_double(self.mfNNratio), _p(m12), C.byref(n)))
        return n.value, m12

    def SearchByBoWKeyFramesDevice(self, kf1, mp1_t, kfs, n_cams, capacity, n_points, bad_t=None, stream=None, out=None):
        """mcs_search_by_bow_keyframes_device: SearchByBoW(KF1, KF_k, vpMatches12) (ref :885-966) for every loop candidate of
        ComputeSim3 in one call (see include/mcs_b200.h).  kf1: (packed uint8 cuda tensor, n_parts, part_images, first_image); mp1_t
        int32 cuda [n_cams * capacity] its map-point ids by slot (-1 none); kfs: [(packed frame, mp_t)] per candidate.  bad_t
        [n_points] u8 cuda or None.  Asynchronous on `stream`.  Returns (matches12 [n_kf, n_cams * capacity], match_slot (same
        shape), nmatches [n_kf], status [1]) as int32 cuda tensors: per KF1 slot the candidate's map-point id matched and its slot,
        -1 = none; slots at or beyond a camera's count are not written."""
        import torch
        dev = mp1_t.device
        nk, ns = len(kfs), n_cams * capacity
        if out is None:
            with _on_stream(stream, dev):
                out = (torch.full((nk, ns), -1, dtype=torch.int32, device=dev), torch.full((nk, ns), -1, dtype=torch.int32, device=dev),
                       torch.zeros(nk, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))
        frames = (PackedFrame * max(nk, 1))(*[PackedFrame(f[0].data_ptr(), *f[1:4]) for f, _ in kfs])
        mps = (C.c_void_p * max(nk, 1))(*[mp_t.data_ptr() for _, mp_t in kfs])
        _check(lib().mcs_search_by_bow_keyframes_device(C.byref(PackedFrame(kf1[0].data_ptr(), *kf1[1:4])), _dptr(mp1_t), frames, mps, nk,
                                                        n_cams, capacity, self.mbFeatDim, n_points, _dptr(bad_t), self.TH_LOW_,
                                                        C.c_double(self.mfNNratio), int(self.havingMasks), _dptr(out[0]), _dptr(out[1]),
                                                        _dptr(out[2]), _dptr(out[3]), _stream_handle(stream, dev)))
        return out

    def SearchByBoWKeyFramesHost(self, kf1, mp1_t, kfs, n_cams, capacity, n_points, bad_t=None, _bf=None):
        """The host route of SearchByBoWKeyFramesDevice, what a caller does without it: read the frames and map-point rows back,
        put them in contiguous order (slots_to_contiguous) and call SearchByBoW (mcs_match_bruteforce) once per candidate.  Same
        arguments; returns (matches12, match_slot, nmatches, status) as numpy arrays of the device call's shapes, with -1 at every
        slot at or beyond a camera's count.  A map-point id >= n_points makes its keypoint no query / database entry and sets
        status to MCS_ERR_INVALID.  _bf: another brute-force matcher with oracle_api.match_bruteforce's arguments (the tests'
        oracle route); the frames may then be CPU tensors."""
        dim, ns = self.mbFeatDim, n_cams * capacity
        bad = None if bad_t is None else bad_t.cpu().numpy()
        status = [MCS_OK]

        def frame(f, mp_t):
            _, d, m, _, _, mp, slots = _contiguous_frame(f, mp_t, n_cams, capacity, dim)
            if (mp >= n_points).any():
                status[0] = MCS_ERR_INVALID
            ok = (mp >= 0) & (mp < n_points)
            if bad is not None:
                ok[ok] = bad[mp[ok]] == 0
            return d, m, ok.astype(np.uint8), mp, slots

        d1, m1, v1, _, s1 = frame(kf1, mp1_t)
        m12 = np.full((len(kfs), ns), -1, np.int32)
        slot12 = np.full((len(kfs), ns), -1, np.int32)
        nm = np.zeros(len(kfs), np.int32)
        for k, (f, mp_t) in enumerate(kfs):
            d2, m2, v2, mp2, s2 = frame(f, mp_t)
            if _bf is None:
                nm[k], b = self.SearchByBoW(d1, d2, m1, m2, v1, v2)
            else:
                nm[k], b = _bf(d1, d2, self.TH_LOW_, self.mfNNratio, *((m1, m2) if self.havingMasks else (None, None)), v1, v2)
            hit = b >= 0
            m12[k, s1[hit]] = mp2[b[hit]]
            slot12[k, s1[hit]] = s2[b[hit]]
        return m12, slot12, nm, np.asarray(status, np.int32)

    def SearchByBoWFrame(self, desc_kf, featvec_kf, desc_f, featvec_f, mask_kf=None, mask_f=None, valid_kf=None):
        """SearchByBoW(cMultiKeyFrame* pKF, cMultiFrame& F, vpMapPointMatches) (ref src/cORBmatcher.cpp:179-324): matching
        restricted to keypoints that fall into the same vocabulary node.  featvec_* = (nodes, offsets, features) as returned
        by ORBVocabulary.transform.  Returns (nmatches, match_of_f) with match_of_f[i] = key-frame keypoint or -1."""
        d1 = np.ascontiguousarray(desc_kf, np.uint8)
        d2 = np.ascontiguousarray(desc_f, np.uint8)
        m1, m2 = self._masks(mask_kf, mask_f)
        v1 = _contig(valid_kf, np.uint8)
        a =[np.ascontiguousarray(x, np.int32) for x in featvec_kf]
        b = [np.ascontiguousarray(x, np.int32) for x in featvec_f]
        out = np.zeros(len(d2), np.int32)
        n = C.c_int32(0)
        _check(lib().mcs_search_by_bow(_p(d1), _p(m1), _p(v1), len(d1), _p(a[0]), _p(a[1]), len(a[0]), _p(a[2]), _p(d2), _p(m2), len(d2),
                                       _p(b[0]), _p(b[1]), len(b[0]), _p(b[2]), d1.shape[1], self.TH_LOW_, C.c_double(self.mfNNratio),
                                       _p(out), C.byref(n)))
        return n.value, out

    def SearchByBoWDevice(self, kfs, cur, n_points, bad_t=None, max_nodes=None, stream=None, out=None):
        """mcs_search_by_bow_device: SearchByBoW(pKF, F, vpMapPointMatches) (ref :179-324) for every candidate key frame of a
        relocalisation in one call, all frames in packed feature buffers.  kfs: [(DeviceBoW, mp_t)] with mp_t the key frame's int32
        cuda [n_cams * capacity] map-point ids by slot (-1 none); cur: the current frame's DeviceBoW (ORBVocabulary.transform_device,
        or built by hand from CSR tensors).  bad_t [n_points] u8 cuda or None; max_nodes: the node lists visited, by default the
        largest max_nodes of the frames.  Asynchronous on `stream`.  Returns (match_mp [n_kf, n_cams * capacity], match_slot (same
        shape), nmatches [n_kf], status [1]) as int32 cuda tensors: per current-frame slot the matched map-point id and the
        key-frame slot it came from, -1 = none; slots at or beyond a camera's count are not written."""
        import torch
        dev = cur.packed[0].device
        nk, ns = len(kfs), cur.n_cams * cur.capacity
        if max_nodes is None:
            max_nodes = max([cur.max_nodes] + [b.max_nodes for b, _ in kfs])
        if out is None:
            with _on_stream(stream, dev):
                out =(torch.full((nk, ns), -1, dtype=torch.int32, device=dev), torch.full((nk, ns), -1, dtype=torch.int32, device=dev),
                       torch.zeros(nk, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))
        frames = (BowFrame * max(nk, 1))(*[b.bow_frame(mp_t) for b, mp_t in kfs])
        fc = cur.bow_frame()
        _check(lib().mcs_search_by_bow_device(frames, nk, C.byref(fc), cur.n_cams, cur.capacity, self.mbFeatDim, max_nodes, n_points,
                                              _dptr(bad_t), self.TH_LOW_, C.c_double(self.mfNNratio), int(self.havingMasks),
                                              _dptr(out[0]), _dptr(out[1]), _dptr(out[2]), _dptr(out[3]), _stream_handle(stream, dev)))
        return out


class DeviceBoW:
    """What ComputeBoW leaves on the device for one frame (ORBVocabulary.transform_device): packed = (uint8 cuda tensor, n_parts,
    part_images, first_image); the FeatureVector as CSR over slots (fv_nodes [max_nodes], fv_offsets [max_nodes + 1], n_fv [1],
    fv_features [n_cams * capacity]); the BowVector (bow_words, bow_values [n_cams * capacity], n_bow [1]); status [1]; word /
    weight / node per slot when they were asked for.  The tensors a search does not read may be None."""

    def __init__(self, packed, n_cams, capacity, fv_nodes, fv_offsets, n_fv, fv_features, bow_words=None, bow_values=None, n_bow=None,
                 status=None, word=None, weight=None, node=None):
        self.packed, self.n_cams, self.capacity = packed, n_cams, capacity
        self.fv_nodes, self.fv_offsets, self.n_fv, self.fv_features = fv_nodes, fv_offsets, n_fv, fv_features
        self.bow_words, self.bow_values, self.n_bow, self.status = bow_words, bow_values, n_bow, status
        self.word, self.weight, self.node = word, weight, node
        self.max_nodes = fv_nodes.shape[0]

    def bow_frame(self, mp_t=None):
        """the mcs_bow_frame of this frame; mp_t: its map-point ids by slot (a key frame's)"""
        f = BowFrame()
        f.frame = PackedFrame(self.packed[0].data_ptr(), *self.packed[1:4])
        f.fv_nodes_dev, f.fv_offsets_dev, f.n_fv_dev = self.fv_nodes.data_ptr(), self.fv_offsets.data_ptr(), self.n_fv.data_ptr()
        f.fv_features_dev = self.fv_features.data_ptr()
        f.mp_dev = mp_t.data_ptr() if mp_t is not None else None
        return f

    def host(self):
        """(bow_words, bow_values, (fv_nodes, fv_offsets, fv_features)) as ORBVocabulary.transform returns them, feature indices
        being slots (synchronises)"""
        nb, nf = int(self.n_bow.item()), int(self.n_fv.item())
        fo = self.fv_offsets[:nf + 1].cpu().numpy()
        return (self.bow_words[:nb].cpu().numpy(), self.bow_values[:nb].cpu().numpy(),
                (self.fv_nodes[:nf].cpu().numpy(), fo, self.fv_features[:int(fo[nf])].cpu().numpy()))


class ORBVocabulary:
    """Mirror of ORBVocabulary = DBoW2::TemplatedVocabulary<FORB::TDescriptor, FORB> (ref include/cORBVocabulary.h:34) for the
    calls the SLAM front end makes: load, transform(features, BowVector, FeatureVector, levelsup), score, size.
    The tree lives on the GPU (mcs_vocabulary_create); `voc` is a mapping with k, L, scoring, weighting, parent, weight,
    desc, word_node and optionally node_order (tools/extract_vocabulary.py writes that layout)."""

    def __init__(self, voc, scoring=None, weighting=None):
        self.k, self.L = int(voc["k"]), int(voc["L"])
        self.scoring = int(voc["scoring"] if scoring is None else scoring)
        self.weighting = int(voc["weighting"] if weighting is None else weighting)
        par = np.ascontiguousarray(voc["parent"], np.int32)
        wt = np.ascontiguousarray(voc["weight"], np.float64)
        ds = np.ascontiguousarray(voc["desc"], np.uint8)
        wn = np.ascontiguousarray(voc["word_node"], np.int32)
        order = _contig(voc["node_order"] if "node_order" in voc else None, np.int32)
        if ds.shape != (len(par), 32) or len(wt) != len(par):
            raise ValueError("vocabulary arrays disagree in size")
        self._n_words = len(wn)
        self._h = C.c_void_p()
        _check(lib().mcs_vocabulary_create(self.k, self.L, self.scoring, self.weighting, len(par), _p(par), _p(wt), _p(ds), _p(order),
                                           len(wn), _p(wn), C.byref(self._h)))

    def __del__(self):
        if getattr(self, "_h", None):
            lib().mcs_vocabulary_destroy(self._h)
            self._h = None

    @staticmethod
    def loadFromTextFile(path, **kw):
        """DBoW2 text layout (ref TemplatedVocabulary.h:1338-1425): 'k L scoring weighting', then one line per node
        'parent isLeaf d0..d31 weight', node ids and word ids in line order."""
        lines = [ln for ln in open(path).read().split("\n") if ln.strip()]
        k, L, sc, wg = (int(t) for t in lines[0].split()[:4])
        n = len(lines)
        parent = np.zeros(n, np.int32); weight = np.zeros(n); desc = np.zeros((n, 32), np.uint8); words = []
        for i, ln in enumerate(lines[1:], start=1):
            t = ln.split()
            parent[i] = int(t[0]); desc[i] = [int(x) for x in t[2:34]]; weight[i] = float(t[34])
            if int(t[1]) > 0:
                words.append(i)
        return ORBVocabulary(dict(k=k, L=L, scoring=sc, weighting=wg, parent=parent, weight=weight, desc=desc,
                                  word_node=np.asarray(words, np.int32)), **kw)

    @staticmethod
    def load(path, **kw):
        """DBoW2 YAML layout as cv::FileStorage writes it (ref TemplatedVocabulary.h:1476-1624)."""
        import re
        txt = open(path).read()
        head = {key: int(re.search(r"\b%s:\s*(\d+)" % key, txt).group(1)) for key in ("k", "L", "scoringType", "weightingType")}
        nodes = re.findall(r"nodeId:(\d+),\s*parentId:(\d+),\s*weight:([-+0-9.eE]+),\s*descriptor:\"([^\"]*)\"", txt)
        words = re.findall(r"wordId:(\d+),\s*nodeId:(\d+)", txt)
        n = len(nodes) + 1
        parent = np.zeros(n, np.int32); weight = np.zeros(n); desc = np.zeros((n, 32), np.uint8); order = np.zeros(n - 1, np.int32)
        for i, (nid, pid, w, d) in enumerate(nodes):
            nid = int(nid); order[i] = nid; parent[nid] = int(pid); weight[nid] = float(w + "0" if w.endswith(".") else w)
            desc[nid] = [int(x) for x in d.split()]
        wn = np.zeros(len(words), np.int32)
        for wid, nid in words:
            wn[int(wid)] = int(nid)
        return ORBVocabulary(dict(k=head["k"], L=head["L"], scoring=head["scoringType"], weighting=head["weightingType"], parent=parent,
                                  weight=weight, desc=desc, node_order=order, word_node=wn), **kw)

    def size(self):
        return self._n_words

    def transform_features(self, desc, levelsup=4):
        """per descriptor: (word id, word weight, node id at level L - levelsup)  (ref :1218-1261)"""
        desc = np.ascontiguousarray(desc, np.uint8)
        if desc.ndim != 2 or desc.shape[1] != 32:
            raise ValueError("the vocabulary works on 32-byte descriptors (FORB::L)")
        n = len(desc)
        w = np.zeros(n, np.int32); wt = np.zeros(n, np.float64); nd = np.zeros(n, np.int32)
        _check(lib().mcs_bow_transform(self._h, _p(desc), n, levelsup, _p(w), _p(wt), _p(nd)))
        return w, wt, nd

    def transform(self, desc, levelsup=4):
        """transform(features, BowVector&, FeatureVector&, levelsup) (ref :1126-1194).
        -> (bow_words, bow_values, (fv_nodes, fv_offsets, fv_features))"""
        desc = np.ascontiguousarray(desc, np.uint8)
        if desc.ndim != 2 or (len(desc) and desc.shape[1] != 32):
            raise ValueError("the vocabulary works on 32-byte descriptors (FORB::L)")
        n = len(desc)
        bw = np.zeros(max(n, 1), np.int32); bv = np.zeros(max(n, 1), np.float64); nb = C.c_int32(0)
        fn = np.zeros(max(n, 1), np.int32); fo = np.zeros(n + 2, np.int32); nf = C.c_int32(0); ff = np.zeros(max(n, 1), np.int32)
        _check(lib().mcs_bow_vectors(self._h, _p(desc), n, levelsup, _p(bw), _p(bv), C.byref(nb), _p(fn), _p(fo), C.byref(nf), _p(ff)))
        k = nf.value
        return bw[:nb.value].copy(), bv[:nb.value].copy(), (fn[:k].copy(), fo[:k + 1].copy(), ff[:fo[k]].copy())

    def level_nodes(self, levelsup=4):
        """mcs_vocabulary_level_nodes: the most node ids a FeatureVector built with `levelsup` can hold"""
        n = C.c_int32(0)
        _check(lib().mcs_vocabulary_level_nodes(self._h, levelsup, C.byref(n)))
        return n.value

    def transform_device(self, packed, n_cams, capacity, levelsup=4, max_nodes=None, per_slot=False, stream=None):
        """mcs_bow_vectors_device: ComputeBoW on a frame that stays in its packed feature buffer.  packed = (uint8 cuda tensor,
        n_parts, part_images, first_image); camera c = image first_image + c.  max_nodes defaults to level_nodes(levelsup);
        per_slot also returns word / weight / node per slot.  Asynchronous on `stream`.  Returns a DeviceBoW of cuda tensors."""
        import torch
        dev = packed[0].device
        ns = n_cams * capacity
        if max_nodes is None:
            max_nodes = self.level_nodes(levelsup)
        i32 = lambda n: torch.zeros(n, dtype=torch.int32, device=dev)  # noqa: E731
        f64 = lambda n: torch.zeros(n, dtype=torch.float64, device=dev)  # noqa: E731
        with _on_stream(stream, dev):
            b =DeviceBoW(packed, n_cams, capacity, i32(max_nodes), i32(max_nodes + 1), i32(1), i32(ns), i32(ns), f64(ns), i32(1), i32(1),
                          *((i32(ns), f64(ns), i32(ns)) if per_slot else ()))
        fr = PackedFrame(packed[0].data_ptr(), *packed[1:4])
        _check(lib().mcs_bow_vectors_device(self._h, C.byref(fr), n_cams, capacity, 32, levelsup, max_nodes, _dptr(b.word), _dptr(b.weight),
                                            _dptr(b.node), _dptr(b.fv_nodes), _dptr(b.fv_offsets), _dptr(b.n_fv), _dptr(b.fv_features),
                                            _dptr(b.bow_words), _dptr(b.bow_values), _dptr(b.n_bow), _dptr(b.status),
                                            _stream_handle(stream, dev)))
        return b

    def score(self, v1, v2):
        """score(BowVector, BowVector) with the vocabulary's scoring type; v = (words, values)."""
        w1 = np.ascontiguousarray(v1[0], np.int32); x1 = np.ascontiguousarray(v1[1], np.float64)
        w2 = np.ascontiguousarray(v2[0], np.int32); x2 = np.ascontiguousarray(v2[1], np.float64)
        s = C.c_double(0)
        _check(lib().mcs_bow_score(self._h, _p(w1), _p(x1), len(w1), _p(w2), _p(x2), len(w2), C.byref(s)))
        return s.value
