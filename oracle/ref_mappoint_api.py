"""ctypes wrapper of oracle/_ref/libmappoint_ref.so: the REFERENCE's own cMapPoint (src/cMapPoint.cpp, ref_mappoint/Makefile).

update() builds one real cMapPoint over stand-in key frames, adds the listed observations, runs UpdateNormalAndDepth() and/or
ComputeDistinctiveDescriptors(havingMasks) and returns what the device tables would hold, plus the order in which mObservations
(a std::map keyed by key-frame address) iterated, so that a test can hand the same order to the host mirror and the device.
Tests reach it through oracle/ref_tape.py, which replays recorded results where the library cannot be built."""
import ctypes as C
import pathlib

import numpy as np

_HERE = pathlib.Path(__file__).resolve().parent
SO = _HERE / "_ref" / "libmappoint_ref.so"
MCS_REF = _HERE / "_ref" / "libmcs_ref.so"
_lib = None


def available():
    return SO.exists() and MCS_REF.exists()


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(SO))
        if _lib.refmp_init(str(MCS_REF).encode()) != 0:
            raise RuntimeError(f"{MCS_REF}: the reference's descriptor distances could not be loaded")
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def update(desc, dmask, octave, ow, kf_bad, scale_factors, obs_kf, obs_slot, ref_kf, X, point_bad, what, having_masks, n_cams, capacity):
    """desc / dmask [n_kf, n_cams * capacity, dim] u8 and octave [n_kf, n_cams * capacity] by slot; ow [n_kf, 3]; kf_bad [n_kf];
    obs_kf / obs_slot: the observations in AddObservation order.  Returns (desc_set, mask_set, desc hex, dmask hex, nd = (normal
    x, y, z, GetMinDistanceInvariance, GetMaxDistanceInvariance) as the hex of its five doubles' bytes (a NaN keeps its sign and
    payload), order: key-frame indices in mObservations order), all of it plain Python values, which a tape keeps verbatim."""
    desc, dmask = np.ascontiguousarray(desc, np.uint8), np.ascontiguousarray(dmask, np.uint8)
    octave, ow = np.ascontiguousarray(octave, np.int32), np.ascontiguousarray(ow, np.float64)
    kf_bad, sf = np.ascontiguousarray(kf_bad, np.int32), np.ascontiguousarray(scale_factors, np.float64)
    obs_kf, obs_slot = np.ascontiguousarray(obs_kf, np.int32), np.ascontiguousarray(obs_slot, np.int32)
    X = np.ascontiguousarray(X, np.float64)
    n_kf, dim = desc.shape[0], desc.shape[2]
    od, om, nd = np.zeros(dim, np.uint8), np.zeros(dim, np.uint8), np.zeros(5)
    order, n_order, ds, ms = np.zeros(max(n_kf, 1), np.int32), C.c_int(), C.c_int(), C.c_int()
    rc = lib().refmp_update(n_kf, n_cams, capacity, dim, _p(desc), _p(dmask), _p(octave), _p(ow), _p(kf_bad), len(sf), _p(sf),
                            len(obs_kf), _p(obs_kf), _p(obs_slot), int(ref_kf), _p(X), int(point_bad), int(what), int(having_masks),
                            C.byref(ds), C.byref(ms), _p(od), _p(om), _p(nd), _p(order), C.byref(n_order))
    if rc != 0:
        raise RuntimeError(f"refmp_update failed ({rc})")
    return (bool(ds.value), bool(ms.value), od.tobytes().hex(), om.tobytes().hex(), nd.tobytes().hex(),
            [int(k) for k in order[:n_order.value]])
