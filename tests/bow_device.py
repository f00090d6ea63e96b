"""The device bag of words on host arrays: frames split into packed cameras, mcs_bow_vectors_device with guarded outputs and its
check against the host transform, and SearchByBoW(KF_i, F) on the device and on the host copies."""
import ctypes as C
import pathlib

import numpy as np

from device_frames import BIG_ID, from_slots, on_device, pack_frames, reversed_image, slot_to_contiguous_index, to_slots

GOLD = pathlib.Path(__file__).resolve().parent / "golden"
TAIL_WORDS, VEC_FILL = 8, -77   # mcs_bow_vectors_device: guard words behind each output, and the value every output word starts at
SEARCH_FILL = -55               # mcs_search_by_bow_device: the value every output starts at
LAYOUTS = ["single", "parts", "shared"]


def split(desc, counts):
    """descriptors -> per-camera (kps, desc, mask) with the given counts"""
    from multicol_slam_b200.ctypes_defs import KEYPOINT_DTYPE
    o, per = 0, []
    for n in counts:
        per.append((np.zeros(n, KEYPOINT_DTYPE), np.ascontiguousarray(desc[o:o + n]), np.full((n, desc.shape[1]), 255, np.uint8)))
        o += n
    assert o == len(desc)
    return per


def pack_bow_frames(frames, cap, dim, layout):
    """frames: list of per-camera [(kps, desc, mask)] -> one packed-frame record per frame, the first frame's fullest camera reversed
    as the decoy.  single: one buffer per frame, a decoy image before and after its cameras; parts: n_cams one-image buffers back to
    back per frame, as the allgather leaves them; shared: all frames' cameras as consecutive images of one buffer"""
    decoy = reversed_image(max(frames[0], key=lambda p: len(p[0])))
    return pack_frames(frames, cap, dim, {"single": "single", "parts": "separate", "shared": "joint"}[layout], decoy=decoy)


def call(api, v, packed, counts, cap, levelsup, max_nodes=None, stream=None):
    """mcs_bow_vectors_device with every output set to VEC_FILL first and TAIL_WORDS guard words behind it -> dict of host arrays"""
    import torch
    nc, ns = len(counts), len(counts) * cap
    max_nodes = v.level_nodes(levelsup) if max_nodes is None else max_nodes
    sizes = dict(word=ns, weight=ns, node=ns, fv_nodes=max_nodes, fv_offsets=max_nodes + 1, n_fv=1, fv_features=ns, bow_words=ns,
                 bow_values=ns, n_bow=1, status=1)
    T = {k: torch.full((n + TAIL_WORDS,), VEC_FILL, dtype=torch.float64 if k in ("weight", "bow_values") else torch.int32, device="cuda")
         for k, n in sizes.items()}
    from multicol_slam_b200.ctypes_defs import PackedFrame
    fr = PackedFrame(packed[0].data_ptr(), *packed[1:4])
    h = C.c_void_p(stream.cuda_stream) if stream is not None else None
    torch.cuda.current_stream().synchronize()                    # the fills above; `stream` keeps whatever it is busy with
    rc =api.lib().mcs_bow_vectors_device(v._h, C.byref(fr), nc, cap, 32, levelsup, max_nodes, *(C.c_void_p(T[k].data_ptr()) for k in sizes), h)
    assert rc == 0, api.lib().mcs_last_error()
    torch.cuda.synchronize()
    H = {k: a.cpu().numpy() for k, a in T.items()}
    for k, n in sizes.items():
        assert np.all(H[k][n:] == VEC_FILL), f"{k}: written beyond the array"
    H["sizes"] = sizes
    return H


def check(api, H, v, desc, counts, cap, levelsup, oracle=None):
    """the device outputs H against mcs_bow_vectors / mcs_bow_transform on the concatenated descriptors (and the oracle)"""
    bw, bv, (fn, fo, ff) = v.transform(desc, levelsup)
    assert H["status"][0] == 0
    nb, nf = int(H["n_bow"][0]), int(H["n_fv"][0])
    assert nb == len(bw) and np.array_equal(H["bow_words"][:nb], bw) and np.array_equal(H["bow_values"][:nb], bv)
    assert nf == len(fn) and np.array_equal(H["fv_nodes"][:nf], fn) and np.array_equal(H["fv_offsets"][:nf + 1], fo)
    assert np.array_equal(slot_to_contiguous_index(H["fv_features"][:fo[nf]], counts, cap), ff)
    ns = len(counts) * cap
    assert np.all(H["bow_words"][nb:ns] == VEC_FILL) and np.all(H["fv_features"][fo[nf]:ns] == VEC_FILL)
    w, wt, nd = v.transform_features(desc, levelsup) if len(desc) else (np.zeros(0, np.int32), np.zeros(0), np.zeros(0, np.int32))
    live = np.zeros(ns, bool)
    for c, n in enumerate(counts):
        live[c * cap:c * cap + n] = True
    for k, ref in (("word", w), ("weight", wt), ("node", nd)):
        assert np.array_equal(H[k][:ns][live], ref), k
        assert np.all(H[k][:ns][~live] == VEC_FILL), k                 # untouched at or beyond a camera's count
    if oracle is not None:
        obw, obv, ofn, ofo, off = oracle.transform(desc, levelsup)
        assert np.array_equal(bw, obw) and np.array_equal(bv, obv) and np.array_equal(fn, ofn) and np.array_equal(fo, ofo) and np.array_equal(ff, off)
    return nb, nf


def counts_of(per):
    return [len(p[0]) for p in per]


def frame_of(per, fv, mp=None):
    """a frame on the host: per-camera (kps, desc, mask), its FeatureVector over contiguous keypoint ids, a key frame's map points"""
    return dict(per=per, fv=tuple(np.asarray(x, np.int32) for x in fv), mp=None if mp is None else np.asarray(mp, np.int32),
                desc=np.concatenate([p[1] for p in per]), mask=np.concatenate([p[2] for p in per]))


def index_to_slots(idx, counts, cap):
    first = np.concatenate([[0], np.cumsum(counts)])
    idx = np.asarray(idx, np.int64)
    c = np.searchsorted(first, idx, side="right") - 1
    return (c * cap + idx - first[c]).astype(np.int32)


def device_bow(api, packed, fr, cap, max_nodes):
    """DeviceBoW from a host FeatureVector: CSR tensors padded to max_nodes, features as slots"""
    nodes, off, feat = fr["fv"]
    counts = counts_of(fr["per"])
    pn = np.full(max_nodes, SEARCH_FILL, np.int32); pn[:len(nodes)] = nodes
    po = np.full(max_nodes + 1, SEARCH_FILL, np.int32); po[:len(off)] = off
    ns = len(counts) * cap
    pf = np.full(max(ns, len(feat)), SEARCH_FILL, np.int32); pf[:len(feat)] = index_to_slots(feat, counts, cap) if len(feat) else feat
    return api.DeviceBoW(packed, len(counts), cap, on_device(pn), on_device(po), on_device(np.array([len(nodes)], np.int32)), on_device(pf))


def mp_slots(api, fr, cap):
    return to_slots(api, counts_of(fr["per"]), fr["mp"], cap, BIG_ID)


def device_bow_search(api, m, kfs, cur, n_points, bad, layout="single", cap=None, stream=None, bows=None):
    """-> ([(nmatches, match_of_f, match_mp)] per key frame in contiguous keypoint ids, status)"""
    import torch
    frames = kfs + [cur]
    dim = cur["desc"].shape[1]
    cap = cap or max(max(counts_of(f["per"])) for f in frames) + 3
    packed = pack_bow_frames([f["per"] for f in frames], cap, dim, layout)
    max_nodes = max(len(f["fv"][0]) for f in frames) + 2
    if bows is None:
        bows = [device_bow(api, p, f, cap, max_nodes) for p, f in zip(packed, frames)]
    ns = len(cur["per"]) * cap
    out = tuple(torch.full(shape, SEARCH_FILL, dtype=torch.int32, device="cuda") for shape in ((len(kfs), ns), (len(kfs), ns), (len(kfs),), (1,)))
    bad_t = None if bad is None else on_device(np.asarray(bad, np.uint8))
    torch.cuda.current_stream().synchronize()
    m.SearchByBoWDevice([(b, mp_slots(api, f, cap)) for b, f in zip(bows[:-1], kfs)], bows[-1], n_points, bad_t, stream=stream, out=out)
    torch.cuda.synchronize()
    mmp, msl, nm, st = (x.cpu().numpy() for x in out)
    cc = counts_of(cur["per"])
    res = []
    for k, kf in enumerate(kfs):
        sl, mp = from_slots(api, msl[k], cc, cap, SEARCH_FILL), from_slots(api, mmp[k], cc, cap, SEARCH_FILL)
        idx = np.where(sl >= 0, slot_to_contiguous_index(np.maximum(sl, 0), counts_of(kf["per"]), cap), -1).astype(np.int32)
        res.append((int(nm[k]), idx, mp))
    return res, int(st[0])


def host_bow_search(api, m, kf, cur, n_points, bad, search=None):
    """mcs_search_by_bow (or the oracle) on the host copies -> (nmatches, match_of_f, match_mp)"""
    mp = kf["mp"]
    valid = (mp >= 0) & (mp < n_points)
    if bad is not None:
        valid &= np.asarray(bad)[np.clip(mp, 0, n_points - 1)] == 0
    use = m.havingMasks
    if search is None:
        n, out = m.SearchByBoWFrame(kf["desc"], kf["fv"], cur["desc"], cur["fv"], kf["mask"] if use else None, cur["mask"] if use else None,
                                    valid.astype(np.uint8))
    else:
        n, out = search(kf["desc"], kf["mask"] if use else None, valid.astype(np.uint8), kf["fv"], cur["desc"], cur["mask"] if use else None,
                        cur["fv"], m.TH_LOW_, m.mfNNratio)
    return n, out, np.where(out >= 0, mp[np.maximum(out, 0)], -1).astype(np.int32)


def same(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
