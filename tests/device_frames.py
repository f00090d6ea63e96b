"""Plumbing shared by the device-search tests: packed feature buffers, slot-indexed rows, the shared fixtures and constants.

Test modules import the fixtures they use by name (pytest finds fixtures in a module's namespace).  torch is imported inside
the functions that need it, so collecting the CPU tests needs no device."""
import pathlib
import re

import numpy as np
import pytest

ROOT = pathlib.Path(__file__).resolve().parents[1]

FAKE = 0x10000              # stands for a device pointer: never dereferenced by the host
FILL = 12345                # frame_mp value of the slots beyond a camera's count: must come back untouched
BIG_ID = 1 << 30            # map-point id of the slots beyond a camera's count: reading one would raise the status
GUARD = -999                # output value of the slots beyond a camera's count, and of rows past an output's end
POISON = 7777               # matches12 at or beyond a camera's count: must survive the call
PREV_FILL = -7777.25        # prev value of the slots beyond a camera's count
INT_MAX = 2**31 - 1
SIZES = [(754, 480)] * 3
TAPE_LIMIT = 1 << 20        # reference results stored whole: the tests compute on them


# ---- fixtures ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rm():
    """the reference's own matcher where oracle/_ref was built, None otherwise"""
    import ref_match_api
    return ref_match_api if ref_match_api.available() else None


def taped_rm(tape, name="ref_match_api", limit=TAPE_LIMIT):
    """a module fixture: the reference module `name`, live while recording and replayed from tests/golden/ref_tape_<tape>.*"""
    @pytest.fixture(scope="module")
    def rm():
        import ref_tape
        return ref_tape.module(name, tape, limit)
    return rm


@pytest.fixture(scope="module")
def frames(oa, cams):
    """two consecutive 3-camera frames of the sliding-texture stream, extracted by the CPU oracle"""
    import multicol_slam_b200.api as api            # plain array holders only
    from multicol_slam_b200 import synth
    ex = oa.OracleExtractor(nfeatures=350, do_dbrief=True, learn_masks=True)
    sf = [float(ex.info.scale_factor[l]) for l in range(8)]
    out = []
    streams = [synth.texture_stream(cams[c], 2, seed=60 + c) for c in range(3)]
    for t in range(2):
        per = [ex.extract(streams[c][t], synth.mirror_mask(cams[c]), cams[c]) for c in range(3)]
        out.append(api.Frame.from_cameras(per, SIZES, sf))
    return out


def declared_symbols():
    """the mcs_* functions include/mcs_b200.h declares"""
    txt = (ROOT / "include" / "mcs_b200.h").read_text()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(mcs_[a-z0-9_]+)\s*\(", txt)))


# ---- frames -----------------------------------------------------------------------------------------------------------------------
def counts(F):
    """keypoints per camera of a Frame"""
    return [int((F.key_cam == c).sum()) for c in range(len(F.cam_w))]


def per_cam(F):
    """a Frame -> per camera (kps, desc, dmask), the images rig.pack takes"""
    return [(F.keys[F.key_cam == c], F.desc[F.key_cam == c], None if F.dmask is None else F.dmask[F.key_cam == c])
            for c in range(len(F.cam_w))]


def keep_cameras(api, F, cams):
    """F with the keypoints of the cameras `cams` alone, and their indices in F"""
    i = np.flatnonzero(np.isin(F.key_cam, cams))
    return api.Frame(F.keys[i], F.key_cam[i], F.desc[i], F.dmask[i], list(zip(F.cam_w, F.cam_h)), F.scale_factors), i


def sizes(F):
    return list(zip(F.cam_w.tolist(), F.cam_h.tolist()))


def on_device(a, device="cuda"):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def flip(rng, d, nbits):
    """descriptor row d with nbits distinct bits flipped"""
    out = d.copy()
    for b in rng.choice(8 * len(d), nbits, replace=False):
        out[b // 8] ^= 1 << (b % 8)
    return out


def flip_bits(rng, desc, kmax):
    """every row of desc with up to kmax distinct bits flipped"""
    d = desc.copy()
    for i in range(len(d)):
        for b in rng.choice(8 * d.shape[1], rng.integers(0, kmax + 1), replace=False):
            d[i, b // 8] ^= 1 << (b % 8)
    return d


def widener(dim):
    """32-byte rows -> dim-byte rows: 16 = the first half of every row, 64 = the row and a variant of it"""
    if dim == 16:
        return lambda d: np.ascontiguousarray(d[:, :16])
    return lambda d: np.ascontiguousarray(np.concatenate([d, d ^ 0x5A], 1))


def widen(api, F, dim):
    """F with dim-byte rows made from its 32-byte ones"""
    if dim == 32:
        return F
    w = widener(dim)
    return api.Frame(F.keys, F.key_cam, w(F.desc), w(F.dmask), list(zip(F.cam_w, F.cam_h)), F.scale_factors)


def reversed_image(im):
    """a decoy image: the keypoints, descriptors and masks of `im` in reverse order"""
    k, d, m = im
    return k[::-1].copy(), d[::-1].copy(), None if m is None else m[::-1].copy()


def pack_frames(frames, capacity, dim=None, layout="single", device="cuda", first_image=1, after=1, decoy=None):
    """Frames (api.Frame or per-camera [(kps, desc, dmask)]) -> one packed-frame record (buffer, n_parts, part_images,
    first_image) per frame.  Layouts:
      single:   each frame alone in a buffer, `first_image` decoy images before its cameras and `after` after them;
      parts:    every camera of every frame a one-image part of one buffer, as the allgather leaves a batch of frames;
      separate: each frame's cameras one-image parts of a buffer of its own;
      joint:    all frames' cameras consecutive images of one single-part buffer.
    The decoy is `decoy` if given, else each frame's first camera reversed.  device None gives numpy buffers."""
    from multicol_slam_b200 import rig
    per = [f if isinstance(f, list) else per_cam(f) for f in frames]
    nc = len(per[0])
    dim = dim or per[0][0][1].shape[1]
    parts = lambda ims: np.concatenate([rig.pack([im], capacity, dim) for im in ims])  # noqa: E731
    if layout == "single":
        out = []
        for p in per:
            dec = decoy or reversed_image(p[0])
            out.append((rig.pack([dec] * first_image + p + [dec] * after, capacity, dim), 1, nc + first_image + after, first_image))
    elif layout == "parts":
        b = parts([im for p in per for im in p])
        out = [(b, nc * len(per), 1, nc * i) for i in range(len(per))]
    elif layout == "separate":
        out = [(parts(p), nc, 1, 0) for p in per]
    else:
        assert layout == "joint", layout
        b = rig.pack([im for p in per for im in p], capacity, dim)
        out = [(b, 1, nc * len(per), nc * i) for i in range(len(per))]
    if device is None:
        return out
    tensors = {id(b): on_device(b, device) for b, *_ in out}           # one tensor per buffer
    return [(tensors[id(b)],) + tuple(r) for b, *r in out]


# ---- slot-indexed rows ------------------------------------------------------------------------------------------------------------
def to_slots(api, F, row, capacity, fill, device="cuda", dtype=np.int32):
    """a row in contiguous keypoint order -> its slot-indexed tensor (slot c * capacity + j), `fill` beyond each camera's count.
    F is a Frame or its per-camera counts."""
    n = F if isinstance(F, (list, tuple, np.ndarray)) else counts(F)
    return on_device(api.contiguous_to_slots(np.asarray(row, np.int32), n, capacity, fill=fill).astype(dtype), device)


def from_slots(api, t, counts, capacity, fill):
    """a slot-indexed row (tensor or array) back to contiguous order, after checking that every slot at or beyond a camera's count
    still holds `fill`"""
    a = np.asarray(t.cpu().numpy() if hasattr(t, "cpu") else t).reshape(-1, capacity)
    for c, n in enumerate(counts):
        assert np.all(a[c, int(n):] == fill), f"camera {c}: a slot beyond the count was written"
    return api.slots_to_contiguous(a.reshape(-1), counts, capacity)


def slot_to_contiguous_index(slots, counts, capacity):
    """slot indices c * capacity + j -> contiguous keypoint indices, checking each j < its camera's count"""
    first = np.concatenate([[0], np.cumsum(counts)])
    slots = np.asarray(slots)
    c, j = slots // capacity, slots % capacity
    assert np.all(j < np.asarray(counts)[c])
    return (first[c] + j).astype(np.int32)
