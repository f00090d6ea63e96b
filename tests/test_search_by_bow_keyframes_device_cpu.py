"""CPU: argument validation of loop closing's device SearchByBoW(KF1, KF_k) (mcs_search_by_bow_keyframes_device) happens on the host
before any launch, and without a device the accepted shapes fail with MCS_ERR_NO_DEVICE.  The host route the device call is compared
with (cORBmatcher.SearchByBoWKeyFramesHost: read back, slots_to_contiguous, one brute-force SearchByBoW per candidate), run here on
the oracle's brute-force matcher, reproduces the reference's own SearchByBoW(KF1, KF2) (recorded in
tests/golden/ref_tape_search_by_bow_keyframes_device_cpu.*) on the scenes the GPU tests use."""
import ctypes as C

import numpy as np
import pytest

import test_ref_match_cpu as T

FAKE = 0x10000      # stands for a device pointer: never dereferenced by the host
BIG_ID = 1 << 30    # map-point id of the slots at or beyond a camera's count: reading one would raise the status
frames = T.frames


@pytest.fixture(scope="module")
def rm():
    """the reference's own matcher, live while recording and replayed from tests/golden/ref_tape_search_by_bow_keyframes_device_cpu.*"""
    import ref_tape
    return ref_tape.module("ref_match_api", "search_by_bow_keyframes_device_cpu", T.TAPE_LIMIT)


def _call(api, kf1=(FAKE, 1, 4, 0), mp1=FAKE, kfs=((FAKE, 1, 4, 0),), mps=None, n_kf=None, n_cams=4, capacity=2000, dim=32, n_points=500,
          bad=None, masks=1, m12=FAKE, slot=FAKE, nm=FAKE, status=FAKE):
    from multicol_slam_b200.ctypes_defs import PackedFrame
    arr = None if kfs is None else (PackedFrame * max(len(kfs), 1))(*[PackedFrame(*f) for f in kfs])
    if mps is None and kfs is not None:
        mps = [FAKE] * len(kfs)
    mp_arr = None if mps is None else (C.c_void_p * max(len(mps), 1))(*mps)
    n_kf = (0 if kfs is None else len(kfs)) if n_kf is None else n_kf
    return api.lib().mcs_search_by_bow_keyframes_device(C.byref(PackedFrame(*kf1)) if kf1 is not None else None, mp1, arr, mp_arr, n_kf,
                                                        n_cams, capacity, dim, n_points, bad, 64, 0.75, masks, m12, slot, nm, status, None)


FRAMES_BAD = [(None, 1, 4, 0), (FAKE, 0, 4, 0), (FAKE, 1, 0, 0), (FAKE, 1, 4, -1), (FAKE, 1, 4, 1), (FAKE, 3, 1, 0)]


def test_validation(api):
    two = ((FAKE, 1, 4, 0), (FAKE, 2, 4, 4))
    bad = [dict(n_kf=-1), dict(kf1=None), dict(mp1=None), dict(kfs=None, n_kf=1), dict(kfs=two, mps=[FAKE, None]), dict(m12=None),
           dict(nm=None), dict(status=None), dict(n_points=-1), dict(n_cams=0), dict(capacity=0), dict(capacity=65536), dict(dim=24),
           dict(dim=0), dict(dim=128)]
    bad += [dict(kf1=f) for f in FRAMES_BAD] + [dict(kfs=((FAKE, 1, 4, 0), f)) for f in FRAMES_BAD]
    for kw in bad:
        assert _call(api, **kw) == api.MCS_ERR_INVALID, kw
    _call(api, kfs=((FAKE, 1, 4, 0), (FAKE, 1, 4, 1)))
    assert b"candidate 1" in api.lib().mcs_last_error()
    # the "taken" bits of one candidate's database in one CTA's shared memory: n_cams * capacity <= 1 622 016
    assert _call(api, n_cams=25, capacity=65535, kf1=(FAKE, 1, 25, 0), kfs=((FAKE, 1, 25, 0),)) == api.MCS_ERR_UNSUPPORTED
    assert _call(api, n_cams=31, capacity=52324, kf1=(FAKE, 1, 31, 0), kfs=((FAKE, 1, 31, 0),)) == api.MCS_ERR_UNSUPPORTED
    # n_kf * n_cams * capacity below 2^31
    many = ((FAKE, 1, 24, 0),) * 1400
    assert _call(api, n_cams=24, capacity=65535, kf1=(FAKE, 1, 24, 0), kfs=many) == api.MCS_ERR_UNSUPPORTED
    assert b"2^31" in api.lib().mcs_last_error()
    # no candidates: a successful no-op, whatever else is passed
    assert _call(api, kfs=(), n_kf=0) == api.MCS_OK and _call(api, kfs=None, n_kf=0, kf1=None, mp1=None, m12=None) == api.MCS_OK
    ok = [dict(), dict(kfs=two), dict(kfs=((FAKE, 4, 1, 0),) * 8), dict(kf1=(FAKE, 2, 4, 4), kfs=((FAKE, 2, 4, 0), (FAKE, 2, 4, 4))),
          dict(slot=None), dict(bad=FAKE), dict(masks=0), dict(dim=16), dict(dim=64), dict(n_points=0), dict(capacity=65535),
          dict(n_cams=32, capacity=50688, kf1=(FAKE, 1, 32, 0), kfs=((FAKE, 1, 32, 0),)),
          dict(n_cams=2, capacity=65535, kf1=(FAKE, 1, 2, 0), kfs=((FAKE, 1, 2, 0),) * 16000)]
    if api.device_count() == 0:
        for kw in ok:
            assert _call(api, **kw) == api.MCS_ERR_NO_DEVICE, kw


def test_symbol_is_declared_and_exported(api):
    from test_cabi_symbols import declared_symbols
    assert "mcs_search_by_bow_keyframes_device" in declared_symbols() and hasattr(api.lib(), "mcs_search_by_bow_keyframes_device")
    assert callable(api.cORBmatcher.SearchByBoWKeyFramesDevice) and callable(api.cORBmatcher.SearchByBoWKeyFramesHost)


# ---- the scenes ------------------------------------------------------------------------------------------------------------------
def counts(F):
    return [int((F.key_cam == c).sum()) for c in range(len(F.cam_w))]


def max_count(s):
    """the most keypoints a camera of the scene's frames holds"""
    return max(max(counts(F)) for F in [s["KF1"]] + s["cands"])


def widen(api, F, dim):
    """F with 16- or 64-byte rows made from its 32-byte ones (first half / row and its bitwise complement-ish variant)"""
    if dim == 32:
        return F
    w = (lambda d: np.ascontiguousarray(d[:, :16])) if dim == 16 else (lambda d: np.ascontiguousarray(np.concatenate([d, d ^ 0x5A], 1)))
    return api.Frame(F.keys, F.key_cam, w(F.desc), w(F.dmask), list(zip(F.cam_w, F.cam_h)), F.scale_factors)


def bow_kf_scene(api, frames, n_kf, seed=5, dim=32):
    """KF1 = the first frame, about 60 % of its keypoints carrying map points 0 ..; candidate k a variant of either frame (a few bits
    flipped per descriptor, more for later candidates) carrying points of its own; about 5 % of all points bad."""
    F1, F2 = frames
    rng = np.random.default_rng(seed)
    KF1 = widen(api, F1, dim)
    n1 = len(F1.keys)
    mp1 = np.where(rng.random(n1) < 0.6, np.arange(n1), -1).astype(np.int32)
    cands, mps, off = [], [], n1
    for k in range(n_kf):
        B = F2 if k % 2 else F1
        F = api.Frame(B.keys, B.key_cam, T.flip_bits(rng, B.desc, 2 + k % 6), B.dmask, list(zip(B.cam_w, B.cam_h)), B.scale_factors)
        cands.append(widen(api, F, dim))
        n = len(B.keys)
        mps.append(np.where(rng.random(n) < 0.6, off + np.arange(n), -1).astype(np.int32))
        off += n
    bad = (rng.random(off) < 0.05).astype(np.uint8)
    return dict(KF1=KF1, mp1=mp1, cands=cands, mps=mps, bad=bad, n_points=off)


def pack_frames(KFs, cap, layout, device="cpu"):
    """one (packed uint8 tensor, n_parts, part_images, first_image) per frame.  single: each frame alone in its buffer with a decoy
    image before and after its cameras; parts: every camera a one-image part of one buffer (an allgather); joint: all frames' cameras
    as images of one single-part buffer."""
    import torch
    from multicol_slam_b200 import rig
    dim = KFs[0].desc.shape[1]
    t = lambda b: torch.from_numpy(b).to(device)  # noqa: E731
    per = [[(F.keys[F.key_cam == c], F.desc[F.key_cam == c], F.dmask[F.key_cam == c]) for c in range(len(F.cam_w))] for F in KFs]
    nc = len(per[0])
    if layout == "single":
        out = []
        for p in per:
            k, d, m = p[0]
            decoy = (k[::-1].copy(), d[::-1].copy(), m[::-1].copy())
            out.append((t(rig.pack([decoy] + p + [decoy], cap, dim)), 1, nc + 2, 1))
        return out
    if layout == "parts":
        b = t(np.concatenate([rig.pack([c], cap, dim) for p in per for c in p]))
        return [(b, nc * len(per), 1, nc * i) for i in range(len(per))]
    b = t(rig.pack([c for p in per for c in p], cap, dim))
    return [(b, 1, nc * len(per), nc * i) for i in range(len(per))]


def slot_row(api, F, mp, cap, fill=BIG_ID, device="cpu"):
    import torch
    return torch.from_numpy(api.contiguous_to_slots(np.asarray(mp, np.int32), counts(F), cap, fill=fill)).to(device)


def host_route(api, m, s, cap, layout="single", device="cpu", _bf=None, cands=None):
    """SearchByBoWKeyFramesHost on the scene -> (matches12, match_slot, nmatches, status)"""
    import torch
    idx = range(len(s["cands"])) if cands is None else cands
    packs = pack_frames([s["KF1"]] + [s["cands"][k] for k in idx], cap, layout, device)
    kfs = [(packs[1 + i], slot_row(api, s["cands"][k], s["mps"][k], cap, device=device)) for i, k in enumerate(idx)]
    return m.SearchByBoWKeyFramesHost(packs[0], slot_row(api, s["KF1"], s["mp1"], cap, device=device), kfs, len(s["KF1"].cam_w), cap,
                                      s["n_points"], torch.from_numpy(s["bad"]).to(device), _bf=_bf)


def reference_bow_kf(rm, cams, s, k, nnratio, masks):
    """the reference's SearchByBoW(KF1, KF_k): (nmatches, map-point id per KF1 keypoint in contiguous order)"""
    table = rm.MPTable(3, np.zeros((s["n_points"], 32), np.uint8), bad=s["bad"])
    return rm.search_by_bow_kfkf(rm.KF(s["KF1"], cams, mp=s["mp1"]), rm.KF(s["cands"][k], cams, mp=s["mps"][k]), table, nnratio, masks)


@pytest.mark.parametrize("masks", [False, True])
def test_host_route_equals_reference(oa, rm, api, frames, cams, masks):
    """the oracle-backed host route == the reference's SearchByBoW(KF1, KF_k), map-point id for map-point id, candidate by
    candidate; one of the candidates is KF1 itself"""
    s = bow_kf_scene(api, frames, 5)
    s["cands"].append(s["KF1"]); s["mps"].append(s["mp1"])
    m = api.cORBmatcher(0.75, False, 32, masks)
    cap = max_count(s) + 3
    m12, slot12, nm, st = host_route(api, m, s, cap, _bf=oa.match_bruteforce)
    assert st[0] == api.MCS_OK
    for k in range(len(s["cands"])):
        rn, rout = reference_bow_kf(rm, cams, s, k, 0.75, masks)
        assert rn == nm[k] > 20, k
        assert np.array_equal(rout, api.slots_to_contiguous(m12[k], counts(s["KF1"]), cap)), k
    # KF1 against itself: every valid keypoint whose own descriptor is not ambiguous matches itself
    self_row = api.slots_to_contiguous(m12[-1], counts(s["KF1"]), cap)
    assert (self_row[self_row >= 0] == s["mp1"][self_row >= 0]).mean() > 0.9
