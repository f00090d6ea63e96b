"""CPU: argument validation of local mapping's device SearchForTriangulationRaw (mcs_search_for_triangulation_device) happens on the
host before any launch, and without a device the accepted shapes fail with MCS_ERR_NO_DEVICE.  The host route the device call is
compared with (cORBmatcher.SearchForTriangulationRawHost: read back, slots_to_contiguous, host rays, SearchForTriangulationRaw), run
here on the oracle's search, reproduces the reference's own SearchForTriangulationRaw(KF1, KF2) (recorded in
tests/golden/ref_tape_search_for_triangulation_device_cpu.*), for one neighbour and along CreateNewMapPoints' sequence of five
neighbours, where the points triangulated with one neighbour leave the next search's queries."""
import ctypes as C

import numpy as np
import pytest

from device_frames import BIG_ID, FAKE, counts, declared_symbols, frames, pack_frames, taped_rm, to_slots  # noqa: F401  (frames: a fixture)
from search_scenes import essential, rays_of, reference_tri, rig_of, tri_scene

rm = taped_rm("search_for_triangulation_device_cpu")


def _call(api, kf1=(FAKE, 1, 4, 0), mp1=FAKE, kf2=(FAKE, 1, 4, 0), mp2=FAKE, n_cams=4, capacity=2000, dim=32, cams=True, E=True,
          epi=1e-2, th_low=32, masks=1, m12=FAKE, nm=FAKE, diag=FAKE):
    from multicol_slam_b200.ctypes_defs import Ocam, PackedFrame
    nc = max(n_cams, 1)
    oc = (Ocam * nc)() if cams else None
    Em = np.zeros((nc, nc, 3, 3)) if E else None
    return api.lib().mcs_search_for_triangulation_device(C.byref(PackedFrame(*kf1)) if kf1 is not None else None, mp1,
                                                         C.byref(PackedFrame(*kf2)) if kf2 is not None else None, mp2, n_cams, capacity,
                                                         dim, oc, api._p(Em), epi, th_low, masks, m12, nm, diag, None)


FRAMES_BAD = [(None, 1, 4, 0), (FAKE, 0, 4, 0), (FAKE, 1, 0, 0), (FAKE, 1, 4, -1), (FAKE, 1, 4, 1), (FAKE, 3, 1, 0)]


def test_validation(api):
    bad = [dict(kf1=None), dict(kf2=None), dict(mp1=None), dict(mp2=None), dict(cams=False), dict(E=False), dict(m12=None), dict(nm=None),
           dict(n_cams=0), dict(n_cams=-1), dict(capacity=0), dict(capacity=-5), dict(dim=24), dict(dim=0), dict(dim=128)]
    bad += [dict(kf1=f) for f in FRAMES_BAD] + [dict(kf2=f) for f in FRAMES_BAD]
    for kw in bad:
        assert _call(api, **kw) == api.MCS_ERR_INVALID, kw
    # a camera's rows and "taken" bits in one CTA, 16-bit segment indices; the device searches' 2^24 query bound
    assert _call(api, capacity=65536) == api.MCS_ERR_UNSUPPORTED
    assert b"65535" in api.lib().mcs_last_error()
    assert _call(api, n_cams=257, capacity=65535, kf1=(FAKE, 1, 257, 0), kf2=(FAKE, 1, 257, 0)) == api.MCS_ERR_UNSUPPORTED
    assert b"2^24" in api.lib().mcs_last_error()
    ok = [dict(), dict(diag=None), dict(masks=0), dict(dim=16), dict(dim=64), dict(capacity=1), dict(capacity=65535), dict(n_cams=1, kf1=(FAKE, 1, 1, 0)),
          dict(kf1=(FAKE, 2, 4, 4), kf2=(FAKE, 2, 4, 0)), dict(kf1=(FAKE, 8, 1, 4), kf2=(FAKE, 8, 1, 0)), dict(th_low=-1), dict(epi=0.0),
          dict(epi=float("nan")), dict(n_cams=256, capacity=65535, kf1=(FAKE, 1, 256, 0), kf2=(FAKE, 1, 256, 0))]
    if api.device_count() == 0:
        for kw in ok:
            assert _call(api, **kw) == api.MCS_ERR_NO_DEVICE, kw


def test_symbol_is_declared_and_exported(api):
    assert "mcs_search_for_triangulation_device" in declared_symbols() and hasattr(api.lib(), "mcs_search_for_triangulation_device")
    assert callable(api.cORBmatcher.SearchForTriangulationRawDevice) and callable(api.cORBmatcher.SearchForTriangulationRawHost)


def host_route(api, m, s, k, cams, cap, mp1, mp2, layout="single", device="cpu", _st=None, epi=1e-2):
    """SearchForTriangulationRawHost(KF1, neighbour k) with the given contiguous map-point rows -> (nmatches, matches12 by slot)"""
    packs = pack_frames([s["KF1"], s["nbs"][k]], cap, layout=layout, device=device)
    E = essential(s["rig1"], s["rigs"][k])
    return m.SearchForTriangulationRawHost(packs[0], to_slots(api, s["KF1"], mp1, cap, BIG_ID, device), packs[1],
                                           to_slots(api, s["nbs"][k], mp2, cap, BIG_ID, device), cams, cap, E, epi, _st=_st)


def pairs_of(api, s, k, m12, cap):
    """the (KF1 index, KF2 index) pairs, contiguous order, of a slot-indexed matches12 row"""
    c1 = api.slots_to_contiguous(m12, counts(s["KF1"]), cap)
    s2 = api.slots_to_contiguous(np.arange(len(m12), dtype=np.int32), counts(s["nbs"][k]), cap)
    inv = {int(v): i for i, v in enumerate(s2)}
    return np.array([(i, inv[int(b)]) for i, b in enumerate(c1) if b >= 0], np.int32).reshape(-1, 2)


def triangulate_stand_in(rng, s, k, m12, cap, mp1_slots, mp2_slots):
    """A seeded stand-in for CreateNewMapPoints' checks (ref src/cLocalMapping.cpp:284-367): about 70 % of the pairs become new map
    points, whose ids go into both slot rows (AddMapPoint on KF1 and on the neighbour)."""
    hit = np.flatnonzero(m12 >= 0)
    keep = hit[rng.random(len(hit)) < 0.7]
    ids = s["next_id"] + np.arange(len(keep), dtype=np.int32)
    s["next_id"] += len(keep)
    mp1_slots[keep] = ids
    mp2_slots[m12[keep]] = ids
    return len(keep)


@pytest.mark.parametrize("masks", [False, True])
def test_host_route_equals_reference(oa, rm, api, frames, cams, masks):
    """the oracle-backed host route == the reference's SearchForTriangulationRaw(KF1, KF_k), pair for pair, for each neighbour
    from the same KF1 state; one neighbour is KF1 itself"""
    s = tri_scene(api, frames, cams, 3)
    s["nbs"].append(s["KF1"]); s["mps"].append(s["mp1"]); s["rigs"].append(rig_of(api, cams, [0.02, 0.0, -0.01]))
    assert np.array_equal(rays_of(api, s["KF1"], cams), oa.frame_prepare(s["KF1"].keys, s["KF1"].key_cam, cams)[0])
    m = api.cORBmatcher(0.6, False, 32, masks)
    cap = max(max(counts(F)) for F in [s["KF1"]] + s["nbs"]) + 3
    for k in range(len(s["nbs"])):
        n, m12 = host_route(api, m, s, k, cams, cap, s["mp1"], s["mps"][k], _st=oa.search_for_triangulation)
        rn, rpairs = reference_tri(rm, api, s, k, cams, s["mp1"], s["mps"][k], masks)
        assert rn == n > 20, k
        assert np.array_equal(rpairs, pairs_of(api, s, k, m12, cap)), k


def sequence(api, oa, m, s, cams, cap, seed, rm=None, masks=False):
    """CreateNewMapPoints' loop over the neighbours (ref src/cLocalMapping.cpp:226-380) on the host route, the stand-in writing the
    new points into KF1's and the neighbour's rows after each search.  Returns the per-neighbour (nmatches, matches12)."""
    rng = np.random.default_rng(seed)
    mp1 = s["mp1"].copy()
    out = []
    for k in range(len(s["nbs"])):
        mp2 = s["mps"][k].copy()
        n, m12 = host_route(api, m, s, k, cams, cap, mp1, mp2, _st=oa.search_for_triangulation)
        if rm is not None:
            rn, rpairs = reference_tri(rm, api, s, k, cams, mp1, mp2, masks)
            assert rn == n and np.array_equal(rpairs, pairs_of(api, s, k, m12, cap)), k
        out.append((n, m12))
        s1 = api.contiguous_to_slots(mp1, counts(s["KF1"]), cap)
        s2 = api.contiguous_to_slots(mp2, counts(s["nbs"][k]), cap)
        triangulate_stand_in(rng, s, k, m12, cap, s1, s2)
        mp1 = api.slots_to_contiguous(s1, counts(s["KF1"]), cap)
    return out


@pytest.mark.parametrize("masks", [False, True])
def test_neighbour_sequence_equals_reference(oa, rm, api, frames, cams, masks):
    """five neighbours in CreateNewMapPoints' order, KF1's row updated between the searches: the host route == the reference at
    every step; the same five searches made from KF1's entry state give another result, so no call over all neighbours at once
    can be the reference's"""
    s = tri_scene(api, frames, cams, 5, seed=11)
    m = api.cORBmatcher(0.6, False, 32, masks)
    cap = max(max(counts(F)) for F in [s["KF1"]] + s["nbs"]) + 3
    seq = sequence(api, oa, m, s, cams, cap, seed=5, rm=rm, masks=masks)
    entry = [host_route(api, m, s, k, cams, cap, s["mp1"], s["mps"][k], _st=oa.search_for_triangulation) for k in range(5)]
    assert seq[0][0] == entry[0][0] and np.array_equal(seq[0][1], entry[0][1])
    differ = [k for k in range(1, 5) if seq[k][0] != entry[k][0] or not np.array_equal(seq[k][1], entry[k][1])]
    assert len(differ) >= 3, differ
    assert all(seq[k][0] > 10 for k in range(5))
