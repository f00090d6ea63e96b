"""GPU: the device Fuse (mcs_fuse_device) on the window edge scenes of tests/fuse_window_scenes.py, for all three overloads, at
16, 32 and 64 bytes with masks on and off, with the key frames alone in a buffer each or as one-image parts of one buffer.

Fuse(pKF, ., th) (:1420) decides in fu_first_kernel, which walks the window with its own copy of window_kbest's cell range,
visiting order and level / radius tests; the other two read the first key of window_kbest's list (fu_best_kernel).  On these
scenes a copy that iterates the cells row by row, tests the radius with `>=` or in float32, filters the levels {l, l + 1} or
stops after a cell's first 32 items gives other hits (tests/test_fuse_window_edges_cpu.py::test_edges_discriminate), and so does
a list that breaks ties by slot or keeps distances `< TH_LOW_`.

The device projection calls CUDA's atan and the host's the libm's, so a device window centre can differ from the host's by a few
ulps (DESIGN.md section 2), and a keypoint built at distance r exactly from the host's centre can then fall outside.  So the device's
centres are read off frustum_kernel, which runs the same cam_project_in_mask, and the device hits must equal, hit for hit, the
walk model (tests/fuse_window_scenes.py::walk, equal to the host window search on the host's centres) on the device's centres,
and the host's window search wherever the centres agree.  The replayed map mutations must equal the host Fuse's and the
reference's (the oracle's window search where the reference did not travel), on the queries whose hits do not move with a
centre."""
import numpy as np
import pytest

from device_frames import counts
from device_frames import rm  # noqa: F401  (a fixture)
from device_searches import dev_map, fuse_device, fuse_replay
from fuse_window_scenes import N_KF, cameras, designed, host_best, model_best, projection_rig, scene, windows
from search_scenes import host_fuse, reference_ops

pytestmark = pytest.mark.gpu


def _device(api, m, KFs, ss, variant, layout, cap):
    return fuse_device(api, m, KFs, [s["sc"]["rig"] for s in ss], [None] * len(KFs), ss[0]["points"], dev_map(ss[0]), cap, layout, variant,
                       Scw=ss[0]["Scw"])


def _device_windows(api, KF, s, variant):
    """the scene's windows with the device's centres: frustum_kernel's proj_x / proj_y for the same pose (viewing angle 0, no
    distance bounds, so that only the projection and the mask decide), and which centres differ from the host's"""
    prig = projection_rig(api, s, variant)
    po = s["world"] - prig.M_t[:3, 3]
    nrm = po / np.linalg.norm(po, axis=1)[:, None]
    n = len(po)
    iv, _, px, py, _ = api.project_mappoints(prig.MtMc_inv, prig.MtMc, prig.cams, np.stack(prig.masks), s["world"], nrm, np.zeros(n),
                                             np.full(n, np.inf), KF.scale_factors)
    win = windows(api, KF, s, variant)
    i, c = win[0][:, 0], win[0][:, 1]
    assert iv[i, c].all()
    return win, (win[0], px[i, c], py[i, c]) + win[3:], (px[i, c] != win[1]) | (py[i, c] != win[2])


@pytest.mark.parametrize("layout", ["single", "parts"])
@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("variant", [0, 1, 2])
def test_device_equals_host(api, oa, rm, variant, masks, dim, layout):
    """one call over the scene's key frames, per key frame: the host window search == the oracle's and decides every designed
    case as built; the device hits == the walk model on the device's centres, == the host's where the centres agree; the
    replayed ops == the host Fuse's == the reference's"""
    KFs, ss = scene(api, oa, variant, dim, masks)
    m = api.cORBmatcher(0.6, False, dim, masks)
    cap = max(max(counts(KF)) for KF in KFs) + 5
    hits, n, status, _ = _device(api, m, KFs, ss, variant, layout, cap)
    assert status == api.MCS_OK and n == len(hits)
    for k, (KF, s) in enumerate(zip(KFs, ss)):
        hb = host_best(api, m, KF, s, variant)
        assert np.array_equal(hb, host_best(api, m, KF, s, variant, _sw=oa.search_windows))
        cases = designed(api, KF, s, variant, k)
        assert all(hb[i, c] == want for _, i, c, want in cases)
        first = np.concatenate([[0], np.cumsum(counts(KF))])
        db = np.full_like(hb, -1)
        for kk, q, sl in hits:
            if kk == k:
                assert db[q, sl // cap] == -1
                db[q, sl // cap] = first[sl // cap] + sl % cap
        win, dwin, div = _device_windows(api, KF, s, variant)
        rows = win[0]
        assert np.array_equal(db, model_best(api, KF, s, variant, m.TH_LOW_, masks, win=dwin))
        agree = rows[~div]
        assert np.array_equal(db[agree[:, 0], agree[:, 1]], hb[agree[:, 0], agree[:, 1]]) and (hb >= 0).sum() > 50
        # most designed windows keep the host's centre on the device, the exact-radius ones included
        same = {(int(i), int(c)) for i, c in agree}
        exact = [(i, c) for kind, i, c, _ in cases if kind.startswith("exact_")]
        assert sum((i, c) in same for i, c in exact) >= len(exact) // 2
        # the replay, on the queries whose hits do not move with a centre (the others made bad, which every route skips)
        moved = np.unique(rows[div & (db[rows[:, 0], rows[:, 1]] != hb[rows[:, 0], rows[:, 1]])][:, 0])
        bad = s["bad"].copy()
        bad[s["points"][moved]] = 1
        s2 = dict(s, bad=bad)
        dn, dops, _ = fuse_replay(m, KF, s2, variant, hits, cap, k=k)
        hn, hops, _ = host_fuse(api, m, KF, s2, variant)
        assert dn == hn and np.array_equal(dops, hops) and len(dops) > 40
        if rm:
            rn, rops = reference_ops(api, rm, cameras(), KF, s2, variant, masks)
        else:
            rn, rops, _ = host_fuse(api, m, KF, s2, variant, _sw=oa.search_windows)
        assert rn == dn and np.array_equal(rops, dops)


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_batch_equals_separate_calls(api, oa, variant):
    """the call over all key frames as one-image parts of one buffer == one call per key frame on a buffer of its own"""
    KFs, ss = scene(api, oa, variant, 32, True)
    m = api.cORBmatcher(0.6, False, 32, True)
    cap = max(max(counts(KF)) for KF in KFs) + 3
    batch, n, status, _ = _device(api, m, KFs, ss, variant, "parts", cap)
    assert status == api.MCS_OK
    sep = []
    for k in range(N_KF):
        h, _, st, _ = _device(api, m, [KFs[k]], [ss[k]], variant, "single", cap)
        assert st == api.MCS_OK
        h = h.copy()
        h[:, 0] = k
        sep.append(h)
    sep = np.concatenate(sep)
    assert n == len(sep) > 100 and np.array_equal(batch, sep)
