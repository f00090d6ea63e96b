"""CPU: the 64x48 keypoint grid and the window searches on hand-built edge scenes, at descriptor sizes 16, 32 and 64.

The scenes place keypoints by hand where GetFeaturesInArea / PosInGrid decide (ref src/cMultiFrame.cpp:272-353): on the inclusive
window border `!(|kx - x| > r)` and one float ulp outside it, on cell borders of the floor / ceil cell range, in windows partly or
wholly off the image, at half-cell positions where cvRound ties to even (and a keypoint rounding to column 64 or row 48 is dropped),
in cells of 31, 32, 33 and 70 keypoints, and in a camera with no keypoints.  One frame has cameras of one size whose grid steps
are exact (1024x768: 16 px cells), the other mixes 1024x768, 754x480 and 1280x720.  Each case is first shown to be reached on the
C++ oracle's output; then the oracle, oracle/pyref_match.py and the reference's own matcher (replayed from
tests/golden/ref_tape_window_edges_cpu.*, see oracle/ref_tape.py) must agree on every call.  tests/test_window_search_widths_gpu.py
builds the same scenes and compares the CUDA kernels with the oracle."""
import numpy as np
import pytest

from device_frames import taped_rm
from window_edge_scenes import CROWD_ROW, CROWDED, EMPTY_CAM, LEVEL_FORMS, SIZES, edge_scene, projection_scene, second_frame

rm = taped_rm("window_edges_cpu", limit=256)     # larger results are stored as digests (oracle/ref_tape.py) and compared with ref_tape.same


def _in_grid(oa, F, cams):
    _, start, items = oa.frame_prepare(F.keys, F.key_cam, cams)
    return start, items


@pytest.mark.parametrize("kind", ["exact", "mixed"])
def test_edge_scene_reaches_every_case(oa, kind):
    """the builder reaches what it is for, read off the oracle's grid and window lists"""
    sc = edge_scene(kind, 32)
    F = sc.frame
    start, items = _in_grid(oa, F, sc.cams)
    per_cell = np.diff(start).reshape(len(F.cam_w), 64, 48)
    assert per_cell[EMPTY_CAM].sum() == 0 and (F.key_cam == EMPTY_CAM).sum() == 0
    gridded = np.zeros(len(F.keys), bool)
    gridded[items] = True
    for c in range(len(F.cam_w)):
        if c == EMPTY_CAM:
            continue
        for ix, m in CROWDED.items():
            assert per_cell[c, ix, CROWD_ROW] >= m
        assert {31, 32, 33}.issubset(set(per_cell[c].ravel().tolist())) and per_cell[c].max() > 64
        mk = sc.marks[c]
        assert not gridded[sc.first[c] + np.array(mk.dropped)].any() and gridded[sc.first[c] + np.array(mk.col0)].all()
        col0 = start[(c * 64 + 0) * 48 + 20], start[(c * 64 + 0) * 48 + 21]
        assert sc.first[c] + mk.col0[0] in items[col0[0]:col0[1]]
    oi, _, oc, rc = oa.window_search(F, sc.queries, sc.qdesc, sc.qmask, max_cand=4096)
    assert rc == 0
    got = [set(oi[i, :oc[i]].tolist()) for i in range(len(sc.queries))]
    q = sc.queries
    nolev = (q["min_level"] == -1) & (q["max_level"] == -1)
    nf = len(LEVEL_FORMS)
    for c in range(len(F.cam_w)):
        mk = sc.marks[c]
        w0 = int(np.flatnonzero(q["cam"] == c)[0]) // nf                # first window of camera c
        for wi, ins, outs in mk.border:                                 # border keypoints in, one ulp beyond out
            i = (w0 + wi) * nf
            assert q["min_level"][i] == -1 and q["max_level"][i] == -1
            assert {sc.first[c] + k for k in ins} <= got[i] and not ({sc.first[c] + k for k in outs} & got[i])
        sel = np.flatnonzero(nolev & (q["cam"] == c))
        for i in sel:
            name = sc.names[i]
            if name == "off":
                assert oc[i] == 0
            if name == "whole":
                assert oc[i] == per_cell[c].sum()
            if name == "partial" and c != EMPTY_CAM:
                assert oc[i] > 0
    # every level form returns candidates somewhere, the l = 0 form included
    for lo, hi in LEVEL_FORMS:
        assert oc[(q["min_level"] == lo) & (q["max_level"] == hi)].sum() > 50
    assert oc[sc.names == "crowded"].max() > 64


@pytest.mark.parametrize("kind", ["exact", "mixed"])
def test_features_in_area_three_ways(oa, rm, kind):
    """GetFeaturesInArea of the reference (both overloads) == the oracle's window lists == pyref_match, on every edge window"""
    import pyref_match as pm
    sc = edge_scene(kind, 32)
    F = sc.frame
    kf = rm.KF(F, sc.cams)
    grid = pm.Grid(F.keys, F.key_cam, SIZES[kind])
    oi, _, oc, rc = oa.window_search(F, sc.queries, sc.qdesc, sc.qmask, max_cand=4096)
    assert rc == 0
    for i, qq in enumerate(sc.queries):
        cam, x, y, r, lo, hi = int(qq["cam"]), float(qq["x"]), float(qq["y"]), float(qq["r"]), int(qq["min_level"]), int(qq["max_level"])
        ref = rm.features_in_area(kf, False, cam, x, y, r, lo, hi)
        assert ref == grid.features_in_area(cam, x, y, r, lo, hi) == list(oi[i, :oc[i]]), (i, sc.names[i])
        if lo == -1 and hi == -1:                                     # the key-frame overload: `<= r`, no level filter
            assert rm.features_in_area(kf, True, cam, x, y, r) == grid.features_in_area_kf(cam, x, y, r) == ref


@pytest.mark.parametrize("kind", ["exact", "mixed"])
def test_frame_prepare_grid_three_ways(oa, rm, kind):
    """the oracle's CSR grid == pyref_match's cells, and per camera its items in cell order == the reference's whole-image window"""
    import pyref_match as pm
    sc = edge_scene(kind, 32)
    F = sc.frame
    _, start, items = oa.frame_prepare(F.keys, F.key_cam, sc.cams)
    grid = pm.Grid(F.keys, F.key_cam, SIZES[kind])
    flat = [grid.cells[c][ix][iy] for c in range(len(F.cam_w)) for ix in range(64) for iy in range(48)]
    assert np.array_equal(np.diff(start), [len(v) for v in flat])
    assert items.tolist() == [k for v in flat for k in v]
    kf = rm.KF(F, sc.cams)
    for c, (w, h) in enumerate(SIZES[kind]):
        lo, hi = start[c * 64 * 48], start[(c + 1) * 64 * 48]
        assert rm.features_in_area(kf, False, c, w / 2, h / 2, 4.0 * max(w, h), -1, -1) == items[lo:hi].tolist()


@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masked", [False, True])
def test_window_search_distances(oa, rm, dim, masked):
    """the oracle's candidate distances at every width == pyref_match's, with a sample against the reference's distance"""
    import pyref_match as pm
    for kind in ("exact", "mixed"):
        sc = edge_scene(kind, dim)
        F = sc.frame
        qm = sc.qmask if masked else None
        oi, od, oc, rc = oa.window_search(F, sc.queries, sc.qdesc, qm, max_cand=4096)
        assert rc == 0
        rng = np.random.default_rng(dim)
        for i in range(len(sc.queries)):
            for j in range(oc[i]):
                k = oi[i, j]
                want = pm.distance(sc.qdesc[i], F.desc[k], qm[i] if masked else None, F.dmask[k] if masked else None)
                assert od[i, j] == want
        hit = np.flatnonzero(oc > 0)
        for i in rng.choice(hit, 12, replace=False):
            k = oi[i, 0]
            ref = rm.distance64_masked(sc.qdesc[i], F.desc[k], sc.qmask[i], F.dmask[k], dim) if masked else \
                rm.distance64(sc.qdesc[i], F.desc[k], dim)
            assert ref == od[i, 0]


def _tables(rm, mps, nc):
    return rm.MPTable(nc, mps.desc, dmask=mps.dmask, bad=mps.bad, in_view=mps.in_view, level=mps.level, proj_x=mps.proj_x,
                      proj_y=mps.proj_y, view_cos=mps.view_cos)


@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("kind", ["exact", "mixed"])
def test_searches_equal_reference(oa, rm, kind, dim, masked):
    """SearchByProjection(F, MapPoints, th), SearchForInitialization and WindowSearch of the reference on the edge scenes ==
    the oracle (and pyref_match for the first two)"""
    import multicol_slam_b200.api as api
    import pyref_match as pm
    from ref_tape import same
    sc = edge_scene(kind, dim)
    F = sc.frame
    nc = len(F.cam_w)
    th_high, th_low = rm.thresholds(dim, masked)
    m = api.cORBmatcher(0.8, False, dim, masked)
    assert (m.TH_HIGH_, m.TH_LOW_) == (th_high, th_low)
    grid = pm.Grid(F.keys, F.key_cam, SIZES[kind])
    mps = projection_scene(F, dim, masked, seed=dim + 2 * masked)
    table = _tables(rm, mps, nc)
    for th, pre in ((3.0, None), (1.0, np.where(np.arange(len(F.keys)) % 4 == 0, 0, -1))):
        start = np.full(len(F.keys), -1, np.int32) if pre is None else pre.astype(np.int32)
        on, ofmp = oa.search_by_projection(F, mps, th, 0.8, th_high, masked, start.copy())
        rn, rfmp = rm.search_by_projection(rm.KF(F, sc.cams, mp=start), table, th, 0.8, masked)
        pn, pfmp = pm.search_by_projection(F, grid, mps, th, 0.8, th_high, masked, start.copy())
        assert on == rn == pn and same(ofmp, rfmp) and np.array_equal(ofmp, pfmp)
        assert on > 100
    F2 = second_frame(F, 10.0, seed=dim)
    prev = np.stack([F.keys["x"], F.keys["y"]], axis=1).astype(np.float64)
    grid2 = pm.Grid(F2.keys, F2.key_cam, SIZES[kind])
    for window in (10, 40):
        on, om12, oprev = oa.search_for_initialization(F, F2, prev, window, 0.9, th_low, masked)
        rn, rm12, rprev = rm.search_for_initialization(rm.KF(F, sc.cams), rm.KF(F2, sc.cams), prev, window, 0.9, masked)
        pn, pm12, pprev = pm.search_for_initialization(F, F2, grid2, prev, window, 0.9, th_low, masked)
        assert on == rn == pn and same(om12, rm12) and np.array_equal(om12, pm12)
        assert same(oprev, rprev) and np.array_equal(oprev, pprev)
        assert on > 100
    rng = np.random.default_rng(dim + masked)
    n1 = len(F.keys)
    has1 = rng.random(n1) < 0.7
    mp1 = np.where(has1, np.arange(n1), -1).astype(np.int32)
    wt = rm.MPTable(nc, np.zeros((n1, dim), np.uint8))
    for minl in (0, 1):
        rn, rout = rm.window_search(rm.KF(F, sc.cams, mp=mp1), rm.KF(F2, sc.cams), wt, 10, minl, 2**31 - 1, 0.8, masked)
        on, o21 = m.WindowSearch(F, F2, 10, has1, minl, _sw=oa.search_windows)
        assert rn == on and same(o21, rout) and rn > 100
