"""CPU: the 64x48 keypoint grid and the window searches on hand-built edge scenes, at descriptor sizes 16, 32 and 64.

The scenes place keypoints by hand where GetFeaturesInArea / PosInGrid decide (ref src/cMultiFrame.cpp:272-353): on the inclusive
window border `!(|kx - x| > r)` and one float ulp outside it, on cell borders of the floor / ceil cell range, in windows partly or
wholly off the image, at half-cell positions where cvRound ties to even (and a keypoint rounding to column 64 or row 48 is dropped),
in cells of 31, 32, 33 and 70 keypoints, and in a camera with no keypoints.  One frame has cameras of one size whose grid steps
are exact (1024x768: 16 px cells), the other mixes 1024x768, 754x480 and 1280x720.  Each case is first shown to be reached on the
C++ oracle's output; then the oracle, oracle/pyref_match.py and the reference's own matcher (replayed from
tests/golden/ref_tape_window_edges_cpu.*, see oracle/ref_tape.py) must agree on every call.  tests/test_window_search_widths_gpu.py
builds the same scenes and compares the CUDA kernels with the oracle."""
import pathlib
import sys

import numpy as np
import pytest

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))

EXACT = [(1024, 768)] * 4                                   # 16 px cells: winv = hinv = 1/16 exactly
MIXED = [(1024, 768), (754, 480), (1280, 720), (754, 480)]
SIZES = {"exact": EXACT, "mixed": MIXED}
EMPTY_CAM = 3                                               # the camera without keypoints in both frames
SF = np.cumprod([1.0] + [1.2000000476837158] * 7)
CROWDED = {20: 31, 21: 32, 22: 33, 23: 70}                  # grid column -> keypoints placed in cell (column, CROWD_ROW)
CROWD_ROW = 30
N_BACKGROUND = 260
TAPE_LIMIT = 256           # larger results are stored as digests (oracle/ref_tape.py) and compared with ref_tape.same
# level filters of a window: none, one level, {l-1, l} with l = 0 (min_level = -1), {l-1, l} with l = 2
LEVEL_FORMS = [(-1, -1), (1, 1), (-1, 0), (1, 2)]


def _f32_boundary(x, r, sign):
    """(inside, outside): the float32 keypoint coordinate farthest from the double x on side `sign` that the window test
    `!(|(double)kx - x| > r)` keeps, and the next float32 beyond it"""
    f = np.float32(x + sign * r)
    step = np.float32(np.inf * sign)
    while abs(float(f) - x) > r:
        f = np.nextafter(f, -step)
    while not abs(float(np.nextafter(f, step)) - x) > r:
        f = np.nextafter(f, step)
    return f, np.nextafter(f, step)


class CamMarks:
    """what the builder placed in one camera: windows (x, y, r, name); border: (window, keypoints on its border, keypoints one
    ulp beyond it); keypoints PosInGrid drops / puts into column 0.  Keypoint indices are camera-local."""

    def __init__(self):
        self.windows, self.border, self.dropped, self.col0 = [], [], [], []


def _camera(rng, w, h, dim):
    """keypoints (x, y, octave) and the windows that reach the edges for one camera of size w x h"""
    cw, ch = w / 64.0, h / 48.0
    bx, by = rng.uniform(-3, w + 3, 300), rng.uniform(-3, h + 3, 300)
    keep = ~((bx > 19.4 * cw) & (bx < 23.6 * cw) & (by > (CROWD_ROW - 0.6) * ch) & (by < (CROWD_ROW + 0.6) * ch))
    xs, ys = list(bx[keep][:N_BACKGROUND]), list(by[keep][:N_BACKGROUND])      # background, the crowded cells left alone
    marks = CamMarks()

    def add(x, y):
        xs.append(float(np.float32(x))); ys.append(float(np.float32(y)))
        return len(xs) - 1
    for ix, m in CROWDED.items():                           # crowded cells: the warp's 32-wide chunk loop changes at 32 and 64
        for _ in range(m):
            add((ix + rng.uniform(-0.45, 0.45)) * cw, (CROWD_ROW + rng.uniform(-0.45, 0.45)) * ch)
    for k in (0, 1, 2, 17, 40, 61, 62):                      # half-cell columns: cvRound ties to even
        add((k + 0.5) * cw, 10.25 * ch)
    for k in (0, 1, 45, 46):                                 # half-cell rows
        add(12.25 * cw, (k + 0.5) * ch)
    marks.dropped += [add(63.5 * cw, 10.25 * ch), add(12.25 * cw, 47.5 * ch)]     # round to column 64 / row 48: outside the grid
    marks.dropped.append(add(float(np.nextafter(np.float32(-0.5 * cw), np.float32(-np.inf))), 20.25 * ch))
    marks.col0.append(add(-0.5 * cw, 20.25 * ch))           # cvRound(-0.5) = 0: a keypoint left of the image in column 0
    # inside the windows that lie partly off the image; the ones within half a cell of the right / bottom edge round to column 64 /
    # row 48 and are never found
    for x, y in ((1.0, h / 2 + 2), (0.0, h / 2 - 5), (w - 0.6 * cw, h / 2 - 3), (w / 2 + 1, 2.0), (w / 2 - 4, 0.0), (w / 2 - 2, h - 0.6 * ch)):
        add(x, y)
    marks.dropped += [add(w - 0.25, h / 2 + 6), add(w / 2 + 3, h - 0.5)]
    # window borders: x +- r and y +- r exactly (dyadic query) and the extreme floats of a non-dyadic one, plus one ulp outside
    probes = [(20 * cw + 0.0, 16 * ch, 10.0), (0.37 * w + 0.3, 0.61 * h + 0.7, 5.7), (0.8 * w + 0.1, 0.2 * h + 0.45, 3.3)]
    probes = [(float(np.float32(x)), float(np.float32(y)), r) for x, y, r in probes]
    for x, y, r in probes:
        ins, outs = [], []
        for sign in (-1, 1):
            ix, ox = _f32_boundary(x, r, sign)
            iy, oy = _f32_boundary(y, r, sign)
            ins += [add(ix, y), add(x, iy), add(ix, iy)]
            outs += [add(ox, y), add(x, oy), add(ox, iy), add(ix, oy)]
        marks.border.append((len(marks.windows), ins, outs))
        marks.windows.append((x, y, r, "border"))
    k0 = add(0.55 * w + 0.123, 0.45 * h + 0.321)             # r = 0: only the keypoint exactly at the centre
    outs = [add(np.nextafter(np.float32(xs[k0]), np.float32(np.inf)), ys[k0]),
            add(xs[k0], np.nextafter(np.float32(ys[k0]), np.float32(-np.inf)))]
    marks.border.append((len(marks.windows), [k0], outs))
    marks.windows.append((xs[k0], ys[k0], 0.0, "r0"))
    # windows whose x +- r / y +- r fall on cell borders, around the crowded cells and the half-cell keypoints
    marks.windows += [(10 * cw, 12 * ch, 2 * cw, "cellborder"), (3 * cw, 5 * ch, 3 * cw, "cellborder"),
                      (40 * cw, 30 * ch, 4 * ch, "cellborder"), (64 * cw - 2 * cw, 48 * ch - ch, 2 * cw, "cellborder")]
    marks.windows += [(ix * cw, CROWD_ROW * ch, 0.5 * cw, "crowded") for ix in CROWDED]
    marks.windows += [(21.5 * cw, CROWD_ROW * ch, 2.5 * cw, "crowded")]
    marks.windows += [(63.5 * cw, 10.25 * ch, 1.5 * cw, "halfcell"), (12.25 * cw, 47.5 * ch, 1.5 * ch, "halfcell"),
                      (1.0 * cw, 10.25 * ch, 1.5 * cw, "halfcell"), (-0.5 * cw, 20.25 * ch, 0.75 * cw, "halfcell")]
    # off the image: wholly and partly, on every side
    r = 10.0
    marks.windows += [(-r - 5, h / 2, r, "off"), (w + r + 5, h / 2, r, "off"), (w / 2, -r - 5, r, "off"), (w / 2, h + r + 5, r, "off")]
    marks.windows += [(-4.0, h / 2, r, "partial"), (w - 3.0, h / 2, r, "partial"), (w / 2, -4.0, r, "partial"), (w / 2, h - 3.0, r, "partial")]
    marks.windows += [(w / 2, h / 2, float(max(w, h)), "whole"), (0.0, 0.0, 2.0 * max(w, h), "whole")]
    marks.windows += [(float(rng.uniform(-20, w + 20)), float(rng.uniform(-20, h + 20)), float(rng.uniform(1, 60)), "random")
                      for _ in range(12)]
    n = len(xs)
    keys = np.zeros(n, _kdtype())
    keys["x"], keys["y"] = xs, ys
    keys["octave"] = rng.integers(0, 4, n)
    keys["size"], keys["response"] = 31.0, rng.uniform(0, 1, n).astype(np.float32)
    return keys, marks


def _kdtype():
    from multicol_slam_b200.ctypes_defs import KEYPOINT_DTYPE
    return KEYPOINT_DTYPE


def _descriptors(rng, n, dim, crowd_at=None):
    """random descriptors and masks; the keypoints of each crowded cell share a base descriptor up to a few bits, so that their
    windows hold many candidates within the matching thresholds"""
    d = rng.integers(0, 256, (n, dim), dtype=np.uint8)
    m = rng.integers(0, 256, (n, dim), dtype=np.uint8) | rng.integers(0, 256, (n, dim), dtype=np.uint8)
    for sl in (crowd_at or []):
        base = rng.integers(0, 256, dim, dtype=np.uint8)
        for i in range(sl.start, sl.stop):
            d[i] = flip(rng, base, int(rng.integers(0, dim // 2)))
    return d, m


def flip(rng, d, nbits):
    out = d.copy()
    for b in rng.choice(8 * len(d), nbits, replace=False):
        out[b // 8] ^= 1 << (b % 8)
    return out


class EdgeScene:
    """frame: api.Frame; marks[c]: CamMarks with camera-local indices; first[c]: contiguous index of camera c's first keypoint;
    queries: window queries (every window of every camera under every level form) with random query descriptors qdesc / qmask"""

    def __init__(self, frame, marks, first, queries, names, qdesc, qmask, cams):
        self.frame, self.marks, self.first, self.queries, self.names = frame, marks, first, queries, names
        self.qdesc, self.qmask, self.cams = qdesc, qmask, cams


def lafida_like_cams(sizes):
    from multicol_slam_b200 import synth
    base = synth.lafida_cams()
    return [synth.scaled_cam(base[c % 3], w, h) for c, (w, h) in enumerate(sizes)]


def edge_scene(kind, dim, seed=0):
    """the edge frame `kind` ("exact" / "mixed") with dim-byte descriptors"""
    import multicol_slam_b200.api as api                  # plain array holders only
    from multicol_slam_b200.ctypes_defs import WINDOW_QUERY_DTYPE
    sizes = SIZES[kind]
    rng = np.random.default_rng(1000 * seed + dim + (7 if kind == "mixed" else 0))
    per, marks, first, o = [], [], [], 0
    for c, (w, h) in enumerate(sizes):
        if c == EMPTY_CAM:
            keys, mk = np.zeros(0, _kdtype()), CamMarks()
            mk.windows = [(w / 2, h / 2, float(max(w, h)), "whole"), (100.0, 100.0, 30.0, "random")]
        else:
            keys, mk = _camera(rng, w, h, dim)
        crowd, s = [], N_BACKGROUND
        for m in CROWDED.values():
            if len(keys):
                crowd.append(slice(s, s + m))
            s += m
        d, m = _descriptors(rng, len(keys), dim, crowd)
        per.append((keys, d, m))
        marks.append(mk)
        first.append(o)
        o += len(keys)
    F = api.Frame.from_cameras(per, sizes, SF)
    rows, names = [], []
    for c, mk in enumerate(marks):
        for x, y, r, name in mk.windows:
            for lo, hi in LEVEL_FORMS:
                rows.append((c, x, y, r, lo, hi))
                names.append(name)
    q = np.zeros(len(rows), WINDOW_QUERY_DTYPE)
    for i, (c, x, y, r, lo, hi) in enumerate(rows):
        q[i]["cam"], q[i]["x"], q[i]["y"], q[i]["r"], q[i]["min_level"], q[i]["max_level"] = c, x, y, r, lo, hi
    q["desc_index"] = np.arange(len(rows))
    qd, qm = _descriptors(rng, len(rows), dim)
    for i in range(0, len(rows), 3):                        # a third of the query descriptors near a frame keypoint: small distances
        qd[i] = flip(rng, F.desc[rng.integers(0, len(F.keys))], int(rng.integers(0, dim)))
    return EdgeScene(F, marks, first, q, np.array(names), qd, qm, lafida_like_cams(sizes))


def projection_scene(F, dim, masked, seed, nmp=700):
    """map points for SearchByProjection(F, vpMapPoints, th) on an edge frame: projections near keypoints (a third of them into the
    crowded cells), levels around the keypoint's octave including level 0, descriptors = the keypoint's with flipped bits"""
    import multicol_slam_b200.api as api
    rng = np.random.default_rng(seed)
    nc = len(F.cam_w)
    cand = np.flatnonzero((F.keys["x"] > 0) & (F.keys["y"] > 0) & (F.keys["x"] < F.cam_w[F.key_cam] - 1) &
                          (F.keys["y"] < F.cam_h[F.key_cam] - 1))
    src = rng.choice(cand, nmp)
    desc = np.stack([flip(rng, F.desc[s], int(rng.integers(0, dim * 2))) for s in src])
    dm = F.dmask[src].copy() if masked else None
    in_view = np.zeros((nmp, nc), np.uint8); level = np.zeros((nmp, nc), np.int32)
    px = np.zeros((nmp, nc)); py = np.zeros((nmp, nc)); vc = np.zeros((nmp, nc))
    r = np.arange(nmp)
    c = F.key_cam[src]
    in_view[r, c] = 1
    level[r, c] = np.clip(F.keys["octave"][src] + rng.integers(-1, 2, nmp), 0, 7)
    px[r, c] = F.keys["x"][src] + rng.normal(0, 1.5, nmp)
    py[r, c] = F.keys["y"][src] + rng.normal(0, 1.5, nmp)
    vc[r, c] = np.where(rng.random(nmp) < 0.5, 0.999, 0.95)
    exact = rng.random(nmp) < 0.15                          # projected exactly onto the keypoint
    px[exact, c[exact]] = F.keys["x"][src[exact]]; py[exact, c[exact]] = F.keys["y"][src[exact]]
    # level-0 points whose window border passes exactly through their keypoint: radius 4 * th (view cosine < 0.998, scale 1) is
    # 4 at th = 1 and 12 at th = 3, and kx -+ radius is exact in double, so |kx - px| == r
    oct0 = np.flatnonzero(F.keys["octave"][src] == 0)
    border = oct0[rng.random(len(oct0)) < 0.5]
    cb, sb = c[border], src[border]
    rad = np.where(rng.random(len(border)) < 0.5, 4.0, 12.0)
    sgn = rng.choice([-1.0, 1.0], (2, len(border)))
    level[border, cb] = 0
    vc[border, cb] = 0.95
    px[border, cb] = F.keys["x"][sb].astype(np.float64) + sgn[0] * rad
    py[border, cb] = F.keys["y"][sb].astype(np.float64) + np.where(rng.random(len(border)) < 0.5, sgn[1] * rad, 0.0)
    desc[border] = F.desc[sb]
    also = np.flatnonzero(rng.random(nmp) < 0.2)            # also in view of the camera without keypoints
    in_view[also, EMPTY_CAM] = 1
    px[also, EMPTY_CAM] = rng.uniform(0, 700, len(also)); py[also, EMPTY_CAM] = rng.uniform(0, 470, len(also))
    vc[also, EMPTY_CAM] = 0.95
    bad = (rng.random(nmp) < 0.05).astype(np.uint8)
    return api.MapPoints(bad, in_view, level, px, py, vc, desc, dm)


def second_frame(F, window, seed):
    """F moved for SearchForInitialization / WindowSearch: a third of the keypoints shifted by exactly +-window (in float32), a few by
    window plus one ulp, the rest by a little; descriptors with a few flipped bits"""
    import multicol_slam_b200.api as api
    rng = np.random.default_rng(seed)
    n = len(F.keys)
    keys = F.keys.copy()
    kind = rng.integers(0, 6, n)
    sx = np.where(kind == 0, window, np.where(kind == 1, -window, rng.normal(0, 2, n)))
    sy = np.where(kind == 2, window, np.where(kind == 3, -window, rng.normal(0, 2, n)))
    keys["x"] = (F.keys["x"].astype(np.float64) + sx).astype(np.float32)
    keys["y"] = (F.keys["y"].astype(np.float64) + sy).astype(np.float32)
    out = kind == 4
    keys["x"][out] = np.nextafter((F.keys["x"][out].astype(np.float64) + window).astype(np.float32), np.float32(np.inf))
    dim = F.desc.shape[1]
    desc = np.stack([flip(rng, F.desc[i], int(rng.integers(0, dim))) for i in range(n)])
    return api.Frame(keys, F.key_cam, desc, F.dmask, list(zip(F.cam_w.tolist(), F.cam_h.tolist())), F.scale_factors)


# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rm():
    import ref_tape
    return ref_tape.module("ref_match_api", "window_edges_cpu", TAPE_LIMIT)


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
