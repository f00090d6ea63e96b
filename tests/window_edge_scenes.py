"""The keypoint grid's and window searches' edge scenes (see tests/test_window_edges_cpu.py), shared by the CPU and GPU tests."""
import pathlib
import sys

import numpy as np

from device_frames import flip

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
# level filters of a window: none, one level, {l-1, l} with l = 0 (min_level = -1), {l-1, l} with l = 2
LEVEL_FORMS = [(-1, -1), (1, 1), (-1, 0), (1, 2)]


def f32_boundary(x, r, sign):
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
            ix, ox = f32_boundary(x, r, sign)
            iy, oy = f32_boundary(y, r, sign)
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
