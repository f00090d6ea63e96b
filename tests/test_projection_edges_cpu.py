"""CPU: the map-point projection (isInFrustum, ref src/cMultiFrame.cpp:218-270) on scenes built to sit on its decisions.

The scenes place world points by a search in host double arithmetic (the pose product in the kernel's order, then
mcs_cam_world_to_img) so that the host projection lands on a decision or on the nearest doubles either side of it:
- image border: u, v on 0.5, 1.5, width - 1.5, width - 0.5 (and the rows); cvRound ties to even, so 0.5 is out and 1.5 is in;
- the mirror-mask circle: the last pixel inside and the first outside along eight directions, and the .5 tie between them;
- distance: dist == minDistance, dist == maxDistance, one ulp either side, minDistance == maxDistance;
- level: ratio == mvScaleFactors[l] for every l (the lower_bound tie), one ulp either side, ratio above the top factor (the
  clamp), in tables of 1, 8 and 16 levels, the extractor's 1.2 table and tables of powers of two (which ratio can hit exactly);
- degenerate points: on the optical axis (norm == 0 -> 1e-14), z == 0, x*x + y*y underflowing, behind the camera, NaN / inf
  coordinates, and, in cameras whose polynomial throws u past the int range, cvRound's out-of-range result.
Cameras: Lafida camera 0 with its mirror mask, the same camera with an all-ones mask (the border decides), the 1920x1080 195 deg
synthetic camera; poses: identity and a random rig.

Each case is shown to be reached on the host values.  Then the C++ oracle (mcso_project_mappoints), oracle/pyref_match.py and a
composition of the reference's own compiled camera functions (WorldToImg, isPointInMirrorMask, replayed from
tests/golden/ref_tape_projection_edges_cpu.* where the reference is absent, see oracle/ref_tape.py) with a transcription of
isInFrustum's remaining lines must agree on every output, bit for bit.  The projections are those of the host libm's atan (the
tape was recorded against glibc 2.39's).  tests/test_projection_edges_gpu.py runs the CUDA kernels on the same scenes.
"""
import functools
import json
import math
import pathlib
import sys
import zlib

import numpy as np
import pytest

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
GOLD = ROOT / "tests" / "golden"
MP200 = GOLD / "projection_edges_mp200.npz"        # tests/golden/make_projection_edges_golden.py
TAPE_LIMIT = 1 << 16
SF12 = np.cumprod([1.0] + [1.2000000476837158] * 7)
SF_TABLES = {"sf12": SF12, "pow2": 2.0 ** np.arange(8), "one": np.array([1.0]), "pow2_16": 2.0 ** np.arange(16)}
INT_WRAP = [2.0 ** 32 + 300.25, -(2.0 ** 32) + 300.25, 2.0 ** 31 + 10.0]     # u where a wrapping (int)lrint would land in the image


def cameras():
    from multicol_slam_b200 import synth
    laf = dict(synth.lafida_cams()[0])
    wide = next(c for c in json.loads((GOLD / "synthetic_cams.json").read_text()) if c["name"] == "wide1920x1080_195")
    wide = {k: v for k, v in wide.items() if k != "name"}
    return {"lafida0": laf, "lafida0_open": dict(laf, mirror_mask=0), "wide1920": wide}


def wrap_cam(target):
    """Lafida camera 0 with a constant rho and e = 0: a point with y = 0, x > 0 projects to u = K c + u0 = target, v = v0"""
    laf = cameras()["lafida0_open"]
    return dict(laf, e=0.0, inv_pol=[(target - laf["u0"]) / laf["c"]] + [0.0] * 11)


def random_pose(seed):
    """MtMc = [R t; 0 1] and its rigid inverse (cConverter::invMat), as tests/test_match_gpu.py::_random_rig"""
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    if np.linalg.det(q) < 0:
        q[:, 0] = -q[:, 0]
    t = rng.normal(0, 0.2, 3)
    m, inv = np.eye(4), np.eye(4)
    m[:3, :3], m[:3, 3] = q, t
    inv[:3, :3], inv[:3, 3] = q.T, -(q.T @ t)
    return m, inv


POSES = {"identity": (np.eye(4), np.eye(4)), "random": random_pose(5)}


def cam_point(inv, P):
    """ptRot = MtMc_inv * (P, 1) in the kernel's order: ((a0 P0 + a1 P1) + a2 P2) + a3, no FMA"""
    with np.errstate(invalid="ignore"):
        return [((inv[k][0] * P[0] + inv[k][1] * P[1]) + inv[k][2] * P[2]) + inv[k][3] * 1.0 for k in range(3)]


def host_uv(cam, inv, P):
    import multicol_slam_b200.api as api
    return api.world_to_img(cam, *(float(x) for x in cam_point(inv, P)))


def distance(mtmc, P):
    o = [P[k] - mtmc[k][3] for k in range(3)]
    return math.sqrt((o[0] * o[0] + o[1] * o[1]) + o[2] * o[2])


def to_world(mtmc, pc):
    return (np.asarray(mtmc) @ np.append(np.asarray(pc, np.float64), 1.0))[:3]


def place(cam, mtmc, inv, tu, tv, axis, depth=2.0, span=40):
    """world points whose host u (axis 0) or v (axis 1) is the largest double below the target, the target itself (None when
    no point of the scan hits it) and the smallest above.  Newton steps along the most sensitive world coordinate, then a scan
    over `span` neighbouring doubles of that coordinate either side."""
    import multicol_slam_b200.api as api
    t = (tu, tv)[axis]
    P = to_world(mtmc, np.array(api.img_to_world(cam, tu, tv)) * depth)

    def f(Q):
        return host_uv(cam, inv, Q)[axis]
    g = []
    for k in range(3):
        e = np.zeros(3); e[k] = 1e-7
        g.append((f(P + e) - f(P - e)) / 2e-7)
    k = int(np.argmax(np.abs(g)))
    for _ in range(8):
        P[k] += (t - f(P)) / g[k]
    below, equal, above = None, None, None
    x0 = P[k]
    for direction in (-np.inf, np.inf):
        Q = P.copy()
        x = x0
        for _ in range(span):
            Q[k] = x
            y = f(Q)
            if y < t and (below is None or y > below[0]):
                below = (y, Q.copy())
            elif y > t and (above is None or y < above[0]):
                above = (y, Q.copy())
            elif y == t:
                equal = (y, Q.copy())
            x = np.nextafter(x, direction)
    return [None if b is None else b[1] for b in (below, equal, above)]


class Scene:
    """one call of isInFrustum over every point and camera: cams, masks [nc,h,w] (one size), poses mtmc / inv [nc,4,4], pos, nrm,
    dmin, dmax, sf, and per point a label (what it is for) and the camera it was built for"""

    def __init__(self, name, cams, mtmc, inv, sf):
        import multicol_slam_b200.api as api
        self.name, self.cams, self.sf = name, cams, np.asarray(sf, np.float64)
        self.mtmc, self.inv = np.stack(mtmc), np.stack(inv)
        self.masks = np.stack([api.mirror_mask(c) for c in cams])
        self.rows = []               # (position, normal, dmin, dmax, label, camera)

    def add(self, P, label, cam=0, dmin=1.0, dmax=1e3, nrm=None):
        n = np.asarray(nrm if nrm is not None else [0.0, 0.0, 1.0], np.float64)
        self.rows.append((np.asarray(P, np.float64), n, float(dmin), float(dmax), label, cam))

    def arrays(self):
        pos = np.stack([r[0] for r in self.rows]); nrm = np.stack([r[1] for r in self.rows])
        dmin = np.array([r[2] for r in self.rows]); dmax = np.array([r[3] for r in self.rows])
        return pos, nrm, dmin, dmax

    @property
    def labels(self):
        return np.array([r[4] for r in self.rows])

    @property
    def home(self):
        return np.array([r[5] for r in self.rows])


def _mask_edges(mask):
    """(inside pixel, outside pixel, direction) at the mirror-mask circle, along those of eight directions from the mask's
    centroid that meet it inside the image"""
    ys, xs = np.nonzero(mask)
    cy, cx = ys.mean(), xs.mean()
    out = []
    for a in np.arange(8) * np.pi / 4:
        last, r = None, 0.0
        while True:
            ur, vr = int(round(cx + r * np.cos(a))), int(round(cy + r * np.sin(a)))
            if not (0 <= ur < mask.shape[1] and 0 <= vr < mask.shape[0]):
                break                                     # the circle leaves the image: the border decides there
            if mask[vr, ur] == 0:
                out.append((last, (ur, vr), a))
                break
            last = (ur, vr)
            r += 0.25
    return out


def _add_border(sc, c, cam, mtmc, inv):
    w, h = cam["width"], cam["height"]
    for axis, n, other in ((0, w, h * 0.5 + 0.25), (1, h, w * 0.5 + 0.25)):
        for t in (0.5, 1.5, n - 1.5, n - 0.5):
            tu, tv = (t, other) if axis == 0 else (other, t)
            for P, side in zip(place(cam, mtmc, inv, tu, tv, axis), ("below", "equal", "above")):
                if P is not None:
                    sc.add(P, f"border{'uv'[axis]}:{t}:{side}", c)


def _add_mask(sc, c, cam, mtmc, inv):
    import multicol_slam_b200.api as api
    for inside, outside, a in _mask_edges(sc.masks[c]):
        for px, tag in ((inside, "in"), (outside, "out")):
            sc.add(to_world(mtmc, np.array(api.img_to_world(cam, float(px[0]), float(px[1]))) * 2.0), f"mask:{tag}", c)
        if (inside[0] == outside[0]) != (inside[1] == outside[1]):     # side by side: the .5 tie between the two pixels
            axis = 0 if inside[1] == outside[1] else 1
            tie = 0.5 * (inside[axis] + outside[axis])
            tu, tv = (tie, float(inside[1])) if axis == 0 else (float(inside[0]), tie)
            for P, side in zip(place(cam, mtmc, inv, tu, tv, axis), ("below", "equal", "above")):
                if P is not None:
                    sc.add(P, f"masktie:{'uv'[axis]}:{tie}:{side}", c)


def _base_point(cam, mtmc, depth):
    import multicol_slam_b200.api as api
    return to_world(mtmc, np.array(api.img_to_world(cam, cam["width"] * 0.43, cam["height"] * 0.56)) * depth)


def _add_distance(sc, c, cam, mtmc):
    P = _base_point(cam, mtmc, 3.0)
    d = distance(mtmc, P)
    up, down = np.nextafter(d, np.inf), np.nextafter(d, -np.inf)
    for dmin, tag in ((d, "dmin=dist"), (up, "dmin=dist+ulp"), (down, "dmin=dist-ulp")):
        sc.add(P, f"dist:{tag}", c, dmin=dmin, dmax=4 * d)
    for dmax, tag in ((d, "dmax=dist"), (down, "dmax=dist-ulp"), (up, "dmax=dist+ulp")):
        sc.add(P, f"dist:{tag}", c, dmin=d / 3, dmax=dmax)
    sc.add(P, "dist:dmin=dmax=dist", c, dmin=d, dmax=d)
    sc.add(P, "dist:dmin=dmax=dist+ulp", c, dmin=up, dmax=up)


def _add_levels(sc, c, cam, mtmc):
    """per level l: a minDistance with ratio == sf[l] exactly, and ones with ratio one ulp below and above"""
    for l, s in enumerate(sc.sf):
        want = {"eq": s, "below": np.nextafter(s, -np.inf), "above": np.nextafter(s, np.inf)}
        if l == 0:
            del want["below"]                                     # ratio < 1 means dist < minDistance
        for depth in np.linspace(3.0, 3.5, 40):
            P = _base_point(cam, mtmc, depth)
            d = distance(mtmc, P)
            found = {}
            for tag, r in want.items():
                x = d / r
                for _ in range(8):
                    x = np.nextafter(x, -np.inf)
                for _ in range(17):
                    if d / x == r:
                        found[tag] = x
                        break
                    x = np.nextafter(x, np.inf)
            if len(found) == len(want):
                for tag, dmin in found.items():
                    sc.add(P, f"level:{l}:{tag}", c, dmin=dmin, dmax=d * 2.0 ** 20)
                break
    P = _base_point(cam, mtmc, 3.0)
    d = distance(mtmc, P)
    sc.add(P, "level:clamp", c, dmin=d / (sc.sf[-1] * 1.5), dmax=2 * d)
    sc.add(P, "level:clamp", c, dmin=d * 1e-9, dmax=2 * d)


def _add_degenerate(sc, c, cam, mtmc):
    import multicol_slam_b200.api as api
    vis = np.array(api.img_to_world(cam, cam["width"] * 0.61, cam["height"] * 0.38)) * 2.5
    pcs = {"axis": [(0.0, 0.0, 2.0), (0.0, 0.0, -2.0), (0.0, -0.0, 1.0)], "z0": [(1.5, -0.7, 0.0), (-0.3, 0.9, -0.0)],
           "underflow": [(1e-170, 0.0, 1.0), (0.0, -1e-200, -1.0)], "behind": [-vis, -0.5 * vis, (vis[0], vis[1], -vis[2])]}
    for label, pts in pcs.items():
        for pc in pts:
            sc.add(to_world(mtmc, pc), f"degenerate:{label}", c)
    for bad in (np.nan, np.inf, -np.inf):
        for k in range(3):
            P = to_world(mtmc, vis)
            P[k] = bad
            sc.add(P, f"degenerate:nonfinite", c)


SCENE_NAMES = [f"{c}/{p}" for c in ("lafida0", "lafida0_open", "wide1920", "levels_pow2", "levels_one", "levels_pow2_16")
               for p in POSES] + ["int_wrap/identity"]


@functools.lru_cache(maxsize=None)
def scenes():
    """name -> Scene, deterministic"""
    cams = cameras()
    out = {}
    rng = np.random.default_rng(77)
    for cname, cam in cams.items():
        for pname, (mtmc, inv) in POSES.items():
            sc = Scene(f"{cname}/{pname}", [cam], [mtmc], [inv], SF12)
            _add_border(sc, 0, cam, mtmc, inv)
            if cam.get("mirror_mask", 1) == 1:
                _add_mask(sc, 0, cam, mtmc, inv)
            _add_distance(sc, 0, cam, mtmc)
            _add_levels(sc, 0, cam, mtmc)
            _add_degenerate(sc, 0, cam, mtmc)
            out[sc.name] = sc
    for sname in ("pow2", "one", "pow2_16"):
        for pname, (mtmc, inv) in POSES.items():
            sc = Scene(f"levels_{sname}/{pname}", [cams["lafida0_open"]], [mtmc], [inv], SF_TABLES[sname])
            _add_levels(sc, 0, cams["lafida0_open"], mtmc)
            out[sc.name] = sc
    # three cameras whose polynomials throw u past the int range, in one call (camera indexing of the pose / mask arrays)
    wc = [wrap_cam(t) for t in INT_WRAP]
    sc = Scene("int_wrap/identity", wc, [np.eye(4)] * 3, [np.eye(4)] * 3, SF12)
    for c in range(3):
        for x in (1.0, 2.5):
            sc.add((x, 0.0, 0.3), "wrap", c)
    out[sc.name] = sc
    for sc in out.values():            # normals: random unit vectors (only view_cos reads them)
        n = rng.normal(size=(len(sc.rows), 3))
        n /= np.linalg.norm(n, axis=1)[:, None]
        sc.rows = [(r[0], n[i], *r[2:]) for i, r in enumerate(sc.rows)]
    return out


def scene_crc(sc):
    """CRC-32 of a scene's inputs, stored with the 200-bit projections to catch a builder that drifted"""
    pos, nrm, dmin, dmax = sc.arrays()
    return zlib.crc32(b"".join(np.ascontiguousarray(a).tobytes() for a in (pos, sc.inv, sc.sf, dmin, dmax)))


def host_projection(sc):
    """per (point, camera): host (u, v) in the kernel's operation order -> [n, nc, 2]"""
    pos = sc.arrays()[0]
    return np.array([[host_uv(sc.cams[c], sc.inv[c], P) for c in range(len(sc.cams))] for P in pos])


def cv_round(x):
    """cvRound(double) of OpenCV on x86-64 (cvtsd2si): round half to even; NaN and results outside int give INT_MIN"""
    if not math.isfinite(x):
        return -2 ** 31
    r = int(np.rint(x))
    return r if -2 ** 31 <= r < 2 ** 31 else -2 ** 31


# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rm():
    import ref_tape
    return ref_tape.module("ref_mcs_api", "projection_edges_cpu", TAPE_LIMIT)


def reference_is_in_frustum(rm, sc):
    """isInFrustum over the scene with the reference's own WorldToImg and isPointInMirrorMask; the lines between them
    transcribed: PO = P - (Tcw(0,3), Tcw(1,3), Tcw(2,3)); dist = cv::norm(PO) (s = 0, s += x*x in index order, sqrt);
    viewCos = PO.dot(Pn) / dist; ratio = dist / minDistance; lower_bound over the std::vector<double>, clamped to n - 1"""
    import bisect
    pos, nrm, dmin, dmax = sc.arrays()
    n, nc = len(pos), len(sc.cams)
    in_view, level = np.zeros((n, nc), np.uint8), np.zeros((n, nc), np.int32)
    px, py, vc = np.zeros((n, nc)), np.zeros((n, nc)), np.zeros((n, nc))
    sf = [float(s) for s in sc.sf]
    for c in range(nc):
        rot = []
        for P in pos:
            r = []
            for k in range(3):                        # cv::Matx<double,4,4> * Vec4d: s = 0; s += a(k,j) b(j)
                s = 0.0
                for j, b in enumerate((P[0], P[1], P[2], 1.0)):
                    s += float(sc.inv[c][k][j]) * float(b)
                r.append(s)
            rot.append(r)
        uv = np.asarray(rm.world_to_img_many(sc.cams[c], np.array(rot)))
        inm = rm.points_in_mask(sc.cams[c], uv)
        T = sc.mtmc[c]
        for i, P in enumerate(pos):
            if not inm[i]:
                continue
            PO = [float(P[k]) - float(T[k][3]) for k in range(3)]
            s = 0.0
            for x in PO:
                s += x * x
            dist = math.sqrt(s)
            if dist < dmin[i] or dist > dmax[i]:
                continue
            dot = 0.0
            for k in range(3):
                dot += PO[k] * float(nrm[i][k])
            lv = bisect.bisect_left(sf, dist / dmin[i])
            lv = min(lv, len(sf) - 1)
            in_view[i, c], px[i, c], py[i, c], level[i, c], vc[i, c] = 1, uv[i, 0], uv[i, 1], lv, dot / dist
    return in_view, level, px, py, vc


def pyref_is_in_frustum(sc):
    import pyref_match as pm
    pos, nrm, dmin, dmax = sc.arrays()
    n, nc = len(pos), len(sc.cams)
    out = [np.zeros((n, nc), np.uint8), np.zeros((n, nc), np.int32), np.zeros((n, nc)), np.zeros((n, nc)), np.zeros((n, nc))]
    for c in range(nc):
        for i in range(n):
            r = pm.is_in_frustum(sc.inv[c], sc.mtmc[c], sc.cams[c], sc.masks[c], pos[i], nrm[i], dmin[i], dmax[i], sc.sf)
            if r is not None:
                out[0][i, c], out[2][i, c], out[3][i, c], out[1][i, c], out[4][i, c] = 1, r[0], r[1], r[2], r[3]
    return tuple(out)


def oracle_is_in_frustum(oa, sc):
    pos, nrm, dmin, dmax = sc.arrays()
    return oa.project_mappoints(sc.inv, sc.mtmc, sc.cams, sc.masks, pos, nrm, dmin, dmax, sc.sf)


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def assert_same(a, b, what):
    names = ("in_view", "level", "proj_x", "proj_y", "view_cos")
    for k in range(5):
        x, y = np.asarray(a[k]), np.asarray(b[k])
        ok = np.array_equal(bits(x), bits(y)) if x.dtype == np.float64 else np.array_equal(x, y)
        bad = np.argwhere(bits(x) != bits(y)) if x.dtype == np.float64 else np.argwhere(x != y)
        assert ok, f"{what}: {names[k]} differs at {bad[:5].tolist()}"


# ---------------------------------------------------------------------------------------------------------------------------------
def test_scenes_reach_every_case(api):
    """what each point is for, read off the host values"""
    sc_all = scenes()
    n_equal = 0
    for sc in sc_all.values():
        uv = host_projection(sc)
        pos, _, dmin, dmax = sc.arrays()
        lab, home = sc.labels, sc.home
        for i, L in enumerate(lab):
            c = home[i]
            u, v = uv[i, c]
            kind = L.split(":")
            if kind[0] in ("borderu", "borderv", "masktie"):
                t = float(kind[-2]) if kind[0] != "masktie" else float(kind[2])
                x = u if (kind[0] == "borderu" or (kind[0] == "masktie" and kind[1] == "u")) else v
                side = kind[-1]
                assert (x < t) if side == "below" else ((x > t) if side == "above" else x == t), (sc.name, L, x)
                if side == "below":
                    assert np.nextafter(x, np.inf) >= t or abs(x - t) < 1e-12, (sc.name, L, x)
                n_equal += side == "equal"
            if kind[0] == "mask":
                ur, vr = cv_round(u), cv_round(v)
                assert (sc.masks[c][vr, ur] > 0) == (kind[1] == "in"), (sc.name, L)
            if kind[0] == "dist":
                d = distance(sc.mtmc[c], pos[i])
                want = {"dmin=dist": d == dmin[i], "dmin=dist+ulp": dmin[i] == np.nextafter(d, np.inf),
                        "dmin=dist-ulp": dmin[i] == np.nextafter(d, -np.inf), "dmax=dist": d == dmax[i],
                        "dmax=dist-ulp": dmax[i] == np.nextafter(d, -np.inf), "dmax=dist+ulp": dmax[i] == np.nextafter(d, np.inf),
                        "dmin=dmax=dist": d == dmin[i] == dmax[i], "dmin=dmax=dist+ulp": dmin[i] == dmax[i] == np.nextafter(d, np.inf)}
                assert want[kind[1]], (sc.name, L)
            if kind[0] == "level" and kind[1] != "clamp":
                ratio = distance(sc.mtmc[c], pos[i]) / dmin[i]
                s = sc.sf[int(kind[1])]
                want = {"eq": s, "below": np.nextafter(s, -np.inf), "above": np.nextafter(s, np.inf)}[kind[2]]
                assert ratio == want, (sc.name, L)
            if kind[0] == "level" and kind[1] == "clamp":
                assert distance(sc.mtmc[c], pos[i]) / dmin[i] > sc.sf[-1]
            if L == "degenerate:nonfinite":
                assert not (math.isfinite(u) and math.isfinite(v))
            if L == "wrap":
                assert abs(u) >= 2 ** 31 and abs(u) < 2 ** 33 and 0 < v < sc.cams[c]["height"]
        labels = set(lab.tolist())
        # every level of every table has its tie, and its neighbours
        for l in range(len(sc.sf)):
            if sc.name.startswith("int_wrap"):
                break
            assert {f"level:{l}:eq", f"level:{l}:above"} <= labels, (sc.name, l)
        if not sc.name.startswith(("levels_", "int_wrap")):
            for t in ("0.5", "1.5"):
                assert {f"borderu:{t}:below", f"borderu:{t}:above", f"borderv:{t}:below", f"borderv:{t}:above"} <= labels, sc.name
            if sc.name.startswith("lafida0/"):
                assert (lab == "mask:in").sum() >= 4 and (lab == "mask:out").sum() >= 4 and sum(L.startswith("masktie") for L in labels) >= 12
    assert n_equal >= 16                     # the host u / v lands exactly on a border or .5 tie target
    # the open camera decides the border: 1.5 in (rounds to 2), 0.5 out (rounds to 0, ties to even)
    sc = sc_all["lafida0_open/identity"]
    uv = host_projection(sc)
    lab = sc.labels
    for L, want in (("borderu:0.5:equal", 0), ("borderu:1.5:equal", 2), ("borderv:0.5:equal", 0), ("borderv:1.5:equal", 2)):
        for i in np.flatnonzero(lab == L):
            assert cv_round(uv[i, 0, int("borderv" in L)]) == want


@pytest.mark.parametrize("name", SCENE_NAMES)
def test_oracle_pyref_and_reference_agree(api, oa, rm, name):
    """mcso_project_mappoints == pyref_match.is_in_frustum == the reference's WorldToImg + isPointInMirrorMask + isInFrustum's
    arithmetic, every output bit for bit"""
    sc = scenes()[name]
    o = oracle_is_in_frustum(oa, sc)
    p = pyref_is_in_frustum(sc)
    r = reference_is_in_frustum(rm, sc)
    assert_same(o, p, f"{name}: oracle vs pyref_match")
    assert_same(o, r, f"{name}: oracle vs reference")
    for c, cam in enumerate(sc.cams):
        from ref_tape import same
        assert same(rm.mirror_mask(cam), sc.masks[c])
    # the host projection is the oracle's wherever a point is in view
    uv = host_projection(sc)
    iv = o[0].astype(bool)
    assert np.array_equal(bits(uv[..., 0][iv]), bits(o[2][iv])) and np.array_equal(bits(uv[..., 1][iv]), bits(o[3][iv]))
    assert o[0].any() != name.startswith("int_wrap")      # the int-wrap points are never in view


def test_decisions_at_the_edges(api, oa):
    """the outcomes the edges must have, stated directly"""
    for name, sc in scenes().items():
        iv, lv = oracle_is_in_frustum(oa, sc)[:2]
        lab, home = sc.labels, sc.home
        for i, L in enumerate(lab):
            c = home[i]
            k = L.split(":")
            if k[0] == "dist":
                want = k[1] in ("dmin=dist", "dmin=dist-ulp", "dmax=dist", "dmax=dist+ulp", "dmin=dmax=dist")
                assert iv[i, c] == want, (name, L)
            if k[0] == "level" and iv[i, c]:
                n = len(sc.sf)
                want = n - 1 if k[1] == "clamp" else min(int(k[1]) + (k[2] == "above"), n - 1)
                assert lv[i, c] == want, (name, L)
            if k[0] == "level":
                assert iv[i, c], (name, L)
            if L in ("degenerate:nonfinite", "wrap"):
                assert not iv[i].any(), (name, L)
            if (k[0] == "borderu" or k[0] == "borderv") and name.startswith("lafida0_open"):
                t, n = float(k[1]), sc.cams[c]["width" if k[0] == "borderu" else "height"]
                r = {"below": t - 0.5, "above": t + 0.5, "equal": t - 0.5 if (t - 0.5) % 2 == 0 else t + 0.5}[k[2]]
                assert iv[i, c] == (1 <= r <= n - 1), (name, L)        # u 0.5 -> 0 out, 1.5 -> 2 in, w - 0.5 -> w out


def test_mp200_golden_matches_the_scenes():
    """the committed 200-bit projections were computed from these scenes' inputs"""
    g = np.load(MP200)
    for name, sc in scenes().items():
        key = name.replace("/", "__")
        assert int(g[f"{key}__crc"]) == scene_crc(sc), name
        assert g[f"{key}__uv"].shape == (len(sc.rows), len(sc.cams), 2)