"""The map-point projection's edge scenes (see tests/test_projection_edges_cpu.py), shared by the CPU and GPU tests."""
import functools
import json
import math
import pathlib
import sys
import zlib

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
GOLD = ROOT / "tests" / "golden"
MP200 = GOLD / "projection_edges_mp200.npz"        # tests/golden/make_projection_edges_golden.py
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
    """MtMc = [R t; 0 1] and its rigid inverse (cConverter::invMat), as match_scenes.random_rig"""
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


def oracle_is_in_frustum(oa, sc):
    pos, nrm, dmin, dmax = sc.arrays()
    return oa.project_mappoints(sc.inv, sc.mtmc, sc.cams, sc.masks, pos, nrm, dmin, dmax, sc.sf)


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)
