"""Fuse's window edge scenes: key frames whose keypoints are built around the windows Fuse's queries open, so that each window
decides at an edge of the walk (see tests/test_fuse_window_edges_cpu.py), and a numpy model of that walk with switchable mistakes.

The cameras are the Lafida ones scaled to 1024x768 (16 px grid cells: winv = hinv = 1/16 exactly) without a mirror mask, so that
projections next to the image border are searched.  Map points are placed on the bearing ray of a chosen pixel; where a case needs
the window's centre exactly (x - r or x + r on a cell border, a keypoint at distance r exactly) the point is moved along the
camera's x or y axis until the projection lands on it.  The window every query opens is then read off the host projection
api._project, and the key frame's keypoints and descriptors are placed around it.  (The device projection calls CUDA's atan, so
its centre can differ from the host's by a few ulps; tests/test_fuse_window_edges_gpu.py reads the device's centres.)

Each key frame of a scene has its own pose and its own map points; the queries of a call are all points of all key frames, so
that a key frame also sees the other key frames' points (incidental windows, decided like any other).  Camera 2 has no keypoints.

mcs_fuse_device reads the mirror masks as one [n_cams][h][w] array and refuses cameras of different sizes, so every image of a
Fuse call has the same size and the same grid steps.
"""
import functools

import numpy as np

from device_frames import flip
from window_edge_scenes import EXACT, SF, f32_boundary, lafida_like_cams

TH = 2.5                                   # Fuse's th
N_KF = 2
W, H = EXACT[0]                            # 1024 x 768
EMPTY_CAM = 2
SHIFTS = [(0.0, 0.0, 0.0), (0.021, -0.013, 0.017)]
# queries per key frame and camera (cameras 0 and 1) of each kind
PLAN = {"radius_x": 3, "radius_y": 3, "exact_x_lo": 2, "exact_x_hi": 2, "exact_y_lo": 2, "exact_y_hi": 2, "tie": 4, "crowded": 2,
        "level0": 2, "leveltop": 2, "levelmid": 3, "th_keep": 2, "th_drop": 2, "nolevel": 2}
EDGES = ("edge_left", "edge_top", "edge_right", "edge_bottom")
N_NOKEYS = 4                               # queries per key frame into the camera without keypoints
LEVEL = {"exact_x_lo": 0, "exact_x_hi": 0, "exact_y_lo": 0, "exact_y_hi": 0, "crowded": 2, "level0": 0, "leveltop": 7,
         "edge_left": 2, "edge_top": 2, "edge_right": 7, "edge_bottom": 7}
# the mistakes the model can make; which of them apply to the first-candidate walk (:1420) and to the best-candidate one
MUTATIONS = ("radius_ge", "radius_f32", "row_major", "slot_ties", "th_lt", "levels_up", "batch32")
FIRST_MUTATIONS = ("radius_ge", "radius_f32", "row_major", "levels_up", "batch32")
BEST_MUTATIONS = ("radius_ge", "radius_f32", "row_major", "slot_ties", "th_lt", "levels_up")


def f32(v):
    return float(np.float32(v))


def cameras():
    return [dict(c, mirror_mask=0) for c in lafida_like_cams(EXACT[:3])]


def thresholds(dim, masks):
    """(TH_LOW_, the largest distance) at a width: cORBmatcher's TH_LOW_"""
    return (dim if masks else 2 * dim), 8 * dim


# ---- placing map points ------------------------------------------------------------------------------------------------------------
def _place(api, prig, cams, c, tu, tv, depth, exact):
    """a world point on the bearing ray of (tu, tv) in camera c of the projection rig; exact "x" / "y": moved along the camera's
    x / y axis until the projection's u / v equals tu / tv exactly"""
    ray = np.array(api.img_to_world(cams[c], tu, tv))
    p = api._mm(prig.MtMc[c], np.append(ray * depth, 1.0))[:3]
    if exact is None:
        return p
    a = 0 if exact == "x" else 1
    axis, target = prig.MtMc[c][:3, a].copy(), (tu, tv)[a]
    proj = lambda q: prig.world_to_cam(c, q)[a]  # noqa: E731
    for _ in range(8):
        e = proj(p) - target
        if e == 0.0:
            return p
        slope = (proj(p + 1e-6 * axis) - proj(p)) / 1e-6
        p = p - (e / slope) * axis
    for i in range(-30, 31):                     # the last ulps: step the point's coordinates
        for j in range(-30, 31):
            q = p.copy()
            q[0] += i * np.spacing(p[0])
            q[2] += j * np.spacing(p[2])
            if proj(q) == target:
                return q
    raise AssertionError(f"no world point projects exactly onto {target}")


def _dist3d(p, ow, float_dist):
    po = p - ow
    d = float(np.sqrt(po[0] * po[0] + po[1] * po[1] + po[2] * po[2]))
    return f32(d) if float_dist else d


def _range_for_level(d, l):
    """(min_d, max_d) whose lower_bound level is l: d / min_d == 1 gives level 0, a ratio just below sf[l] gives l"""
    if l == 0:
        return d, 10.0 * d
    return d / (SF[l] * 0.995), 10.0 * d


# ---- keypoints around a window -----------------------------------------------------------------------------------------------------
def _case_keys(kind, x, y, r, l, first):
    """the keypoints of one case kind around window (x, y, r) on levels {l - 1, l}, in the order they are added (their index
    order within the camera): (kx, ky, octave, distance) with distance an int, ("th", d) = TH_LOW_ + d or "max" = 8 * dim, and
    the position in that list of the keypoint the window must decide for (None: no hit)"""
    x32, y32 = f32(x), f32(y)
    if kind in ("radius_x", "radius_y"):
        out = []
        for sign in (-1, 1):
            ins, outs = f32_boundary(x if kind == "radius_x" else y, r, sign)
            pos = (lambda v: (float(v), y32)) if kind == "radius_x" else (lambda v: (x32, float(v)))
            out += [pos(outs) + (l, 1 if sign < 0 else 2), pos(ins) + (l, 6 if sign < 0 else 5)]
        # outside one first in visiting order: the first-candidate walk takes the near-side inside one, the best one the far side's
        return out, (1 if first else 3)
    if kind.startswith("exact_"):
        # the window's x - r / x + r (or y's) is a multiple of 16 exactly: a keypoint on it, at distance r exactly, in the cell of
        # the range's bound, visited before a second candidate inside
        on = f32(x - r if kind.endswith("_lo") else x + r) if kind.startswith("exact_x") else f32(y - r if kind.endswith("_lo") else y + r)
        a = (on, y32) if kind.startswith("exact_x") else (x32, on)
        return [a + (0, 2), (x32, y32, 0, 4)], 0
    if kind == "tie":
        # the corner of cells (ix, iy + 1) and (ix + 1, iy): Q in (ix + 1, iy) is added first (lower slot), P in (ix, iy + 1) is
        # visited first (column-major).  Equal distances for the best candidate, the later one nearer for the first; R fails the
        # level test (passes on {l, l + 1}).
        ix, iy = int(np.floor((x - 8) / 16 + 0.5)), int(np.floor((y - 8) / 16 + 0.5))
        q = (f32(16 * ix + 9), f32(16 * iy + 7), l, 1 if first else 4)
        p = (f32(16 * ix + 7), f32(16 * iy + 9), l, 6 if first else 4)
        return [q, p, (x32, y32, min(l + 1, 7), 0)], 1
    if kind == "crowded":
        # 36 items of the window's cell fail (30 on the level, 6 outside the radius), item 37 passes, 4 more fail, and a
        # second candidate lies in the next column
        keys = []
        for t in range(36):
            if t % 6 == 5:
                keys.append((f32(x - r - 0.3 - 0.02 * t), f32(y - 0.9 + 0.05 * t), l, 0))
            else:
                keys.append((f32(x - 1.5 + 0.08 * t), f32(y - 1.0 + 0.05 * t), l + 1 if t % 2 else l - 2, 0))
        keys.append((f32(x - 0.7), f32(y + 0.4), l, 3))
        keys += [(f32(x - 1.2 + 0.1 * t), f32(y - 0.5), l + 1, 0) for t in range(4)]
        keys.append((f32(16 * np.floor(x / 16 + 0.5) + 8.6), y32, l, 5))
        return keys, 36
    if kind == "level0":
        return [(f32(x - 1.5), y32, 1, 1), (f32(x - 0.5), y32, 0, 4), (f32(x + 1.0), y32, 2, 2)], 1
    if kind == "leveltop":
        return [(f32(x - 6.0), y32, 5, 1), (f32(x - 4.0), y32, 6, 3), (f32(x - 2.0), y32, 7, 5)], 1
    if kind == "levelmid":
        return [(f32(x + o * r), y32, l + dl, d) for o, dl, d in ((-0.5, -2, 1), (-0.25, -1, 3), (0.0, 0, 5), (0.25, 1, 2))], 1
    if kind == "th_keep":
        # TH_LOW_ is kept (<=), TH_LOW_ + 1 is not; the first-candidate walk ignores the distance: 8 * dim still wins
        return [(f32(x - 0.5), y32, l, "max" if first else ("th", 0)), (f32(x + 0.5), y32, l, "max" if first else ("th", 1))], 0
    if kind == "th_drop":
        return [(f32(x - 0.5), y32, l, "max" if first else ("th", 1))], (0 if first else None)
    if kind == "nolevel":
        # every item fails the level test: the list counts none and the window has no hit
        return [(f32(x - 0.6), y32, l + 1, 1), (f32(x + 0.4), y32, l + 2, 2), (f32(x + 0.9), y32, l - 2, 3)], None
    if kind == "edge_left":       # a keypoint left of the image (column 0) and one inside
        return [(-1.5, y32, l, 2), (f32(x + 0.8), y32, l, 4)], 0
    if kind == "edge_top":
        return [(x32, -1.5, l, 2), (x32, f32(y + 0.8), l, 4)], 0
    if kind == "edge_right":      # 1020 rounds to column 64 and is not in the grid; 1015 is in column 63
        return [(1020.0, y32, l, 0), (1015.0, y32, l, 2), (1014.2, y32, l - 1, 4)], 1
    if kind == "edge_bottom":
        return [(x32, 763.0, l, 0), (x32, 759.0, l, 2), (x32, 758.2, l - 1, 4)], 1
    raise ValueError(kind)


def _targets(kind, ax, ay, rng):
    """(tu, tv, exact axis) of a case around the lattice anchor (ax, ay) (multiples of 64)"""
    if kind == "exact_x_lo":
        return ax + TH, ay + 5.3, "x"
    if kind == "exact_x_hi":
        return ax - TH, ay + 5.3, "x"
    if kind == "exact_y_lo":
        return ax + 5.3, ay + TH, "y"
    if kind == "exact_y_hi":
        return ax + 5.3, ay - TH, "y"
    if kind == "tie":
        return ax + 8.2, ay + 7.9, None
    if kind == "crowded":
        return ax + 5.5, ay + 0.3, None
    return ax + 3.3 + rng.uniform(0, 4), ay + 2.7 + rng.uniform(0, 4), None


@functools.lru_cache(maxsize=None)
def geometry(variant):
    """the variant's poses, map points and keypoint layout (descriptors come with the width, see scene)"""
    import multicol_slam_b200.api as api
    from search_scenes import rig_of
    cams = cameras()
    rigs = [rig_of(api, cams, sh) for sh in SHIFTS[:N_KF]]
    Scw = None
    if variant == 2:
        Scw = api.inv_rigid(rigs[0].M_t).copy()
        Scw[:3, :3] *= 1.3
        Scw[:3, 3] *= 1.3
    prigs = [r if variant != 2 else api._sim3_rig(r, Scw) for r in rigs]
    float_dist = variant != 2
    rng = np.random.default_rng(90 + variant)
    world, min_d, max_d, cam_of, kf_of, kinds, levels = [], [], [], [], [], [], []
    # per key frame and camera: (kx, ky, octave, point, best-candidate distance, first-candidate distance)
    keys = [[[] for _ in cams] for _ in range(N_KF)]
    expect = {}                                          # (k, point) -> the designed hits of both walks (camera-local, -1 none)
    anchors = [(64 * i + 64, 64 * j + 64) for i in range(14) for j in range(10)]
    for k in range(N_KF):
        prig, ow = prigs[k], prigs[k].M_t[:3, 3].copy()
        mine = [a for n, a in enumerate(anchors) if (n + k) % 2 == 0]
        cases = []
        for c in (0, 1):
            order = [kind for kind, m in PLAN.items() for _ in range(m)]
            cases += [(c, kind, _targets(kind, *mine[n], rng)) for n, kind in enumerate(order)]
            yy = 150 + 260 * k + 40 * c
            cases += [(c, "edge_left", (1.2, yy + 3.1, None)), (c, "edge_top", (yy + 5.3, 1.2, None)),
                      (c, "edge_right", (W - 1.4, yy + 7.7, None)), (c, "edge_bottom", (yy + 9.9, H - 1.4, None))]
        cases += [(EMPTY_CAM, "nokeys", _targets("nokeys", *mine[n], rng)) for n in range(N_NOKEYS)]
        for c, kind, (tu, tv, exact) in cases:
            p = _place(api, prig, cams, c, tu, tv, rng.uniform(2.0, 5.0), exact)
            u, v, _ = prig.world_to_cam(c, p)
            if exact == "x":
                assert u == tu
            if exact == "y":
                assert v == tv
            l = LEVEL.get(kind) if kind in LEVEL else int(rng.integers(*{"nolevel": (2, 6), "levelmid": (2, 7)}.get(kind, (1, 7))))
            lo, hi = _range_for_level(_dist3d(p, ow, float_dist), l)
            i = len(world)
            world.append(p); min_d.append(lo); max_d.append(hi); cam_of.append(c); kf_of.append(k); kinds.append(kind); levels.append(l)
            if kind == "nokeys":
                expect[(k, i)] = (-1, -1)
                continue
            r = TH * SF[l]
            kb, hb = _case_keys(kind, u, v, r, l, False)
            kf, hf = _case_keys(kind, u, v, r, l, True)
            assert [a[:3] for a in kb] == [a[:3] for a in kf]
            base = len(keys[k][c])
            # (best-candidate hit, first-candidate hit) as camera-local keypoint indices
            expect[(k, i)] = tuple(-1 if h is None else base + h for h in (hb, hf))
            keys[k][c] += [(kx, ky, o, i, db, dfi) for (kx, ky, o, db), (*_, dfi) in zip(kb, kf)]
    return dict(cams=cams, rigs=rigs, prigs=prigs, Scw=Scw, world=np.array(world), min_d=np.array(min_d), max_d=np.array(max_d),
                cam_of=np.array(cam_of), kf_of=np.array(kf_of), kinds=np.array(kinds), levels=np.array(levels), keys=keys, expect=expect)


# ---- the scene at a width ------------------------------------------------------------------------------------------------------------
def _distance(spec, th_low, dmax):
    if spec == "max":
        return dmax
    if isinstance(spec, tuple):
        return th_low + spec[1]
    return spec


def scene(api, oa, variant, dim=32, masks=False):
    """-> (key frames, per key frame the scene dict of tests/search_scenes.py's helpers: host_fuse, reference_ops, fuse_replay,
    dev_map).  Descriptors: dim bytes, masks all ones (so that the masked distance is the plain one); a keypoint's descriptor is
    its query point's with as many bits flipped as the case asks (TH_LOW_ of this width and masks where it asks for the
    threshold)."""
    from multicol_slam_b200.ctypes_defs import KEYPOINT_DTYPE
    g = geometry(variant)
    th_low, dmax = thresholds(dim, masks)
    rng = np.random.default_rng(1000 * variant + 2 * dim + int(masks))
    n = len(g["world"])
    desc = rng.integers(0, 256, (n, dim), dtype=np.uint8)
    dmask = np.full((n, dim), 255, np.uint8)
    pick = 5 if variant == 1 else 4
    KFs, ss = [], []
    for k in range(N_KF):
        per = []
        for c in range(len(g["cams"])):
            ks = g["keys"][k][c]
            kp = np.zeros(len(ks), KEYPOINT_DTYPE)
            kp["x"] = [a[0] for a in ks]
            kp["y"] = [a[1] for a in ks]
            kp["octave"] = [a[2] for a in ks]
            kp["size"], kp["response"] = 31.0, 1.0
            d = np.stack([flip(rng, desc[a[3]], _distance(a[pick], th_low, dmax)) for a in ks]) if ks else np.zeros((0, dim), np.uint8)
            per.append((kp, d, np.full_like(d, 255)))
        KF = api.Frame.from_cameras(per, EXACT[:3], list(SF))
        rig = g["rigs"][k]
        rays, _, _ = oa.frame_prepare(KF.keys, KF.key_cam, g["cams"])
        sc = dict(rig=rig, M_c=rig.M_c, M_t=rig.M_t, rays=rays, src=(np.arange(n) % len(KF.keys)).astype(np.int64))
        cur = None
        if variant == 0:
            # curKF: a rig pose a few centimetres away whose keypoint i carries point i, its ray the point's bearing from there
            M_t2 = rig.M_t.copy()
            M_t2[:3, 3] += [0.03, -0.01, 0.02]
            cur_rig = api.Rig(g["cams"], rig.M_c, M_t2)
            cr = np.zeros((n, 3))
            for i in range(n):
                pc = api._mm(cur_rig.MtMc_inv[g["cam_of"][i]], np.append(g["world"][i], 1.0))[:3]
                cr[i] = pc / np.linalg.norm(pc)
            cur = dict(rig=cur_rig, M_t=M_t2, rays=cr, key_cam=g["cam_of"].astype(np.int32))
        ss.append(dict(sc=sc, n=n, kf_mp=np.full(len(KF.keys), -1, np.int32), occupied=np.zeros(0, np.int64), bad=np.zeros(n, np.uint8),
                       in_kf=np.zeros(n, bool), points=np.arange(n, dtype=np.int32), world=g["world"], min_d=g["min_d"], max_d=g["max_d"],
                       desc=desc, dmask=dmask, Scw=g["Scw"], cur=cur))
        KFs.append(KF)
    return KFs, ss


def projection_rig(api, s, variant):
    return s["sc"]["rig"] if variant != 2 else api._sim3_rig(s["sc"]["rig"], s["Scw"])


def host_best(api, m, KF, s, variant, _sw=None):
    """FuseCandidates on every query point (none is bad or in the key frame) -> best [n, n_cams] contiguous keypoint or -1"""
    nc = len(KF.cam_w)
    ids = s["points"]
    uv, ok, lvl = api._project(projection_rig(api, s, variant), KF.scale_factors, s["world"], s["min_d"], s["max_d"], ids,
                               np.tile(np.arange(nc), (len(ids), 1)), float_dist=variant != 2)
    return m.FuseCandidates(KF, uv, ok, lvl, TH, s["desc"], s["dmask"], first_wins=(variant == 1), points=ids, _sw=_sw)


# ---- a numpy model of the walk -----------------------------------------------------------------------------------------------------
def windows(api, KF, s, variant):
    """the windows Fuse's queries open, as FuseCandidates builds them: (rows (point, camera), x, y, r, min_level, max_level)"""
    nc = len(KF.cam_w)
    ids = s["points"]
    uv, ok, lvl = api._project(projection_rig(api, s, variant), KF.scale_factors, s["world"], s["min_d"], s["max_d"], ids,
                               np.tile(np.arange(nc), (len(ids), 1)), float_dist=variant != 2)
    i, c = np.nonzero(ok)
    lv = lvl[i, c]
    return np.stack([i, c], 1), uv[i, c, 0], uv[i, c, 1], TH * np.asarray(KF.scale_factors)[lv], lv - 1, lv


def _grid(KF):
    """PosInGrid: cvRound of the position times the inverse cell size; cells outside the 64 x 48 grid are dropped"""
    cells = {}
    for j, (x, y, c) in enumerate(zip(KF.keys["x"].astype(np.float64), KF.keys["y"].astype(np.float64), KF.key_cam)):
        ix, iy = int(np.rint(x * 64.0 / KF.cam_w[c])), int(np.rint(y * 48.0 / KF.cam_h[c]))
        if 0 <= ix < 64 and 0 <= iy < 48:
            cells.setdefault((int(c), ix, iy), []).append(j)
    return cells


def _dist(a, b, ma, mb):
    x = a ^ b
    if ma is None:
        return int(np.unpackbits(x).sum())
    return (int(np.unpackbits(x & ma).sum()) + int(np.unpackbits(x & mb).sum())) >> 1


def walk(KF, win, qdesc, qmask, first, th_low, mut=()):
    """the hit (contiguous keypoint or -1) of every window: the cells of the floor / ceil range column by column, each cell's
    items in keypoint order, the level filter and the inclusive radius test in double; first: the first candidate that passes,
    else the best (distance, visiting position) kept when its distance is <= th_low.  mut: mistakes of MUTATIONS to make."""
    rows, xs, ys, rs, los, his = win
    cells = _grid(KF)
    kx, ky, koct = KF.keys["x"], KF.keys["y"], KF.keys["octave"]
    out = np.full(len(rows), -1, np.int64)
    for t, ((i, c), x, y, r, lo, hi) in enumerate(zip(rows, xs, ys, rs, los, his)):
        x, y, r = float(x), float(y), float(r)
        if "levels_up" in mut:
            lo, hi = hi, hi + 1
        wi, hi_ = 64.0 / KF.cam_w[c], 48.0 / KF.cam_h[c]
        cx0, cx1 = max(0, int(np.floor((x - r) * wi))), min(63, int(np.ceil((x + r) * wi)))
        cy0, cy1 = max(0, int(np.floor((y - r) * hi_))), min(47, int(np.ceil((y + r) * hi_)))
        if "row_major" in mut:
            seq = [(ix, iy) for iy in range(cy0, cy1 + 1) for ix in range(cx0, cx1 + 1)]
        else:
            seq = [(ix, iy) for ix in range(cx0, cx1 + 1) for iy in range(cy0, cy1 + 1)]
        check = not (lo == -1 and hi == -1)
        same = check and lo == hi
        best, pos = None, 0
        for cell in seq:
            items = cells.get((int(c), cell[0], cell[1]), [])
            if first and "batch32" in mut:
                items = items[:32]
            for j in items:
                o = int(koct[j])
                if (check and not same and (o < lo or o > hi)) or (same and o != lo):
                    continue
                if "radius_f32" in mut:
                    dx, dy, rr = abs(np.float32(kx[j]) - np.float32(x)), abs(np.float32(ky[j]) - np.float32(y)), np.float32(r)
                else:
                    dx, dy, rr = abs(float(kx[j]) - x), abs(float(ky[j]) - y), r
                if (dx >= rr or dy >= rr) if "radius_ge" in mut else (dx > rr or dy > rr):
                    continue
                if first:
                    best = (0, 0, j)
                    break
                d = _dist(qdesc[i], KF.desc[j], None if qmask is None else qmask[i], None if qmask is None else KF.dmask[j])
                key = (d, j if "slot_ties" in mut else pos, j)
                pos += 1
                if best is None or key < best:
                    best = key
            if first and best is not None:
                break
        if best is not None and (first or (best[0] < th_low if "th_lt" in mut else best[0] <= th_low)):
            out[t] = best[2]
    return out


def model_best(api, KF, s, variant, th_low, masks, mut=(), win=None):
    """walk() over every window of the scene -> best [n, n_cams] as host_best gives it"""
    win = windows(api, KF, s, variant) if win is None else win
    hits = walk(KF, win, s["desc"], s["dmask"] if masks else None, variant == 1, th_low, mut)
    best = np.full((s["n"], len(KF.cam_w)), -1, np.int32)
    best[win[0][:, 0], win[0][:, 1]] = hits
    return best


def designed(api, KF, s, variant, k):
    """(kind, point, camera, contiguous keypoint the window was built to decide for or -1) of key frame k's own queries"""
    g = geometry(variant)
    first = np.concatenate([[0], np.cumsum([int((KF.key_cam == c).sum()) for c in range(len(KF.cam_w))])])
    out = []
    for (kk, i), want in g["expect"].items():
        if kk == k:
            w = want[1 if variant == 1 else 0]
            c = int(g["cam_of"][i])
            out.append((str(g["kinds"][i]), i, c, -1 if w < 0 else int(first[c] + w)))
    return out
