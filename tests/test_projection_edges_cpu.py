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
import math

import numpy as np
import pytest

from device_frames import taped_rm
from projection_edge_scenes import MP200, SCENE_NAMES, bits, cv_round, distance, host_projection, oracle_is_in_frustum, scene_crc, scenes
# tests/golden/make_projection_edges_golden.py reads cam_point, scenes, scene_crc and MP200 from this module
from projection_edge_scenes import cam_point  # noqa: F401

rm = taped_rm("projection_edges_cpu", "ref_mcs_api", 1 << 16)


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