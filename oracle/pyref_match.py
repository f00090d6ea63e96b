"""pyref_match.py -- second, independent restatement of the matcher half of the path in plain Python (TEST INFRASTRUCTURE).

Written from the reference sources, not from oracle/mcs_oracle.cpp, so that the two restatements check each other
(tests/test_oracle_match_pyref.py), the way oracle/pyref.py does for the extractor:

  grid            cMultiFrame ctor / PosInGrid / GetFeaturesInArea      src/cMultiFrame.cpp:143-184, :272-353
  distances       DescriptorDistance64[Masked]                          src/cORBmatcher.cpp:2438-2474
  search_by_projection        SearchByProjection(F, vpMapPoints, th)     src/cORBmatcher.cpp:67-176
  search_for_initialization   SearchForInitialization                    src/cORBmatcher.cpp:579-726
  search_by_bow_kf            SearchByBoW(KF1, KF2, vpMatches12)         src/cORBmatcher.cpp:885-966
  search_for_triangulation    SearchForTriangulationRaw                  src/cORBmatcher.cpp:968-1156, src/misc.cpp:53-69
  is_in_frustum               cMultiFrame::isInFrustum                   src/cMultiFrame.cpp:218-270,
                              WorldToCamHom_fast src/cam_system_omni.cpp:92-112, isPointInMirrorMask src/cam_model_omni.cpp:163-178
(mbCheckOrientation is compiled out in the reference, include/cORBmatcher.h:40.)"""
import math

import numpy as np

GRID_COLS, GRID_ROWS = 64, 48          # include/cMultiFrame.h:47-48
INT_MAX = 2**31 - 1


def cv_round(v):
    """cvRound(double): round half to even (lrint)"""
    return int(np.rint(np.float64(v)))


def popcount_bytes(a):
    return int(np.unpackbits(np.asarray(a, np.uint8)).sum())


def distance(d1, d2, m1=None, m2=None):
    x = np.bitwise_xor(d1, d2)
    if m1 is None:
        return popcount_bytes(x)                                   # :2438-2450
    return (popcount_bytes(x & m1) + popcount_bytes(x & m2)) // 2   # :2452-2474 (integer division)


class Grid:
    """mGrids[cam][col][row] -> keypoint ids in insertion order, for a frame with mnMin = 0, mnMax = sensor size"""

    def __init__(self, keys, key_cam, cam_sizes):
        self.keys, self.key_cam = keys, key_cam
        self.winv = [float(GRID_COLS) / float(w) for w, h in cam_sizes]
        self.hinv = [float(GRID_ROWS) / float(h) for w, h in cam_sizes]
        self.cells = [[[[] for _ in range(GRID_ROWS)] for _ in range(GRID_COLS)] for _ in cam_sizes]
        for i in range(len(keys)):
            c = int(key_cam[i])
            # kp.pt.x is float, mnMinX int -> float difference, times a double
            px = cv_round(float(np.float32(keys["x"][i]) - np.float32(0)) * self.winv[c])
            py = cv_round(float(np.float32(keys["y"][i]) - np.float32(0)) * self.hinv[c])
            if px < 0 or px >= GRID_COLS or py < 0 or py >= GRID_ROWS:
                continue
            self.cells[c][px][py].append(i)

    def features_in_area(self, cam, x, y, r, min_level=-1, max_level=-1):
        out = []
        x, y, r = float(x), float(y), float(r)
        c0 = max(0, int(math.floor((x - 0 - r) * self.winv[cam])))
        if c0 >= GRID_COLS:
            return out
        c1 = min(GRID_COLS - 1, int(math.ceil((x - 0 + r) * self.winv[cam])))
        if c1 < 0:
            return out
        r0 = max(0, int(math.floor((y - 0 - r) * self.hinv[cam])))
        if r0 >= GRID_ROWS:
            return out
        r1 = min(GRID_ROWS - 1, int(math.ceil((y - 0 + r) * self.hinv[cam])))
        if r1 < 0:
            return out
        check = not (min_level == -1 and max_level == -1)
        same = check and min_level == max_level
        for ix in range(c0, c1 + 1):
            for iy in range(r0, r1 + 1):
                for k in self.cells[cam][ix][iy]:
                    octv = int(self.keys["octave"][k])
                    if check and not same:
                        if octv < min_level or octv > max_level:
                            continue
                    elif same:
                        if octv != min_level:
                            continue
                    if abs(float(self.keys["x"][k]) - x) > r or abs(float(self.keys["y"][k]) - y) > r:
                        continue
                    out.append(k)
        return out

    def features_in_area_kf(self, cam, x, y, r):
        """the cMultiKeyFrame overload (src/cMultiKeyFrame.cpp:694-737): same cell range, no level filter, `<= r` in place of
        `!(> r)`"""
        x, y, r = float(x), float(y), float(r)
        c0 = max(0, int(math.floor((x - 0 - r) * self.winv[cam])))
        c1 = min(GRID_COLS - 1, int(math.ceil((x - 0 + r) * self.winv[cam])))
        r0 = max(0, int(math.floor((y - 0 - r) * self.hinv[cam])))
        r1 = min(GRID_ROWS - 1, int(math.ceil((y - 0 + r) * self.hinv[cam])))
        if c0 >= GRID_COLS or c1 < 0 or r0 >= GRID_ROWS or r1 < 0:
            return []
        return [k for ix in range(c0, c1 + 1) for iy in range(r0, r1 + 1) for k in self.cells[cam][ix][iy]
                if abs(float(self.keys["x"][k]) - x) <= r and abs(float(self.keys["y"][k]) - y) <= r]


def radius_by_viewing_cos(view_cos):
    return 2.5 if view_cos > 0.998 else 4.0


def search_by_projection(F, grid, mps, th, nnratio, th_high, having_masks, frame_mp):
    """F: Frame holder; mps: MapPoints holder ([point, cam] arrays); frame_mp[k] >= 0 <=> keypoint k already has a map point.
    Returns (nmatches, frame_mp) with the matched map point index written in."""
    frame_mp = np.array(frame_mp, np.int64).copy()
    n_cams = len(F.cam_w)
    nmatches = 0
    use_factor = th != 1.0
    for i in range(len(mps.bad)):
        if mps.bad[i]:
            continue
        for cam in range(n_cams):
            if not mps.in_view[i, cam]:
                continue
            level = int(mps.level[i, cam])
            r = radius_by_viewing_cos(float(mps.view_cos[i, cam]))
            if use_factor:
                r *= th
            near = grid.features_in_area(cam, mps.proj_x[i, cam], mps.proj_y[i, cam], r * float(F.scale_factors[level]), level - 1, level)
            if not near:
                continue
            best, best2, lvl, lvl2, besti = INT_MAX, INT_MAX, -1, -1, -1
            for k in near:
                if frame_mp[k] >= 0:
                    continue
                d = distance(mps.desc[i], F.desc[k], mps.dmask[i] if having_masks else None, F.dmask[k] if having_masks else None)
                if d < best:
                    best2, best, lvl2, lvl, besti = best, d, lvl, int(F.keys["octave"][k]), k
                elif d < best2:
                    lvl2, best2 = int(F.keys["octave"][k]), d
            if best <= th_high:
                if lvl == lvl2 and best > nnratio * best2:
                    continue
                frame_mp[besti] = i
                nmatches += 1
    return nmatches, frame_mp


def search_for_initialization(F1, F2, grid2, prev_matched, window, nnratio, th_low, having_masks):
    prev = np.array(prev_matched, np.float64).copy()
    n1, n2 = len(F1.keys), len(F2.keys)
    m12 = np.full(n1, -1, np.int64)
    m21 = np.full(n2, -1, np.int64)
    matched_dist = np.full(n2, INT_MAX, np.int64)
    nmatches = 0
    for i1 in range(n1):
        level1 = int(F1.keys["octave"][i1])
        cam1 = int(F1.key_cam[i1])
        cand = grid2.features_in_area(cam1, prev[i1, 0], prev[i1, 1], window, level1, level1)
        if not cand:
            continue
        best, best2, besti = INT_MAX, INT_MAX, -1
        for i2 in cand:
            d = distance(F1.desc[i1], F2.desc[i2], F1.dmask[i1] if having_masks else None, F2.dmask[i2] if having_masks else None)
            if matched_dist[i2] <= d:
                continue
            if d < best:
                best2, best, besti = best, d, i2
            elif d < best2:
                best2 = d
        if best <= th_low and best < float(best2) * nnratio:
            if m21[besti] >= 0:
                m12[m21[besti]] = -1
                nmatches -= 1
            m12[i1] = besti
            m21[besti] = i1
            matched_dist[besti] = best
            nmatches += 1
    for i1 in range(n1):
        if m12[i1] >= 0:
            prev[i1] = (float(F2.keys["x"][m12[i1]]), float(F2.keys["y"][m12[i1]]))
    return nmatches, m12, prev


def search_by_bow_kf(d1, d2, th_low, nnratio, m1=None, m2=None, valid1=None, valid2=None):
    n1, n2 = len(d1), len(d2)
    m12 = np.full(n1, -1, np.int64)
    matched2 = np.zeros(n2, bool)
    nmatches = 0
    for i1 in range(n1):
        if valid1 is not None and not valid1[i1]:
            continue
        best, best2, besti = INT_MAX, INT_MAX, -1
        for i2 in range(n2):
            if matched2[i2] or (valid2 is not None and not valid2[i2]):
                continue
            d = distance(d1[i1], d2[i2], None if m1 is None else m1[i1], None if m2 is None else m2[i2])
            if d < best:
                best2, best, besti = best, d, i2
            elif d < best2:
                best2 = d
        if best < th_low and float(best) < nnratio * float(best2):
            m12[i1] = besti
            matched2[besti] = True
            nmatches += 1
    return nmatches, m12


def check_dist_epipolar_line(ray1, ray2, E, thresh):
    E = [[float(E[i][j]) for j in range(3)] for i in range(3)]
    r1, r2 = [float(v) for v in ray1], [float(v) for v in ray2]

    def dot3(a, b):                            # cv::Matx products: s = 0; s += a_k * b_k in index order
        s = 0.0
        for k in range(3):
            s += a[k] * b[k]
        return s
    t = [dot3(r2, [E[0][j], E[1][j], E[2][j]]) for j in range(3)]          # ray2^T * E12
    nom = dot3(t, r1)                                                       # (ray2^T * E12) * ray1
    ex1 = [dot3(E[i], r1) for i in range(3)]                                # E12 * ray1
    etx2 = [dot3([E[0][i], E[1][i], E[2][i]], r2) for i in range(3)]        # E12^T * ray2
    den = float(ex1[0] * ex1[0] + ex1[1] * ex1[1] + ex1[2] * ex1[2] + etx2[0] * etx2[0] + etx2[1] * etx2[1] + etx2[2] * etx2[2])
    if den == 0.0:
        return False
    return (nom * nom) / den < thresh


def search_for_triangulation(d1, m1, cam1, free1, rays1, d2, m2, cam2, free2, rays2, E, th_low, epi_thresh=1e-2):
    """free[i]: the keypoint has no map point yet.  E[c1][c2]: essential matrices."""
    n1, n2 = len(d1), len(d2)
    m12 = np.full(n1, -1, np.int64)
    matched2 = np.zeros(n2, bool)
    nmatches = 0
    for i1 in range(n1):
        if not free1[i1]:
            continue
        cand = []
        for i2 in range(n2):
            if matched2[i2] or not free2[i2]:
                continue
            if cam1[i1] != cam2[i2]:
                continue
            d = distance(d1[i1], d2[i2], None if m1 is None else m1[i1], None if m2 is None else m2[i2])
            if d > th_low:
                continue
            cand.append((d, i2))
        if not cand:
            continue
        cand.sort()                              # pair<int, size_t>: by distance, then index
        dist_th = cv_round(2 * cand[0][0])
        for d, i2 in cand:
            if d > dist_th:
                break
            if check_dist_epipolar_line(rays1[i1], rays2[i2], E[int(cam1[i1])][int(cam2[i2])], epi_thresh):
                matched2[i2] = True
                m12[i1] = i2
                nmatches += 1
                break
    return nmatches, m12


def world_to_img(cam, x, y, z):
    """cCamModelGeneral_::WorldToImg, src/cam_model_omni.cpp:146-161"""
    norm = math.sqrt(x * x + y * y)
    if norm == 0.0:
        norm = 1e-14
    theta = math.atan(-z / norm)
    rho = 0.0
    for c in reversed(cam["inv_pol"]):
        rho = rho * theta + c
    uu, vv = x / norm * rho, y / norm * rho
    return uu * cam["c"] + vv * cam["d"] + cam["u0"], uu * cam["e"] + vv + cam["v0"]


def img_to_world(cam, u, v):
    """cCamModelGeneral_::ImgToWorld, src/cam_model_omni.cpp:49-67"""
    inv_aff = cam["c"] - cam["d"] * cam["e"]
    ut, vt = u - cam["u0"], v - cam["v0"]
    x = (ut - cam["d"] * vt) / inv_aff
    y = (-cam["e"] * ut + cam["c"] * vt) / inv_aff
    x2, y2 = x * x, y * y
    rho = math.sqrt(x2 + y2)
    z = 0.0
    for c in reversed(list(cam["pol"])[:5]):
        z = z * rho + c
    z = -z
    n = math.sqrt(x2 + y2 + z * z)
    return x / n, y / n, z / n


def is_in_frustum(mtmc_inv, mtmc, cam, mask, P, normal, min_dist, max_dist, scale_factors):
    """one (map point, camera): returns None or (proj_x, proj_y, level, view_cos)"""
    p4 = np.array([P[0], P[1], P[2], 1.0])
    rot = np.array([sum(mtmc_inv[r][k] * p4[k] for k in range(4)) for r in range(4)])     # cv::Matx product: index order
    u, v = world_to_img(cam, rot[0], rot[1], rot[2])
    if not (math.isfinite(u) and math.isfinite(v)):
        return None
    ur, vr = cv_round(u), cv_round(v)
    if ur >= mask.shape[1] or ur <= 0 or vr >= mask.shape[0] or vr <= 0:
        return None
    if not mask[vr, ur] > 0:
        return None
    po = np.array([P[0] - mtmc[0][3], P[1] - mtmc[1][3], P[2] - mtmc[2][3]])
    dist = math.sqrt(po[0] * po[0] + po[1] * po[1] + po[2] * po[2])
    if dist < min_dist or dist > max_dist:
        return None
    view_cos = (po[0] * normal[0] + po[1] * normal[1] + po[2] * normal[2]) / dist
    ratio = dist / min_dist
    level = int(np.searchsorted(np.asarray(scale_factors, np.float64), ratio, side="left"))      # std::lower_bound
    level = min(level, len(scale_factors) - 1)
    return u, v, level, view_cos


# ---- the other window searches (M4): matching cores, projections supplied by the caller -----------------------------
def window_search(F1, F2, grid2, window, valid1, nnratio, th_high, having_masks, min_level=0, max_level=INT_MAX):
    """WindowSearch(F1, F2, windowSize, vpMapPointMatches2, minScaleLevel, maxScaleLevel)  src/cORBmatcher.cpp:326-474.
    valid1[i1]: keypoint i1 of F1 carries a non-bad map point.  Returns (nmatches, vnMatches21)."""
    m21 = np.full(len(F2.keys), -1, np.int64)
    nmatches = 0
    for i1 in range(len(F1.keys)):
        if not valid1[i1]:
            continue
        level1 = int(F1.keys["octave"][i1])
        if min_level > 0 and level1 < min_level:
            continue
        if max_level < INT_MAX and level1 > max_level:
            continue
        cam1 = int(F1.key_cam[i1])
        # kp1.pt.x (float) is passed as const double&
        cand = grid2.features_in_area(cam1, float(F1.keys["x"][i1]), float(F1.keys["y"][i1]), float(window))
        if not cand:
            continue
        best, best2, besti = INT_MAX, INT_MAX, -1
        for i2 in cand:
            if m21[i2] >= 0:
                continue
            d = distance(F1.desc[i1], F2.desc[i2], F1.dmask[i1] if having_masks else None, F2.dmask[i2] if having_masks else None)
            if d < best:
                best2, best, besti = best, d, i2
            elif d < best2:
                best2 = d
        if best <= best2 * nnratio and best <= th_high:
            m21[besti] = i1
            nmatches += 1
    return nmatches, m21


def search_by_projection_frames(F1, F2, grid2, window, valid1, uv, in_mask, assigned2, nnratio, th_high, having_masks):
    """SearchByProjection(F1, F2, windowSize, vpMapPointMatches2)  src/cORBmatcher.cpp:476-573.  valid1: the caller's map-point
    bookkeeping (:487-497); uv[i1, c], in_mask[i1, c]: projection of the map point into camera c of F2 and its mirror-mask test."""
    a2 = np.array(assigned2, np.int64).copy()
    nmatches = 0
    for i1 in range(len(F1.keys)):
        if not valid1[i1]:
            continue
        level1 = int(F1.keys["octave"][i1])
        for c in range(len(F2.cam_w)):
            if not in_mask[i1, c]:
                continue
            cand = grid2.features_in_area(c, uv[i1, c, 0], uv[i1, c, 1], float(window), level1, level1)
            if not cand:
                continue
            best, best2, besti = INT_MAX, INT_MAX, -1
            for i2 in cand:
                if a2[i2] >= 0:
                    continue
                d = distance(F1.desc[i1], F2.desc[i2], F1.dmask[i1] if having_masks else None, F2.dmask[i2] if having_masks else None)
                if d < best:
                    best2, best, besti = best, d, i2
                elif d < best2:
                    best2 = d
            if float(best) <= float(best2) * nnratio and best <= th_high:
                a2[besti] = i1
                nmatches += 1
    return nmatches, a2


def search_by_projection_last(Cur, grid_cur, Last, th, valid_last, uv, in_mask, assigned_cur, th_high, having_masks):
    """SearchByProjection(CurrentFrame, LastFrame, th)  src/cORBmatcher.cpp:1990-2118 (motion model)."""
    a = np.array(assigned_cur, np.int64).copy()
    nmatches = 0
    for i in range(len(Last.keys)):
        if not valid_last[i] or not in_mask[i]:
            continue
        cam = int(Last.key_cam[i])
        octave = int(Last.keys["octave"][i])
        radius = th * float(Cur.scale_factors[octave])
        cand = grid_cur.features_in_area(cam, uv[i, 0], uv[i, 1], radius, octave - 1, octave + 1)
        if not cand:
            continue
        best, besti = INT_MAX, -1
        for i2 in cand:
            if a[i2] >= 0:
                continue
            d = distance(Last.desc[i], Cur.desc[i2], Last.dmask[i] if having_masks else None, Cur.dmask[i2] if having_masks else None)
            if d < best:
                best, besti = d, i2
        if best <= th_high:
            a[besti] = i
            nmatches += 1
    return nmatches, a


def fuse_candidates(KF, grid, uv, in_mask, level, th, mp_desc, mp_dmask, th_low, having_masks):
    """Matching core of Fuse(pKF, curKF, vpMapPoints, th)  src/cORBmatcher.cpp:1265-1418 (same core in :1420, :1570 and
    SearchBySim3 :1721): per (map point i, camera c) passing the mirror-mask / distance tests (in_mask), the key-frame keypoint
    with the smallest distance inside radius th * scale[level] whose level is level-1 or level; kept if <= TH_LOW_.
    The key-frame flavour of GetFeaturesInArea (src/cMultiKeyFrame.cpp:694-737) has no level argument; the level test is in the loop."""
    best = np.full(in_mask.shape, -1, np.int64)
    for i in range(in_mask.shape[0]):
        for c in range(in_mask.shape[1]):
            if not in_mask[i, c]:
                continue
            lvl = int(level[i, c])
            radius = th * float(KF.scale_factors[lvl])
            bd, bi = INT_MAX, -1
            for k in grid.features_in_area(c, uv[i, c, 0], uv[i, c, 1], radius):
                kl = int(KF.keys["octave"][k])
                if kl < lvl - 1 or kl > lvl:
                    continue
                d = distance(mp_desc[i], KF.desc[k], mp_dmask[i] if having_masks else None, KF.dmask[k] if having_masks else None)
                if d < bd:
                    bd, bi = d, k
            if bi >= 0 and bd <= th_low:
                best[i, c] = bi
    return best
