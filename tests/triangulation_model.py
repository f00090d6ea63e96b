"""A plain-Python model of local mapping's device SearchForTriangulationRaw (mcs_search_for_triangulation_device,
multicol_slam_b200/csrc/match_kernels.cu, DESIGN.md "Local mapping's triangulation search on the device") and a seeded catalogue
of planted scenes that put its walk on each of its decision edges.

The model restates the kernels one for one: lists() is seg_lists_kernel<CamSegs> with topk_merge_kernel, flags() is tr_epi_kernel
and walk() is tr_walk_kernel with its exact rescan (tr_scan).  Its output is what the device writes -- matches12 by slot, nmatches and
diag = [queries, rescans] -- plus a record of the rule that decided each query, which the scene classes assert on.  `mutant`
switches one rule to a plausible wrong one; the tests show that some scene tells each of them from the sequential loop.

A scene is three Lafida-sized cameras.  Descriptor distances are planted by flipping bits of a cluster's base row (in masked
scenes one flipped bit is masked out on the candidate's side, so the masked sum is odd and its halving matters); epipolar pass or
fail is planted by geometry: the neighbour is KF1's rig moved a few centimetres, a passing candidate sits on the query's epipolar
curve (the query ray projected onto the plane E[c][c] * ray1 is normal to, residual about 0) and a failing one on a pixel far off
that curve.  (Only camera 0's pose is the rig's, so E[c][c] of the other cameras does not map a pixel onto itself.)"""
import ctypes as C

import numpy as np

from device_frames import counts
from search_scenes import epipolar_residual, essential, rig_of

K = 8                        # kTopKMax: list length per query
TOPK_THREADS, DB_TILE = 128, 256     # kTopkThreads (query rows per list CTA), kDbTile
SCAN_THREADS = 256 - 32      # tr_scan's scanning threads (warps 1 .. of the walk's CTA)
H100_SMS = 132
SIZES = [(754, 480)] * 3
SF = np.cumprod([1.0] + [1.2000000476837158] * 7)
PIX = [(400.25, 300.75), (301.5, 201.25), (455.75, 250.5)]      # per camera: the queries' pixel
POPC = np.array([bin(i).count("1") for i in range(256)], np.int64)

MUTANTS = ("wd_lt", "dK_lt", "full8_complete", "no_open_none", "best_first_listed", "list_th_low_lt", "rescan_ignores_taken",
           "rescan_smallest_only", "ties_larger_index", "shared_taken")


# ------------------------------------------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------------------------------------------
def distances(dq, mq, dd, md):
    """DescriptorDistance64 / DescriptorDistance64Masked of every (query row, database row): popcount of the xor, or the sum of
    its popcounts under either mask halved once (integer division)"""
    out = np.empty((len(dq), len(dd)), np.int64)
    for i in range(len(dq)):
        x = dq[i][None, :] ^ dd
        if mq is None:
            out[i] = POPC[x].sum(1)
        else:
            out[i] = (POPC[x & mq[i][None, :]].sum(1) + POPC[x & md].sum(1)) // 2
    return out


def segments(F, free):
    """per camera, the contiguous indices of its free rows in order: the device's compact segment (slot order inside a camera)"""
    return [np.flatnonzero((F.key_cam == c) & free) for c in range(len(F.cam_w))]


def lists(dist, th_low, mutant=None):
    """seg_lists_kernel<CamSegs> + topk_merge_kernel for one camera: per query row, the K smallest (distance, segment index) keys
    with distance <= th_low, as (index, distance) lists padded with (-1, INT_MAX)"""
    out = []
    for row in dist:
        ok = row < th_low if mutant == "list_th_low_lt" else row <= th_low
        ids = np.flatnonzero(ok)
        order = sorted(ids.tolist(), key=lambda j: (int(row[j]), -j if mutant == "ties_larger_index" else j))[:K]
        out.append([(j, int(row[j])) for j in order] + [(-1, 2**31 - 1)] * (K - len(order)))
    return out


def epipolar_ok(oa, r1, r2, E, epi):
    """CheckDistEpipolarLine (ref src/misc.cpp:53-69) as the oracle computes it, pinned to the reference by test_ref_pin_cpu"""
    lib = oa.lib()
    lib.mcso_check_epipolar.restype = C.c_int
    a, b, e = (np.ascontiguousarray(v, np.float64) for v in (r1, r2, E))
    return bool(lib.mcso_check_epipolar(a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), e.ctypes.data_as(C.c_void_p),
                                        C.c_double(epi)))


def flags(oa, lst, q_rays, d_rays, E, epi):
    """tr_epi_kernel for one camera: per list entry, 1 when the pair passes the epipolar test, 0 for a failing or empty entry"""
    return [[0 if j < 0 else int(epipolar_ok(oa, q_rays[i], d_rays[j], E, epi)) for j, _ in l] for i, l in enumerate(lst)]


def walk(oa, dist, lst, flg, q_rays, d_rays, E, epi, th_low, taken, mutant=None):
    """tr_walk_kernel for one camera: its queries in segment order against the camera's `taken` set (a set of segment indices,
    updated).  -> (winner segment index or -1 per query, rescans, record per query)"""
    win_of, rescans, rec = [], 0, []
    for t, l in enumerate(lst):
        ids = [j for j, _ in l]
        ds = [d for _, d in l]
        open_ = [j >= 0 and j not in taken for j in ids]
        passing = [o and f == 1 for o, f in zip(open_, flg[t])]
        n_valid = sum(j >= 0 for j in ids)
        best = ds[0] if mutant == "best_first_listed" else (ds[open_.index(True)] if any(open_) else ds[0])
        dK = ds[K - 1]
        info = dict(best=best, dK=dK, n_listed=n_valid, n_cand=int((dist[t] <= th_low).sum()))
        if any(passing):
            wl = passing.index(True)
            wd = ds[wl]
            ok = wd < 2 * best if mutant == "wd_lt" else wd <= 2 * best
            code, win, rule = (1, ids[wl], "list_win") if ok else (0, -1, "list_window_reject")
            info.update(wd=wd, wpos=wl)
        elif n_valid != K or (mutant == "full8_complete" and info["n_cand"] <= K):
            code, win, rule = 0, -1, "list_short_none"
        elif not any(open_):
            code, win, rule = (0, -1, "list_no_open_none") if mutant == "no_open_none" else (2, -1, "rescan_no_open")
        else:
            again = dK < 2 * best if mutant == "dK_lt" else dK <= 2 * best
            code, win, rule = (2, -1, "rescan_no_pass") if again else (0, -1, "list_dK_none")
        if code == 2:
            rescans += 1
            keys = [(int(dist[t][j]), j) for j in range(dist.shape[1])
                    if dist[t][j] <= th_low and (mutant == "rescan_ignores_taken" or j not in taken)]
            keys.sort(key=lambda k: (k[0], -k[1]) if mutant == "ties_larger_index" else k)
            B = keys[0] if keys else None
            if mutant == "rescan_smallest_only":
                W = B if B is not None and epipolar_ok(oa, q_rays[t], d_rays[B[1]], E, epi) else None
            else:
                W = next((k for k in keys if epipolar_ok(oa, q_rays[t], d_rays[k[1]], E, epi)), None)
            ok = W is not None and W[0] <= 2 * B[0]
            win = W[1] if ok else -1
            info.update(rescan_best=None if B is None else B[0], rescan_wd=None if W is None else W[0])
            rule = rule + ("_win" if ok else "_none")
        if win >= 0:
            taken.add(win)
        win_of.append(win)
        rec.append(dict(info, rule=rule, win=win))
    return win_of, rescans, rec


def predict(oa, s, mutant=None):
    """the device call on scene s -> dict(n, m12: contiguous KF2 index per KF1 row or -1, slots: matches12 by KF1 slot (-1 below
    the counts, None beyond), diag = [queries, rescans], record: per camera the per-query records, lists: per camera the lists)"""
    KF1, KF2 = s["KF1"], s["nbs"][0]
    nc = len(KF1.cam_w)
    q_seg, d_seg = segments(KF1, s["mp1"] == -1), segments(KF2, s["mps"][0] == -1)
    masked = s["masked"]
    m12 = np.full(len(KF1.keys), -1, np.int32)
    shared = set()
    diag, record, all_lists = [0, 0], [], []
    for c in range(nc):
        qi, di = q_seg[c], d_seg[c]
        dist = distances(KF1.desc[qi], KF1.dmask[qi] if masked else None, KF2.desc[di], KF2.dmask[di] if masked else None)
        E = s["E"][c, c]
        qr, dr = s["rays1"][qi], s["rays2"][di]
        lst = lists(dist, s["th_low"], mutant)
        flg = flags(oa, lst, qr, dr, E, s["epi"])
        taken = shared if mutant == "shared_taken" else set()
        win, rs, rec = walk(oa, dist, lst, flg, qr, dr, E, s["epi"], s["th_low"], taken, mutant)
        for t, w in enumerate(win):
            if w >= 0:
                m12[qi[t]] = di[w]
        diag[0] += len(qi)
        diag[1] += rs
        record.append(rec)
        all_lists.append(lst)
    return dict(n=int((m12 >= 0).sum()), m12=m12, slots=to_slots(s, m12), diag=diag, record=record, lists=all_lists)


def to_slots(s, m12):
    """a contiguous matches12 as the device writes it: per KF1 slot the KF2 slot, -1 below a camera's count, None beyond"""
    cap, KF1, KF2 = s["cap"], s["KF1"], s["nbs"][0]
    slot = lambda F: np.concatenate([c * cap + np.arange(n) for c, n in enumerate(counts(F))]).astype(np.int64)   # noqa: E731
    s1, s2 = slot(KF1), slot(KF2)
    out = np.full(len(KF1.cam_w) * cap, None, object)
    out[s1] = -1
    hit = m12 >= 0
    out[s1[hit]] = s2[m12[hit]]
    return out


def chunk_of(capacity, n_cams, sms=H100_SMS):
    """launch_search_for_triangulation's database chunk of seg_lists_kernel<CamSegs> (a multiple of kDbTile) and the number of
    chunks: list_plan(sms, ceil(capacity / 128) * n_cams, capacity) in match_kernels.cu, the one plan of the K-best list kernels"""
    qblocks, tiles = -(-capacity // TOPK_THREADS), -(-capacity // DB_TILE)
    cta_q = qblocks * n_cams
    splits = max(1, min(tiles, -(-(4 * sms * 8) // cta_q)))
    chunk = -(-tiles // splits) * DB_TILE
    return chunk, -(-capacity // chunk)


def scan_warp(j):
    """the scanning warp (1 ..) of tr_scan that holds database row j of a rescan"""
    return 1 + (j % SCAN_THREADS) // 32


# ------------------------------------------------------------------------------------------------------------------------------
# planted scenes
# ------------------------------------------------------------------------------------------------------------------------------
class Planter:
    """Builds one scene camera by camera.  Rows are added in walk order (KF1) and segment order (KF2); a KF1 query is a cluster's
    base row at the camera's pixel, a KF2 candidate is the base at a planted distance, at the query's pixel (passes) or at the
    camera's failing pixel (fails)."""

    def __init__(self, api, cams, rng, dim, masked, th_low, pass_pix, fail_pix):
        self.api, self.cams, self.rng, self.dim, self.masked, self.th_low = api, cams, rng, dim, masked, th_low
        self.pass_pix, self.fail_pix = pass_pix, fail_pix
        self.q = [[] for _ in range(3)]          # per camera: (x, y, desc, mask, map-point id)
        self.d = [[] for _ in range(3)]

    def base(self):
        return self.rng.integers(0, 256, self.dim, dtype=np.uint8)

    def at(self, b, dist):
        """(desc, mask) at exactly `dist` from the query b (full mask): in a masked scene dist + 1 bits flipped and one of them
        masked out on this side, (dist + 1 + dist) // 2 == dist"""
        nb = dist + (1 if self.masked else 0)
        bits = self.rng.choice(8 * self.dim, nb, replace=False)
        d, m = b.copy(), np.full(self.dim, 255, np.uint8)
        for x in bits:
            d[x // 8] ^= np.uint8(1 << (x % 8))
        if self.masked:
            m[bits[0] // 8] ^= np.uint8(1 << (bits[0] % 8))
        return d, m

    def query(self, c, b, free=True, pix=None):
        x, y = PIX[c] if pix is None else pix
        self.q[c].append((x, y, b, np.full(self.dim, 255, np.uint8), -1 if free else 10**6))
        return len(self.q[c]) - 1

    def cand(self, c, b, dist, passes=True, free=True, pix=None):
        """a KF2 row at `dist` from b -> its position in the camera's rows"""
        d, m = self.at(b, dist)
        x, y = pix if pix is not None else (self.pass_pix[c] if passes else self.fail_pix[c])
        self.d[c].append((x, y, d, m, -1 if free else 10**6))
        return len(self.d[c]) - 1

    def filler(self, c, n, free=True):
        """n KF2 rows of random descriptors, far beyond th_low from every query"""
        for _ in range(n):
            self.d[c].append((PIX[c][0], PIX[c][1], self.base(), np.full(self.dim, 255, np.uint8), -1 if free else 10**6))

    def frame(self, rows):
        api = self.api
        flat = [(c, r) for c in range(3) for r in rows[c]]
        keys = np.zeros(len(flat), api.KEYPOINT_DTYPE)
        keys["x"] = [r[0] for _, r in flat]
        keys["y"] = [r[1] for _, r in flat]
        cam = np.array([c for c, _ in flat], np.int32)
        desc = np.array([r[2] for _, r in flat], np.uint8).reshape(-1, self.dim)
        mask = np.array([r[3] for _, r in flat], np.uint8).reshape(-1, self.dim)
        mp = np.array([r[4] for _, r in flat], np.int32)
        return api.Frame(keys, cam, desc, mask, SIZES, SF), mp


def f32(x, y):
    """a pixel as the keypoints hold it"""
    return float(np.float32(x)), float(np.float32(y))


def pass_pixels(api, cams, E):
    """per camera, a pixel on the epipolar curve of the camera's query pixel: the query ray made normal to E[c][c] * ray1"""
    out = []
    for c in range(3):
        r1 = np.array(api.img_to_world(cams[c], *PIX[c]))
        n = E[c, c] @ r1
        r2 = r1 - (r1 @ n) / (n @ n) * n
        px = f32(*api.world_to_img(cams[c], *r2))
        res = epipolar_residual(api, r1, np.array(api.img_to_world(cams[c], *px)), E[c, c])
        assert res < 1e-9, (c, res)
        out.append(px)
    return out


def fail_pixels(api, cams, E):
    """per camera, a pixel whose pair with the camera's query pixel has a large residual: far off the query's epipolar curve"""
    out = []
    for c in range(3):
        r1 = np.array(api.img_to_world(cams[c], *PIX[c]))
        best, bp = -1.0, None
        for x in range(60, 700, 40):
            for y in range(40, 450, 40):
                r2 = np.array(api.img_to_world(cams[c], float(x), float(y)))
                v = epipolar_residual(api, r1, r2, E[c, c])
                if v > best:
                    best, bp = v, (float(x), float(y))
        assert best > 0.05, best
        out.append(bp)
    return out


def finish(api, oa, P, cams, rig1, rig2, E, cap_extra=0, epi=1e-2, cap=None, **info):
    KF1, mp1 = P.frame(P.q)
    KF2, mp2 = P.frame(P.d)
    cap = cap if cap is not None else max(counts(KF1) + counts(KF2)) + cap_extra
    return dict(KF1=KF1, mp1=mp1, nbs=[KF2], mps=[mp2], rig1=rig1, rigs=[rig2], E=E, dim=P.dim, masked=P.masked, th_low=P.th_low,
                epi=epi, cap=cap, rays1=oa.frame_prepare(KF1.keys, KF1.key_cam, cams)[0],
                rays2=oa.frame_prepare(KF2.keys, KF2.key_cam, cams)[0], **info)


def th_low_of(dim, masked):
    """cORBmatcher's TH_LOW_ (ref src/cORBmatcher.cpp:52-64)"""
    return dim if masked else 2 * dim


def _geometry(api, cams, seed):
    rng = np.random.default_rng(1000 + seed)
    rig1 = rig_of(api, cams, [0, 0, 0])
    rig2 = rig_of(api, cams, rng.uniform(0.02, 0.05, 3) * rng.choice([-1, 1], 3))
    E = essential(rig1, rig2)
    return rig1, rig2, E


def make(api, oa, cams, spec):
    """spec = (class, dim, masked, variant) -> scene dict (the fields the triangulation tests' helpers read, plus the model's)"""
    cls, dim, masked, var = spec
    seed = hash_spec((cls, dim, masked, ""))             # the variants of a class share their geometry and draws
    rig1, rig2, E = _geometry(api, cams, seed)
    P = Planter(api, cams, np.random.default_rng(seed), dim, masked, th_low_of(dim, masked), pass_pixels(api, cams, E),
                fail_pixels(api, cams, E))
    return BUILD[cls](api, oa, cams, P, rig1, rig2, E, var)


def hash_spec(spec):
    return sum((i + 1) * ord(ch) for i, ch in enumerate(spec_id(spec))) % 100000


def spec_id(spec):
    cls, dim, masked, var = spec
    return f"{cls}-{dim}{'m' if masked else 'u'}-{var}"


def _taker(P, c, x_desc):
    """a KF1 query equal to a KF2 row: it takes that row (distance 0, passing) before the queries that follow it"""
    P.query(c, x_desc)


def _window(api, oa, cams, P, rig1, rig2, E, var):
    """class 1: the winner is the first open passing entry behind a taken entry and a failing one, at wd == 2 * best (accepted)
    or 2 * best + 1 (rejected); in the list (camera 0) and in a rescan (camera 1).  Camera 2 holds the same pair with best taken
    the same pair without the taken entry."""
    extra = 0 if var == "eq" else 1
    for c in (0, 2):
        b = P.base()
        x = P.cand(c, b, 2) if c == 0 else None                       # taken by the taker below
        P.cand(c, b, 3, passes=False)                                 # best = 3, fails
        P.cand(c, b, 6 + extra)                                       # wd = 6 (+1)
        P.cand(c, b, 2 * 6 + 2, passes=True)                          # beyond any window
        if x is not None:
            _taker(P, c, P.d[c][x][2])
        P.query(c, b)
    # camera 1: a full list of a taken entry and 7 failing ones, dK = best = 3; the winner is not listed
    b = P.base()
    x = P.cand(1, b, 2)
    for _ in range(7):
        P.cand(1, b, 3, passes=False)
    P.cand(1, b, 5)                                                   # a taken row beyond the list: the rescan must skip it
    y = len(P.d[1]) - 1
    P.cand(1, b, 6 + extra)
    P.filler(1, 20)
    _taker(P, 1, P.d[1][x][2])
    _taker(P, 1, P.d[1][y][2])
    P.query(1, b)
    return finish(api, oa, P, cams, rig1, rig2, E, cap_extra=3, cls="window", var=var)


def _length(api, oa, cams, P, rig1, rig2, E, var):
    """class 2: 7, 8 and 9 candidates.  var 7: none passes, the short list decides "no match".  var 8: none passes; camera 0
    dK == 2 * best (rescan, none), camera 1 dK > 2 * best (no rescan), camera 2 dK < 2 * best (rescan, none).  var 9: the ninth
    candidate ties with dK at a larger index, is the only one that passes and lies within 2 * best: only a rescan finds it."""
    n = int(var)
    plans = {7: [[3] * 7, [3, 4, 4, 5, 5, 6, 6], [2] * 7],
             8: [[3, 3, 4, 4, 5, 5, 6, 6], [2, 2, 3, 3, 4, 4, 5, 5], [4] * 8],
             9: [[3, 3, 4, 4, 5, 5, 6, 6, 6], [3] * 9, [2, 3, 3, 3, 4, 4, 4, 4, 4]]}[n]
    for c in range(3):
        b = P.base()
        P.filler(c, 3)
        for i, d in enumerate(plans[c]):
            P.cand(c, b, d, passes=(n == 9 and i == 8))
        P.filler(c, 2)
        P.query(c, b)
        P.query(c, P.base())                                         # no candidate at all
    return finish(api, oa, P, cams, rig1, rig2, E, cls="length", var=var)


def _chains(api, oa, cams, P, rig1, rig2, E, var):
    """class 3: chains of identical queries against one cluster: from the ninth query on every listed entry is taken and the
    camera is rescanned, until the cluster runs out (rescans with no winner).  Some members fail the epipolar test."""
    n_q = {"a": [12, 9, 14], "b": [16, 10, 11]}[var]
    for c in range(3):
        b = P.base()
        ds = sorted(P.rng.integers(1, 6, n_q[c] - 2 + 2 * c).tolist())
        for i, d in enumerate(ds):
            P.cand(c, b, d, passes=i < K or i % 3 != 0)               # the 8 smallest pass: the first 8 queries take them
            if i % 4 == 0:
                P.filler(c, 1)
        for _ in range(n_q[c]):
            P.query(c, b)
    return finish(api, oa, P, cams, rig1, rig2, E, cls="chains", var=var)


def _th_low(api, oa, cams, P, rig1, rig2, E, var):
    """class 4: candidates at th_low (listed, taken) and th_low + 1 (never listed, never taken), from the list and in a rescan
    whose window 2 * best reaches past th_low"""
    T = P.th_low
    lo = T // 2 + 1                                                  # 2 * lo > T
    for c in range(3):
        b = P.base()                                                 # the only candidate at T: matched from the list
        P.cand(c, b, T)
        P.query(c, b)
        b = P.base()                                                 # the only candidate at T + 1: none
        P.cand(c, b, T + 1)
        P.query(c, b)
        b = P.base()                                                 # 8 failing at lo, unlisted passing at T + 1 (and at T in var "in")
        for _ in range(8):
            P.cand(c, b, lo, passes=False)
        P.cand(c, b, T + 1)
        if var == "in":
            P.cand(c, b, T)
        P.query(c, b)
    return finish(api, oa, P, cams, rig1, rig2, E, cls="th_low", var=var)


def _ties(api, oa, cams, P, rig1, rig2, E, var):
    """class 5: ten equal-distance passing candidates on both sides of a database chunk boundary of seg_lists_kernel (camera 0), taken
    by a chain of identical queries in index order; camera 1: equal-distance passing candidates that different scanning warps of a
    rescan hold, taken by a chain of rescanning queries in index order"""
    b = P.base()
    P.filler(0, DB_TILE - 5)
    for _ in range(10):                                              # segment rows 251 .. 260
        P.cand(0, b, 4)
    P.filler(0, 20)
    for _ in range(11):
        P.query(0, b)
    b = P.base()
    for _ in range(8):
        P.cand(1, b, 3, passes=False)                                # best = dK = 3, all failing: every query rescans
    pos = [40, 70, 100, 230, 264, 301]                               # warps 2, 3, 4, 1, 2, 3 of the scan
    for p in pos:
        P.filler(1, p - len(P.d[1]))
        P.cand(1, b, 5)
    P.filler(1, 10)
    for _ in range(len(pos) + 1):
        P.query(1, b)
    b = P.base()
    P.cand(2, b, 0)
    P.query(2, b)
    return finish(api, oa, P, cams, rig1, rig2, E, cls="ties", var=var, tie_rows=list(range(DB_TILE - 5, DB_TILE + 5)), warp_rows=pos)


def _epi(api, oa, cams, P, rig1, rig2, E, var):
    """class 6: a pair only a rescan reaches, with epi_thresh = its host residual (rejected) or the next double (accepted)"""
    near = f32(P.pass_pix[0][0] + 1.5, P.pass_pix[0][1] - 0.75)
    b = P.base()
    for _ in range(8):
        P.cand(0, b, 3, passes=False)
    j = P.cand(0, b, 4, pix=near)
    P.query(0, b)
    for c in (1, 2):
        b = P.base()
        P.cand(c, b, 1)
        P.query(c, b)
    r1 = np.array(api.img_to_world(cams[0], *PIX[0]))
    r2 = np.array(api.img_to_world(cams[0], *near))
    res = epipolar_residual(api, r1, r2, E[0, 0])
    assert 1e-8 < res < 1e-3, res
    epi = res if var == "at" else float(np.nextafter(res, np.inf))
    return finish(api, oa, P, cams, rig1, rig2, E, epi=epi, cls="epi", var=var, near_row=j)


def _rescan_query(P, c):
    """a query whose list is 8 failing entries at best = dK = 3 and whose one passing candidate at 5 only a rescan finds"""
    b = P.base()
    for _ in range(8):
        P.cand(c, b, 3, passes=False)
    P.cand(c, b, 5)
    P.query(c, b)


def _blocks(api, oa, cams, P, rig1, rig2, E, var):
    """class 7: per-camera query counts at the walk's 32-query chunks and the lists' 128-row blocks, with rescans at t = 31 and the
    next chunk's t = 0 (queries 31, 32, 63, 64, 127, 128); var "edge": a camera with queries and no free KF2 row, one with no query"""
    n_of = {"a": [31, 32, 33], "b": [65, 127, 128], "edge": [129, 5, 0]}[var]
    for c, n in enumerate(n_of):
        if var == "edge" and c == 1:
            for _ in range(n):
                b = P.base()
                P.cand(c, b, 1, free=False)                          # its only candidate carries a map point
                P.query(c, b)
            continue
        for t in range(n):
            if t in (31, 32, 63, 64, 127, 128):
                _rescan_query(P, c)
            else:
                b = P.base()
                P.cand(c, b, int(P.rng.integers(0, 6)), passes=bool(t % 7))
                if t % 3 == 0:
                    P.query(c, P.base(), free=False)                 # rows carrying a map point are not queries
                P.query(c, b)
    if var == "edge":
        P.filler(2, 7)
    return finish(api, oa, P, cams, rig1, rig2, E, cls="blocks", var=var, n_queries=n_of)


CAPACITY = 65535


def _capacity(api, oa, cams, P, rig1, rig2, E, var):
    """class 8: camera 0 with count == capacity == 65535 free KF2 rows and a few dozen queries.  One query's only candidate is the
    last row (compact index 65534, the last chunk), decided from its list; another's list is 8 failing entries and its passing
    candidate lies in the last stride of tr_scan, found by a rescan."""
    last_stride = CAPACITY - CAPACITY % SCAN_THREADS                 # 65408: rows of the scan's 293rd stride .. 65534
    plan = {}
    b_list, b_scan = P.base(), P.base()
    fails = [100 + 4000 * i for i in range(8)]
    for r in fails:
        plan[r] = (b_scan, 3, False)
    plan[last_stride + 60] = (b_scan, 6, True)
    plan[CAPACITY - 1] = (b_list, 2, True)
    others = []
    spread = P.rng.choice(np.setdiff1d(np.arange(CAPACITY - 1), list(plan)), 24, replace=False)
    for i, r in enumerate(spread):                                   # more queries, each with a candidate spread over the camera
        bo = P.base()
        plan[int(r)] = (bo, int(P.rng.integers(0, 5)), bool(i % 4))
        others.append(bo)
    rows, fill, full = P.d[0], P.rng.integers(0, 256, (CAPACITY, P.dim), dtype=np.uint8), np.full(P.dim, 255, np.uint8)
    for r in range(CAPACITY):
        if r in plan:
            bb, d, ok = plan[r]
            P.cand(0, bb, d, passes=ok)
        else:
            rows.append((PIX[0][0], PIX[0][1], fill[r], full, -1))
    P.query(0, b_list)
    for bo in others[:12]:
        P.query(0, bo)
    P.query(0, b_scan)
    for bo in others[12:]:
        P.query(0, bo)
    for c in (1, 2):
        b = P.base()
        P.cand(c, b, 2)
        P.filler(c, 5)
        P.query(c, b)
    return finish(api, oa, P, cams, rig1, rig2, E, cap=CAPACITY, cls="capacity", var=var, list_row=CAPACITY - 1,
                  scan_row=last_stride + 60)


BUILD = dict(window=_window, length=_length, chains=_chains, th_low=_th_low, ties=_ties, epi=_epi, blocks=_blocks, capacity=_capacity)
VARIANTS = dict(window=["eq", "over"], length=["7", "8", "9"], chains=["a", "b"], th_low=["out", "in"], ties=["x"], epi=["at", "next"],
                blocks=["a", "b", "edge"], capacity=["x"])
WIDE = ("window", "length", "chains", "th_low")          # at 16, 32 and 64 bytes, masked and not; the rest at 32 bytes, masked


def catalogue():
    out = []
    for cls, vs in VARIANTS.items():
        forms = [(d, m) for d in (16, 32, 64) for m in (False, True)] if cls in WIDE else [(32, True)]
        out += [(cls, d, m, v) for d, m in forms for v in vs]
    return out
