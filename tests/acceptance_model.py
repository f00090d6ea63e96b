"""A plain-Python model of the device searches' ordered acceptance (multicol_slam_b200/csrc/proj_search_kernels.cu, DESIGN.md
section 4) and a seeded generator of dense contention scenes for the five device searches that use it.

The model restates the kernels one for one: lists() is ps_list_kernel, decide() is ps_decide, rounds() is ps_round_kernel run up to
the round cap together with ps_finalize_kernel, walk() is ps_walk_kernel and init_walk() is pi_walk_kernel.  Its input is what the
reference's GetFeaturesInArea visits: per query, the candidates in visiting order with their distances and octaves (oracle
window_search), plus the keypoints taken on entry.  Its output is what the device computes, including the diagnostics (rounds run,
walk start, queries, rescans), so the tests can tell a correct acceptance from one that only ends at the right answer."""
import numpy as np

from device_frames import flip

K = 8                       # kPsK in proj_search_kernels.cu: list length per query
INT_MAX = 2**31 - 1
RULE_RATIO, RULE_BEST, RULE_LEVEL_RATIO = 0, 1, 2          # MCS_RULE_* (include/mcs_b200.h)
RULE_INIT = 100                                             # kRuleInit: SearchForInitialization's acceptance
SIZES = [(754, 480)] * 3
SF = np.cumprod([1.0] + [1.2000000476837158] * 7)
CENTRE = (300.0, 200.0)


# ------------------------------------------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------------------------------------------
class Query:
    """one query: its camera and the window's candidates in visiting order (slot = contiguous keypoint index of the searched
    frame, distance, octave)"""

    def __init__(self, cam, slots, dists, octs):
        self.cam, self.slots, self.dists, self.octs = int(cam), [int(s) for s in slots], [int(d) for d in dists], [int(o) for o in octs]

    def keys(self):
        return sorted((d << 16) | p for p, d in enumerate(self.dists))


def lists(q):
    """ps_list_kernel: the K smallest (distance << 16 | visiting position) keys and the true candidate count"""
    return q.keys()[:K], len(q.dists)


def decide(rule, q, taken, th_high, nnratio):
    """ps_decide -> (accepted slot or -1, best distance or None, rescanned).  taken(slot, distance): the rule's predicate; the
    list decides when it holds as many free keys as the rule reads (1 for MCS_RULE_BEST, else 2) or every candidate, otherwise
    the whole window is scanned again with the predicate."""
    nb = 1 if rule == RULE_BEST else 2
    lk, cnt = lists(q)
    free = [k for k in lk if not taken(q.slots[k & 0xFFFF], k >> 16)]
    rescan = not (len(free) >= nb or cnt <= K)
    if rescan:
        free = [k for k in q.keys() if not taken(q.slots[k & 0xFFFF], k >> 16)][:nb]
    if not free:
        return -1, None, rescan
    d0, p0 = free[0] >> 16, free[0] & 0xFFFF
    s0 = q.slots[p0]
    d1 = free[1] >> 16 if len(free) > 1 else INT_MAX
    if rule == RULE_BEST:
        ok = d0 <= th_high
    elif rule == RULE_RATIO:
        ok = float(d0) <= float(d1) * nnratio and d0 <= th_high
    elif rule == RULE_INIT:
        ok = d0 <= th_high and float(d0) < float(d1) * nnratio
    else:
        l0, l1 = q.octs[p0], (q.octs[free[1] & 0xFFFF] if len(free) > 1 else -1)
        ok = d0 <= th_high and not (l0 == l1 and float(d0) > nnratio * float(d1))
    return (s0 if ok else -1), d0, rescan


def rounds(rule, queries, taken0, cap, th_high, nnratio):
    """ps_round_kernel for r = 0 .. cap - 1, then ps_finalize_kernel.  Round r decides every query at or above `settled` (the
    first query whose decision changed in round r - 1, 0 for r < 2) with a keypoint taken when it was taken on entry or a smaller
    query accepted it in round r - 1; queries below `settled` republish what their buffer holds (round r - 2's decision).  A round
    whose `settled` is "no change" returns at once.  Decisions live in two buffers by round parity, exactly as on the device.
    -> dict(history: per round the decision buffer as that round left it, chg, rounds: rounds run, start: the walk start S (n when
    none), dec: the last round's buffer, rescans)"""
    n = len(queries)
    buf = [[None] * n, [None] * n]
    chg = [None] * cap
    own_prev, ran, rescans, history = {}, 0, 0, []
    for r in range(cap):
        settled = chg[r - 1] if r >= 2 else 0
        if settled is None:
            break
        ran = r + 1
        cur, prev = buf[r & 1], buf[(r + 1) & 1]
        own_cur = {}
        for qi, q in enumerate(queries):
            if qi < settled:
                d = cur[qi]
            else:
                def taken(s, _d, qi=qi):
                    return s in taken0 or (r > 0 and own_prev.get(s, n) < qi)
                d, _, resc = decide(rule, q, taken, th_high, nnratio)
                rescans += resc
                if r >= 1 and d != prev[qi] and chg[r] is None:
                    chg[r] = qi
                cur[qi] = d
            if d >= 0:
                own_cur[d] = min(own_cur.get(d, n), qi)
        own_prev = own_cur
        history.append(list(cur))
    rl = ran - 1
    S = (chg[rl] if rl >= 1 else 0) if n else None
    if S is None or S > n:
        S = n
    return dict(history=history, chg=chg, rounds=ran, start=S, dec=list(buf[rl & 1]) if n else [], rescans=rescans)


def walk(rule, queries, taken0, R, th_high, nnratio, n_cams):
    """ps_finalize_kernel's writes of the settled prefix, then ps_walk_kernel: per camera, the queries from S on in order against
    the camera's taken keypoints.  -> (decision per query, rescans of the walk)"""
    S, out, rescans = R["start"], list(R["dec"][:R["start"]]) + [-1] * (len(queries) - R["start"]), 0
    for c in range(n_cams):
        taken = set(taken0) | {d for q, d in enumerate(out[:S]) if d >= 0 and queries[q].cam == c}
        for qi in range(S, len(queries)):
            if queries[qi].cam != c:
                continue
            d, _, resc = decide(rule, queries[qi], lambda s, _d: s in taken, th_high, nnratio)
            rescans += resc
            out[qi] = d
            if d >= 0:
                taken.add(d)
    return out, rescans


def search(rule, queries, taken0, cap, th_high, nnratio, n_cams):
    """the rounds and the walk -> (decision per query, diag as ps_diag_kernel writes it, the rounds' record)"""
    R = rounds(rule, queries, set(taken0), cap, th_high, nnratio)
    dec, wr = walk(rule, queries, set(taken0), R, th_high, nnratio, n_cams)
    n = len(queries)
    diag = [R["rounds"], R["start"] if R["start"] < n else -1, n, R["rescans"] + wr]
    return dec, diag, R


def init_walk(queries, th_low, nnratio, n_cams):
    """pi_walk_kernel: per camera, the queries in order with MD (the smallest distance any earlier query accepted a keypoint
    at) as the skip predicate (MD[s] <= d); the last accepter of a keypoint owns it.  -> (decision per query, the survivors'
    slot or -1 per query, rescans)"""
    dec, owner, rescans = [-1] * len(queries), {}, 0
    for c in range(n_cams):
        md = {}
        for qi, q in enumerate(queries):
            if q.cam != c:
                continue
            d, d0, resc = decide(RULE_INIT, q, lambda s, dist: md.get(s, 0xFFFF) <= dist, th_low, nnratio)
            rescans += resc
            dec[qi] = d
            if d >= 0:
                md[d] = d0
                owner[d] = qi
    keep = [d if d >= 0 and owner[d] == qi else -1 for qi, d in enumerate(dec)]
    return dec, keep, rescans


def evicted(queries, th_low, nnratio, n_cams):
    """(queries whose acceptance a later query took back, acceptances skipped over an equal MD) of init_walk's run"""
    ties = []
    dec, keep, _ = init_walk(queries, th_low, nnratio, n_cams)
    md = {}
    for qi, q in enumerate(queries):
        ties.append(any(md.get(s) == d for s, d in zip(q.slots, q.dists)))
        if dec[qi] >= 0:
            md[dec[qi]] = q.dists[q.slots.index(dec[qi])]
    return sum(d >= 0 and k < 0 for d, k in zip(dec, keep)), sum(ties)


def oscillating(R):
    """queries whose decision returns to an earlier value after changing, over the rounds the model ran"""
    hist = R["history"]
    n = len(hist[0]) if hist else 0
    count = 0
    for q in range(n):
        seq = [h[q] for h in hist]
        changes = [seq[0]] + [b for a, b in zip(seq, seq[1:]) if a != b]
        count += len(changes) != len(set(changes))
    return count


# ------------------------------------------------------------------------------------------------------------------------------
# model inputs from a search's queries
# ------------------------------------------------------------------------------------------------------------------------------
def model_queries(oa, frame, q, qdesc, qmask):
    """the oracle's GetFeaturesInArea for each window query -> [Query]"""
    if len(q) == 0:
        return []
    mc = 512
    idx, dist, cnt, rc = oa.window_search(frame, q, qdesc, qmask, max_cand=mc)
    assert rc == 0 and cnt.max() <= mc
    oct_ = frame.keys["octave"]
    return [Query(q["cam"][i], idx[i, :cnt[i]], dist[i, :cnt[i]], oct_[idx[i, :cnt[i]]]) for i in range(len(q))]


def local_queries(api, F, mps, th):
    """MapPointQueries: entry point * n_cams + cam when the point is not bad and in view -> (query array, descriptor row per query)"""
    rows = []
    nc = len(F.cam_w)
    for i in range(len(mps.bad)):
        if mps.bad[i]:
            continue
        for c in range(nc):
            if not mps.in_view[i, c]:
                continue
            lvl = int(mps.level[i, c])
            r = 2.5 if mps.view_cos[i, c] > 0.998 else 4.0
            if th != 1.0:
                r *= th
            rows.append((c, mps.proj_x[i, c], mps.proj_y[i, c], r * float(F.scale_factors[lvl]), lvl - 1, lvl, i))
    a = np.array(rows, dtype=object).reshape(-1, 7)
    return api._queries(a[:, 0].astype(np.int32), a[:, 1].astype(np.float64), a[:, 2].astype(np.float64), a[:, 3].astype(np.float64),
                        a[:, 4].astype(np.int32), a[:, 5].astype(np.int32), a[:, 6].astype(np.int32))


class Capture:
    """a stand-in for search_windows that records what a host entry point asks for and answers with the oracle's replay"""

    def __init__(self, oa):
        self.oa, self.calls = oa, []

    def __call__(self, frame, q, qdesc, qmask, tags, rule, nnratio, threshold, assigned):
        self.calls.append(dict(frame=frame, q=np.array(q), qdesc=qdesc, qmask=qmask, tags=np.array(tags), rule=rule, nnratio=nnratio,
                               threshold=threshold, assigned=np.array(assigned)))
        return self.oa.search_windows(frame, q, qdesc, qmask, tags, rule, nnratio, threshold, assigned)


def predict_windows(api, oa, call):
    """the device result of one recorded search_windows call -> (nmatches, assigned, diag, rounds record)"""
    qs = model_queries(oa, call["frame"], call["q"], call["qdesc"], call["qmask"])
    taken0 = set(np.flatnonzero(call["assigned"] >= 0).tolist())
    cap = api.lib().mcs_search_by_projection_max_rounds()
    dec, diag, R = search(call["rule"], qs, taken0, cap, call["threshold"], call["nnratio"], len(call["frame"].cam_w))
    R["queries"] = qs
    out = call["assigned"].copy()
    for qi, d in enumerate(dec):
        if d >= 0:
            out[d] = call["tags"][qi]
    return sum(d >= 0 for d in dec), out, diag, R


def predict_local(api, oa, m, F, mps, th, pre=None):
    """SearchByProjection(F, vpMapPoints, th) as the device computes it -> (nmatches, frame_mp, diag, rounds record)"""
    q = local_queries(api, F, mps, th)
    fm = np.full(len(F.keys), -1, np.int32) if pre is None else np.array(pre, np.int32)
    call = dict(frame=F, q=q, qdesc=mps.desc, qmask=m._masks(mps.dmask), tags=q["desc_index"], rule=RULE_LEVEL_RATIO, nnratio=m.mfNNratio,
                threshold=m.TH_HIGH_, assigned=fm)
    return predict_windows(api, oa, call)


def predict_init(oa, m, F1, F2, prev, window):
    """SearchForInitialization as pi_walk_kernel computes it -> (nmatches, matches12, prev after the call, diag [queries, rescans])"""
    import multicol_slam_b200.api as api
    prev = np.array(prev, np.float64, copy=True)
    lv = F1.keys["octave"]
    q = api._queries(F1.key_cam, prev[:, 0], prev[:, 1], float(window), lv, lv, np.arange(len(F1.keys)))
    qs = model_queries(oa, F2, q, F1.desc, m._masks(F1.dmask))
    _, keep, resc = init_walk(qs, m.TH_LOW_, m.mfNNratio, len(F2.cam_w))
    keep = np.asarray(keep, np.int32)
    for i in np.flatnonzero(keep >= 0):
        prev[i] = (float(F2.keys["x"][keep[i]]), float(F2.keys["y"][keep[i]]))
    return int((keep >= 0).sum()), keep, prev, [len(qs), resc], qs


# ------------------------------------------------------------------------------------------------------------------------------
# the scene generator
# ------------------------------------------------------------------------------------------------------------------------------
class Abstract:
    """a search-independent scene: keypoints of the searched frame per camera, queries in the order the search makes them, the
    searched keypoints taken on entry, and the descriptor masks (None: unmasked)"""

    def __init__(self, dim, n_cams=3):
        self.dim, self.n_cams = dim, n_cams
        self.kps = [[] for _ in range(n_cams)]        # (x, y, octave, desc, mask)
        self.queries = []                              # (cam, x, y, level, desc, mask)
        self.taken = set()                             # (cam, j)
        self.R = 40                                    # the window radius every search is given, in pixels at octave 1

    def kp(self, cam, x, y, octave, desc, mask=None):
        self.kps[cam].append((float(x), float(y), int(octave), desc, mask))
        return len(self.kps[cam]) - 1

    def query(self, cam, x, y, level, desc, mask=None):
        self.queries.append((int(cam), float(x), float(y), int(level), desc, mask))

    def frame(self, api, items_per_cam, masked):
        per = []
        for items in items_per_cam:
            k = np.zeros(len(items), api.KEYPOINT_DTYPE)
            if items:
                k["x"] = [i[0] for i in items]; k["y"] = [i[1] for i in items]; k["octave"] = [i[2] for i in items]
            d = np.stack([i[3] for i in items]) if items else np.zeros((0, self.dim), np.uint8)
            mk = None
            if masked:
                mk = np.stack([i[4] if i[4] is not None else np.full(self.dim, 255, np.uint8) for i in items]) if items else \
                    np.zeros((0, self.dim), np.uint8)
            per.append((k, d, mk))
        return api.Frame.from_cameras(per, SIZES[:self.n_cams], SF)

    def target(self, api, masked):
        return self.frame(api, self.kps, masked)

    def taken_contiguous(self):
        off = np.concatenate([[0], np.cumsum([len(k) for k in self.kps])])
        return sorted(int(off[c] + j) for c, j in self.taken)


def _ray_point(api, cams, rig, cam, x, y, depth):
    ray = np.array(api.img_to_world(cams[cam], x, y)) * depth
    return np.asarray(api._mm(rig.MtMc[cam], np.append(ray, 1.0))[:3], np.float64)


def realise(api, kind, A, masked):
    """Abstract -> the inputs of one search.  kind: 'local' (SearchByProjection(F, vpMapPoints)), 'last' (the motion model),
    'window' (WindowSearch), 'frames' (SearchByProjection(F1, F2)), 'init' (SearchForInitialization).  Queries of the two-frame
    searches come from last-frame keypoints, whose order is camera-major: their queries are taken in that order."""
    from multicol_slam_b200 import synth
    cams = synth.lafida_cams()[:A.n_cams]
    if kind in ("frames", "init"):              # these searches read the query's octave alone: every keypoint at octave 1
        A.kps = [[(x, y, 1, d, mk) for x, y, _, d, mk in items] for items in A.kps]
    F = A.target(api, masked)
    s = dict(kind=kind, F=F, masked=masked, dim=A.dim, abstract=A)
    qs = A.queries
    if kind == "local":
        n = len(qs)
        in_view = np.zeros((n, A.n_cams), np.uint8); level = np.zeros((n, A.n_cams), np.int32)
        px = np.zeros((n, A.n_cams)); py = np.zeros((n, A.n_cams)); vc = np.full((n, A.n_cams), 0.9)
        for i, (c, x, y, lv, _, _) in enumerate(qs):
            in_view[i, c], level[i, c], px[i, c], py[i, c] = 1, lv, x, y
        desc = np.stack([q[4] for q in qs])
        dm = np.stack([q[5] if q[5] is not None else np.full(A.dim, 255, np.uint8) for q in qs]) if masked else None
        s.update(mps=api.MapPoints(np.zeros(n, np.uint8), in_view, level, px, py, vc, desc, dm), th=A.R / (4.0 * SF[1]))
        pre = np.full(len(F.keys), -1, np.int32)
        pre[A.taken_contiguous()] = 7
        s["pre"] = pre
        return s
    order = sorted(range(len(qs)), key=lambda i: qs[i][0])
    last_items = [[] for _ in range(A.n_cams)]
    for i in order:
        c, x, y, lv, d, mk = qs[i]
        last_items[c].append((x, y, lv, d, mk))
    Fl = A.frame(api, last_items, masked)
    if kind == "init":
        prev = np.stack([Fl.keys["x"], Fl.keys["y"]], axis=1).astype(np.float64)
        s.update(F1=Fl, F2=F, prev=prev, window=int(A.R))
        return s
    rig = api.Rig(cams)
    rng = np.random.default_rng(len(qs))
    world = np.stack([_ray_point(api, cams, rig, int(Fl.key_cam[i]), float(Fl.keys["x"][i]), float(Fl.keys["y"][i]), rng.uniform(2.0, 8.0))
                      for i in range(len(Fl.keys))]) if len(Fl.keys) else np.zeros((0, 3))
    mp_last = np.arange(len(Fl.keys), dtype=np.int32)
    mp_cur = np.full(len(F.keys), -1, np.int32)
    mp_cur[A.taken_contiguous()] = len(Fl.keys) + 5
    s.update(Fl=Fl, rig=rig, world=world, mp_last=mp_last, mp_cur=mp_cur, bad=np.zeros(len(Fl.keys) + 8, np.uint8),
             th=A.R / SF[1] if kind == "last" else int(A.R))
    return s


def predict(api, oa, m, s):
    """the device result of a realised scene from the model -> dict(n, out, diag, R or None, host oracle result)"""
    k = s["kind"]
    if k == "local":
        n, out, diag, R = predict_local(api, oa, m, s["F"], s["mps"], s["th"], s["pre"])
        on, oout = oa.search_by_projection(s["F"], s["mps"], s["th"], m.mfNNratio, m.TH_HIGH_, s["masked"], s["pre"].copy())
        return dict(n=n, out=out, diag=diag, R=R, oracle=(on, oout))
    if k == "init":
        n, keep, prev, diag, qs = predict_init(oa, m, s["F1"], s["F2"], s["prev"], s["window"])
        o = oa.search_for_initialization(s["F1"], s["F2"], s["prev"], s["window"], m.mfNNratio, m.TH_LOW_, s["masked"])
        return dict(n=n, out=keep, prev=prev, diag=diag, R=dict(queries=qs), oracle=o)
    cap = Capture(oa)
    on, oout = host_call(m, s, cap)
    if not cap.calls:                                  # nothing in any mask: no query at all
        return dict(n=0, out=oout, diag=None, R=None, oracle=(on, oout))
    call = cap.calls[0]
    n, assigned, diag, R = predict_windows(api, oa, call)
    out = assigned if k != "window" else np.where(assigned >= 0, s["mp_last"][np.maximum(assigned, 0)], -1).astype(np.int32)
    return dict(n=n, out=out, diag=diag, R=R, oracle=(on, oout))


def host_call(m, s, sw=None):
    """the host entry point of a realised two-frame scene (search_windows replay: `sw`, default the library's) -> (n, out)"""
    k = s["kind"]
    if k == "last":
        return m.SearchByProjectionLastRig(s["F"], s["rig"], s["mp_cur"], s["Fl"], s["mp_last"], None, s["world"], s["bad"], s["th"], _sw=sw)
    if k == "frames":
        return m.SearchByProjectionFramesRig(s["Fl"], s["mp_last"], s["F"], s["rig"], s["mp_cur"], s["world"], s["bad"], s["th"], _sw=sw)
    valid1 = np.ones(len(s["Fl"].keys), bool)
    n, v21 = m.WindowSearch(s["Fl"], s["F"], s["th"], valid1, 0, INT_MAX, _sw=sw)
    return n, np.where(v21 >= 0, s["mp_last"][np.maximum(v21, 0)], -1).astype(np.int32)


# ---- scene classes ----
def _mask(rng, dim, masked, p=0.1):
    if not masked:
        return None
    return np.packbits(rng.random(8 * dim) >= p).astype(np.uint8)


def dense(rng, dim, masked):
    """20-80 keypoints of camera 0 over a few grid cells, 50-300 queries whose windows cover them all; descriptors are noisy
    copies of 2-4 prototypes, so equal distances at different visiting positions are frequent"""
    A = Abstract(dim)
    protos = [rng.integers(0, 256, dim).astype(np.uint8) for _ in range(rng.integers(2, 5))]
    cx, cy = CENTRE
    for _ in range(rng.integers(20, 81)):
        A.kp(0, cx + rng.uniform(-14, 14), cy + rng.uniform(-12, 12), rng.integers(0, 2), flip(rng, protos[rng.integers(len(protos))],
             int(rng.integers(0, 5))), _mask(rng, dim, masked))
    for j in rng.choice(len(A.kps[0]), len(A.kps[0]) // 10, replace=False):
        A.taken.add((0, int(j)))
    for _ in range(rng.integers(50, 301)):
        A.query(0, cx + rng.uniform(-2, 2), cy + rng.uniform(-2, 2), 1, flip(rng, protos[rng.integers(len(protos))], int(rng.integers(0, 4))),
                _mask(rng, dim, masked))
    return A


def oscillation(rng, dim, masked, groups=24):
    """groups far apart, each of three queries with one descriptor over four keypoints a (octave 0), x = a + 1 (octave 1),
    y = a + 2 (octave 0) and b > a (octave 1), 8 < a < 16, placed so that query 0 sees x alone, query 1 sees a, x and y, and
    query 2 sees a and b.  Query 1 accepts a in round 0 (second best x on another octave); in round 1 query 0 has taken x, the
    second best is y on a's octave and a > 0.8 y rejects.  Query 2 so takes a, then b (a taken by query 1), then a again."""
    A = Abstract(dim)
    A.R = 4
    for g in range(groups):
        x0, y0 = 60.0 + 50.0 * (g % 12), 120.0 + 200.0 * (g // 12)
        base = rng.integers(0, 256, dim).astype(np.uint8)
        a = int(rng.integers(9, 16))
        for (dx, dy), d, o in (((0.5, 0.0), a, 0), ((-6.0, 0.5), a + 1, 1), ((-3.0, 3.0), a + 2, 0), ((7.0, -0.5), a + int(rng.integers(2, 10)), 1)):
            A.kp(0, x0 + dx, y0 + dy, o, flip(rng, base, d))
        for dx in (-9.5, -3.0, 4.0):
            A.query(0, x0 + dx, y0, 1, base)
    return A


def chain(A, rng, cam, n_cand, centre):
    """n_cand keypoints at distinct distances 1..n_cand from one descriptor, with octaves alternating along the distance order:
    identical queries with that descriptor take them one after the other, a dependency chain in which best and second best
    always differ in octave (the level-ratio test never applies) -> the descriptor"""
    base = rng.integers(0, 256, A.dim).astype(np.uint8)
    for k in rng.permutation(n_cand):
        A.kp(cam, centre[0] + rng.uniform(-20, 20), centre[1] + rng.uniform(-15, 15), int(k) % 2, flip(rng, base, int(k) + 1))
    return base


def depth(rng, dim, masked, n_chain, walk_mod=None):
    """a chain of n_chain queries in camera 0 (converges in n_chain + 1 rounds) interleaved, in map-point-major order, with
    independent queries of camera 1; walk_mod: the number of camera-1 queries before the chain's eighth query is chosen so that
    the walk starts at that residue mod 32"""
    A = Abstract(dim)
    base = chain(A, rng, 0, n_chain + 6, CENTRE)
    n_other = 40
    others = []
    for i in range(n_other):
        x, y = 60.0 + 80.0 * (i % 8), 60.0 + 90.0 * (i // 8)
        d = rng.integers(0, 256, dim).astype(np.uint8)
        A.kp(1, x, y, 1, d)
        others.append((x, y, flip(rng, d, int(rng.integers(0, 8)))))
    # where the chain's queries go among the others: spread, then shifted so that chain query 7 lands on walk_mod (mod 32)
    before7 = int(rng.integers(3, 20)) if walk_mod is None else (walk_mod - 7) % 32
    pos = sorted(rng.choice(before7 + 1, 7, replace=True).tolist()) + [before7] * (n_chain - 7 if n_chain > 7 else 0)
    pos = pos[:n_chain]
    oi = 0
    for k in range(n_chain):
        while oi < pos[k]:
            x, y, d = others[oi]; A.query(1, x, y, 1, d); oi += 1
        A.query(0, CENTRE[0], CENTRE[1], 1, base)
    for x, y, d in others[oi:]:
        A.query(1, x, y, 1, d)
    return A


def list_edges(rng, dim, masked, n_cand, tie, taken_mode):
    """groups whose windows hold exactly n_cand keypoints (8 or 9); tie: the 8th and 9th smallest keys at one distance;
    taken_mode 'entry': every listed keypoint but one taken on entry, 'queries': taken by earlier queries of the group"""
    A = Abstract(dim)
    A.R = 20
    for g in range(12):
        x0, y0 = 70.0 + 55.0 * (g % 8), 120.0 + 160.0 * (g // 8)
        base = rng.integers(0, 256, dim).astype(np.uint8)
        ds = sorted(rng.choice(np.arange(2, 40), n_cand, replace=False).tolist())
        if tie and n_cand >= 9:
            ds[8] = ds[7]
        first = len(A.kps[0])
        for i, dd in enumerate(rng.permutation(ds)):
            A.kp(0, x0 + rng.uniform(-3, 3), y0 + rng.uniform(-3, 3), int(rng.integers(0, 2)), flip(rng, base, int(dd)))
        js = list(range(first, first + n_cand))
        if taken_mode == "entry":
            keep = int(rng.integers(n_cand))
            for j in js:
                if j != first + keep:
                    A.taken.add((0, j))
            A.query(0, x0, y0, 1, base)
        else:
            # exact copies of the listed keypoints take them one by one, then the query of interest
            order = sorted(js, key=lambda j: int(np.unpackbits(A.kps[0][j][3] ^ base).sum()))
            for j in order[:min(7, n_cand - 1)]:
                A.query(0, x0, y0, 1, A.kps[0][j][3].copy())
            A.query(0, x0, y0, 1, base)
    return A


def ratio_pairs(nnratio, th_high):
    """(d0, d1) with d0 == d1 * nnratio exactly in double, d0 <= th_high, and the pairs one below and one above"""
    out = []
    for d1 in range(2, 200):
        p = float(d1) * nnratio
        if p == int(p) and 1 <= p <= th_high - 1 and d1 > p:
            out.append((int(p), d1))
    return out


def rule_edges(rng, dim, masked, nnratio, th_high):
    """isolated single queries: best / second best at d0 == nnratio * d1 (and one apart) with equal and with different octaves;
    d0 == th_high and th_high + 1 with no second candidate"""
    A = Abstract(dim)
    A.R = 5
    cases = []
    for d0, d1 in ratio_pairs(nnratio, th_high)[:6]:
        for dd in (0, -1, 1):
            for same in (True, False):
                cases.append((d0 + dd, d1, same))
    for d in (th_high, th_high + 1):
        cases.append((d, None, True))
    for g, (d0, d1, same) in enumerate(cases):
        x0, y0 = 40.0 + 30.0 * (g % 22), 60.0 + 40.0 * (g // 22)
        base = rng.integers(0, 256, dim).astype(np.uint8)
        A.kp(0, x0 + 1.0, y0, 1, flip(rng, base, d0))
        if d1 is not None:
            A.kp(0, x0 - 1.0, y0 + 1.0, 1 if same else 0, flip(rng, base, d1))
        A.query(0, x0, y0, 1, base)
    return A


def evictions(rng, dim, masked):
    """SearchForInitialization contention: a few keypoints, many queries at random distances, so that later queries take
    keypoints back with strictly smaller distances, equal distances are skipped, and lists fill with skipped entries"""
    A = Abstract(dim)
    A.R = 20
    for g in range(6):
        x0, y0 = 100.0 + 100.0 * (g % 6), 150.0 + 150.0 * (g // 6)
        base = rng.integers(0, 256, dim).astype(np.uint8)
        for _ in range(int(rng.integers(6, 14))):
            A.kp(0, x0 + rng.uniform(-6, 6), y0 + rng.uniform(-6, 6), 1, flip(rng, base, int(rng.integers(0, 10))), _mask(rng, dim, masked))
        for _ in range(int(rng.integers(20, 40))):
            A.query(0, x0 + rng.uniform(-2, 2), y0 + rng.uniform(-2, 2), 1, flip(rng, base, int(rng.integers(0, 12))), _mask(rng, dim, masked))
    return A


def catalogue(cap):
    """every generated scene: (scene class, search, seed, descriptor bytes, masked, nnratio, builder).  Every class runs masked and
    unmasked at 32 bytes, and one seed per class at 16 and 64 bytes."""
    out = []

    def add(cls, kinds, nn, seeds, build):
        for kind in kinds:
            for seed in seeds:
                for masked in (False, True):
                    out.append((cls, kind, seed, 32, masked, nn, build))
            out.append((cls, kind, seeds[0], 16, True, nn, build))
            out.append((cls, kind, seeds[0], 64, False, nn, build))

    add("dense", ["local", "last", "window", "frames", "init"], 0.8, [0, 1, 2], lambda rng, dim, mk, th: dense(rng, dim, mk))
    add("oscillation", ["local"], 0.8, [0, 1], lambda rng, dim, mk, th: oscillation(rng, dim, mk))
    for n_chain, wm in ((cap - 2, None), (cap - 1, None), (cap, 0), (cap, 1), (cap, 31)):
        add(f"depth{n_chain}" + ("" if wm is None else f"_s{wm}"), ["local"], 0.8, [0],
            lambda rng, dim, mk, th, n=n_chain, w=wm: depth(rng, dim, mk, n, w))
    for n_cand, tie, mode in ((8, False, "entry"), (8, False, "queries"), (9, True, "entry"), (9, True, "queries")):
        add(f"list{n_cand}_{mode}", ["local", "last"], 0.8, [0], lambda rng, dim, mk, th, n=n_cand, t=tie, m=mode: list_edges(rng, dim, mk, n, t, m))
    for kind, ratios in (("local", (0.6, 0.75, 0.8, 0.9)), ("window", (0.6, 0.75, 0.8, 0.9)), ("last", (0.8,)), ("init", (0.6, 0.75, 0.8, 0.9))):
        for nn in ratios:
            add(f"rule{nn}", [kind], nn, [0], lambda rng, dim, mk, th, nn=nn: rule_edges(rng, dim, mk, nn, th))
    add("evictions", ["init"], 0.9, [0, 1, 2], lambda rng, dim, mk, th: evictions(rng, dim, mk))
    return out


def make(api, spec):
    """spec from catalogue() -> (matcher, realised scene)"""
    cls, kind, seed, dim, masked, nn, build = spec
    m = api.cORBmatcher(nn, False, dim, masked)
    th = m.TH_LOW_ if kind == "init" else m.TH_HIGH_
    rng = np.random.default_rng(1000 * seed + dim + 7 * masked + sum(map(ord, cls + kind)))
    return m, realise(api, kind, build(rng, dim, masked, th), masked)


def spec_id(spec):
    cls, kind, seed, dim, masked, nn, _ = spec
    return f"{cls}-{kind}-s{seed}-{dim}B" + ("-masked" if masked else "")
