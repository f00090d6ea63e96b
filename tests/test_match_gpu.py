"""GPU parity of the matcher half: Hamming top-K / brute force (M2), grid window search (G1) and the
SearchByProjection / SearchForInitialization replays (M1, M3) vs the CPU oracle.  Integer work: bit-exact."""
import numpy as np
import pytest

from match_scenes import make_frames, random_rig

pytestmark = pytest.mark.gpu


def popcount_dist(q, d):
    x = np.bitwise_xor(q[:, None, :], d[None, :, :])
    return np.unpackbits(x, axis=2).sum(axis=2).astype(np.int32)


def rand_desc(rng, n, dim=32):
    return rng.integers(0, 256, (n, dim)).astype(np.uint8)


@pytest.mark.parametrize("dim,K", [(16, 4), (32, 4), (64, 4), (16, 5), (64, 7)], ids=["16", "32", "64", "16-K5", "64-K7"])
@pytest.mark.parametrize("masked", [False, True])
def test_topk_vs_numpy(api, dim, masked, K):
    rng = np.random.default_rng(dim + masked)
    q, d = rand_desc(rng, 300, dim), rand_desc(rng, 1777, dim)
    d[5] = d[900] = q[7]                        # exact duplicates in different database splits: ties must keep the lower index
    if masked:
        qm, dm = rand_desc(rng, 300, dim) | rand_desc(rng, 300, dim), rand_desc(rng, 1777, dim) | rand_desc(rng, 1777, dim)
        x = np.bitwise_xor(q[:, None, :], d[None, :, :])
        dist = (np.unpackbits(x & qm[:, None, :], axis=2).sum(axis=2) + np.unpackbits(x & dm[None, :, :], axis=2).sum(axis=2)) // 2
        idx, dd = api.hamming_topk(q, d, K, qm, dm)
    else:
        dist = popcount_dist(q, d)
        idx, dd = api.hamming_topk(q, d, K)
    order = np.lexsort((np.broadcast_to(np.arange(d.shape[0]), dist.shape), dist), axis=1)[:, :K]
    assert np.array_equal(idx, order.astype(np.int32))
    assert np.array_equal(dd, np.take_along_axis(dist, order, axis=1).astype(np.int32))
    if not masked:
        assert idx[7, 0] == 5 and idx[7, 1] == 900 and dd[7, 0] == 0


def test_topk_skip_and_small(api):
    rng = np.random.default_rng(3)
    q, d = rand_desc(rng, 10), rand_desc(rng, 3)
    skip = np.array([0, 1, 0], np.uint8)
    idx, dd = api.hamming_topk(q, d, 4, db_skip=skip)
    dist = popcount_dist(q, d)
    for i in range(10):
        cand = sorted([(dist[i, j], j) for j in (0, 2)])
        assert list(idx[i, :2]) == [c[1] for c in cand] and list(idx[i, 2:]) == [-1, -1]
        assert list(dd[i, :2]) == [c[0] for c in cand]


@pytest.mark.parametrize("masked", [False, True])
def test_bruteforce_search_by_bow(api, oa, masked):
    """SearchByBoW(KF,KF) semantics incl. the greedy one-use rule under heavy contention."""
    rng = np.random.default_rng(11)
    nd, nq = 3000, 1200
    d = rand_desc(rng, nd)
    # many queries planted on few database entries -> contention for the same best match
    target = rng.integers(0, 40, nq)
    q = d[target].copy()
    flips = rng.integers(0, 30, nq)
    for i in range(nq):
        bits = rng.choice(256, flips[i], replace=False)
        for b in bits:
            q[i, b // 8] ^= 1 << (b % 8)
    qm = dm = None
    if masked:
        qm = (rng.random((nq, 256)) < 0.85)
        dm = (rng.random((nd, 256)) < 0.85)
        qm, dm = np.packbits(qm, axis=1, bitorder="little"), np.packbits(dm, axis=1, bitorder="little")
    v1 = (rng.random(nq) < 0.9).astype(np.uint8)
    v2 = (rng.random(nd) < 0.95).astype(np.uint8)
    matcher = api.cORBmatcher(0.9, False, 32, masked)
    n, m12 = matcher.SearchByBoW(q, d, qm, dm, v1, v2)
    on, om12 = oa.match_bruteforce(q, d, matcher.TH_LOW_, 0.9, qm, dm, v1, v2)
    assert n == on and np.array_equal(m12, om12)
    assert n > 20


def test_window_search_candidates(api, oa, cams):
    from multicol_slam_b200.ctypes_defs import WINDOW_QUERY_DTYPE
    F = make_frames(api, oa, cams, [1, 2, 3])
    rng = np.random.default_rng(0)
    nq = 700
    qs = np.zeros(nq, WINDOW_QUERY_DTYPE)
    qs["cam"] = rng.integers(0, 3, nq)
    lv = rng.integers(0, 8, nq)
    kind = rng.integers(0, 3, nq)
    qs["min_level"] = np.where(kind == 0, -1, np.where(kind == 1, lv, lv - 1))
    qs["max_level"] = np.where(kind == 0, -1, lv)
    qs["desc_index"] = rng.integers(0, len(F.keys), nq)
    qs["x"] = rng.uniform(-30, 790, nq)
    qs["y"] = rng.uniform(-30, 510, nq)
    qs["r"] = rng.uniform(1, 60, nq)
    gi, gd, gc, rc = api.window_search(F, qs, F.desc, F.dmask, max_cand=512)
    oi, od, oc, orc = oa.window_search(F, qs, F.desc, F.dmask, max_cand=512)
    assert rc == 0 and orc == 0
    assert np.array_equal(gc, oc)
    for i in range(nq):
        assert np.array_equal(gi[i, :gc[i]], oi[i, :oc[i]]) and np.array_equal(gd[i, :gc[i]], od[i, :oc[i]])
    assert gc.max() > 20
    # overflow is reported, true counts are still returned
    gi2, gd2, gc2, rc2 = api.window_search(F, qs, F.desc, F.dmask, max_cand=4)
    assert rc2 == api.MCS_ERR_CAPACITY and np.array_equal(gc2, oc)


@pytest.mark.parametrize("masks", [False, True])
def test_search_by_projection(api, oa, cams, masks):
    F = make_frames(api, oa, cams, [4, 5, 6], masks=masks)
    rng = np.random.default_rng(2)
    nmp, nc = 4000, 3
    src = rng.integers(0, len(F.keys), nmp)
    desc = F.desc[src].copy()
    for i in range(nmp):
        for b in rng.choice(256, rng.integers(0, 41), replace=False):
            desc[i, b // 8] ^= 1 << (b % 8)
    dm = F.dmask[src].copy() if masks else None
    in_view = np.zeros((nmp, nc), np.uint8)
    level = np.zeros((nmp, nc), np.int32)
    px = np.zeros((nmp, nc)); py = np.zeros((nmp, nc)); vc = np.zeros((nmp, nc))
    for i in range(nmp):
        c = F.key_cam[src[i]]
        in_view[i, c] = 1
        level[i, c] = min(7, max(0, F.keys[src[i]]["octave"] + rng.integers(-1, 2)))
        px[i, c] = F.keys[src[i]]["x"] + rng.normal(0, 2)
        py[i, c] = F.keys[src[i]]["y"] + rng.normal(0, 2)
        vc[i, c] = rng.uniform(0.9, 1.0)
        if rng.random() < 0.2:      # also visible in a second camera
            c2 = (c + 1) % nc
            in_view[i, c2] = 1; level[i, c2] = rng.integers(0, 8)
            px[i, c2] = rng.uniform(0, 754); py[i, c2] = rng.uniform(0, 480); vc[i, c2] = rng.uniform(0.9, 1.0)
    bad = (rng.random(nmp) < 0.05).astype(np.uint8)
    mps = api.MapPoints(bad, in_view, level, px, py, vc, desc, dm)
    matcher = api.cORBmatcher(0.8, False, 32, masks)
    n, fmp = matcher.SearchByProjection(F, mps, 3.0)
    on, ofmp = oa.search_by_projection(F, mps, 3.0, 0.8, matcher.TH_HIGH_, masks)
    assert n == on and np.array_equal(fmp, ofmp)
    assert n > 500
    # pre-assigned keypoints are skipped (greedy rule, ref :121)
    pre = np.full(len(F.keys), -1, np.int32)
    pre[::3] = 0
    n2, fmp2 = matcher.SearchByProjection(F, mps, 1.0, pre.copy())
    on2, ofmp2 = oa.search_by_projection(F, mps, 1.0, 0.8, matcher.TH_HIGH_, masks, pre.copy())
    assert n2 == on2 and np.array_equal(fmp2, ofmp2)


@pytest.mark.parametrize("masks", [False, True])
def test_search_for_initialization(api, oa, cams, masks):
    from multicol_slam_b200 import synth
    ex = api.mdBRIEFextractorOct(nfeatures=800, fastThreshold=5, do_dBrief=True, learnMasks=masks)
    sf = [ex.info.scale_factor[l] for l in range(8)]
    fr = []
    for t in range(2):
        per = []
        for c in range(3):
            stream = synth.texture_stream(cams[c], 2, seed=40 + c)
            per.append(ex(stream[t], synth.mirror_mask(cams[c]), cams[c]))
        fr.append(api.Frame.from_cameras(per, [(754, 480)] * 3, sf))
    F1, F2 = fr
    prev = np.stack([F1.keys["x"], F1.keys["y"]], axis=1).astype(np.float64)
    matcher = api.cORBmatcher(0.9, False, 32, masks)
    p1 = prev.copy()
    n, m12 = matcher.SearchForInitialization(F1, F2, p1, 50)
    on, om12, oprev = oa.search_for_initialization(F1, F2, prev, 50, 0.9, matcher.TH_LOW_, masks)
    assert n == on and np.array_equal(m12, om12) and np.array_equal(p1, oprev)
    assert n > 200
    # matched keypoints moved by the stream's (3,2) px/frame motion
    ok = m12 >= 0
    dx = F1.keys["x"][ok] - F2.keys["x"][m12[ok]]
    assert np.median(np.abs(dx - 3.0)) < 1.5


@pytest.mark.parametrize("masks", [False, True])
def test_extract_match_stream(api, oa, cams, masks):
    """The combined stream entry point: extraction identical to per-image calls, matches identical to an
    all-pairs numpy evaluation of the reference distance (frame t vs t-1, same camera)."""
    from multicol_slam_b200 import synth
    F, Cn, K = 3, 3, 2
    imgs = np.stack([np.stack([synth.texture_stream(cams[c], F, seed=70 + c)[t] for c in range(Cn)]) for t in range(F)])
    mk = np.stack([synth.mirror_mask(c) for c in cams])
    ex = api.mdBRIEFextractorOct(nfeatures=500, do_dBrief=True, learnMasks=masks)
    r = ex.extract_match_stream(imgs, mk, cams, K=K)
    oe = oa.OracleExtractor(nfeatures=500, do_dbrief=True, learn_masks=masks)
    per = {}
    for t in range(F):
        for c in range(Cn):
            i = t * Cn + c
            ok, od, om = oe.extract(imgs[t, c], mk[c], cams[c])
            n = r["counts"][i]
            assert n == len(ok) and r["kps"][i, :n].tobytes() == ok.tobytes()
            assert np.array_equal(r["desc"][i, :n], od) and np.array_equal(r["dmask"][i, :n], om)
            per[(t, c)] = (od, om)
    for t in range(F):
        for c in range(Cn):
            i = t * Cn + c
            n = r["counts"][i]
            if t == 0:
                assert np.all(r["match_idx"][i] == -1) and np.all(r["match_dist"][i] == 0x7FFFFFFF)
                continue
            q, qm = per[(t, c)]
            d, dm = per[(t - 1, c)]
            x = np.bitwise_xor(q[:, None, :], d[None, :, :])
            if masks:
                dist = (np.unpackbits(x & qm[:, None, :], axis=2).sum(axis=2) + np.unpackbits(x & dm[None, :, :], axis=2).sum(axis=2)) // 2
            else:
                dist = np.unpackbits(x, axis=2).sum(axis=2)
            order = np.lexsort((np.broadcast_to(np.arange(len(d)), dist.shape), dist), axis=1)[:, :K]
            assert np.array_equal(r["match_idx"][i, :n], order.astype(np.int32))
            assert np.array_equal(r["match_dist"][i, :n], np.take_along_axis(dist, order, axis=1).astype(np.int32))
            assert np.all(r["match_idx"][i, n:] == -1)


def test_config4_full_size_bruteforce(api):
    """BASELINE config 4 size: 32 000 queries vs a 200 000-descriptor database (loop-closure path), with masks.
    Size-independent properties: every query is planted once with <= 30 flipped bits and must come back as the
    best match at exactly its planted (masked) distance; the second best is a random descriptor, far away."""
    rng = np.random.default_rng(4)
    nd, nq = 200_000, 32_000
    d = rng.integers(0, 256, (nd, 32), dtype=np.uint8)
    dm = np.packbits(rng.random((nd, 256)) < 0.85, axis=1, bitorder="little")
    where = rng.permutation(nd)[:nq]
    q = d[where].copy()
    qm = np.packbits(rng.random((nq, 256)) < 0.85, axis=1, bitorder="little")
    nflip = rng.integers(0, 31, nq)
    flips = np.zeros((nq, 256), bool)
    for i in range(nq):
        flips[i, rng.choice(256, nflip[i], replace=False)] = True
    fl = np.packbits(flips, axis=1, bitorder="little")
    q ^= fl
    idx, dist = api.hamming_topk(q, d, 2, qm, dm)
    expect = (np.unpackbits(fl & qm, axis=1).sum(axis=1).astype(np.int64) + np.unpackbits(fl & dm[where], axis=1).sum(axis=1)) // 2
    assert np.array_equal(idx[:, 0], where.astype(np.int32))
    assert np.array_equal(dist[:, 0], expect.astype(np.int32))
    assert dist[:, 1].min() > 60 and np.all(dist[:, 1] >= dist[:, 0])
    # unmasked as well
    idx2, dist2 = api.hamming_topk(q, d, 1)
    assert np.array_equal(idx2[:, 0], where.astype(np.int32)) and np.array_equal(dist2[:, 0], nflip.astype(np.int32))


def test_config3_full_size_search_by_projection(api, oa, cams):
    """BASELINE config 3 size: 4 fisheye cameras 1280x720, 2000 feat/cam, SearchByProjection against 50 000 map points."""
    from multicol_slam_b200 import synth
    cam4 = [synth.scaled_cam(cams[i % 3], 1280, 720) for i in range(4)]
    ex = api.mdBRIEFextractorOct(nfeatures=2000, do_dBrief=True, learnMasks=True)
    imgs = np.stack([synth.frame(cam4[c], 300 + c) for c in range(4)])
    mk = np.stack([synth.mirror_mask(c) for c in cam4])
    kps, desc, dmask, counts = ex.extract_batch(imgs, mk, cam4, [0, 1, 2, 3])
    per = [(kps[c, :counts[c]], desc[c, :counts[c]], dmask[c, :counts[c]]) for c in range(4)]
    F = api.Frame.from_cameras(per, [(1280, 720)] * 4, [ex.info.scale_factor[l] for l in range(8)])
    rng = np.random.default_rng(3)
    nmp = 50_000
    src = rng.integers(0, len(F.keys), nmp)
    mdesc = F.desc[src].copy()
    flips = rng.integers(0, 41, nmp)
    for i in range(nmp):
        b = rng.choice(256, flips[i], replace=False)
        np.bitwise_xor.at(mdesc[i], b // 8, (1 << (b % 8)).astype(np.uint8))
    in_view = np.zeros((nmp, 4), np.uint8); level = np.zeros((nmp, 4), np.int32)
    px = np.zeros((nmp, 4)); py = np.zeros((nmp, 4)); vc = np.zeros((nmp, 4))
    c = F.key_cam[src]
    r = np.arange(nmp)
    in_view[r, c] = 1
    level[r, c] = rng.integers(0, 8, nmp)
    px[r, c] = F.keys["x"][src] + rng.normal(0, 2, nmp)
    py[r, c] = F.keys["y"][src] + rng.normal(0, 2, nmp)
    vc[r, c] = rng.uniform(0.9, 1.0, nmp)
    mps = api.MapPoints(np.zeros(nmp, np.uint8), in_view, level, px, py, vc, mdesc, F.dmask[src].copy())
    matcher = api.cORBmatcher(0.8, False, 32, True)
    n, fmp = matcher.SearchByProjection(F, mps, 3.0)
    on, ofmp = oa.search_by_projection(F, mps, 3.0, 0.8, matcher.TH_HIGH_, True)
    assert n == on and np.array_equal(fmp, ofmp) and n > 2000


@pytest.mark.parametrize("masks", [False, True])
def test_m4_window_searches(api, oa, cams, masks):
    """The remaining projection-window searches (SURVEY 8a row M4) through mcs_search_windows: WindowSearch (:326),
    SearchByProjection(F1,F2,win) (:476), SearchByProjection(Current,Last,th) (:1990) vs the oracle's generic loop."""
    from multicol_slam_b200 import synth
    from multicol_slam_b200.api import RULE_BEST, RULE_RATIO, _queries
    ex = api.mdBRIEFextractorOct(nfeatures=700, do_dBrief=True, learnMasks=masks)
    sf = [ex.info.scale_factor[l] for l in range(8)]
    fr = []
    for t in range(2):
        per = [ex(synth.texture_stream(cams[c], 2, seed=60 + c)[t], synth.mirror_mask(cams[c]), cams[c]) for c in range(3)]
        fr.append(api.Frame.from_cameras(per, [(754, 480)] * 3, sf))
    F1, F2 = fr
    rng = np.random.default_rng(8)
    valid1 = (rng.random(len(F1.keys)) < 0.8).astype(np.uint8)
    m = api.cORBmatcher(0.8, False, 32, masks)
    qm = F1.dmask if masks else None

    # WindowSearch
    n, m21 = m.WindowSearch(F1, F2, 60, valid1, 0, 5)
    lv = F1.keys["octave"]
    sel = np.flatnonzero((valid1 != 0) & (lv <= 5))
    q = _queries(F1.key_cam[sel], F1.keys["x"][sel].astype(np.float64), F1.keys["y"][sel].astype(np.float64), 60.0, -1, -1, sel)
    on, om21 = oa.search_windows(F2, q, F1.desc, qm, sel, RULE_RATIO, 0.8, m.TH_HIGH_, np.full(len(F2.keys), -1, np.int32))
    assert n == on and np.array_equal(m21, om21) and n > 300

    # SearchByProjection(F1, F2, windowSize): projections = F1 keypoint position moved by the stream motion, all cameras tried
    uv = np.zeros((len(F1.keys), 3, 2))
    in_mask = np.zeros((len(F1.keys), 3), np.uint8)
    for c in range(3):
        uv[:, c, 0] = F1.keys["x"] - 3.0 + rng.normal(0, 1, len(F1.keys))
        uv[:, c, 1] = F1.keys["y"] - 2.0 + rng.normal(0, 1, len(F1.keys))
        in_mask[:, c] = (F1.key_cam == c) | (rng.random(len(F1.keys)) < 0.1)
    pre = np.full(len(F2.keys), -1, np.int32)
    pre[::7] = 0
    n2, a2 = m.SearchByProjectionFrames(F1, F2, 40, valid1, uv, in_mask, pre.copy())
    i1, c = np.nonzero((valid1 != 0)[:, None] & (in_mask != 0))
    q = _queries(c, uv[i1, c, 0], uv[i1, c, 1], 40.0, lv[i1], lv[i1], i1)
    on2, oa2 = oa.search_windows(F2, q, F1.desc, qm, i1, RULE_RATIO, 0.8, m.TH_HIGH_, pre.copy())
    assert n2 == on2 and np.array_equal(a2, oa2) and n2 > 300

    # SearchByProjection(CurrentFrame = F2, LastFrame = F1, th)
    uvl = np.stack([F1.keys["x"] - 3.0, F1.keys["y"] - 2.0], axis=1).astype(np.float64)
    inm = (rng.random(len(F1.keys)) < 0.95).astype(np.uint8)
    n3, a3 = m.SearchByProjectionLast(F2, F1, 50.0, valid1, uvl, inm)
    sel = np.flatnonzero((valid1 != 0) & (inm != 0))
    l3 = lv[sel]
    q = _queries(F1.key_cam[sel], uvl[sel, 0], uvl[sel, 1], 50.0 * F2.scale_factors[l3], l3 - 1, l3 + 1, sel)
    on3, oa3 = oa.search_windows(F2, q, F1.desc, qm, sel, RULE_BEST, 0.8, m.TH_HIGH_, np.full(len(F2.keys), -1, np.int32))
    assert n3 == on3 and np.array_equal(a3, oa3) and n3 > 300

    # the generic entry point with the level rule reproduces the dedicated SearchByProjection(F, MapPoints) oracle
    nmp = 1500
    src = rng.integers(0, len(F2.keys), nmp)
    nc = 3
    in_view = np.zeros((nmp, nc), np.uint8); level = np.zeros((nmp, nc), np.int32)
    px = np.zeros((nmp, nc)); py = np.zeros((nmp, nc)); vc = np.full((nmp, nc), 0.95)
    cc = F2.key_cam[src]; r = np.arange(nmp)
    in_view[r, cc] = 1; level[r, cc] = F2.keys["octave"][src]
    px[r, cc] = F2.keys["x"][src]; py[r, cc] = F2.keys["y"][src]
    mps = api.MapPoints(np.zeros(nmp, np.uint8), in_view, level, px, py, vc, F2.desc[src], F2.dmask[src] if masks else None)
    n4, f4 = m.SearchByProjection(F2, mps, 3.0)
    on4, of4 = oa.search_by_projection(F2, mps, 3.0, 0.8, m.TH_HIGH_, masks)
    assert n4 == on4 and np.array_equal(f4, of4)


def test_project_mappoints_and_search(api, oa, cams):
    """Projection front-end (isInFrustum batched, SURVEY 8f row 2) vs the oracle, then the full chain
    projection -> SearchByProjection on the GPU against the oracle's chain."""
    from multicol_slam_b200 import synth
    rng = np.random.default_rng(12)
    nc, n = 3, 20000
    mtmc, inv = random_rig(rng, nc)
    masks = np.stack([synth.mirror_mask(c) for c in cams])
    pos = rng.normal(size=(n, 3)); pos *= (rng.uniform(1.5, 12.0, n) / np.linalg.norm(pos, axis=1))[:, None]
    nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    dmin = rng.uniform(0.5, 4.0, n); dmax = dmin * rng.uniform(1.5, 6.0, n)
    sf = np.cumprod([1.0] + [1.2000000476837158] * 7)
    g = api.project_mappoints(inv, mtmc, cams, masks, pos, nrm, dmin, dmax, sf)
    o = oa.project_mappoints(inv, mtmc, cams, masks, pos, nrm, dmin, dmax, sf)
    assert np.array_equal(g[0], o[0]) and np.array_equal(g[1], o[1])            # in_view, level: exact
    assert np.array_equal(g[4], o[4])                                              # view cosine: sqrt/div only -> exact
    assert np.abs(g[2] - o[2]).max() < 1e-9 and np.abs(g[3] - o[3]).max() < 1e-9   # projections: atan() differs in the last ulp
    assert 0.1 < g[0].mean() < 0.9
    # chain: a frame + map points whose descriptors are noisy copies of frame descriptors near their projections
    ex = api.mdBRIEFextractorOct(nfeatures=1000, do_dBrief=True, learnMasks=True)
    per = [ex(synth.frame(cams[c], 200 + c), masks[c], cams[c]) for c in range(3)]
    F = api.Frame.from_cameras(per, [(754, 480)] * 3, [ex.info.scale_factor[l] for l in range(8)])
    desc = F.desc[rng.integers(0, len(F.keys), n)].copy()
    mps_g = api.MapPoints(np.zeros(n, np.uint8), g[0], g[1], g[2], g[3], g[4], desc, F.dmask[rng.integers(0, len(F.keys), n)])
    mps_o = api.MapPoints(np.zeros(n, np.uint8), o[0], o[1], o[2], o[3], o[4], mps_g.desc, mps_g.dmask)
    m = api.cORBmatcher(0.8, False, 32, True)
    ng, fg = m.SearchByProjection(F, mps_g, 3.0)
    no, fo = oa.search_by_projection(F, mps_o, 3.0, 0.8, m.TH_HIGH_, True)
    assert ng == no and np.array_equal(fg, fo)


@pytest.mark.parametrize("masks", [False, True])
def test_search_for_triangulation(api, oa, cams, masks):
    """SearchForTriangulationRaw (ref :968-1156): all-pairs same-camera scan with the epipolar test, incl. the case of more than
    K candidates inside the thresholds (paging) via many near-duplicate descriptors."""
    from multicol_slam_b200 import synth
    rng = np.random.default_rng(21)
    ex = api.mdBRIEFextractorOct(nfeatures=600, do_dBrief=True, learnMasks=masks)
    fr = []
    for t in range(2):
        per = [ex(synth.texture_stream(cams[c], 2, seed=80 + c)[t], synth.mirror_mask(cams[c]), cams[c]) for c in range(3)]
        fr.append(api.Frame.from_cameras(per, [(754, 480)] * 3, [ex.info.scale_factor[l] for l in range(8)]))
    F1, F2 = fr

    def rays(F):
        out = np.zeros((len(F.keys), 3))
        for i, k in enumerate(F.keys):
            out[i] = api.img_to_world(cams[F.key_cam[i]], float(k["x"]), float(k["y"]))
        return out
    r1, r2 = rays(F1), rays(F2)
    # a small sideways translation between the two keyframes: E = [t]x R with R = I
    t = np.array([1.0, 0.1, 0.0]); t /= np.linalg.norm(t)
    Ex = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    E = np.tile(Ex, (3, 3, 1, 1))
    free1 = (rng.random(len(F1.keys)) < 0.7).astype(np.uint8)
    free2 = (rng.random(len(F2.keys)) < 0.7).astype(np.uint8)
    d2 = F2.desc.copy()
    d2[100:140] = F1.desc[50]                      # 40 database entries identical to one query: > K candidates at distance ~0
    d2[100:140, 5] ^= rng.integers(0, 4, 40).astype(np.uint8)
    m = api.cORBmatcher(0.8, False, 32, masks)
    for thr in (1e-2, 1e-4):
        n, m12 = m.SearchForTriangulationRaw(F1.desc, F1.dmask, F1.key_cam, free1, r1, d2, F2.dmask, F2.key_cam, free2, r2, E, thr)
        on, om12 = oa.search_for_triangulation(F1.desc, F1.dmask if masks else None, F1.key_cam, free1, r1, d2, F2.dmask if masks else None,
                                               F2.key_cam, free2, r2, E, m.TH_LOW_, thr)
        assert n == on and np.array_equal(m12, om12)
    assert n > 20


def test_frame_prepare_rays_and_grid(api, oa, cams):
    """Bearing rays + 64x48 grid of the cMultiFrame constructor on the GPU (SURVEY 8f row 3): rays bit-identical to the host
    evaluation (no libm call involved), CSR grid identical to the reference's per-cell insertion order."""
    F = make_frames(api, oa, cams, [7, 8, 9], nf=2000)
    keys = F.keys.copy()
    keys["x"][::97] = -3.0          # out-of-grid keypoints are dropped by PosInGrid
    keys["y"][5::89] = 481.0
    g = api.frame_prepare(keys, F.key_cam, cams)
    o = oa.frame_prepare(keys, F.key_cam, cams)
    assert np.array_equal(g[0].view(np.uint64), o[0].view(np.uint64))
    assert np.array_equal(g[1], o[1]) and np.array_equal(g[2], o[2])
    assert len(g[2]) < len(keys) and len(g[2]) > 0.9 * len(keys)
    assert np.allclose(np.linalg.norm(g[0], axis=1), 1.0)


def test_fuse_candidates_stateless_rule(api, oa, cams):
    """MCS_RULE_BEST_FREE: the matching core of Fuse / SearchBySim3 (best candidate in {l-1,l}, nothing skipped or marked)."""
    from multicol_slam_b200.api import RULE_BEST_FREE, _queries
    KF = make_frames(api, oa, cams, [31, 32, 33], nf=900)
    rng = np.random.default_rng(5)
    n = 3000
    src = rng.integers(0, len(KF.keys), n)
    uv = np.zeros((n, 3, 2)); in_mask = np.zeros((n, 3), np.uint8); level = np.zeros((n, 3), np.int64)
    c = KF.key_cam[src]; r = np.arange(n)
    uv[r, c, 0] = KF.keys["x"][src] + rng.normal(0, 1.5, n); uv[r, c, 1] = KF.keys["y"][src] + rng.normal(0, 1.5, n)
    in_mask[r, c] = 1; level[r, c] = np.clip(KF.keys["octave"][src] + rng.integers(0, 2, n), 0, 7)
    m = api.cORBmatcher(0.8, False, 32, True)
    best = m.FuseCandidates(KF, uv, in_mask, level, 2.5, KF.desc[src], KF.dmask[src])
    i, cc = np.nonzero(in_mask)
    lv = level[i, cc]
    q = _queries(cc, uv[i, cc, 0], uv[i, cc, 1], 2.5 * KF.scale_factors[lv], lv - 1, lv, i)
    on, ores = oa.search_windows(KF, q, KF.desc[src], KF.dmask[src], np.zeros(len(q), np.int32), RULE_BEST_FREE, 0.8, m.TH_LOW_,
                                 np.full(max(len(q), len(KF.keys)), -1, np.int32))
    assert np.array_equal(best[i, cc], ores[:len(q)])
    assert (best[i, cc] == src).mean() > 0.5 and (best[i, cc] >= 0).sum() == on


def test_packed_extraction_replay_and_device_bruteforce(api, oa, cams):
    """Round-2 device-resident pieces in one flow: K3 writing straight into the packed exchange buffer (mcs_packed_layout), the
    stream matcher's K-best lists, the on-device greedy acceptance (mcs_match_stream_replay_device) and the device-resident
    brute-force entry (mcs_match_bruteforce_device) -- all against the oracle's SearchByBoW(KF1, KF2) per image pair."""
    import torch
    from multicol_slam_b200 import rig, synth
    Fn, nc = 5, 3
    streams = [synth.texture_stream(cams[c], Fn, seed=70 + c) for c in range(nc)]
    imgs = np.ascontiguousarray(np.stack(streams, axis=1)).reshape(Fn * nc, 480, 754)        # frame-major
    masks = np.stack([synth.mirror_mask(c) for c in cams])
    ex = api.mdBRIEFextractorOct(nfeatures=600, do_dBrief=True, learnMasks=True)
    cap, ds, B = ex.capacity, 32, Fn * nc
    dev = torch.device("cuda", 0)
    pitched = torch.zeros((B, 480, 768), dtype=torch.uint8, device=dev)
    pitched[:, :, :754] = torch.from_numpy(imgs).to(dev)
    coi = np.tile(np.arange(nc, dtype=np.int32), Fn)
    packed = torch.zeros(rig.packed_layout(B, cap, ds)[1], dtype=torch.uint8, device=dev)
    st = torch.cuda.Stream(dev)
    with torch.cuda.stream(st):
        out = ex.extract_batch_packed_device(pitched, masks, cams, coi, packed, stream=st, width=754)
        ref = ex.extract_batch_device(pitched, masks, cams, coi, stream=st, width=754)
        idx, dist = api.match_stream_device(out["desc"], out["dmask"], out["counts"], Fn, nc, K=4, stream=st)
        m12, nm, redo = api.match_stream_replay_device(idx, dist, out["counts"], out["desc"], out["dmask"], Fn, nc, 32, 0.9, stream=st)
        # short lists force the in-kernel rescan of undecidable queries: the result must not depend on K
        idx1, dist1 = api.match_stream_device(out["desc"], out["dmask"], out["counts"], Fn, nc, K=1, stream=st)
        m12b, nmb, _ = api.match_stream_replay_device(idx1, dist1, out["counts"], out["desc"], out["dmask"], Fn, nc, 32, 0.9, stream=st)
        idx8, dist8 = api.match_stream_device(out["desc"], out["dmask"], out["counts"], Fn, nc, K=8, stream=st)      # the 8-entry list kernel
        m12d, nmd, _ = api.match_stream_replay_device(idx8, dist8, out["counts"], out["desc"], out["dmask"], Fn, nc, 32, 0.9, stream=st)
        # lists + replay as one call, the lists cut at the relevance bound of (th_low, nnratio): same matches; also for other
        # thresholds, including ones where the bound exceeds every possible distance
        m12c, nmc = api.match_stream_greedy_device(out["desc"], out["dmask"], out["counts"], Fn, nc, 32, 0.9, stream=st)
        other = []
        for th, nn in ((50, 0.6), (100, 0.8), (20, 0.99), (300, 0.05)):
            i2, d2 = api.match_stream_device(out["desc"], out["dmask"], out["counts"], Fn, nc, K=3, stream=st)
            a = api.match_stream_replay_device(i2, d2, out["counts"], out["desc"], out["dmask"], Fn, nc, th, nn, stream=st)
            b = api.match_stream_greedy_device(out["desc"], out["dmask"], out["counts"], Fn, nc, th, nn, stream=st)
            other.append((a, b))
    torch.cuda.synchronize(dev)
    ex.check_status(st)                                   # asynchronous calls report overflows here: none in this configuration
    assert torch.equal(m12, m12b) and torch.equal(nm, nmb)
    assert torch.equal(m12, m12c) and torch.equal(nm, nmc)
    assert torch.equal(m12, m12d) and torch.equal(nm, nmd)
    assert torch.equal(idx8[:, :, :4], idx) and torch.equal(dist8[:, :, :4], dist)        # the first four of eight = the four-entry lists
    for a, b in other:
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert len({int(a[1].sum().item()) for a, _ in other} | {int(nm.sum().item())}) >= 4     # the sweep is not vacuous: the rules differ
    for k in ("counts", "kps", "desc", "dmask"):
        assert torch.equal(out[k], ref[k]), k
    # the numpy unpacker reads the same buffer
    per_img = rig.unpack(packed.cpu().numpy(), B, cap, ds)
    counts = out["counts"].cpu().numpy()
    assert [len(p[0]) for p in per_img] == counts.tolist()
    assert redo.sum().item() == 0
    m12, nm = m12.cpu().numpy(), nm.cpu().numpy()
    for img in range(B):
        if img < nc:
            assert nm[img] == 0 and (m12[img] == -1).all()
            continue
        q, d = per_img[img], per_img[img - nc]
        on, om = oa.match_bruteforce(q[1], d[1], 32, 0.9, q[2], d[2])
        assert on == nm[img] and np.array_equal(om, m12[img, :counts[img]])
        # the same pair through the device-resident brute-force entry point
        gn, gm = api.match_bruteforce_device(out["desc"][img, :counts[img]].contiguous(), out["dmask"][img, :counts[img]].contiguous(), None,
                                             out["desc"][img - nc, :counts[img - nc]].contiguous(),
                                             out["dmask"][img - nc, :counts[img - nc]].contiguous(), None, 32, 0.9)
        assert gn == on and np.array_equal(gm, om)
    assert nm.sum() > 1000


def test_bruteforce_batch_equals_separate_calls(api, oa):
    """mcs_match_bruteforce_batch_device: key frames of a batch against one database, each with its own matched-entry state -- the
    same matches as one mcs_match_bruteforce_device call (and the oracle's SearchByBoW(KF1, KF2)) per key frame; the sets share
    database entries on purpose (near-duplicate queries across sets), which a shared state would hand out only once"""
    import torch
    rng = np.random.default_rng(5)
    nd, per, nseg = 3000, 400, 4
    db = rng.integers(0, 256, (nd, 32), dtype=np.uint8)
    dbm = np.packbits(rng.random((nd, 256)) < 0.8, axis=1, bitorder="little")
    base = db[rng.choice(nd, per, replace=False)].copy()
    qs, qms = [], []
    for s in range(nseg):
        q = base.copy()
        for i in range(per):
            for b in rng.choice(256, rng.integers(0, 25), replace=False):
                q[i, b // 8] ^= 1 << (b % 8)
        qs.append(q)
        qms.append(np.packbits(rng.random((per, 256)) < 0.7, axis=1, bitorder="little"))
    q, qm = np.concatenate(qs), np.concatenate(qms)
    valid1 = (rng.random(len(q)) < 0.9).astype(np.uint8)
    valid2 = (rng.random(nd) < 0.95).astype(np.uint8)
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(a).to(dev)
    seg = np.arange(nseg + 1) * per
    nms, m12 = api.match_bruteforce_batch_device(t(q), t(qm), valid1, seg, t(db), t(dbm), valid2, 60, 0.8)
    total = 0
    for s in range(nseg):
        sl = slice(seg[s], seg[s + 1])
        n1, m1 = api.match_bruteforce_device(t(q[sl]), t(qm[sl]), valid1[sl], t(db), t(dbm), valid2, 60, 0.8)
        on, om = oa.match_bruteforce(q[sl], db, 60, 0.8, qm[sl], dbm, valid1[sl], valid2)
        assert n1 == on == nms[s] and np.array_equal(m1, om) and np.array_equal(m12[sl], om)
        total += on
    assert total > 0.5 * valid1.sum()
    # a single shared state would differ: the sets compete for the same planted entries
    n_shared, _ = api.match_bruteforce_device(t(q), t(qm), valid1, t(db), t(dbm), valid2, 60, 0.8)
    assert n_shared < total


def test_bruteforce_large_database_cooperative_rescans(api, oa):
    """a database large enough (>= 32768 entries) for the acceptance kernel to spread every rescan over helper CTAs; the data is
    built so that rescans happen: every query set holds clusters of near-identical queries and the database 12 near copies of each
    cluster centre, so the 8-entry lists of later cluster members are used up by the earlier ones"""
    import torch
    rng = np.random.default_rng(11)
    nd, nseg, ncl, per_cl = 40000, 3, 60, 6
    centres = rng.integers(0, 256, (ncl, 32), dtype=np.uint8)

    def near(src, kmax):
        out = src.copy()
        for i in range(len(out)):
            for b in rng.choice(256, rng.integers(0, kmax + 1), replace=False):
                out[i, b // 8] ^= 1 << (b % 8)
        return out
    db = rng.integers(0, 256, (nd, 32), dtype=np.uint8)
    slots = rng.choice(nd, ncl * 12, replace=False)
    db[slots] = near(np.repeat(centres, 12, axis=0), 10)
    dbm = np.packbits(rng.random((nd, 256)) < 0.9, axis=1, bitorder="little")
    qs = [near(np.repeat(centres, per_cl, axis=0)[rng.permutation(ncl * per_cl)], 8) for _ in range(nseg)]
    q = np.concatenate(qs)
    qm = np.packbits(rng.random((len(q), 256)) < 0.9, axis=1, bitorder="little")
    valid2 = (rng.random(nd) < 0.97).astype(np.uint8)
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(a).to(dev)
    seg = np.arange(nseg + 1) * (ncl * per_cl)
    # a permissive ratio so that cluster members keep taking entries (the strict 0.9 would reject most of them as ambiguous)
    nms, m12 = api.match_bruteforce_batch_device(t(q), t(qm), None, seg, t(db), t(dbm), valid2, 40, 1.01)
    for s in range(nseg):
        sl = slice(seg[s], seg[s + 1])
        on, om = oa.match_bruteforce(q[sl], db, 40, 1.01, qm[sl], dbm, None, valid2)
        assert on == nms[s] and np.array_equal(m12[sl], om)
        assert on > 0.8 * (seg[s + 1] - seg[s])


@pytest.mark.parametrize("masked", [True, False])
def test_stream_greedy_clustered_descriptors(api, oa, masked):
    """mcs_match_stream_greedy_device on clustered descriptors -- dozens of near-duplicates per query, i.e. K-best lists that are
    exhausted by earlier queries and force the exact in-kernel rescan all the time: same matches as the reference's sequential
    SearchByBoW(KF1, KF2) (oracle), and as the separate lists + replay calls with a different list length."""
    import torch
    rng = np.random.default_rng(5)
    F, nc, cap, ds = 3, 2, 700, 32
    B = F * nc
    desc = np.zeros((B, cap, ds), np.uint8)
    dmask = np.zeros((B, cap, ds), np.uint8)
    counts = np.array([640, 700, 655, 690, 700, 610], np.int32)
    centres = rng.integers(0, 256, (12, ds), dtype=np.uint8)
    for b in range(B):
        n = counts[b]
        # 8 big clusters (60+ members each), 4 small ones (<= 20 members), the rest unrelated
        which = rng.choice(13, n, p=[0.09] * 8 + [0.025] * 4 + [0.18])
        base = np.where((which < 12)[:, None], centres[np.minimum(which, 11)], rng.integers(0, 256, (n, ds), dtype=np.uint8))
        flips = np.zeros((n, ds * 8), np.uint8)
        for i in range(n):
            flips[i, rng.choice(ds * 8, rng.integers(0, 14), replace=False)] = 1
        desc[b, :n] = base ^ np.packbits(flips, axis=1, bitorder="little")
        dmask[b, :n] = rng.integers(0, 256, (n, ds), dtype=np.uint8) | rng.integers(0, 256, (n, ds), dtype=np.uint8)
    dev = torch.device("cuda", 0)
    d_t, m_t, c_t = torch.from_numpy(desc).to(dev), torch.from_numpy(dmask).to(dev) if masked else None, torch.from_numpy(counts).to(dev)
    for th, nn in ((32, 0.9), (20, 0.99), (40, 0.7)):
        m12, nm = api.match_stream_greedy_device(d_t, m_t, c_t, F, nc, th, nn)
        idx, dist = api.match_stream_device(d_t, m_t, c_t, F, nc, K=3)
        m12l, nml, _ = api.match_stream_replay_device(idx, dist, c_t, d_t, m_t, F, nc, th, nn)
        torch.cuda.synchronize(dev)
        assert torch.equal(m12, m12l) and torch.equal(nm, nml), (th, nn)
        m12, nm = m12.cpu().numpy(), nm.cpu().numpy()
        for img in range(nc, B):
            q, d = slice(0, counts[img]), slice(0, counts[img - nc])
            on, om = oa.match_bruteforce(desc[img, q], desc[img - nc, d], th, nn, dmask[img, q] if masked else None,
                                         dmask[img - nc, d] if masked else None)
            assert on == nm[img] and np.array_equal(om, m12[img, :counts[img]]), (th, nn, img)
        assert nm.sum() > 30
