"""GPU: the grid-window searches and the device SearchByProjection at descriptor sizes 16, 32 and 64, masked and unmasked, on
natural frames (mdBRIEFextractorOct(descSize=dim)) and on the edge scenes of tests/test_window_edges_cpu.py (window borders to the
float ulp, cell borders, windows off the image, half-cell keypoints, crowded cells, mixed camera sizes, a camera without
keypoints), which pins the oracle against the reference on those scenes.  Every comparison with the oracle is exact."""
import re

import numpy as np
import pytest

import acceptance_model as am
from device_frames import flip, on_device, per_cam, sizes
from device_searches import device_projection
from match_scenes import random_rig
from window_edge_scenes import EMPTY_CAM, SF, edge_scene, projection_scene, second_frame

pytestmark = pytest.mark.gpu

DIMS = [16, 32, 64]
KINDS = ["exact", "mixed"]
width = pytest.mark.parametrize("dim", DIMS)
masking = pytest.mark.parametrize("masked", [False, True])


def _extractor_frames(api, cams, dim, masked, seed, nf=600):
    """two consecutive frames of the sliding-texture stream (3 cameras 754x480) extracted at descriptor size dim"""
    from multicol_slam_b200 import synth
    ex = api.mdBRIEFextractorOct(nfeatures=nf, do_dBrief=True, learnMasks=masked, descSize=dim)
    sf = [ex.info.scale_factor[l] for l in range(8)]
    out = []
    for t in range(2):
        per = [ex(synth.texture_stream(cams[c], 2, seed=seed + c)[t], synth.mirror_mask(cams[c]), cams[c]) for c in range(3)]
        out.append(api.Frame.from_cameras(per, [(754, 480)] * 3, sf))
    assert out[0].desc.shape[1] == dim
    return out


_NATURAL = {}


def natural(api, cams, dim, masked):
    key = (dim, masked)
    if key not in _NATURAL:
        _NATURAL[key] = _extractor_frames(api, cams, dim, masked, seed=60 + dim)
    return _NATURAL[key]


def _random_queries(rng, F, nq):
    from multicol_slam_b200.ctypes_defs import WINDOW_QUERY_DTYPE
    qs = np.zeros(nq, WINDOW_QUERY_DTYPE)
    qs["cam"] = rng.integers(0, len(F.cam_w), nq)
    lv = rng.integers(0, 8, nq)
    kind = rng.integers(0, 3, nq)
    qs["min_level"] = np.where(kind == 0, -1, np.where(kind == 1, lv, lv - 1))
    qs["max_level"] = np.where(kind == 0, -1, lv)
    qs["desc_index"] = rng.integers(0, len(F.keys), nq)
    qs["x"] = rng.uniform(-30, 790, nq); qs["y"] = rng.uniform(-30, 510, nq); qs["r"] = rng.uniform(1, 60, nq)
    return qs


def _window_cases(api, cams, dim, masked):
    """(frame, queries, qdesc, qmask) of both edge scenes and of a natural frame"""
    out = []
    for kind in KINDS:
        sc = edge_scene(kind, dim)
        out.append((sc.frame, sc.queries, sc.qdesc, sc.qmask if masked else None))
    F = natural(api, cams, dim, masked)[0]
    out.append((F, _random_queries(np.random.default_rng(dim), F, 600), F.desc, F.dmask if masked else None))
    return out


@width
@masking
def test_window_search_lists_and_overflow(api, oa, cams, dim, masked):
    """mcs_window_search: candidate lists, distances and counts; with short lists the MCS_ERR_CAPACITY report, the true counts and
    the first max_cand entries"""
    longest = 0
    for F, q, qd, qm in _window_cases(api, cams, dim, masked):
        gi, gd, gc, rc = api.window_search(F, q, qd, qm, max_cand=4096)
        oi, od, oc, orc = oa.window_search(F, q, qd, qm, max_cand=4096)
        assert rc == 0 and orc == 0 and np.array_equal(gc, oc)
        for i in range(len(q)):
            assert np.array_equal(gi[i, :gc[i]], oi[i, :oc[i]]) and np.array_equal(gd[i, :gc[i]], od[i, :oc[i]]), i
        longest = max(longest, int(gc.max()))
        mc = 33
        gi2, gd2, gc2, rc2 = api.window_search(F, q, qd, qm, max_cand=mc)
        assert rc2 == api.MCS_ERR_CAPACITY and np.array_equal(gc2, oc)
        n = np.minimum(oc, mc)
        for i in range(len(q)):
            assert np.array_equal(gi2[i, :n[i]], oi[i, :n[i]]) and np.array_equal(gd2[i, :n[i]], od[i, :n[i]])
    assert longest > 64                                     # the crowded cells: more than two 32-wide chunks in one cell


@pytest.mark.parametrize("kind", KINDS)
def test_frame_prepare_on_edge_keypoints(api, oa, kind):
    """rays and CSR grid of the edge keypoints (half-cell ties, column 64 / row 48, left of the image), mixed camera sizes and an
    empty camera included"""
    sc = edge_scene(kind, 32)
    g = api.frame_prepare(sc.frame.keys, sc.frame.key_cam, sc.cams)
    o = oa.frame_prepare(sc.frame.keys, sc.frame.key_cam, sc.cams)
    assert np.array_equal(g[0].view(np.uint64), o[0].view(np.uint64))
    assert np.array_equal(g[1], o[1]) and np.array_equal(g[2], o[2])
    assert len(g[2]) < len(sc.frame.keys)


def _same_with(monkeypatch, api, oa, fn):
    """fn() through the CUDA mcs_search_windows and through the oracle's, as the cORBmatcher wrappers call it"""
    got = fn()
    with monkeypatch.context() as mp:
        mp.setattr(api, "search_windows", oa.search_windows)
        want = fn()
    return got, want


@width
@masking
def test_search_windows_every_rule(api, oa, cams, monkeypatch, dim, masked):
    """mcs_search_windows under RATIO (WindowSearch, SearchByProjection(F1, F2)), BEST (SearchByProjection(Current, Last)),
    LEVEL_RATIO, BEST_FREE / FIRST_FREE (Fuse cores) and SCW, on natural frames and the edge scenes"""
    from multicol_slam_b200.api import RULE_LEVEL_RATIO, _queries
    m = api.cORBmatcher(0.8, False, dim, masked)
    F1n, F2n = natural(api, cams, dim, masked)
    sc = edge_scene("mixed", dim)
    pairs = [(F1n, F2n), (sc.frame, second_frame(sc.frame, 10.0, seed=dim))]
    rng = np.random.default_rng(dim + masked)
    for F1, F2 in pairs:
        n1, nc = len(F1.keys), len(F2.cam_w)
        valid1 = (rng.random(n1) < 0.8).astype(np.uint8)
        lv = F1.keys["octave"]
        g, o = _same_with(monkeypatch, api, oa, lambda: m.WindowSearch(F1, F2, 10, valid1, 0, 5))
        assert g[0] == o[0] and np.array_equal(g[1], o[1]) and g[0] > 30
        uv = np.zeros((n1, nc, 2))
        in_mask = np.zeros((n1, nc), np.uint8)
        for c in range(nc):
            uv[:, c, 0] = F1.keys["x"] + rng.normal(0, 1, n1); uv[:, c, 1] = F1.keys["y"] + rng.normal(0, 1, n1)
            in_mask[:, c] = (F1.key_cam == c) | (rng.random(n1) < 0.1)
        pre = np.full(len(F2.keys), -1, np.int32)
        pre[::7] = 0
        g, o = _same_with(monkeypatch, api, oa, lambda: m.SearchByProjectionFrames(F1, F2, 12, valid1, uv, in_mask, pre.copy()))
        assert g[0] == o[0] and np.array_equal(g[1], o[1]) and g[0] > 30
        uvl = np.stack([F1.keys["x"], F1.keys["y"]], axis=1).astype(np.float64)
        g, o = _same_with(monkeypatch, api, oa, lambda: m.SearchByProjectionLast(F2, F1, 5.0, valid1, uvl, valid1))
        assert g[0] == o[0] and np.array_equal(g[1], o[1]) and g[0] > 30
        sel = np.flatnonzero(valid1)
        q = _queries(F1.key_cam[sel], uvl[sel, 0], uvl[sel, 1], 4.0 * F2.scale_factors[lv[sel]], lv[sel] - 1, lv[sel], sel)
        qm = F1.dmask if masked else None
        start = np.full(len(F2.keys), -1, np.int32)
        gn, ga = api.search_windows(F2, q, F1.desc, qm, sel, RULE_LEVEL_RATIO, 0.8, m.TH_HIGH_, start.copy())
        on, oa_ = oa.search_windows(F2, q, F1.desc, qm, sel, RULE_LEVEL_RATIO, 0.8, m.TH_HIGH_, start.copy())
        assert gn == on and np.array_equal(ga, oa_) and gn > 30
        level = np.clip(lv[:, None] + rng.integers(0, 2, (n1, nc)), 0, 7)
        for first in (False, True):
            g, o = _same_with(monkeypatch, api, oa, lambda: m.FuseCandidates(F2, uv, in_mask, level, 2.5, F1.desc, F1.dmask, first_wins=first))
            assert np.array_equal(g, o) and (g >= 0).sum() > 30
        matched = np.full(len(F2.keys), -1, np.int32)
        matched[rng.choice(len(F2.keys), 30, replace=False)] = 5
        qcam = np.minimum(F1.key_cam, nc - 1)
        g, o = _same_with(monkeypatch, api, oa, lambda: m.SearchByProjectionScw(F2, qcam, uvl, np.clip(lv, 0, 7), 4.0, valid1, F1.desc,
                                                                               F1.dmask, matched.copy()))
        assert g[0] == o[0] and np.array_equal(g[1], o[1]) and g[0] > 5


@width
@masking
def test_host_projection_searches(api, oa, cams, dim, masked):
    """SearchByProjection(F, MapPoints, th) at th 3 and 1, with and without pre-assigned keypoints, and SearchForInitialization,
    on both edge scenes and natural frames"""
    m = api.cORBmatcher(0.8, False, dim, masked)
    frames = [edge_scene(k, dim).frame for k in KINDS] + [natural(api, cams, dim, masked)[0]]
    for j, F in enumerate(frames):
        mps = projection_scene(F, dim, masked, seed=dim + j) if j < 2 else _natural_mappoints(api, F, dim, masked, seed=dim)
        pre = np.where(np.arange(len(F.keys)) % 3 == 0, 0, -1).astype(np.int32)
        for th, start in ((3.0, None), (1.0, pre), (3.0, pre)):
            n, fmp = m.SearchByProjection(F, mps, th, None if start is None else start.copy())
            on, ofmp = oa.search_by_projection(F, mps, th, 0.8, m.TH_HIGH_, masked, None if start is None else start.copy())
            assert n == on and np.array_equal(fmp, ofmp) and n > 50
        F2 = second_frame(F, 10.0, seed=dim + 5)
        prev = np.stack([F.keys["x"], F.keys["y"]], axis=1).astype(np.float64)
        for window in (10, 40):
            p1 = prev.copy()
            n, m12 = m.SearchForInitialization(F, F2, p1, window)
            on, om12, oprev = oa.search_for_initialization(F, F2, prev, window, m.mfNNratio, m.TH_LOW_, masked)
            assert n == on and np.array_equal(m12, om12) and np.array_equal(p1, oprev) and n > 50


def _natural_mappoints(api, F, dim, masked, seed, nmp=3000):
    rng = np.random.default_rng(seed)
    nc = len(F.cam_w)
    src = rng.integers(0, len(F.keys), nmp)
    desc = np.stack([flip(rng, F.desc[s], int(rng.integers(0, dim + 1))) for s in src])
    in_view = np.zeros((nmp, nc), np.uint8); level = np.zeros((nmp, nc), np.int32)
    px = np.zeros((nmp, nc)); py = np.zeros((nmp, nc)); vc = np.zeros((nmp, nc))
    r, c = np.arange(nmp), F.key_cam[src]
    in_view[r, c] = 1
    level[r, c] = np.clip(F.keys["octave"][src] + rng.integers(-1, 2, nmp), 0, 7)
    px[r, c] = F.keys["x"][src] + rng.normal(0, 2, nmp); py[r, c] = F.keys["y"][src] + rng.normal(0, 2, nmp)
    vc[r, c] = rng.uniform(0.9, 1.0, nmp)
    return api.MapPoints((rng.random(nmp) < 0.05).astype(np.uint8), in_view, level, px, py, vc, desc, F.dmask[src].copy() if masked else None)


@width
@masking
def test_search_for_triangulation_paging(api, oa, cams, dim, masked):
    """SearchForTriangulationRaw with more than 8 candidates inside both thresholds for some queries (the paged candidate lists)"""
    rng = np.random.default_rng(21 + dim)
    F1, F2 = natural(api, cams, dim, masked)

    def rays(F):
        return np.stack([api.img_to_world(cams[F.key_cam[i]], float(k["x"]), float(k["y"])) for i, k in enumerate(F.keys)])
    r1, r2 = rays(F1), rays(F2)
    t = np.array([1.0, 0.1, 0.0]); t /= np.linalg.norm(t)
    E = np.tile(np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]]), (3, 3, 1, 1))
    free1 = (rng.random(len(F1.keys)) < 0.7).astype(np.uint8)
    free2 = (rng.random(len(F2.keys)) < 0.7).astype(np.uint8)
    d2 = F2.desc.copy()
    for q, at in ((50, 0), (51, 40)):                       # 40 near copies of two queries in the same camera: > 8 candidates each
        same_cam = np.flatnonzero(F2.key_cam == F1.key_cam[q])[at:at + 40]
        d2[same_cam] = F1.desc[q]
        d2[same_cam, 1] ^= rng.integers(0, 4, len(same_cam)).astype(np.uint8)
        free1[q] = 1
        free2[same_cam] = 1
    m = api.cORBmatcher(0.8, False, dim, masked)
    for thr in (1e-2, 1e-4):
        n, m12 = m.SearchForTriangulationRaw(F1.desc, F1.dmask, F1.key_cam, free1, r1, d2, F2.dmask, F2.key_cam, free2, r2, E, thr)
        on, om12 = oa.search_for_triangulation(F1.desc, F1.dmask if masked else None, F1.key_cam, free1, r1, d2, F2.dmask if masked else None,
                                               F2.key_cam, free2, r2, E, m.TH_LOW_, thr)
        assert n == on and np.array_equal(m12, om12)
    assert n > 10


def _featvec(rng, n, n_nodes):
    """a hand-built CSR feature vector: keypoint -> node, skewed so that the first nodes hold more than 32 keypoints"""
    node = np.minimum(rng.geometric(0.12, n) - 1, n_nodes - 1) * 3 + 2        # sparse, increasing node ids
    nodes = np.unique(node)
    features = np.concatenate([np.flatnonzero(node == v) for v in nodes]).astype(np.int32)
    offsets = np.concatenate([[0], np.cumsum([(node == v).sum() for v in nodes])]).astype(np.int32)
    return nodes.astype(np.int32), offsets, features


@width
@masking
def test_search_by_bow_frame_widths(api, oa, dim, masked):
    """SearchByBoW(KF, F) (group_distance_kernel) with hand-built feature vectors: the vocabulary is 32-byte only"""
    rng = np.random.default_rng(3 + dim + masked)
    n1, n2 = 900, 1000
    d1 = rng.integers(0, 256, (n1, dim), dtype=np.uint8)
    src = rng.integers(0, n1, n2)
    d2 = np.stack([flip(rng, d1[s], int(rng.integers(0, dim))) for s in src])
    m1 = rng.integers(0, 256, (n1, dim), dtype=np.uint8) | rng.integers(0, 256, (n1, dim), dtype=np.uint8)
    m2 = rng.integers(0, 256, (n2, dim), dtype=np.uint8) | rng.integers(0, 256, (n2, dim), dtype=np.uint8)
    fv1 = _featvec(rng, n1, 30)
    node1 = np.empty(n1, np.int32)
    for k in range(len(fv1[0])):
        node1[fv1[2][fv1[1][k]:fv1[1][k + 1]]] = fv1[0][k]
    node2 = np.where(rng.random(n2) < 0.8, node1[src], rng.choice(fv1[0], n2))              # mostly the node of the source keypoint
    nodes2 = np.unique(node2)
    fv2 = (nodes2.astype(np.int32), np.concatenate([[0], np.cumsum([(node2 == v).sum() for v in nodes2])]).astype(np.int32),
           np.concatenate([np.flatnonzero(node2 == v) for v in nodes2]).astype(np.int32))
    assert np.diff(fv1[1]).max() > 64 and np.diff(fv2[1]).max() > 64
    valid1 = (rng.random(n1) < 0.9).astype(np.uint8)
    m = api.cORBmatcher(0.7, False, dim, masked)
    n, out = m.SearchByBoWFrame(d1, fv1, d2, fv2, m1, m2, valid1)
    on, oout = oa.search_by_bow(d1, m1 if masked else None, valid1, fv1, d2, m2 if masked else None, fv2, m.TH_LOW_, 0.7)
    assert n == on and np.array_equal(out, oout) and n > 100


# ---- device SearchByProjection --------------------------------------------------------------------------------------------------
@width
@masking
@pytest.mark.parametrize("layout", ["single", "parts"])
def test_device_search_on_edge_scenes(api, oa, dim, masked, layout):
    """mcs_search_by_projection_device on both edge scenes (mixed sizes, crowded cells, the camera without keypoints, whose slots
    must come back untouched) == the host call == the oracle; capacities that are not a multiple of 32"""
    m = api.cORBmatcher(0.8, False, dim, masked)
    for j, kind in enumerate(KINDS):
        sc = edge_scene(kind, dim)
        F = sc.frame
        mps = projection_scene(F, dim, masked, seed=dim + j)
        per = per_cam(F)
        assert len(per[EMPTY_CAM][0]) == 0
        cap = max(len(p[0]) for p in per) + 7 + 10 * j
        assert cap % 32 != 0
        pre = np.where(np.arange(len(F.keys)) % 4 == 0, 0, -1).astype(np.int32)
        for th, start in ((3.0, None), (1.0, pre)):
            s = None if start is None else start.copy()
            n, fmp = m.SearchByProjection(F, mps, th, s)
            on, ofmp = oa.search_by_projection(F, mps, th, 0.8, m.TH_HIGH_, masked, None if start is None else start.copy())
            gn, gfmp, status, diag = device_projection(api, m, per, sizes(F), F.scale_factors, mps, th,
                                                    pre=None if start is None else start.copy(), layout=layout, cap=cap)
            assert status == api.MCS_OK and n == on == gn and np.array_equal(fmp, ofmp) and np.array_equal(gfmp, fmp)
            assert n > 100 and diag[2] == int(((mps.in_view != 0) & (mps.bad[:, None] == 0)).sum())


@width
@masking
def test_device_search_from_the_extractor(api, oa, cams, dim, masked):
    """the frame is the packed buffer the extractor wrote at descriptor size dim (packed_layout(..., dim))"""
    import torch
    from multicol_slam_b200 import rig, synth
    ex = api.mdBRIEFextractorOct(nfeatures=1200, do_dBrief=True, learnMasks=masked, descSize=dim)
    imgs = on_device(np.stack([synth.frame(cams[c], 400 + c) for c in range(3)]))
    mk = np.stack([synth.mirror_mask(c) for c in cams])
    cap = ex.capacity
    packed = torch.zeros(rig.packed_layout(3, cap, dim)[1], dtype=torch.uint8, device="cuda")
    v = ex.extract_batch_packed_device(imgs, mk, cams, [0, 1, 2], packed)
    torch.cuda.synchronize()
    counts = v["counts"].cpu().numpy()
    kps = v["kps"].cpu().numpy().view(api.KEYPOINT_DTYPE).reshape(3, cap)
    per = [(kps[c, :counts[c]], v["desc"][c, :counts[c]].cpu().numpy(), v["dmask"][c, :counts[c]].cpu().numpy()) for c in range(3)]
    sf = [ex.info.scale_factor[l] for l in range(8)]
    F = api.Frame.from_cameras(per, [(754, 480)] * 3, sf)
    assert F.desc.shape[1] == dim
    mps = _natural_mappoints(api, F, dim, masked, seed=dim, nmp=6000)
    m = api.cORBmatcher(0.8, False, dim, masked)
    n, fmp = m.SearchByProjection(F, mps, 3.0)
    on, ofmp = oa.search_by_projection(F, mps, 3.0, 0.8, m.TH_HIGH_, masked)
    assert n == on and np.array_equal(fmp, ofmp) and n > 500
    fm_t = torch.full((3 * cap,), -1, dtype=torch.int32, device="cuda")
    gn, st, fm_t = m.SearchByProjectionDevice(packed, 1, 3, 0, 3, cap, [(754, 480)] * 3, sf, api.MapPointsDevice.from_host(mps, packed.device),
                                              3.0, fm_t)
    torch.cuda.synchronize()
    assert int(st.item()) == api.MCS_OK and int(gn.item()) == n
    assert np.array_equal(api.slots_to_contiguous(fm_t.cpu().numpy(), counts, cap), fmp)


@width
def test_device_projection_chain(api, oa, cams, dim):
    """project_mappoints_device -> the device search == project_mappoints -> the host search, at descriptor size dim"""
    from multicol_slam_b200 import synth
    rng = np.random.default_rng(12 + dim)
    n = 15000
    mtmc, inv = random_rig(rng, 3)
    masks = np.stack([synth.mirror_mask(c) for c in cams])
    pos = rng.normal(size=(n, 3)); pos *= (rng.uniform(1.5, 12.0, n) / np.linalg.norm(pos, axis=1))[:, None]
    nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    dmin = rng.uniform(0.5, 4.0, n); dmax = dmin * rng.uniform(1.5, 6.0, n)
    F = natural(api, cams, dim, True)[0]
    sf = F.scale_factors
    g = api.project_mappoints(inv, mtmc, cams, masks, pos, nrm, dmin, dmax, sf)
    d = api.project_mappoints_device(inv, mtmc, cams, on_device(masks), on_device(pos), on_device(nrm), on_device(dmin), on_device(dmax), sf)
    src = rng.integers(0, len(F.keys), n)
    desc, dmask = F.desc[src].copy(), F.dmask[rng.integers(0, len(F.keys), n)].copy()
    m = api.cORBmatcher(0.8, False, dim, True)
    ng, fg = m.SearchByProjection(F, api.MapPoints(np.zeros(n, np.uint8), *g, desc, dmask), 3.0)
    mdev = api.MapPointsDevice(None, *d, on_device(desc), on_device(dmask))
    gn, gf, status, _ = device_projection(api, m, per_cam(F), sizes(F), sf, mdev, 3.0)
    assert status == api.MCS_OK and gn == ng and np.array_equal(gf, fg) and ng > 50


@width
def test_device_long_dependency_chain(api, oa, dim):
    """the chain of test_search_projection_device_gpu.py::test_long_dependency_chains_run_the_walk at descriptor size dim: deeper
    than the round cap, so the walk runs, and windows whose lists are used up, so decisions rescan"""
    rng = np.random.default_rng(5 + dim)
    m = api.cORBmatcher(0.8, False, dim, False)
    nk = min(70, m.TH_HIGH_ - 1)                             # distances 1..nk, all within TH_HIGH
    ntaken = nk // 5
    nmp = nk - ntaken - 4
    W, H = 640, 480
    base = rng.integers(0, 256, dim).astype(np.uint8)
    keys = np.zeros(nk, api.KEYPOINT_DTYPE)
    keys["x"] = rng.uniform(92, 108, nk); keys["y"] = rng.uniform(93, 107, nk)
    kd = np.stack([flip(rng, base, k + 1) for k in rng.permutation(nk)])
    dist = np.array([int(np.unpackbits(base ^ kd[k]).sum()) for k in range(nk)])
    taken0 = np.zeros(nk, bool)
    taken0[rng.choice(nk, ntaken, replace=False)] = True
    free_by_dist = [k for k in np.argsort(dist) if not taken0[k]]
    keys["octave"][free_by_dist] = np.arange(len(free_by_dist)) % 2
    keys["octave"][taken0] = 1
    keys2 = np.zeros(200, api.KEYPOINT_DTYPE)
    keys2["x"] = rng.uniform(20, 620, 200); keys2["y"] = rng.uniform(20, 460, 200); keys2["octave"] = rng.integers(0, 3, 200)
    kd2 = rng.integers(0, 256, (200, dim)).astype(np.uint8)
    F = api.Frame.from_cameras([(keys, kd, None), (keys2, kd2, None)], [(W, H)] * 2, SF)
    n2 = 150
    nall = nmp + n2
    in_view = np.zeros((nall, 2), np.uint8); level = np.zeros((nall, 2), np.int32)
    px = np.zeros((nall, 2)); py = np.zeros((nall, 2)); vc = np.full((nall, 2), 0.9)
    desc = np.zeros((nall, dim), np.uint8)
    chain = np.sort(rng.choice(nall, nmp, replace=False))
    other = np.setdiff1d(np.arange(nall), chain)
    in_view[chain, 0] = 1; level[chain, 0] = 1; px[chain, 0] = 100.0; py[chain, 0] = 100.0; desc[chain] = base
    src = rng.integers(0, 200, n2)
    in_view[other, 1] = 1; level[other, 1] = keys2["octave"][src]
    px[other, 1] = keys2["x"][src] + rng.normal(0, 1, n2); py[other, 1] = keys2["y"][src] + rng.normal(0, 1, n2)
    desc[other] = np.stack([flip(rng, kd2[s], int(rng.integers(0, dim // 2))) for s in src])
    mps = api.MapPoints(np.zeros(nall, np.uint8), in_view, level, px, py, vc, desc, None)
    pre = np.full(len(F.keys), -1, np.int32)
    pre[:nk][taken0] = 7
    n, fmp = m.SearchByProjection(F, mps, 3.0, pre.copy())
    on, ofmp = oa.search_by_projection(F, mps, 3.0, 0.8, m.TH_HIGH_, False, pre.copy())
    assert n == on and np.array_equal(fmp, ofmp) and n >= nmp
    pn, pfmp, pdiag, _ = am.predict_local(api, oa, m, F, mps, 3.0, pre.copy())
    cap_rounds = api.lib().mcs_search_by_projection_max_rounds()
    assert pn == n and np.array_equal(pfmp, fmp) and pdiag[0] == cap_rounds and pdiag[1] >= 0 and pdiag[3] > 0
    for layout in ("single", "parts"):
        gn, gfmp, status, diag = device_projection(api, m, per_cam(F), sizes(F), SF, mps, 3.0, pre=pre.copy(), layout=layout)
        assert status == api.MCS_OK and gn == n and np.array_equal(gfmp, fmp)
        assert diag.tolist() == pdiag


@width
@masking
@pytest.mark.parametrize("n_cand", [8, 9])
@pytest.mark.parametrize("taken", [False, True])
def test_device_list_edge(api, oa, dim, masked, n_cand, taken):
    """one query whose window holds exactly 8 or 9 candidates.  With the 7 nearest taken, 9 candidates leave one free entry in the
    8-entry list, so the decision must rescan the window to find the second best: it sits at the same level, close enough for the
    ratio test to reject the best.  8 candidates are all in the list, which then decides alone."""
    rng = np.random.default_rng(dim + 10 * n_cand + taken)
    base = rng.integers(0, 256, dim).astype(np.uint8)
    dists = [2, 3, 4, 5, 6, 7, 8, 20, 22][:n_cand]
    keys = np.zeros(n_cand + 30, api.KEYPOINT_DTYPE)
    keys["x"][:n_cand] = 300.0 + rng.uniform(-3, 3, n_cand); keys["y"][:n_cand] = 200.0 + rng.uniform(-3, 3, n_cand)
    keys["x"][n_cand:] = rng.uniform(350, 700, 30); keys["y"][n_cand:] = rng.uniform(250, 450, 30)     # far from the window
    keys["octave"] = 1
    perm = rng.permutation(n_cand)                          # visiting order unrelated to distance
    kd = rng.integers(0, 256, (len(keys), dim)).astype(np.uint8)
    for i, k in enumerate(perm):
        kd[k] = flip(rng, base, dists[i])
    full = np.full((len(keys), dim), 0xFF, np.uint8) if masked else None      # full masks: masked distance == Hamming distance
    F = api.Frame.from_cameras([(keys, kd, full)], [(754, 480)], SF)
    mps = api.MapPoints(np.zeros(1, np.uint8), np.ones((1, 1), np.uint8), np.ones((1, 1), np.int32), np.full((1, 1), 300.0),
                        np.full((1, 1), 200.0), np.full((1, 1), 0.95), base[None].copy(), np.full((1, dim), 0xFF, np.uint8) if masked else None)
    m = api.cORBmatcher(0.8, False, dim, masked)
    pre = np.full(len(keys), -1, np.int32)
    if taken:
        pre[perm[:7]] = 3
    n, fmp = m.SearchByProjection(F, mps, 1.0, pre.copy())
    on, ofmp = oa.search_by_projection(F, mps, 1.0, 0.8, m.TH_HIGH_, masked, pre.copy())
    assert n == on and np.array_equal(fmp, ofmp)
    assert n == (0 if (taken and n_cand == 9) else 1)
    gn, gfmp, status, diag = device_projection(api, m, per_cam(F), sizes(F), SF, mps, 1.0, pre=pre.copy())
    assert status == api.MCS_OK and gn == n and np.array_equal(gfmp, fmp)
    assert (diag[3] > 0) == (taken and n_cand == 9)


@width
def test_device_full_capacity_whole_image(api, oa, dim):
    """one camera filled to capacity 65535 and windows covering the whole image: visiting positions reach 65534, the top of the
    key's 16-bit field.  The best candidates are identical pairs in the last cell visited, so the position decides between them."""
    rng = np.random.default_rng(dim)
    cap, W, H = 65535, 754, 480
    cw, ch = W / 64.0, H / 48.0
    keys = np.zeros(cap, api.KEYPOINT_DTYPE)
    keys["x"] = rng.uniform(1, 0.98 * 63.5 * cw, cap); keys["y"] = rng.uniform(1, 0.98 * 47.5 * ch, cap)
    keys["octave"] = 1
    kd = rng.integers(0, 256, (cap, dim), dtype=np.uint8)
    nmp = 24
    last = rng.choice(cap, 2 * nmp, replace=False)          # moved into the last cell (63, 47), pairs with one descriptor
    keys["x"][last] = (63 + rng.uniform(-0.4, 0.4, 2 * nmp)) * cw; keys["y"][last] = (47 + rng.uniform(-0.4, 0.4, 2 * nmp)) * ch
    kd[last[1::2]] = kd[last[0::2]]
    F = api.Frame.from_cameras([(keys, kd, None)], [(W, H)], SF)
    mdesc = kd[last[0::2]].copy()                          # distance 0 to both keypoints of its pair
    th = 200.0                                              # 4 * 200 * 1.2 = 960 px: the whole image
    mps = api.MapPoints(np.zeros(nmp, np.uint8), np.ones((nmp, 1), np.uint8), np.ones((nmp, 1), np.int32), np.full((nmp, 1), W / 2),
                        np.full((nmp, 1), H / 2), np.full((nmp, 1), 0.95), mdesc, None)
    m = api.cORBmatcher(0.8, False, dim, False)
    n, fmp = m.SearchByProjection(F, mps, th)
    on, ofmp = oa.search_by_projection(F, mps, th, 0.8, m.TH_HIGH_, False)
    assert n == on and np.array_equal(fmp, ofmp) and n == nmp
    _, start, items = oa.frame_prepare(F.keys, F.key_cam, _one_cam(W, H))
    assert len(items) == cap and start[-1] == cap
    gn, gfmp, status, diag = device_projection(api, m, per_cam(F), sizes(F), SF, mps, th, cap=cap, first_image=1)
    assert status == api.MCS_OK and gn == n and np.array_equal(gfmp, fmp)


def _one_cam(W, H):
    from multicol_slam_b200 import synth
    return [synth.scaled_cam(synth.lafida_cams()[0], W, H)]


# ---- every instantiation launched ----------------------------------------------------------------------------------------------
# ps_round_kernel / ps_walk_kernel take the acceptance rule first; the local-map search runs MCS_RULE_LEVEL_RATIO (2), and only
# that rule's instantiations match here
_KERNEL = re.compile(r"(window_search_kernel|ps_list_kernel|ps_round_kernel|ps_walk_kernel|group_distance_kernel)<(?:2, )?(\d+), (true|false)>")


def test_every_window_and_level_ratio_instantiation_launched(api):
    """torch.profiler over one small case per width and masking: every instantiation of window_search_kernel, ps_list_kernel,
    ps_round / ps_walk_kernel under MCS_RULE_LEVEL_RATIO and group_distance_kernel was launched"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        # after an earlier profiling session in the process, the first kernel records of this one can go missing: start with
        # launches that are not counted
        warm = torch.zeros(64, device="cuda")
        for _ in range(8):
            warm.add_(1)
        torch.cuda.synchronize()
        for dim in DIMS:
            for masked in (False, True):
                sc = edge_scene("exact", dim)
                F = sc.frame
                api.window_search(F, sc.queries[:64], sc.qdesc, sc.qmask if masked else None, max_cand=4096)
                m = api.cORBmatcher(0.8, False, dim, masked)
                mps = projection_scene(F, dim, masked, seed=1, nmp=200)
                device_projection(api, m, per_cam(F), sizes(F), F.scale_factors, mps, 3.0)
                rng = np.random.default_rng(0)
                d1, d2 = F.desc[:200], F.desc[200:400]
                fv = (np.array([2], np.int32), np.array([0, 200], np.int32), np.arange(200, dtype=np.int32))
                m.SearchByBoWFrame(d1, fv, d2, fv, F.dmask[:200], F.dmask[200:400], (rng.random(200) < 0.9).astype(np.uint8))
        torch.cuda.synchronize()
    seen = set()
    for e in prof.key_averages():
        for k in _KERNEL.finditer(e.key):
            seen.add((k.group(1), int(k.group(2)), k.group(3) == "true"))
    want = {(k, w, msk) for k in ("window_search_kernel", "ps_list_kernel", "ps_round_kernel", "ps_walk_kernel", "group_distance_kernel")
            for w in (4, 8, 16) for msk in (False, True)}
    missing = sorted(want - seen)
    assert not missing, f"never launched: {missing}"
    assert len(want) == 30
