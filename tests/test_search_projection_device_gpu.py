"""GPU: the device-resident SearchByProjection (mcs_project_mappoints_device -> mcs_search_by_projection_device) against the host
entry points and the CPU oracle.  Frames come from packed feature buffers in both layouts (one buffer holding every camera at a
non-zero first image, and one one-image buffer per camera as the allgather leaves them); results are compared after the slot ->
contiguous conversion.  Integer work: bit-exact."""
import numpy as np
import pytest

import acceptance_model as am
from device_frames import flip, on_device, per_cam, sizes
from device_searches import collect, device_projection, launch_projection, projection_inputs
from match_scenes import make_frames, random_rig

pytestmark = pytest.mark.gpu


def _projection_scene(api, cams, masks, seed=2, nmp=4000):
    """the inputs of test_match_gpu.py::test_search_by_projection"""
    F = make_frames(api, None, cams, [4, 5, 6], masks=masks)
    rng = np.random.default_rng(seed)
    nc = 3
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
    return F, api.MapPoints(bad, in_view, level, px, py, vc, desc, dm)


@pytest.mark.parametrize("layout", ["single", "parts"])
@pytest.mark.parametrize("masks", [False, True])
def test_search_by_projection_device_matches_host(api, oa, cams, masks, layout):
    F, mps = _projection_scene(api, cams, masks)
    m = api.cORBmatcher(0.8, False, 32, masks)
    n, fmp = m.SearchByProjection(F, mps, 3.0)
    on, ofmp = oa.search_by_projection(F, mps, 3.0, 0.8, m.TH_HIGH_, masks)
    gn, gfmp, status, diag = device_projection(api, m, per_cam(F), sizes(F), F.scale_factors, mps, 3.0, layout=layout)
    assert status == api.MCS_OK and n == on == gn and np.array_equal(fmp, ofmp) and np.array_equal(gfmp, fmp)
    assert gn > 500 and diag[2] == int(((mps.in_view != 0) & (mps.bad[:, None] == 0)).sum())
    # pre-assigned keypoints are skipped (ref :121), th = 1 keeps the radius unscaled
    pre = np.full(len(F.keys), -1, np.int32)
    pre[::3] = 0
    n2, fmp2 = m.SearchByProjection(F, mps, 1.0, pre.copy())
    on2, ofmp2 = oa.search_by_projection(F, mps, 1.0, 0.8, m.TH_HIGH_, masks, pre.copy())
    gn2, gfmp2, status2, _ = device_projection(api, m, per_cam(F), sizes(F), F.scale_factors, mps, 1.0, pre=pre.copy(), layout=layout,
                                            first_image=1)
    assert status2 == api.MCS_OK and n2 == on2 == gn2 and np.array_equal(fmp2, ofmp2) and np.array_equal(gfmp2, fmp2)


def test_config3_size_from_the_extractor(api, oa, cams):
    """BASELINE config 3 size: 4 cameras 1280x720, 2000 features each, 50 000 map points; the frame is the packed buffer the
    extractor wrote on the device."""
    import torch
    from multicol_slam_b200 import synth
    cam4 = [synth.scaled_cam(cams[i % 3], 1280, 720) for i in range(4)]
    ex = api.mdBRIEFextractorOct(nfeatures=2000, do_dBrief=True, learnMasks=True)
    imgs = on_device(np.stack([synth.frame(cam4[c], 300 + c) for c in range(4)]))
    mk = np.stack([synth.mirror_mask(c) for c in cam4])
    from multicol_slam_b200 import rig
    cap = ex.capacity
    packed = torch.zeros(rig.packed_layout(4, cap, 32)[1], dtype=torch.uint8, device="cuda")
    v = ex.extract_batch_packed_device(imgs, mk, cam4, [0, 1, 2, 3], packed)
    torch.cuda.synchronize()
    counts = v["counts"].cpu().numpy()
    kps = v["kps"].cpu().numpy().view(api.KEYPOINT_DTYPE).reshape(4, cap)
    per = [(kps[c, :counts[c]], v["desc"][c, :counts[c]].cpu().numpy(), v["dmask"][c, :counts[c]].cpu().numpy()) for c in range(4)]
    sf = [ex.info.scale_factor[l] for l in range(8)]
    F = api.Frame.from_cameras(per, [(1280, 720)] * 4, sf)
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
    m = api.cORBmatcher(0.8, False, 32, True)
    n, fmp = m.SearchByProjection(F, mps, 3.0)
    on, ofmp = oa.search_by_projection(F, mps, 3.0, 0.8, m.TH_HIGH_, True)
    assert n == on and np.array_equal(fmp, ofmp) and n > 2000
    fm_t = torch.full((4 * cap,), -1, dtype=torch.int32, device="cuda")
    gn, st, fm_t = m.SearchByProjectionDevice(packed, 1, 4, 0, 4, cap, [(1280, 720)] * 4, sf, api.MapPointsDevice.from_host(mps, packed.device),
                                              3.0, fm_t)
    torch.cuda.synchronize()
    assert int(st.item()) == api.MCS_OK and int(gn.item()) == n
    assert np.array_equal(api.slots_to_contiguous(fm_t.cpu().numpy(), counts, cap), fmp)


def test_project_device_then_search_device(api, oa, cams):
    """the chain mcs_project_mappoints_device -> mcs_search_by_projection_device against project_mappoints -> SearchByProjection,
    and skip_dev leaving the flagged points' entries untouched"""
    import torch
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
    masks_t, pos_t, nrm_t, dmin_t, dmax_t = on_device(masks), on_device(pos), on_device(nrm), on_device(dmin), on_device(dmax)
    d = api.project_mappoints_device(inv, mtmc, cams, masks_t, pos_t, nrm_t, dmin_t, dmax_t, sf)
    torch.cuda.synchronize()
    for a, b in zip(g, d):
        assert np.array_equal(a, b.cpu().numpy())                 # same kernel, same arithmetic: every output identical
    # skip: flagged points keep what the output arrays held before the call
    skip = (rng.random(n) < 0.3).astype(np.uint8)
    before = [x.clone() for x in d]
    mt2, inv2 = random_rig(rng, nc)
    d2 = api.project_mappoints_device(inv2, mt2, cams, masks_t, pos_t, nrm_t, dmin_t, dmax_t, sf, skip_t=on_device(skip), out=d)
    g2 = api.project_mappoints(inv2, mt2, cams, masks, pos, nrm, dmin, dmax, sf)
    torch.cuda.synchronize()
    for a, b, o in zip(g2, d2, before):
        b, o = b.cpu().numpy(), o.cpu().numpy()
        assert np.array_equal(b[skip != 0], o[skip != 0]) and np.array_equal(b[skip == 0], a[skip == 0])
    # the search on top of the device projection
    ex = api.mdBRIEFextractorOct(nfeatures=1000, do_dBrief=True, learnMasks=True)
    per = [ex(synth.frame(cams[c], 200 + c), masks[c], cams[c]) for c in range(3)]
    F = api.Frame.from_cameras(per, [(754, 480)] * 3, [ex.info.scale_factor[l] for l in range(8)])
    desc = F.desc[rng.integers(0, len(F.keys), n)].copy()
    dmask = F.dmask[rng.integers(0, len(F.keys), n)].copy()
    mps_h = api.MapPoints(np.zeros(n, np.uint8), g[0], g[1], g[2], g[3], g[4], desc, dmask)
    m = api.cORBmatcher(0.8, False, 32, True)
    ng, fg = m.SearchByProjection(F, mps_h, 3.0)
    mdev = api.MapPointsDevice(None, *d_fresh(api, inv, mtmc, cams, masks_t, pos_t, nrm_t, dmin_t, dmax_t, sf), on_device(desc), on_device(dmask))
    gn, gf, status, _ = device_projection(api, m, per_cam(F), sizes(F), F.scale_factors, mdev, 3.0)
    assert status == api.MCS_OK and gn == ng and np.array_equal(gf, fg) and ng > 100


def d_fresh(api, inv, mtmc, cams, masks_t, pos_t, nrm_t, dmin_t, dmax_t, sf):
    return api.project_mappoints_device(inv, mtmc, cams, masks_t, pos_t, nrm_t, dmin_t, dmax_t, sf)


def test_long_dependency_chains_run_the_walk(api, oa):
    """Many map points share one window whose keypoints lie at strictly increasing distance with alternating octaves: every
    acceptance moves every later query to the next keypoint, so the chain is deeper than the round cap and the sequential walk
    finishes it; the windows hold more than K candidates with most of them taken, so the decisions rescan their windows."""
    rng = np.random.default_rng(5)
    W, H, nk, nmp, dim = 640, 480, 70, 48, 32
    base = rng.integers(0, 256, dim).astype(np.uint8)
    keys = np.zeros(nk, api.KEYPOINT_DTYPE)
    keys["x"] = rng.uniform(92, 108, nk)                 # spread over several grid cells: visiting order != index order
    keys["y"] = rng.uniform(93, 107, nk)
    kd = np.stack([flip(rng, base, k + 1) for k in rng.permutation(nk)])       # distance to `base` = k + 1, in shuffled order
    dist = np.array([int(np.unpackbits(base ^ kd[k]).sum()) for k in range(nk)])
    taken0 = np.zeros(nk, bool)
    taken0[rng.choice(nk, 14, replace=False)] = True     # keypoints of the chain taken on entry
    # levels alternate along the free keypoints in distance order: best and second best always differ, the ratio test never applies
    free_by_dist = [k for k in np.argsort(dist) if not taken0[k]]
    keys["octave"][free_by_dist] = np.arange(len(free_by_dist)) % 2
    keys["octave"][taken0] = 1
    # a second camera with an ordinary scene so that independent chains run side by side
    keys2 = np.zeros(200, api.KEYPOINT_DTYPE)
    keys2["x"] = rng.uniform(20, 620, 200); keys2["y"] = rng.uniform(20, 460, 200); keys2["octave"] = rng.integers(0, 3, 200)
    kd2 = rng.integers(0, 256, (200, dim)).astype(np.uint8)
    sf = np.cumprod([1.0] + [1.2000000476837158] * 7)
    F = api.Frame.from_cameras([(keys, kd, None), (keys2, kd2, None)], [(W, H)] * 2, sf)
    n2 = 150
    nall = nmp + n2
    in_view = np.zeros((nall, 2), np.uint8); level = np.zeros((nall, 2), np.int32)
    px = np.zeros((nall, 2)); py = np.zeros((nall, 2)); vc = np.full((nall, 2), 0.9)
    desc = np.zeros((nall, dim), np.uint8)
    # interleave the chain's points with the second camera's so that both chains share the query order
    chain = np.sort(rng.choice(nall, nmp, replace=False))
    other = np.setdiff1d(np.arange(nall), chain)
    in_view[chain, 0] = 1; level[chain, 0] = 1; px[chain, 0] = 100.0; py[chain, 0] = 100.0; desc[chain] = base
    src = rng.integers(0, 200, n2)
    in_view[other, 1] = 1; level[other, 1] = keys2["octave"][src]
    px[other, 1] = keys2["x"][src] + rng.normal(0, 1, n2); py[other, 1] = keys2["y"][src] + rng.normal(0, 1, n2)
    desc[other] = np.stack([flip(rng, kd2[s], int(rng.integers(0, 20))) for s in src])
    mps = api.MapPoints(np.zeros(nall, np.uint8), in_view, level, px, py, vc, desc, None)
    m = api.cORBmatcher(0.8, False, dim, False)
    pre = np.full(len(F.keys), -1, np.int32)
    pre[:nk][taken0] = 7
    n, fmp = m.SearchByProjection(F, mps, 3.0, pre.copy())
    on, ofmp = oa.search_by_projection(F, mps, 3.0, 0.8, m.TH_HIGH_, False, pre.copy())
    assert n == on and np.array_equal(fmp, ofmp) and n >= nmp
    pn, pfmp, pdiag, _ = am.predict_local(api, oa, m, F, mps, 3.0, pre.copy())
    cap_rounds = api.lib().mcs_search_by_projection_max_rounds()
    assert pn == n and np.array_equal(pfmp, fmp) and pdiag[0] == cap_rounds and pdiag[1] >= 0 and pdiag[3] > 0
    for layout in ("single", "parts"):
        gn, gfmp, status, diag = device_projection(api, m, per_cam(F), sizes(F), sf, mps, 3.0, pre=pre.copy(), layout=layout)
        assert status == api.MCS_OK and gn == n and np.array_equal(gfmp, fmp)
        assert diag.tolist() == pdiag          # rounds run, walk start, queries and rescans as the model of the rounds and walk has them


def test_out_of_range_levels_are_flagged_and_skipped(api, oa, cams):
    F, mps = _projection_scene(api, cams, True, seed=9, nmp=3000)
    rng = np.random.default_rng(4)
    iv = np.argwhere(mps.in_view != 0)
    pick = iv[rng.choice(len(iv), 40, replace=False)]
    lv = mps.level.copy()
    lv[pick[:20, 0], pick[:20, 1]] = 8
    lv[pick[20:, 0], pick[20:, 1]] = -1
    broken = api.MapPoints(mps.bad, mps.in_view, lv, mps.proj_x, mps.proj_y, mps.view_cos, mps.desc, mps.dmask)
    m = api.cORBmatcher(0.8, False, 32, True)
    with pytest.raises(api.McsError):                   # the host call refuses such input
        m.SearchByProjection(F, broken, 3.0)
    gn, gfmp, status, _ = device_projection(api, m, per_cam(F), sizes(F), F.scale_factors, broken, 3.0)
    assert status == api.MCS_ERR_INVALID
    iv2 = mps.in_view.copy()
    iv2[pick[:, 0], pick[:, 1]] = 0
    removed = api.MapPoints(mps.bad, iv2, mps.level, mps.proj_x, mps.proj_y, mps.view_cos, mps.desc, mps.dmask)
    n, fmp = m.SearchByProjection(F, removed, 3.0)
    assert gn == n and np.array_equal(gfmp, fmp)


def test_calls_do_not_wait_for_the_stream(api, oa, cams):
    import torch
    F, mps = _projection_scene(api, cams, True, seed=3, nmp=3000)
    m = api.cORBmatcher(0.8, False, 32, True)
    n, fmp = m.SearchByProjection(F, mps, 3.0)
    rng = np.random.default_rng(1)
    nc, npt = 3, 5000
    from multicol_slam_b200 import synth
    mtmc, inv = random_rig(rng, nc)
    masks = np.stack([synth.mirror_mask(c) for c in cams])
    pos = rng.normal(size=(npt, 3)) * 4.0
    nrm = rng.normal(size=(npt, 3)); nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    dmin = rng.uniform(0.5, 2.0, npt); dmax = dmin * 8.0
    sf = F.scale_factors
    g = api.project_mappoints(inv, mtmc, cams, masks, pos, nrm, dmin, dmax, sf)
    args = (on_device(masks), on_device(pos), on_device(nrm), on_device(dmin), on_device(dmax))
    prep = projection_inputs(api, per_cam(F), mps)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(400_000_000)                  # a few hundred milliseconds of work ahead of both calls
        d = api.project_mappoints_device(inv, mtmc, cams, *args, sf, stream=s)
        n_t, st_t, fm_t, _ = launch_projection(m, prep, sizes(F), sf, 3.0, stream=s)
        busy = s.query()
    assert busy is False
    s.synchronize()
    for a, b in zip(g, d):
        assert np.array_equal(a, b.cpu().numpy())
    gn, gfmp, status = collect(api, prep, n_t, st_t, fm_t)
    assert gn == n and status == api.MCS_OK and np.array_equal(gfmp, fmp)
