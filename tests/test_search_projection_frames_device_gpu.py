"""GPU: the device-resident SearchByProjection(F1 = LastFrame, F2 = CurrentFrame, window, vpMapPointMatches2) of TrackPreviousFrame
(mcs_search_by_projection_frames_device), against the host composition SearchByProjectionFramesRig (projection on the host, window
search through the GPU mcs_search_windows or the CPU oracle) and, where oracle/_ref travelled, the reference's own method.  Both
frames come from packed feature buffers in every layout.  Results are compared after the slot -> contiguous conversion.  Integer
work: bit-exact."""
import numpy as np
import pytest

import acceptance_model as am
from device_frames import INT_MAX, SIZES, frames, keep_cameras, on_device, rm  # noqa: F401  (frames, rm: fixtures)
from device_searches import collect, device_search_frames, launch_frames
from search_scenes import CHAIN_DISTS, host_window_search, make_scene, parity_scene, ratio_chain_scene

pytestmark = pytest.mark.gpu


def _host(m, s, window=40, oa=None, mp1=None, mp2=None, F1=None, world=None):
    return m.SearchByProjectionFramesRig(s["F1"] if F1 is None else F1, s["mp1"] if mp1 is None else mp1, s["F2"], s["rig2"],
                                         s["mp2"] if mp2 is None else mp2, s["sc"]["world"] if world is None else world, s["sc"]["bad"],
                                         window, _sw=None if oa is None else oa.search_windows)


def _dev(api, m, s, window=40, **kw):
    kw.setdefault("mp_cur", s["mp2"]); kw.setdefault("mp_last", s["mp1"]); kw.setdefault("world", s["sc"]["world"])
    return device_search_frames(api, m, s["F2"], s["F1"], s["rig2"], bad=s["sc"]["bad"], window=window, **kw)


@pytest.mark.parametrize("layout", ["single", "parts", "shared"])
@pytest.mark.parametrize("masks", [False, True])
def test_parity_with_host_oracle_and_reference(api, oa, rm, frames, cams, masks, layout):
    s = parity_scene(api, oa, cams, frames)
    m = api.cORBmatcher(0.8, False, 32, masks)
    hn, hout = _host(m, s)
    on, oout = _host(m, s, oa=oa)
    assert hn == on and np.array_equal(hout, oout)
    if rm:
        sc = s["sc"]
        table = rm.MPTable(3, sc["desc"], dmask=sc["dmask"], bad=sc["bad"], world_pos=sc["world"], min_dist=sc["min_d"], max_dist=sc["max_d"])
        k1 = rm.KF(s["F1"], cams, M_c=sc["M_c"], M_t=sc["M_t"], mp=s["mp1"])
        k2 = rm.KF(s["F2"], cams, M_c=sc["M_c"], M_t=s["M_t2"], mp=s["mp2"])
        rn, rout = rm.search_by_projection_frames(k1, k2, table, 40, 0.8, masks)
        assert rn == hn and np.array_equal(rout, hout)
    gn, gout, status, diag = _dev(api, m, s, layout=layout)
    assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)
    pre = s["mp2"] >= 0
    assert np.array_equal(gout[pre], s["mp2"][pre])                          # pre-assigned keypoints keep their map point
    assert not np.isin(gout[~pre & (gout >= 0)], s["mp2"][pre]).any()        # and their points, already found, are not searched
    assert hn > 50 and diag[2] > hn


def test_first_occurrence_and_every_camera(api, oa, frames, cams):
    """the map point on two last-frame keypoints is searched once, from its first keypoint; a point may be accepted in several
    cameras of the current frame"""
    s = parity_scene(api, oa, cams, frames)
    m = api.cORBmatcher(0.8, False, 32, True)
    src = s["sc"]["src"]
    p = int(s["mp1"][src[4]])
    assert s["mp1"][src[5]] == p
    mp1 = s["mp1"].copy()
    mp1[max(src[4], src[5])] = -1                              # the point's later keypoint removed: same queries, same result
    hn, hout = _host(m, s)
    gn, gout, status, diag = _dev(api, m, s)
    hn1, hout1 = _host(m, s, mp1=mp1)
    gn1, gout1, _, diag1 = _dev(api, m, s, mp_last=mp1)
    assert status == api.MCS_OK and gn == hn == gn1 == hn1 and np.array_equal(gout, hout) and np.array_equal(gout1, hout)
    assert np.array_equal(hout1, hout) and diag[2] == diag1[2]
    # cameras that overlap: at identity poses the chain's map points are in front of camera 1 too; copies of the current keypoints
    # around their projection there make every point query both cameras, and a point may be accepted in both
    Fc, Fl, rig, world, mp_last = ratio_chain_scene(api, cams, np.random.default_rng(8))
    u1, v1, _ = rig.world_to_cam(1, world[0])
    assert rig.in_mirror_mask(1, u1, v1)
    k1 = Fc.keys.copy()
    k1["x"] += np.float32(u1 - 300.0); k1["y"] += np.float32(v1 - 200.0)
    both = api.Frame(np.concatenate([Fc.keys, k1]), np.concatenate([Fc.key_cam, Fc.key_cam + 1]), np.concatenate([Fc.desc, Fc.desc]),
                     None, list(zip(Fc.cam_w, Fc.cam_h)), Fc.scale_factors)
    m2 = api.cORBmatcher(0.8, False, 32, False)
    bad = np.zeros(len(world), np.uint8)
    free = np.full(len(both.keys), -1, np.int32)
    hn, hout = m2.SearchByProjectionFramesRig(Fl, mp_last, both, rig, free, world, bad, 50)
    gn, gout, status, diag = device_search_frames(api, m2, both, Fl, rig, free, mp_last, world, bad, 50)
    assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)
    acc = gout[gout >= 0]
    assert len(acc) > len(np.unique(acc))                      # some point accepted in both cameras


def test_empty_cameras_and_untouched_slots(api, oa, frames, cams):
    """camera 1 has no keypoints in either frame, camera 2 none in the last frame; slots beyond each count stay as they were"""
    s = parity_scene(api, oa, cams, frames)
    F1, i1 = keep_cameras(api, s["F1"], [0])
    F2, i2 = keep_cameras(api, s["F2"], [0, 2])
    s.update(F1=F1, F2=F2, mp1=s["mp1"][i1], mp2=s["mp2"][i2])
    m = api.cORBmatcher(0.8, False, 32, True)
    hn, hout = _host(m, s)
    for layout in ("single", "parts", "shared"):
        gn, gout, status, _ = _dev(api, m, s, layout=layout)
        assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout) and hn > 10


def test_edge_queries(api, oa, frames, cams):
    """last-frame octaves -1 (no level filter) and n_levels (no candidate); map points behind the rig, outside every mask, at
    non-finite positions and at the rig centre; windows without candidates"""
    s = parity_scene(api, oa, cams, frames, seed=62)
    rng = np.random.default_rng(23)
    F1 = s["F1"]
    keys = F1.keys.copy()
    pick = rng.permutation(np.flatnonzero(s["mp1"] >= 0))
    keys["octave"][pick[:60]] = -1
    keys["octave"][pick[60:90]] = 8
    world = s["sc"]["world"].copy()
    pts = s["mp1"][pick[120:200]]
    centre = s["rig2"].M_t[:3, 3]
    world[pts[:20]] = 2 * centre - world[pts[:20]]                              # mirrored through the rig centre: behind
    world[pts[20:40]] = centre + 50.0 * rng.normal(size=(20, 3))               # anywhere, mostly outside every mirror mask
    world[pts[40:50]] = np.nan
    world[pts[50:60], 0] = np.inf
    world[pts[60:70]] = centre
    F1e = api.Frame(keys, F1.key_cam, F1.desc, F1.dmask, list(zip(F1.cam_w, F1.cam_h)), F1.scale_factors)
    for masks in (False, True):
        m = api.cORBmatcher(0.8, False, 32, masks)
        for window in (40, 1):
            hn, hout = _host(m, s, window, F1=F1e, world=world)
            on, oout = _host(m, s, window, oa=oa, F1=F1e, world=world)
            assert hn == on and np.array_equal(hout, oout)
            gn, gout, status, _ = _dev(api, m, s, window, world=world, last_keys=keys)
            assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)
            assert window != 40 or hn > 50


@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("dim", [16, 64])
def test_descriptor_sizes(api, oa, cams, dim, masks):
    from multicol_slam_b200 import synth
    ex = oa.OracleExtractor(nfeatures=350, do_dbrief=True, learn_masks=True, desc_size=dim)
    streams = [synth.texture_stream(cams[c], 2, seed=60 + c) for c in range(3)]
    sf = [float(ex.info.scale_factor[l]) for l in range(8)]
    fr = [api.Frame.from_cameras([ex.extract(streams[c][t], synth.mirror_mask(cams[c]), cams[c]) for c in range(3)], SIZES, sf)
          for t in range(2)]
    s = parity_scene(api, oa, cams, fr, seed=63 + dim)
    m = api.cORBmatcher(0.8, False, dim, masks)
    hn, hout = _host(m, s)
    on, oout = _host(m, s, oa=oa)
    assert hn == on and np.array_equal(hout, oout) and hn > 20
    for layout in ("single", "parts"):
        gn, gout, status, _ = _dev(api, m, s, layout=layout)
        assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)


def test_long_dependency_chain_runs_the_walk(api, oa):
    from multicol_slam_b200 import synth
    cams = synth.lafida_cams()
    Fc, Fl, rig, world, mp_last = ratio_chain_scene(api, cams, np.random.default_rng(31))
    m = api.cORBmatcher(0.8, False, 32, False)
    bad = np.zeros(len(world), np.uint8)
    free = np.full(len(Fc.keys), -1, np.int32)
    hn, hout = m.SearchByProjectionFramesRig(Fl, mp_last, Fc, rig, free, world, bad, 40)
    on, oout = m.SearchByProjectionFramesRig(Fl, mp_last, Fc, rig, free, world, bad, 40, _sw=oa.search_windows)
    assert hn == on and np.array_equal(hout, oout) and hn == len(CHAIN_DISTS)
    rec = am.Capture(oa)
    m.SearchByProjectionFramesRig(Fl, mp_last, Fc, rig, free, world, bad, 40, _sw=rec)
    pn, _, pdiag, _ = am.predict_windows(api, oa, rec.calls[0])
    cap_rounds = api.lib().mcs_search_by_projection_max_rounds()
    assert pn == hn and pdiag[0] == cap_rounds and pdiag[1] >= 0 and pdiag[3] > 0
    for layout in ("single", "parts", "shared"):
        gn, gout, status, diag = device_search_frames(api, m, Fc, Fl, rig, free, mp_last, world, bad, 40, layout=layout)
        assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)
        assert diag.tolist() == pdiag          # rounds run, walk start, queries and rescans as the model of the rounds and walk has them


def test_invalid_ids(api, oa, frames, cams):
    """last-frame ids >= n_points drop their keypoint and raise status; current-frame ids >= n_points only mark their keypoint taken"""
    s = parity_scene(api, oa, cams, frames)
    m = api.cORBmatcher(0.8, False, 32, True)
    rng = np.random.default_rng(3)
    ids = rng.choice(np.flatnonzero(s["mp1"] >= 0), 8, replace=False)
    mp1 = s["mp1"].copy()
    mp1[ids] = 600 + 7
    dropped = s["mp1"].copy()
    dropped[ids] = -1
    hn, hout = _host(m, s, mp1=dropped)
    gn, gout, status, _ = _dev(api, m, s, mp_last=mp1)
    assert status == api.MCS_ERR_INVALID and gn == hn and np.array_equal(gout, hout)
    mp2 = s["mp2"].copy()
    mp2[rng.choice(np.flatnonzero(mp2 < 0), 40, replace=False)] = 600 + 9
    hn, hout = _host(m, s, mp2=mp2)
    gn, gout, status, _ = _dev(api, m, s, mp_cur=mp2)
    assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)


def test_track_previous_frame_chain_from_the_extractor(api, oa, cams):
    """TrackPreviousFrame on two consecutive frames extracted on the device into one packed buffer: the last frame's frame_mp from
    the local-map device search, WindowSearch, a stand-in for PoseOptimization (some accepted slots set to -1 on the device, the
    pose moved), SearchByProjection(F1, F2) at the new pose, then the local-map device search on the current frame; every step
    against the host composition on the same data"""
    import torch
    from multicol_slam_b200 import rig as rigmod
    from multicol_slam_b200 import synth
    ex = api.mdBRIEFextractorOct(nfeatures=1000, do_dBrief=True, learnMasks=True)
    W, H = 754, 480
    pitch = (W + 63) // 64 * 64
    streams = [synth.texture_stream(cams[c], 2, seed=80 + c) for c in range(3)]
    imgs = torch.zeros((6, H, pitch), dtype=torch.uint8, device="cuda")
    for t in range(2):
        for c in range(3):
            imgs[3 * t + c, :, :W] = on_device(np.ascontiguousarray(streams[c][t]).reshape(H, W))
    masks = np.stack([synth.mirror_mask(c) for c in cams])
    cap = ex.capacity
    packed = torch.zeros(rigmod.packed_layout(6, cap, 32)[1], dtype=torch.uint8, device="cuda")
    v = ex.extract_batch_packed_device(imgs, masks, cams, [0, 1, 2, 0, 1, 2], packed, width=W)
    torch.cuda.synchronize()
    counts = v["counts"].cpu().numpy()
    kps = v["kps"].cpu().numpy().view(api.KEYPOINT_DTYPE).reshape(6, cap)
    sf = [float(ex.info.scale_factor[l]) for l in range(8)]
    Fs = [api.Frame.from_cameras([(kps[i, :counts[i]], v["desc"][i, :counts[i]].cpu().numpy(), v["dmask"][i, :counts[i]].cpu().numpy())
                                  for i in range(3 * t, 3 * t + 3)], SIZES, sf) for t in range(2)]
    Fl, Fc = Fs
    sc = make_scene(api, oa, cams, Fl, 71, npts=min(700, len(Fl.keys)))
    rig1 = sc["rig"]
    world, n = sc["world"], len(sc["world"])
    nrm = world - rig1.M_t[:3, 3]
    nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    m = api.cORBmatcher(0.8, False, 32, True)
    masks_t, world_t, nrm_t, dmin_t, dmax_t = on_device(masks), on_device(world), on_device(nrm), on_device(sc["min_d"]), on_device(sc["max_d"])
    desc_t, dmask_t = on_device(sc["desc"]), on_device(sc["dmask"])
    zeros = np.zeros(n, np.uint8)
    zeros_t = on_device(zeros)
    cur, last = (packed, 1, 6, 3), (packed, 1, 6, 0)
    as_contig = lambda x, k: api.slots_to_contiguous(x.cpu().numpy(), counts[3 * k:3 * k + 3], cap)  # noqa: E731
    # 1. the last frame's map points: local-map search at the last pose
    g = api.project_mappoints(rig1.MtMc_inv, rig1.MtMc, cams, masks, world, nrm, sc["min_d"], sc["max_d"], sf)
    n1, fmp_last = m.SearchByProjection(Fl, api.MapPoints(zeros, *g, sc["desc"], sc["dmask"]), 3.0)
    proj = api.project_mappoints_device(rig1.MtMc_inv, rig1.MtMc, cams, masks_t, world_t, nrm_t, dmin_t, dmax_t, sf)
    fm_last_t = torch.full((3 * cap,), -1, dtype=torch.int32, device="cuda")
    gn1, st1, _ = m.SearchByProjectionDevice(packed, 1, 6, 0, 3, cap, SIZES, sf, api.MapPointsDevice(None, *proj, desc_t, dmask_t), 3.0,
                                             fm_last_t)
    torch.cuda.synchronize()
    assert int(st1.item()) == api.MCS_OK and int(gn1.item()) == n1 and n1 > 100
    assert np.array_equal(as_contig(fm_last_t, 0), fmp_last)
    # 2. WindowSearch(LastFrame, CurrentFrame, 60, ., 1): the device frame_mp of the last frame is last_mp as it stands
    n2, mp_cur = host_window_search(m, Fl, Fc, fmp_last, zeros, 60, 1, INT_MAX)
    cur_mp_t = torch.full((3 * cap,), -1, dtype=torch.int32, device="cuda")
    gn2, st2, _ = m.WindowSearchDevice(cur, last, cap, SIZES, fm_last_t, 60, cur_mp_t, min_level=1, bad_t=zeros_t)
    torch.cuda.synchronize()
    assert int(st2.item()) == api.MCS_OK and int(gn2.item()) == n2 and n2 > 50
    assert np.array_equal(as_contig(cur_mp_t, 1), mp_cur)
    # 3. stand-in for PoseOptimization: every fifth accepted keypoint an outlier (set to -1 on the device), the pose moved
    acc = np.flatnonzero(mp_cur >= 0)[::5]
    mp_cur[acc] = -1
    slot = np.concatenate([c * cap + np.arange(counts[3 + c]) for c in range(3)])[acc]
    cur_mp_t[on_device(slot.astype(np.int64))] = -1
    M_t2 = sc["M_t"].copy()
    M_t2[:3, 3] += [0.003, 0.002, -0.004]
    rig2 = api.Rig(cams, sc["M_c"], M_t2)
    # 4. SearchByProjection(LastFrame, CurrentFrame, 40, .) at the optimised pose
    n4, mp_cur4 = m.SearchByProjectionFramesRig(Fl, fmp_last, Fc, rig2, mp_cur, world, zeros, 40)
    gn4, st4, _ = m.SearchByProjectionFramesDevice(cur, last, cap, rig2, masks_t, fm_last_t, world_t, 40, cur_mp_t, bad_t=zeros_t)
    torch.cuda.synchronize()
    assert int(st4.item()) == api.MCS_OK and int(gn4.item()) == n4 and n4 > 10
    assert np.array_equal(as_contig(cur_mp_t, 1), mp_cur4)
    # 5. local-map search on the current frame with those assignments pre-assigned
    g2 = api.project_mappoints(rig2.MtMc_inv, rig2.MtMc, cams, masks, world, nrm, sc["min_d"], sc["max_d"], sf)
    n5, fmp_cur = m.SearchByProjection(Fc, api.MapPoints(zeros, *g2, sc["desc"], sc["dmask"]), 3.0, mp_cur4.copy())
    proj2 = api.project_mappoints_device(rig2.MtMc_inv, rig2.MtMc, cams, masks_t, world_t, nrm_t, dmin_t, dmax_t, sf)
    gn5, st5, _ = m.SearchByProjectionDevice(packed, 1, 6, 3, 3, cap, SIZES, sf, api.MapPointsDevice(None, *proj2, desc_t, dmask_t), 3.0,
                                             cur_mp_t)
    torch.cuda.synchronize()
    assert int(st5.item()) == api.MCS_OK and int(gn5.item()) == n5
    assert np.array_equal(as_contig(cur_mp_t, 1), fmp_cur)


def test_call_does_not_wait_for_the_stream(api, oa, frames, cams):
    import torch
    s = parity_scene(api, oa, cams, frames)
    m = api.cORBmatcher(0.8, False, 32, True)
    hn, hout = _host(m, s)
    d = _dev(api, m, s, run=False)
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda._sleep(400_000_000)                  # a few hundred milliseconds of work ahead of the call
        res = launch_frames(m, d, stream=st)
        busy = st.query()
    assert busy is False
    st.synchronize()
    gn, gout, status, _ = collect(api, d, *res)
    assert gn == hn and status == api.MCS_OK and np.array_equal(gout, hout)
