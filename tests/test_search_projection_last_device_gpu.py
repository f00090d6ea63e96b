"""GPU: the device-resident motion-model search, SearchByProjection(CurrentFrame, LastFrame, th) (mcs_search_by_projection_last_device),
against the host composition SearchByProjectionLastRig (projection on the host, window search through the GPU mcs_search_windows or
the CPU oracle) and, where oracle/_ref travelled, the reference's own method.  Both frames come from packed feature buffers in
every layout: one extraction buffer with decoy images around, one one-image buffer per camera, and both frames in one buffer.
Results are compared after the slot -> contiguous conversion.  Integer work: bit-exact."""
import numpy as np
import pytest

import acceptance_model as am
from device_frames import SIZES, flip, frames, keep_cameras, on_device, rm  # noqa: F401  (frames, rm: fixtures)
from device_searches import collect, device_last, launch_last
from search_scenes import make_scene, parity_scene

pytestmark = pytest.mark.gpu


def _host(m, s, th, oa=None, mp1=None, F1=None, world=None):
    return m.SearchByProjectionLastRig(s["F2"], s["rig2"], s["mp2"], F1 if F1 is not None else s["F1"], s["mp1"] if mp1 is None else mp1,
                                       s["outlier"], s["sc"]["world"] if world is None else world, s["sc"]["bad"], th,
                                       _sw=None if oa is None else oa.search_windows)


@pytest.mark.parametrize("th", [50.0, 5.0])
@pytest.mark.parametrize("layout", ["single", "parts", "shared"])
@pytest.mark.parametrize("masks", [False, True])
def test_parity_with_host_oracle_and_reference(api, oa, rm, frames, cams, masks, layout, th):
    s = parity_scene(api, oa, cams, frames)
    m = api.cORBmatcher(0.8, False, 32, masks)
    hn, hout = _host(m, s, th)
    on, oout = _host(m, s, th, oa=oa)
    assert hn == on and np.array_equal(hout, oout)
    if rm:
        sc = s["sc"]
        table = rm.MPTable(3, sc["desc"], dmask=sc["dmask"], bad=sc["bad"], world_pos=sc["world"], min_dist=sc["min_d"], max_dist=sc["max_d"])
        k1 = rm.KF(s["F1"], cams, M_c=sc["M_c"], M_t=sc["M_t"], mp=s["mp1"], outlier=s["outlier"])
        k2 = rm.KF(s["F2"], cams, M_c=sc["M_c"], M_t=s["M_t2"], mp=s["mp2"])
        rn, rout = rm.search_by_projection_last(k2, k1, table, th, 0.8, masks)
        assert rn == hn and np.array_equal(rout, hout)
    gn, gout, status, diag = device_last(api, m, s["F2"], s["F1"], s["rig2"], s["mp2"], s["mp1"], s["outlier"], s["sc"]["world"],
                                          s["sc"]["bad"], th, layout=layout)
    assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)
    assert np.array_equal(gout[s["mp2"] >= 0], s["mp2"][s["mp2"] >= 0])        # pre-assigned keypoints keep their map point
    assert hn > (100 if th == 50.0 else 10) and diag[2] > hn


def test_empty_cameras_and_untouched_slots(api, oa, frames, cams):
    """camera 1 has no keypoints in either frame, camera 2 none in the last frame; slots beyond each count stay as they were"""
    s = parity_scene(api, oa, cams, frames)
    F1, i1 = keep_cameras(api, s["F1"], [0])
    F2, i2 = keep_cameras(api, s["F2"], [0, 2])
    s.update(F1=F1, F2=F2, mp1=s["mp1"][i1], mp2=s["mp2"][i2], outlier=s["outlier"][i1])
    m = api.cORBmatcher(0.8, False, 32, True)
    hn, hout = _host(m, s, 50.0)
    for layout in ("single", "parts", "shared"):
        gn, gout, status, _ = device_last(api, m, F2, F1, s["rig2"], s["mp2"], s["mp1"], s["outlier"], s["sc"]["world"], s["sc"]["bad"],
                                           50.0, layout=layout)
        assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout) and hn > 20


def test_edge_queries(api, oa, frames, cams):
    """last-frame keypoints at octave 0 (min_level -1) and at the top octave; map points behind the camera, outside the mask and at
    non-finite positions; windows without candidates (th = 1)"""
    s = parity_scene(api, oa, cams, frames, seed=62)
    rng = np.random.default_rng(23)
    F1 = s["F1"]
    keys = F1.keys.copy()
    has = np.flatnonzero(s["mp1"] >= 0)
    pick = rng.permutation(has)
    keys["octave"][pick[:60]] = 0
    keys["octave"][pick[60:120]] = 7
    world = s["sc"]["world"].copy()
    pts = s["mp1"][pick[120:200]]
    centre = s["rig2"].M_t[:3, 3]
    world[pts[:20]] = 2 * centre - world[pts[:20]]                              # mirrored through the rig centre: behind
    world[pts[20:40]] = centre + 50.0 * rng.normal(size=(20, 3))               # anywhere, mostly outside the mirror mask
    world[pts[40:50]] = np.nan
    world[pts[50:60], 0] = np.inf
    world[pts[60:70]] = centre                                                  # at the camera system's centre
    F1e = api.Frame(keys, F1.key_cam, F1.desc, F1.dmask, list(zip(F1.cam_w, F1.cam_h)), F1.scale_factors)
    assert (keys["octave"][s["mp1"] >= 0] == 7).sum() >= 60
    for masks in (False, True):
        m = api.cORBmatcher(0.8, False, 32, masks)
        for th in (50.0, 1.0):
            hn, hout = _host(m, s, th, F1=F1e, world=world)
            on, oout = _host(m, s, th, oa=oa, F1=F1e, world=world)
            assert hn == on and np.array_equal(hout, oout)
            gn, gout, status, _ = device_last(api, m, s["F2"], F1e, s["rig2"], s["mp2"], s["mp1"], s["outlier"], world, s["sc"]["bad"], th)
            assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)
            assert th != 50.0 or hn > 50


@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("dim", [16, 64])
def test_descriptor_sizes(api, oa, cams, dim, masks):
    from multicol_slam_b200 import synth
    ex = oa.OracleExtractor(nfeatures=350, do_dbrief=True, learn_masks=True, desc_size=dim)
    streams = [synth.texture_stream(cams[c], 2, seed=60 + c) for c in range(3)]
    sf = [float(ex.info.scale_factor[l]) for l in range(8)]
    fr = [api.Frame.from_cameras([ex.extract(streams[c][t], synth.mirror_mask(cams[c]), cams[c]) for c in range(3)], SIZES, sf)
          for t in range(2)]
    assert fr[0].desc.shape[1] == dim
    s = parity_scene(api, oa, cams, fr, seed=63 + dim)
    m = api.cORBmatcher(0.8, False, dim, masks)
    hn, hout = _host(m, s, 50.0)
    on, oout = _host(m, s, 50.0, oa=oa)
    assert hn == on and np.array_equal(hout, oout) and hn > 20
    for layout in ("single", "parts"):
        gn, gout, status, _ = device_last(api, m, s["F2"], s["F1"], s["rig2"], s["mp2"], s["mp1"], s["outlier"], s["sc"]["world"],
                                           s["sc"]["bad"], 50.0, layout=layout)
        assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)


def _chain_scene(api, cams, rng, n_last=20, n_cur=30, dim=32):
    """n_last last-frame keypoints with one descriptor whose map points all project to one spot of camera 0, and n_cur current
    keypoints in that window at distinct distances <= TH_HIGH_: every query takes the next free candidate"""
    base = rng.integers(0, 256, dim).astype(np.uint8)
    rig = api.Rig(cams)                                          # identity poses: the camera frame is the world frame
    u0, v0 = 300.0, 200.0
    assert rig.in_mirror_mask(0, u0, v0)
    ray = np.array(api.img_to_world(cams[0], u0, v0))
    world = ray[None, :] * rng.uniform(2.0, 8.0, n_last)[:, None]
    kl = np.zeros(n_last, api.KEYPOINT_DTYPE)
    kl["x"] = rng.uniform(250, 350, n_last); kl["y"] = rng.uniform(150, 250, n_last); kl["octave"] = 1
    kc = np.zeros(n_cur, api.KEYPOINT_DTYPE)
    kc["x"] = u0 + rng.uniform(-40, 40, n_cur); kc["y"] = v0 + rng.uniform(-40, 40, n_cur)        # over several grid cells
    kc["octave"] = rng.integers(0, 3, n_cur)
    dc = np.stack([flip(rng, base, k + 1) for k in rng.permutation(n_cur)])
    # camera 1: an ordinary independent scene; camera 2: no keypoints in either frame
    k1 = np.zeros(120, api.KEYPOINT_DTYPE)
    k1["x"] = rng.uniform(100, 650, 120); k1["y"] = rng.uniform(60, 420, 120); k1["octave"] = rng.integers(0, 4, 120)
    d1 = rng.integers(0, 256, (120, dim)).astype(np.uint8)
    e = np.zeros(0, api.KEYPOINT_DTYPE), np.zeros((0, dim), np.uint8), None
    sf = np.cumprod([1.0] + [1.2000000476837158] * 7)
    Fl = api.Frame.from_cameras([(kl, np.tile(base, (n_last, 1)), None), (k1, d1, None), e], SIZES, sf)
    Fc = api.Frame.from_cameras([(kc, dc, None), (k1[::-1].copy(), d1[::-1].copy(), None), e], SIZES, sf)
    # camera-1 map points: on the rays of their last keypoints, seen again in the current frame
    rays = np.array([api.img_to_world(cams[1], float(k["x"]), float(k["y"])) for k in k1])
    w1 = rays * rng.uniform(2.0, 8.0, 120)[:, None]
    w1 = np.stack([api._mm(rig.MtMc[1], np.append(p, 1.0))[:3] for p in w1])
    mp_last = np.concatenate([np.arange(n_last), n_last + np.arange(120)]).astype(np.int32)
    return Fc, Fl, rig, np.concatenate([world, w1]), mp_last


def test_long_dependency_chain_runs_the_walk(api, oa):
    from multicol_slam_b200 import synth
    cams = synth.lafida_cams()
    rng = np.random.default_rng(31)
    Fc, Fl, rig, world, mp_last = _chain_scene(api, cams, rng)
    m = api.cORBmatcher(0.8, False, 32, False)
    mp_cur = np.full(len(Fc.keys), -1, np.int32)
    mp_cur[[3, 11]] = 500                                        # two of the chain's candidates taken on entry
    bad = np.zeros(len(world), np.uint8)
    hn, hout = m.SearchByProjectionLastRig(Fc, rig, mp_cur, Fl, mp_last, None, world, bad, 50.0)
    on, oout = m.SearchByProjectionLastRig(Fc, rig, mp_cur, Fl, mp_last, None, world, bad, 50.0, _sw=oa.search_windows)
    assert hn == on and np.array_equal(hout, oout)
    assert (hout[:30] >= 0).sum() == 22                          # 20 acceptances along the chain + the 2 taken on entry
    rec = am.Capture(oa)
    m.SearchByProjectionLastRig(Fc, rig, mp_cur, Fl, mp_last, None, world, bad, 50.0, _sw=rec)
    pn, _, pdiag, _ = am.predict_windows(api, oa, rec.calls[0])
    cap_rounds = api.lib().mcs_search_by_projection_max_rounds()
    assert pn == hn and pdiag[0] == cap_rounds and pdiag[1] >= 0 and pdiag[3] > 0
    for layout in ("single", "parts", "shared"):
        gn, gout, status, diag = device_last(api, m, Fc, Fl, rig, mp_cur, mp_last, None, world, bad, 50.0, layout=layout)
        assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)
        assert diag.tolist() == pdiag          # rounds run, walk start, queries and rescans as the model of the rounds and walk has them


def test_invalid_ids_and_octaves_drop_only_their_query(api, oa, frames, cams):
    s = parity_scene(api, oa, cams, frames)
    m = api.cORBmatcher(0.8, False, 32, True)
    rig2, F1, sc = s["rig2"], s["F1"], s["sc"]
    live = [i for i in range(len(F1.keys)) if s["mp1"][i] >= 0 and not sc["bad"][s["mp1"][i]] and not s["outlier"][i] and
            rig2.in_mirror_mask(int(F1.key_cam[i]), *rig2.world_to_cam(int(F1.key_cam[i]), sc["world"][s["mp1"][i]])[:2])]
    rng = np.random.default_rng(3)
    pick = rng.choice(live, 10, replace=False)
    ids, octs = pick[:5], pick[5:]
    for kind in ("id", "octave", "both"):
        mp1 = s["mp1"].copy()
        keys = F1.keys.copy()
        if kind in ("id", "both"):
            mp1[ids] = 600 + 7                                   # >= n_points
        if kind in ("octave", "both"):
            keys["octave"][octs[:3]] = 8                          # = n_levels
            keys["octave"][octs[3:]] = -1
        dropped = s["mp1"].copy()
        dropped[ids if kind == "id" else (octs if kind == "octave" else pick)] = -1
        hn, hout = _host(m, s, 50.0, mp1=dropped)
        gn, gout, status, _ = device_last(api, m, s["F2"], F1, rig2, s["mp2"], mp1, s["outlier"], sc["world"], sc["bad"], 50.0,
                                           last_keys=keys)
        assert status == api.MCS_ERR_INVALID and gn == hn and np.array_equal(gout, hout), kind


def test_tracking_chain_from_the_extractor(api, oa, cams):
    """two consecutive frames extracted on the device into one packed buffer: the last frame's frame_mp from the local-map device
    search, then the motion-model search for the current frame, then the local-map device search on the current frame with that
    result pre-assigned; every step against the host composition on the same data"""
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
    M_t2 = sc["M_t"].copy()
    M_t2[:3, 3] += [0.003, 0.002, -0.004]
    rig2 = api.Rig(cams, sc["M_c"], M_t2)
    world, n = sc["world"], len(sc["world"])
    nrm = world - rig1.M_t[:3, 3]
    nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    m = api.cORBmatcher(0.8, False, 32, True)
    masks_t, world_t, nrm_t, dmin_t, dmax_t = on_device(masks), on_device(world), on_device(nrm), on_device(sc["min_d"]), on_device(sc["max_d"])
    desc_t, dmask_t = on_device(sc["desc"]), on_device(sc["dmask"])
    zeros = np.zeros(n, np.uint8)
    # 1. the last frame's map points: local-map search at the last pose
    g = api.project_mappoints(rig1.MtMc_inv, rig1.MtMc, cams, masks, world, nrm, sc["min_d"], sc["max_d"], sf)
    n1, fmp_last = m.SearchByProjection(Fl, api.MapPoints(zeros, *g, sc["desc"], sc["dmask"]), 3.0)
    proj = api.project_mappoints_device(rig1.MtMc_inv, rig1.MtMc, cams, masks_t, world_t, nrm_t, dmin_t, dmax_t, sf)
    fm_last_t = torch.full((3 * cap,), -1, dtype=torch.int32, device="cuda")
    gn1, st1, _ = m.SearchByProjectionDevice(packed, 1, 6, 0, 3, cap, SIZES, sf, api.MapPointsDevice(None, *proj, desc_t, dmask_t), 3.0,
                                             fm_last_t)
    torch.cuda.synchronize()
    assert int(st1.item()) == api.MCS_OK and int(gn1.item()) == n1 and n1 > 100
    assert np.array_equal(api.slots_to_contiguous(fm_last_t.cpu().numpy(), counts[:3], cap), fmp_last)
    # 2. motion model: the last frame's device frame_mp is last_mp as it stands
    n2, mp_cur = m.SearchByProjectionLastRig(Fc, rig2, np.full(len(Fc.keys), -1, np.int32), Fl, fmp_last, None, world, zeros, 50.0)
    cur_mp_t = torch.full((3 * cap,), -1, dtype=torch.int32, device="cuda")
    gn2, st2, _ = m.SearchByProjectionLastDevice((packed, 1, 6, 3), (packed, 1, 6, 0), cap, rig2, masks_t, sf, fm_last_t, world_t, 50.0,
                                                 cur_mp_t)
    torch.cuda.synchronize()
    assert int(st2.item()) == api.MCS_OK and int(gn2.item()) == n2 and n2 > 50
    assert np.array_equal(api.slots_to_contiguous(cur_mp_t.cpu().numpy(), counts[3:], cap), mp_cur)
    # 3. local-map search on the current frame, the motion model's assignments pre-assigned
    g2 = api.project_mappoints(rig2.MtMc_inv, rig2.MtMc, cams, masks, world, nrm, sc["min_d"], sc["max_d"], sf)
    n3, fmp_cur = m.SearchByProjection(Fc, api.MapPoints(zeros, *g2, sc["desc"], sc["dmask"]), 3.0, mp_cur.copy())
    proj2 = api.project_mappoints_device(rig2.MtMc_inv, rig2.MtMc, cams, masks_t, world_t, nrm_t, dmin_t, dmax_t, sf)
    gn3, st3, _ = m.SearchByProjectionDevice(packed, 1, 6, 3, 3, cap, SIZES, sf, api.MapPointsDevice(None, *proj2, desc_t, dmask_t), 3.0,
                                             cur_mp_t)
    torch.cuda.synchronize()
    assert int(st3.item()) == api.MCS_OK and int(gn3.item()) == n3
    assert np.array_equal(api.slots_to_contiguous(cur_mp_t.cpu().numpy(), counts[3:], cap), fmp_cur)


def test_call_does_not_wait_for_the_stream(api, oa, frames, cams):
    import torch
    s = parity_scene(api, oa, cams, frames)
    m = api.cORBmatcher(0.8, False, 32, True)
    hn, hout = _host(m, s, 50.0)
    d = device_last(api, m, s["F2"], s["F1"], s["rig2"], s["mp2"], s["mp1"], s["outlier"], s["sc"]["world"], s["sc"]["bad"], 50.0,
                     run=False)
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda._sleep(400_000_000)                  # a few hundred milliseconds of work ahead of the call
        res = launch_last(m, d, s["rig2"], s["F2"].scale_factors, 50.0, stream=st)
        busy = st.query()
    assert busy is False
    st.synchronize()
    gn, gout, status, _ = collect(api, d, *res)
    assert gn == hn and status == api.MCS_OK and np.array_equal(gout, hout)
