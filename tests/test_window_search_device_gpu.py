"""GPU: the device-resident WindowSearch(F1 = LastFrame, F2 = CurrentFrame, window, ., minOctave, maxOctave) of TrackPreviousFrame
(mcs_window_search_device), against the host composition cORBmatcher.WindowSearch (window search through the GPU mcs_search_windows
or the CPU oracle, vnMatches21 mapped to map-point ids) and, where oracle/_ref travelled, the reference's own method.  Both frames
come from packed feature buffers in every layout.  Results are compared after the slot -> contiguous conversion.  Integer work:
bit-exact."""
import numpy as np
import pytest

import acceptance_model as am
import test_ref_match_cpu as T
from test_search_projection_device_gpu import FILL, _flip
from test_search_projection_last_device_gpu import BIG_ID, _pack, _parity_scene

pytestmark = pytest.mark.gpu
frames = T.frames
INT_MAX = 2**31 - 1
# the windows and level filters of TrackPreviousFrame (ref src/cTracking.cpp:737-750), and one upper level bound
WINDOWS = [(60, 4, INT_MAX), (60, 1, INT_MAX), (50, 0, INT_MAX), (60, 0, 3)]


@pytest.fixture(scope="module")
def rm():
    import ref_match_api
    return ref_match_api if ref_match_api.available() else None


def host_window_search(m, F1, F2, mp1, bad, window, lo, hi, sw=None):
    """cORBmatcher.WindowSearch with its vnMatches21 mapped to map-point ids through mp1 -> (nmatches, cur_mp)"""
    valid1 = (mp1 >= 0) & (np.asarray(bad)[np.maximum(mp1, 0)] == 0)
    n, v21 = m.WindowSearch(F1, F2, window, valid1, lo, hi, _sw=sw)
    return n, np.where(v21 >= 0, mp1[np.maximum(v21, 0)], -1).astype(np.int32)


def _counts(F):
    return [int((F.key_cam == c).sum()) for c in range(len(F.cam_w))]


def _device_ws(api, m, Fc, Fl, mp_last, bad, window, lo=0, hi=INT_MAX, layout="single", cap=None, stream=None, last_keys=None, run=True,
               seed=5):
    """mcs_window_search_device on host arrays -> (nmatches, contiguous cur_mp, status, diag).  cur_mp starts from arbitrary ids: the
    call must overwrite every slot below each camera's count and leave the others (FILL) alone."""
    import torch
    cc, cl = _counts(Fc), _counts(Fl)
    cap = cap or max(cc + cl) + 5
    if last_keys is not None:
        Fl = api.Frame(last_keys, Fl.key_cam, Fl.desc, Fl.dmask, list(zip(Fl.cam_w, Fl.cam_h)), Fl.scale_factors)
    cur, last = _pack(Fc, Fl, layout, cap, Fc.desc.shape[1])
    junk = np.random.default_rng(seed).integers(-1, 600, len(Fc.keys)).astype(np.int32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    d = dict(cur=cur, last=last, cap=cap, cc=cc, sizes=list(zip(Fc.cam_w.tolist(), Fc.cam_h.tolist())),
             last_mp_t=t(api.contiguous_to_slots(mp_last, cl, cap, fill=BIG_ID)), bad_t=t(np.asarray(bad, np.uint8)),
             cur_mp_t=t(api.contiguous_to_slots(junk, cc, cap, fill=FILL)), window=window, lo=lo, hi=hi)
    if not run:
        return d
    res = _launch(m, d, stream)
    torch.cuda.synchronize()
    return _collect(api, d, *res)


def _launch(m, d, stream=None):
    return m.WindowSearchDevice(d["cur"], d["last"], d["cap"], d["sizes"], d["last_mp_t"], d["window"], d["cur_mp_t"], min_level=d["lo"],
                                max_level=d["hi"], bad_t=d["bad_t"], stream=stream, diag=True)


def _collect(api, d, n_t, st_t, fm_t, diag_t):
    out, cap, cc = fm_t.cpu().numpy(), d["cap"], d["cc"]
    assert np.all(np.concatenate([out[c * cap + cc[c]:(c + 1) * cap] for c in range(len(cc))]) == FILL)
    return int(n_t.item()), api.slots_to_contiguous(out, cc, cap), int(st_t.item()), diag_t.cpu().numpy()


def _n_queries(F1, mp1, bad, lo, hi):
    lv = F1.keys["octave"]
    ok = (mp1 >= 0) & (np.asarray(bad)[np.maximum(mp1, 0)] == 0)
    if lo > 0:
        ok &= lv >= lo
    if hi < INT_MAX:
        ok &= lv <= hi
    return int(ok.sum())


@pytest.mark.parametrize("win", WINDOWS)
@pytest.mark.parametrize("layout", ["single", "parts", "shared"])
@pytest.mark.parametrize("masks", [False, True])
def test_parity_with_host_oracle_and_reference(api, oa, rm, frames, cams, masks, layout, win):
    s = _parity_scene(api, oa, cams, frames)
    F1, F2, mp1, bad = s["F1"], s["F2"], s["mp1"], s["sc"]["bad"]
    m = api.cORBmatcher(0.8, False, 32, masks)
    hn, hout = host_window_search(m, F1, F2, mp1, bad, *win)
    on, oout = host_window_search(m, F1, F2, mp1, bad, *win, sw=oa.search_windows)
    assert hn == on and np.array_equal(hout, oout)
    if rm:
        sc = s["sc"]
        table = rm.MPTable(3, sc["desc"], dmask=sc["dmask"], bad=bad, world_pos=sc["world"], min_dist=sc["min_d"], max_dist=sc["max_d"])
        rn, rout = rm.window_search(rm.KF(F1, cams, mp=mp1), rm.KF(F2, cams), table, *win, 0.8, masks)
        assert rn == hn and np.array_equal(rout, hout)
    gn, gout, status, diag = _device_ws(api, m, F2, F1, mp1, bad, *win, layout=layout)
    assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)
    # the map point on two last-frame keypoints makes two queries (no first-occurrence rule here)
    assert mp1[s["sc"]["src"][5]] == mp1[s["sc"]["src"][4]] and diag[2] == _n_queries(F1, mp1, bad, win[1], win[2])
    assert hn > (0 if win[1] == 4 else 50)


def test_empty_cameras_and_untouched_slots(api, oa, frames, cams):
    """camera 1 has no keypoints in either frame, camera 2 none in the last frame; slots beyond each count stay as they were"""
    s = _parity_scene(api, oa, cams, frames)

    def sub(F, keep):
        i = np.flatnonzero(np.isin(F.key_cam, keep))
        return api.Frame(F.keys[i], F.key_cam[i], F.desc[i], F.dmask[i], list(zip(F.cam_w, F.cam_h)), F.scale_factors), i
    F1, i1 = sub(s["F1"], [0])
    F2, _ = sub(s["F2"], [0, 2])
    mp1, bad = s["mp1"][i1], s["sc"]["bad"]
    m = api.cORBmatcher(0.8, False, 32, True)
    hn, hout = host_window_search(m, F1, F2, mp1, bad, 60, 0, INT_MAX)
    for layout in ("single", "parts", "shared"):
        gn, gout, status, _ = _device_ws(api, m, F2, F1, mp1, bad, 60, layout=layout)
        assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout) and hn > 20
        assert np.all(gout[F2.key_cam == 2] == -1)           # a camera with no queries is still cleared


@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("dim", [16, 64])
def test_descriptor_sizes(api, oa, cams, dim, masks):
    from multicol_slam_b200 import synth
    ex = oa.OracleExtractor(nfeatures=350, do_dbrief=True, learn_masks=True, desc_size=dim)
    streams = [synth.texture_stream(cams[c], 2, seed=60 + c) for c in range(3)]
    sf = [float(ex.info.scale_factor[l]) for l in range(8)]
    fr = [api.Frame.from_cameras([ex.extract(streams[c][t], synth.mirror_mask(cams[c]), cams[c]) for c in range(3)], T.SIZES, sf)
          for t in range(2)]
    assert fr[0].desc.shape[1] == dim
    s = _parity_scene(api, oa, cams, fr, seed=63 + dim)
    m = api.cORBmatcher(0.8, False, dim, masks)
    for win in ((60, 1, INT_MAX), (50, 0, INT_MAX)):
        hn, hout = host_window_search(m, s["F1"], s["F2"], s["mp1"], s["sc"]["bad"], *win)
        on, oout = host_window_search(m, s["F1"], s["F2"], s["mp1"], s["sc"]["bad"], *win, sw=oa.search_windows)
        assert hn == on and np.array_equal(hout, oout) and hn > 20
        for layout in ("single", "parts"):
            gn, gout, status, _ = _device_ws(api, m, s["F2"], s["F1"], s["mp1"], s["sc"]["bad"], *win, layout=layout)
            assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)


# distances of the chain candidates: each one passes the ratio test against the next (d_k <= 0.8 d_k+1, never equal), the last
# one has no second candidate; all <= TH_HIGH_ = 96 (32 bytes, no masks)
CHAIN_DISTS = [1, 3, 5, 7, 10, 14, 19, 25, 33, 43, 55, 70, 89]


def ratio_chain_scene(api, cams, rng, n_last=16, dim=32):
    """n_last last-frame keypoints of camera 0 with one descriptor, next to each other, whose map points lie on the bearing ray of
    (u0, v0) at identity poses; len(CHAIN_DISTS) current keypoints around (u0, v0) at those distances from it.  Every query
    accepts the best free candidate, so query k takes the k-th: a dependency chain as long as CHAIN_DISTS.  Cameras 1 and 2 have no
    keypoints.  -> (Fc, Fl, rig, world, mp_last)"""
    base = rng.integers(0, 256, dim).astype(np.uint8)
    rig = api.Rig(cams)
    u0, v0 = 300.0, 200.0
    assert rig.in_mirror_mask(0, u0, v0)
    ray = np.array(api.img_to_world(cams[0], u0, v0))
    world = ray[None, :] * rng.uniform(2.0, 8.0, n_last)[:, None]
    kl = np.zeros(n_last, api.KEYPOINT_DTYPE)
    kl["x"] = u0 + rng.uniform(-3, 3, n_last); kl["y"] = v0 + rng.uniform(-3, 3, n_last); kl["octave"] = 1
    n_cur = len(CHAIN_DISTS)
    kc = np.zeros(n_cur, api.KEYPOINT_DTYPE)
    kc["x"] = u0 + rng.uniform(-35, 35, n_cur); kc["y"] = v0 + rng.uniform(-35, 35, n_cur); kc["octave"] = 1   # over several cells
    dc = np.stack([_flip(rng, base, d) for d in rng.permutation(CHAIN_DISTS)])
    e = np.zeros(0, api.KEYPOINT_DTYPE), np.zeros((0, dim), np.uint8), None
    sf = np.cumprod([1.0] + [1.2000000476837158] * 7)
    Fl = api.Frame.from_cameras([(kl, np.tile(base, (n_last, 1)), None), e, e], T.SIZES, sf)
    Fc = api.Frame.from_cameras([(kc, dc, None), e, e], T.SIZES, sf)
    return Fc, Fl, rig, world, np.arange(n_last, dtype=np.int32)


def test_long_dependency_chain_runs_the_walk(api, oa):
    from multicol_slam_b200 import synth
    cams = synth.lafida_cams()
    Fc, Fl, _, world, mp_last = ratio_chain_scene(api, cams, np.random.default_rng(31))
    m = api.cORBmatcher(0.8, False, 32, False)
    bad = np.zeros(len(world), np.uint8)
    hn, hout = host_window_search(m, Fl, Fc, mp_last, bad, 50, 0, INT_MAX)
    on, oout = host_window_search(m, Fl, Fc, mp_last, bad, 50, 0, INT_MAX, sw=oa.search_windows)
    assert hn == on and np.array_equal(hout, oout) and hn == len(CHAIN_DISTS)
    rec = am.Capture(oa)
    host_window_search(m, Fl, Fc, mp_last, bad, 50, 0, INT_MAX, sw=rec)
    pn, _, pdiag, _ = am.predict_windows(api, oa, rec.calls[0])
    cap_rounds = api.lib().mcs_search_by_projection_max_rounds()
    assert len(CHAIN_DISTS) > cap_rounds and pn == hn and pdiag[0] == cap_rounds and pdiag[1] >= 0 and pdiag[3] > 0
    for layout in ("single", "parts", "shared"):
        gn, gout, status, diag = _device_ws(api, m, Fc, Fl, mp_last, bad, 50, layout=layout)
        assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)
        assert diag.tolist() == pdiag          # rounds run, walk start, queries and rescans as the model of the rounds and walk has them


def test_invalid_ids_drop_only_their_query(api, oa, frames, cams):
    s = _parity_scene(api, oa, cams, frames)
    m = api.cORBmatcher(0.8, False, 32, True)
    F1, mp1, bad = s["F1"], s["mp1"], s["sc"]["bad"]
    live = np.flatnonzero((mp1 >= 0) & (bad[np.maximum(mp1, 0)] == 0))
    ids = np.random.default_rng(3).choice(live, 8, replace=False)
    mp_bad = mp1.copy()
    mp_bad[ids] = 600 + 7                                        # >= n_points
    dropped = mp1.copy()
    dropped[ids] = -1
    keys = F1.keys.copy()
    keys["octave"][np.random.default_rng(4).choice(live, 10, replace=False)] = -1    # no level filter applies to WindowSearch
    F1e = api.Frame(keys, F1.key_cam, F1.desc, F1.dmask, list(zip(F1.cam_w, F1.cam_h)), F1.scale_factors)
    for win in ((60, 0, INT_MAX), (60, 1, INT_MAX)):
        hn, hout = host_window_search(m, F1e, s["F2"], dropped, bad, *win)
        gn, gout, status, _ = _device_ws(api, m, s["F2"], F1, mp_bad, bad, *win, last_keys=keys)
        assert status == api.MCS_ERR_INVALID and gn == hn and np.array_equal(gout, hout)
        gn, gout, status, _ = _device_ws(api, m, s["F2"], F1, dropped, bad, *win, last_keys=keys)
        assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)


def test_call_does_not_wait_for_the_stream(api, oa, frames, cams):
    import torch
    s = _parity_scene(api, oa, cams, frames)
    m = api.cORBmatcher(0.8, False, 32, True)
    hn, hout = host_window_search(m, s["F1"], s["F2"], s["mp1"], s["sc"]["bad"], 60, 1, INT_MAX)
    d = _device_ws(api, m, s["F2"], s["F1"], s["mp1"], s["sc"]["bad"], 60, 1, run=False)
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda._sleep(400_000_000)                  # a few hundred milliseconds of work ahead of the call
        res = _launch(m, d, stream=st)
        busy = st.query()
    assert busy is False
    st.synchronize()
    gn, gout, status, _ = _collect(api, d, *res)
    assert gn == hn and status == api.MCS_OK and np.array_equal(gout, hout)
