"""GPU: the device-resident WindowSearch(F1 = LastFrame, F2 = CurrentFrame, window, ., minOctave, maxOctave) of TrackPreviousFrame
(mcs_window_search_device), against the host composition cORBmatcher.WindowSearch (window search through the GPU mcs_search_windows
or the CPU oracle, vnMatches21 mapped to map-point ids) and, where oracle/_ref travelled, the reference's own method.  Both frames
come from packed feature buffers in every layout.  Results are compared after the slot -> contiguous conversion.  Integer work:
bit-exact."""
import numpy as np
import pytest

import acceptance_model as am
from device_frames import INT_MAX, SIZES, frames, keep_cameras, rm  # noqa: F401  (frames, rm: fixtures)
from device_searches import collect, device_ws, launch_ws
from search_scenes import CHAIN_DISTS, host_window_search, parity_scene, ratio_chain_scene

pytestmark = pytest.mark.gpu
# the windows and level filters of TrackPreviousFrame (ref src/cTracking.cpp:737-750), and one upper level bound
WINDOWS = [(60, 4, INT_MAX), (60, 1, INT_MAX), (50, 0, INT_MAX), (60, 0, 3)]


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
    s = parity_scene(api, oa, cams, frames)
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
    gn, gout, status, diag = device_ws(api, m, F2, F1, mp1, bad, *win, layout=layout)
    assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)
    # the map point on two last-frame keypoints makes two queries (no first-occurrence rule here)
    assert mp1[s["sc"]["src"][5]] == mp1[s["sc"]["src"][4]] and diag[2] == _n_queries(F1, mp1, bad, win[1], win[2])
    assert hn > (0 if win[1] == 4 else 50)


def test_empty_cameras_and_untouched_slots(api, oa, frames, cams):
    """camera 1 has no keypoints in either frame, camera 2 none in the last frame; slots beyond each count stay as they were"""
    s = parity_scene(api, oa, cams, frames)
    F1, i1 = keep_cameras(api, s["F1"], [0])
    F2, _ = keep_cameras(api, s["F2"], [0, 2])
    mp1, bad = s["mp1"][i1], s["sc"]["bad"]
    m = api.cORBmatcher(0.8, False, 32, True)
    hn, hout = host_window_search(m, F1, F2, mp1, bad, 60, 0, INT_MAX)
    for layout in ("single", "parts", "shared"):
        gn, gout, status, _ = device_ws(api, m, F2, F1, mp1, bad, 60, layout=layout)
        assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout) and hn > 20
        assert np.all(gout[F2.key_cam == 2] == -1)           # a camera with no queries is still cleared


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
    for win in ((60, 1, INT_MAX), (50, 0, INT_MAX)):
        hn, hout = host_window_search(m, s["F1"], s["F2"], s["mp1"], s["sc"]["bad"], *win)
        on, oout = host_window_search(m, s["F1"], s["F2"], s["mp1"], s["sc"]["bad"], *win, sw=oa.search_windows)
        assert hn == on and np.array_equal(hout, oout) and hn > 20
        for layout in ("single", "parts"):
            gn, gout, status, _ = device_ws(api, m, s["F2"], s["F1"], s["mp1"], s["sc"]["bad"], *win, layout=layout)
            assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)


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
        gn, gout, status, diag = device_ws(api, m, Fc, Fl, mp_last, bad, 50, layout=layout)
        assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)
        assert diag.tolist() == pdiag          # rounds run, walk start, queries and rescans as the model of the rounds and walk has them


def test_invalid_ids_drop_only_their_query(api, oa, frames, cams):
    s = parity_scene(api, oa, cams, frames)
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
        gn, gout, status, _ = device_ws(api, m, s["F2"], F1, mp_bad, bad, *win, last_keys=keys)
        assert status == api.MCS_ERR_INVALID and gn == hn and np.array_equal(gout, hout)
        gn, gout, status, _ = device_ws(api, m, s["F2"], F1, dropped, bad, *win, last_keys=keys)
        assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout)


def test_call_does_not_wait_for_the_stream(api, oa, frames, cams):
    import torch
    s = parity_scene(api, oa, cams, frames)
    m = api.cORBmatcher(0.8, False, 32, True)
    hn, hout = host_window_search(m, s["F1"], s["F2"], s["mp1"], s["sc"]["bad"], 60, 1, INT_MAX)
    d = device_ws(api, m, s["F2"], s["F1"], s["mp1"], s["sc"]["bad"], 60, 1, run=False)
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda._sleep(400_000_000)                  # a few hundred milliseconds of work ahead of the call
        res = launch_ws(m, d, stream=st)
        busy = st.query()
    assert busy is False
    st.synchronize()
    gn, gout, status, _ = collect(api, d, *res)
    assert gn == hn and status == api.MCS_OK and np.array_equal(gout, hout)
