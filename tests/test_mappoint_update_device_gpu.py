"""GPU: mcs_update_mappoints_device (ComputeDistinctiveDescriptors / UpdateNormalAndDepth for many map points) writes exactly the
bytes the host mirrors write (api.update_mappoints_host, which tests/test_mappoint_update_device_cpu.py checks against the
reference's own cMapPoint): every scene of tests/mappoint_scenes.py, each packed layout, each `what`, masks on and off, invalid
inputs, repeated ids and a busy stream.  The tables it writes feed mcs_project_mappoints_device unchanged."""
import numpy as np
import pytest

import mappoint_scenes as S
from device_frames import on_device
from mappoint_scenes import SCENES, named_scene

pytestmark = pytest.mark.gpu


def _device(api, sc, layout, ids, what, masks, obs=None, ref=None, stream=None, busy=False):
    import torch
    kfs = [(fr, sc["ow"][k], sc["kf_bad"][k]) for k, fr in enumerate(S.packed_frames(sc, layout))]
    off, okf, oslot = api.mappoint_obs_csr(sc["obs"] if obs is None else obs)
    tables = [on_device(t) for t in S.fill_tables(len(off) - 1, sc["dim"])]
    args = [on_device(np.asarray(ids, np.int32)), on_device(off), on_device(okf), on_device(oslot)]
    ref_t, world_t, bad_t = on_device(sc["ref"] if ref is None else ref), on_device(sc["X"]), on_device(sc["bad"])
    torch.cuda.synchronize()
    if busy:
        with torch.cuda.stream(stream):
            torch.cuda._sleep(50_000_000)                  # the call is queued behind ~tens of ms of work on its stream
    st = api.update_mappoints_device(kfs, sc["n_cams"], sc["capacity"], sc["sf"], *args, what=what, having_masks=masks, desc_t=tables[0],
                                     dmask_t=tables[1], normal_t=tables[2], min_dist_t=tables[3], max_dist_t=tables[4], ref_kf_t=ref_t,
                                     world_t=world_t, bad_t=bad_t, dim=sc["dim"], stream=stream)
    torch.cuda.synchronize()
    return int(st.item()), [t.cpu().numpy() for t in tables]


def _same(a, b):
    return all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def _all_ids(n, seed=0):
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.permutation(n), rng.integers(0, n, 9)])  # every point, in a shuffled order, and repeats


@pytest.mark.parametrize("layout", ["one", "parts", "separate"])
@pytest.mark.parametrize("name", sorted(SCENES))
def test_device_equals_mirror(api, name, layout):
    sc, masks = named_scene(name)
    ids = _all_ids(len(sc["obs"]))
    st_h, t_h = S.host_update(api, sc, ids, 3, masks)
    st_d, t_d = _device(api, sc, layout, ids, 3, masks)
    assert st_h == st_d == api.MCS_OK
    assert _same(t_h, t_d), name


@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("what", [1, 2, 3])
def test_what_selects_the_arrays(api, what, masks):
    """each `what` writes only its arrays, dmask only with masks; a subset of the points, the others keep their rows"""
    sc, _ = named_scene("d32_masks")
    ids = np.arange(0, len(sc["obs"]), 2)
    st_h, t_h = S.host_update(api, sc, ids, what, masks)
    st_d, t_d = _device(api, sc, "one", ids, what, masks)
    assert st_h == st_d == api.MCS_OK and _same(t_h, t_d)
    fresh = S.fill_tables(len(sc["obs"]), sc["dim"])
    untouched = ([] if what & 1 else [0, 1]) + ([] if masks and what & 1 else [1]) + ([] if what & 2 else [2, 3, 4])
    for i in untouched:
        assert t_d[i].tobytes() == fresh[i].tobytes(), i
    if what & 1:
        assert t_d[0].tobytes() != fresh[0].tobytes()


def test_invalid_points_are_left_untouched(api):
    sc, masks = named_scene("d32_masks")
    n = len(sc["obs"])
    obs = [list(o) for o in sc["obs"]]
    cand = [i for i in range(n) if len({k for k, _ in obs[i]}) >= 2 and not sc["bad"][i] and sc["ref"][i] in {k for k, _ in obs[i]}]
    a, b, c, d, e, f, g = cand[:7]
    obs[a] = obs[a] + [obs[a][0]]                                       # a key frame's observations not adjacent
    obs[b] = [(len(sc["ow"]), 0)] + obs[b][1:]                          # obs_kf out of range
    k, s = obs[c][0]
    cam = s // sc["capacity"]
    obs[c] = [(k, cam * sc["capacity"] + int(sc["kf_counts"][k, cam]))] + obs[c][1:]     # slot at its camera's count
    ref = sc["ref"].copy()
    ref[d] = len(sc["ow"])                                              # ref_kf out of range
    sc = dict(sc, octave=sc["octave"].copy())
    kk, ss = next(x for x in obs[e] if x[0] == ref[e])
    sc["octave"][kk, ss] = sc["n_levels"]                               # the level read lies outside [0, n_levels)
    kk, ss = next(x for x in obs[f] if x[0] == ref[f])
    sc["octave"][kk, ss] = -1
    sc["ref"] = ref
    ids = np.array([a, b, c, d, e, f, g, n, -3, g], np.int32)           # g is valid; n and -3 are ids out of range
    st_h, t_h = S.host_update(api, sc, ids, 3, masks, obs=obs)
    st_d, t_d = _device(api, sc, "parts", ids, 3, masks, obs=obs)
    assert st_h == st_d == api.MCS_ERR_INVALID and _same(t_h, t_d)
    fresh = S.fill_tables(n, sc["dim"])
    for i in (a, b, c, d, e, f):
        assert all(x[i].tobytes() == y[i].tobytes() for x, y in zip(t_d, fresh)), i
    assert all(x[g].tobytes() != y[g].tobytes() for x, y in zip(t_d, fresh))
    # each refusal alone raises the status
    for bad_id in (a, b, c, d, e, f, n):
        st, _ = _device(api, sc, "one", np.array([g, bad_id], np.int32), 3, masks, obs=obs)
        assert st == api.MCS_ERR_INVALID, bad_id
    st, _ = _device(api, sc, "one", np.array([g], np.int32), 3, masks, obs=obs)
    assert st == api.MCS_OK
    st, _ = _device(api, sc, "one", np.array([d, e, f], np.int32), 1, masks, obs=obs)   # ref / level only read by NORMAL_DEPTH
    assert st == api.MCS_OK


def test_busy_stream_and_empty_call(api):
    import torch
    sc, masks = named_scene("ties")
    ids = _all_ids(len(sc["obs"]), 1)
    s = torch.cuda.Stream()
    st_h, t_h = S.host_update(api, sc, ids, 3, masks)
    st_d, t_d = _device(api, sc, "separate", ids, 3, masks, stream=s, busy=True)
    assert st_h == st_d == api.MCS_OK and _same(t_h, t_d)
    st_d, t_d = _device(api, sc, "one", np.zeros(0, np.int32), 3, masks)
    assert st_d == api.MCS_OK and _same(t_d, S.fill_tables(len(sc["obs"]), sc["dim"]))


def test_tables_feed_the_projection(api, cams):
    """mcs_project_mappoints_device gives the same outputs from the device-written normal / min / max tables as from the host's"""
    import torch
    sc, masks = named_scene("d32")
    ids = np.arange(len(sc["obs"]))
    keep = ~sc["bad"].astype(bool) & np.array([len(o) > 0 for o in sc["obs"]])      # rows the update writes with finite normals
    _, t_h = S.host_update(api, sc, ids, 3, masks)
    _, t_d = _device(api, sc, "one", ids, 3, masks)
    masks_t = on_device(np.stack([api.mirror_mask(c) for c in cams[:3]]))
    mi = np.tile(np.eye(4), (3, 1, 1))
    outs = []
    for t in (t_h, t_d):
        X = on_device(sc["X"][keep])
        outs.append(api.project_mappoints_device(mi, mi, cams[:3], masks_t, X, on_device(t[2][keep]), on_device(t[3][keep]), on_device(t[4][keep]), sc["sf"]))
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
