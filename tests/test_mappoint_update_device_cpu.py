"""CPU: mcs_update_mappoints_device checks its arguments on the host before any launch, and without a device the accepted shapes fail
with MCS_ERR_NO_DEVICE.  The host mirrors the device call is compared with, api.ComputeDistinctiveDescriptors and
api.UpdateNormalAndDepth, reproduce the reference's own cMapPoint methods bit for bit (recorded in
tests/golden/ref_tape_mappoint_update_device_cpu.*) on the scenes the GPU tests use."""
import ctypes as C
import math

import numpy as np
import pytest

import mappoint_scenes as S
from device_frames import FAKE, taped_rm
from mappoint_scenes import SCENES, named_scene

rm = taped_rm("mappoint_update_device_cpu", "ref_mappoint_api", 256)


def test_exported_symbol_and_layout(api):
    from multicol_slam_b200.ctypes_defs import MpKeyFrame, PackedFrame
    assert hasattr(api.lib(), "mcs_update_mappoints_device")
    assert C.sizeof(PackedFrame) == 24 and C.sizeof(MpKeyFrame) == 24 + 24 + 8
    assert MpKeyFrame.ow.offset == 24 and MpKeyFrame.bad.offset == 48


def _call(api, n_kf=2, frame=(FAKE, 1, 6, 0), n_cams=3, capacity=64, dim=32, n_levels=8, sf=True, what=3, masks=1, ids=FAKE, n_upd=5,
          n_points=100, off=FAKE, okf=FAKE, oslot=FAKE, ref=FAKE, bad=None, world=FAKE, desc=FAKE, dmask=FAKE, normal=FAKE, dmin=FAKE,
          dmax=FAKE, status=FAKE, kfs=True):
    from multicol_slam_b200.ctypes_defs import MpKeyFrame, PackedFrame
    ks = (MpKeyFrame * max(n_kf, 1))()
    for i, k in enumerate(ks):
        k.frame = PackedFrame(frame[0], frame[1], frame[2], frame[3] if i == 0 else min(frame[3] + 3, frame[1] * frame[2] - n_cams))
    s = np.ascontiguousarray([1.2 ** i for i in range(max(n_levels, 1))], np.float64)
    return api.lib().mcs_update_mappoints_device(ks if kfs else None, n_kf, n_cams, capacity, dim, n_levels, api._p(s) if sf else None,
                                                 what, masks, ids, n_upd, n_points, off, okf, oslot, ref, bad, world, desc, dmask, normal,
                                                 dmin, dmax, status, None)


def test_refusals_before_any_launch(api):
    bad = [dict(kfs=False), dict(sf=False), dict(ids=None), dict(off=None), dict(okf=None), dict(oslot=None), dict(status=None),
           dict(desc=None), dict(dmask=None), dict(ref=None), dict(world=None), dict(normal=None), dict(dmin=None), dict(dmax=None),
           dict(what=0), dict(what=4), dict(what=-1), dict(n_kf=0), dict(n_levels=0), dict(n_levels=17), dict(n_upd=-1),
           dict(n_points=-1), dict(n_cams=0), dict(capacity=0), dict(capacity=65536), dict(dim=24), dict(dim=0),
           dict(frame=(0, 1, 6, 0)), dict(frame=(FAKE, 1, 6, 4)), dict(frame=(FAKE, 0, 6, 0)), dict(frame=(FAKE, 1, 6, -1)),
           dict(what=2, ref=None), dict(what=1, desc=None), dict(what=1, masks=1, dmask=None)]
    for kw in bad:
        assert _call(api, **kw) == api.MCS_ERR_INVALID, kw
    # what the selection leaves out may be NULL; dmask without masks; ids without entries
    ok = [dict(), dict(what=1, ref=None, world=None, normal=None, dmin=None, dmax=None), dict(what=2, desc=None, dmask=None),
          dict(what=1, masks=0, dmask=None, ref=None, world=None, normal=None, dmin=None, dmax=None), dict(ids=None, n_upd=0),
          dict(bad=FAKE), dict(dim=16), dict(dim=64), dict(frame=(FAKE, 6, 1, 3))]
    if api.device_count() == 0:
        for kw in ok:
            assert _call(api, **kw) == api.MCS_ERR_NO_DEVICE, kw


def _ref_order(obs, order):
    """obs regrouped into the key-frame order mObservations iterated in (each key frame's slots keep their order)"""
    return [e for k in order for e in obs if e[0] == k]


def _reference(rm, sc, masks):
    """per point: (obs in the reference's order, desc_set, mask_set, desc, dmask, nd) from the reference's own cMapPoint"""
    out = []
    for p, obs in enumerate(sc["obs"]):
        ds, ms, d, m, nd, order = rm.update(sc["desc"], sc["dmask"], sc["octave"], sc["ow"], sc["kf_bad"], sc["sf"],
                                            np.array([k for k, _ in obs], np.int32), np.array([s for _, s in obs], np.int32),
                                            int(sc["ref"][p]), sc["X"][p], int(sc["bad"][p]), 3, int(masks), sc["n_cams"], sc["capacity"])
        d, m = (np.frombuffer(bytes.fromhex(h), np.uint8) for h in (d, m))
        out.append((_ref_order(obs, order) if not sc["bad"][p] else obs, ds, ms, d, m, np.frombuffer(bytes.fromhex(nd), np.float64)))
    return out


@pytest.mark.parametrize("name", sorted(SCENES))
def test_mirrors_equal_reference(api, rm, name):
    sc, masks = named_scene(name)
    for p, (obs, ds, ms, d, m, nd) in enumerate(_reference(rm, sc, masks)):
        b = api.ComputeDistinctiveDescriptors(obs, sc["desc"], sc["kf_bad"], masks, sc["dmask"], bad=bool(sc["bad"][p]))
        assert (b is not None) == ds, (name, p)
        if b is not None:
            k, s = obs[b]
            assert np.array_equal(sc["desc"][k, s], d), (name, p)
            assert ms == masks and (not masks or np.array_equal(sc["dmask"][k, s], m)), (name, p)
        r = api.UpdateNormalAndDepth(obs, sc["ow"], int(sc["ref"][p]), sc["X"][p], sc["octave"], sc["sf"], bad=bool(sc["bad"][p]))
        if r is None:
            assert nd.tobytes() == np.zeros(5).tobytes(), (name, p)          # the constructor's values: nothing changed
        else:
            got = np.array([*r[0], r[1], r[2]])
            assert got.tobytes() == nd.tobytes(), (name, p, got, nd)          # bit for bit, NaN included


def test_scenes_reach_their_edges(api):
    """the scenes hold a point where only the upper-triangle median gives the mirror's (= the reference's) row, a median tie the
    first row wins, a point whose normal differs when Vec / n is a true division, points without observations (NaN normal) and
    ref key frames that do not observe their point"""
    upper_only = ties = division = nan = level1 = 0
    for name in sorted(SCENES):
        sc, masks = named_scene(name)
        for p, obs in enumerate(sc["obs"]):
            if sc["bad"][p]:
                continue
            rows = [e for e in obs if not sc["kf_bad"][e[0]]]
            if len(rows) > 2:
                b = obs[api.ComputeDistinctiveDescriptors(obs, sc["desc"], sc["kf_bad"], masks, sc["dmask"])]
                dist = [[api._dist64(sc["desc"][a], sc["desc"][b], *((sc["dmask"][a], sc["dmask"][b]) if masks else ()))
                         for b in rows] for a in rows]
                full = [sorted(dist[i][:i] + dist[i][i + 1:])[(len(rows) - 1) // 2] for i in range(len(rows))]
                upper = [sorted(dist[i][i + 1:])[(len(rows) - 1 - i) // 2] for i in range(len(rows) - 1)]
                assert rows[upper.index(min(upper))] == b
                upper_only += not np.array_equal(sc["desc"][rows[full.index(min(full))]], sc["desc"][b])
                ties += upper.count(min(upper)) > 1
            nd = api.UpdateNormalAndDepth(obs, sc["ow"], int(sc["ref"][p]), sc["X"][p], sc["octave"], sc["sf"])[0]
            kfs = list(dict.fromkeys(k for k, _ in obs))
            if kfs:
                X, acc = sc["X"][p], np.zeros(3)
                for k in kfs:
                    v = [float(X[i] - sc["ow"][k][i]) for i in range(3)]
                    nr = math.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])
                    acc = [acc[i] + v[i] / nr for i in range(3)]
                division += np.array([a / len(kfs) for a in acc]).tobytes() != nd.tobytes()
            nan += bool(not kfs and np.isnan(nd).all())
            level1 += int(sc["ref"][p]) not in {k for k, _ in obs}
    assert upper_only > 0 and ties > 0 and division > 0 and nan > 0 and level1 > 0, (upper_only, ties, division, nan, level1)


def test_host_route_checks(api):
    """update_mappoints_host: the refusals of the device kernel, the point left untouched and the others written"""
    sc = S.scene(7, n_random=4)
    n = len(sc["obs"])
    obs = [list(o) for o in sc["obs"]]
    ok_ids = [i for i in range(n) if len({k for k, _ in obs[i]}) >= 2 and not sc["bad"][i]]
    a, b, c, d, e = ok_ids[:5]
    obs[a] = obs[a] + [obs[a][0]]                                      # key frame's observations not adjacent
    obs[b] = [(len(sc["ow"]), 0)] + obs[b][1:]                         # key frame out of range
    k, s = obs[c][0]
    obs[c] = [(k, (s // sc["capacity"]) * sc["capacity"] + int(sc["kf_counts"][k, s // sc["capacity"]]))] + obs[c][1:]   # beyond count
    sc["ref"][d] = -1                                                  # ref key frame out of range
    ids = np.array([a, b, c, d, e, n, -1], np.int32)
    st, t = S.host_update(api, sc, ids, 3, True, obs=obs)
    assert st == api.MCS_ERR_INVALID
    fresh = S.fill_tables(n, sc["dim"])
    for i in (a, b, c, d):
        assert all(np.array_equal(x[i], y[i]) for x, y in zip(t, fresh)), i
    assert not np.array_equal(t[2][e], fresh[2][e])
    st, t = S.host_update(api, sc, np.array([d], np.int32), 1, False)  # the ref key frame is read by MCS_MP_NORMAL_DEPTH only
    assert st == api.MCS_OK
