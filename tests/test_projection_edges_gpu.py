"""GPU: the projection kernels (frustum_kernel through mcs_project_mappoints and mcs_project_mappoints_device, pl_project_kernel
through mcs_search_by_projection_last_device; both call cam_project_in_mask) on the edge scenes of tests/test_projection_edges_cpu.py,
and the device-vs-host divergence of the projection measured on dense ray grids.

The device atan is CUDA's, the host's is the libm's, so proj_x / proj_y are not bit-identical.  What is asserted:
- in_view, level and view_cos equal the oracle's exactly, except where an in_view decision flips; a flip must be explained by the
  device u / v (the side that has one) differing from the host's and rounding differently, or by a host u / v within the measured
  bound of a cvRound tie;
- proj_x / proj_y within MAX_ULPS_EDGES / MAX_ULPS_GRID of the host's (the largest distance measured on an H100, see DESIGN.md section 2), reported
  next to the distances of both from the 200-bit projections of tests/golden/projection_edges_mp200.npz;
- the motion-model search on map points at the mask, border and .5-tie edges and current keypoints on its window borders equals
  the host composition, except for queries whose device centre differs from the host's.
"""
import json
import pathlib

import numpy as np
import pytest

import test_projection_edges_cpu as E

pytestmark = pytest.mark.gpu
GOLD = pathlib.Path(__file__).resolve().parent / "golden"
# device vs host proj_x / proj_y, the largest distances measured on an H100 (DESIGN.md section 2).  Counted in ulps of u / v
# itself, so they are large where u or v is near 0: the absolute differences are printed next to them.
MAX_ULPS_EDGES = 512
MAX_ULPS_GRID = 2048
TIE_SLACK = 1e-9               # a host u / v this close to a .5 tie may round the other way on the device


def ordered(a):
    i = np.ascontiguousarray(a, np.float64).view(np.int64).astype(object)
    return np.where(i < 0, -(2 ** 63) - i, i)


def ulps(a, b):
    """distance in units in the last place between finite doubles"""
    return np.abs(ordered(a) - ordered(b)).astype(np.float64)


def near_tie(x):
    return np.isfinite(x) & (np.abs(np.abs(x - np.floor(x)) - 0.5) < TIE_SLACK)


def _device(api, sc, skip=None, out=None, dmax=None):
    import torch
    pos, nrm, dmin, dmx = sc.arrays()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    d = api.project_mappoints_device(sc.inv, sc.mtmc, sc.cams, t(sc.masks), t(pos), t(nrm), t(dmin), t(dmx if dmax is None else dmax),
                                     sc.sf, skip_t=None if skip is None else t(skip), out=out)
    torch.cuda.synchronize()
    return d


def _np(d):
    return tuple(x.cpu().numpy() for x in d)


def compare(o, g, host_uv):
    """-> (n points where device u / v != host, largest ulp distance, largest absolute difference, in_view flips, unexplained
    flips); o oracle, g device outputs"""
    ov, gv = o[0].astype(bool), g[0].astype(bool)
    both = ov & gv
    assert np.array_equal(o[1][both], g[1][both]) and np.array_equal(E.bits(o[4][both]), E.bits(g[4][both]))
    du = E.bits(o[2][both]) != E.bits(g[2][both])
    dv = E.bits(o[3][both]) != E.bits(g[3][both])
    n_diff = int((du | dv).sum())
    worst, worst_px = 0.0, 0.0
    if both.any():
        worst = max(ulps(o[2][both], g[2][both]).max(), ulps(o[3][both], g[3][both]).max())
        worst_px = float(max(np.abs(o[2][both] - g[2][both]).max(), np.abs(o[3][both] - g[3][both]).max()))
    bad = []
    for i, c in np.argwhere(ov != gv):
        hu, hv = host_uv[i, c]
        if gv[i, c]:               # device in view: its u / v must round to another pixel than the host's
            explained = (E.cv_round(g[2][i, c]), E.cv_round(g[3][i, c])) != (E.cv_round(hu), E.cv_round(hv))
        else:                      # device out: the host value sits on a tie the device may round the other way
            explained = bool(near_tie(hu) or near_tie(hv))
        if not explained:
            bad.append((int(i), int(c), hu, hv))
    return n_diff, worst, worst_px, int((ov != gv).sum()), bad


@pytest.mark.parametrize("name", E.SCENE_NAMES)
def test_edge_scenes_against_oracle_host_and_mp200(api, oa, name):
    sc = E.scenes()[name]
    o = E.oracle_is_in_frustum(oa, sc)
    huv = E.host_projection(sc)
    g = api.project_mappoints(sc.inv, sc.mtmc, sc.cams, sc.masks, *sc.arrays(), sc.sf)
    d = _np(_device(api, sc))
    for k in range(5):                               # the two entry points run the same kernel
        assert np.array_equal(g[k], d[k]) if g[k].dtype != np.float64 else np.array_equal(E.bits(g[k]), E.bits(d[k]))
    n_diff, worst, worst_px, flips, bad = compare(o, g, huv)
    assert not bad, f"{name}: in_view differs without a differing projection: {bad[:5]}"
    assert worst <= MAX_ULPS_EDGES, (name, worst)
    # skip: flagged points keep what the previous call left (here: everything out of range, all zeros)
    rng = np.random.default_rng(len(name))
    skip = (rng.random(len(sc.rows)) < 0.5).astype(np.uint8)
    first = _device(api, sc, dmax=np.zeros(len(sc.rows)))
    s = _np(_device(api, sc, skip=skip, out=first))
    for k in range(5):
        assert not s[k][skip == 1].any() and np.array_equal(s[k][skip == 0], d[k][skip == 0])
    # against the 200-bit projections
    mp = np.load(E.MP200)[f"{name.replace('/', '__')}__uv"]
    iv = g[0].astype(bool)
    host_mp = ulps(huv[..., 0][iv], mp[..., 0][iv]).max(initial=0), ulps(huv[..., 1][iv], mp[..., 1][iv]).max(initial=0)
    dev_mp = ulps(g[2][iv], mp[..., 0][iv]).max(initial=0), ulps(g[3][iv], mp[..., 1][iv]).max(initial=0)
    print(f"\n{name}: {iv.sum()} in view, {n_diff} with device u/v != host (max {worst:.0f} ulp, {worst_px:.2e} px), {flips} in_view flips; "
          f"ulp from 200-bit: host {max(host_mp):.0f}, device {max(dev_mp):.0f}")


def _grid_cameras():
    from multicol_slam_b200 import synth
    syn = [{k: v for k, v in c.items() if k != "name"} for c in json.loads((GOLD / "synthetic_cams.json").read_text())]
    return [dict(c, mirror_mask=0) for c in list(synth.lafida_cams()) + syn]


def test_divergence_on_dense_ray_grids(api, oa):
    """rays through a grid of pixels over each camera's whole image (Lafida's three, the seven synthetic ones), at two depths and
    behind the camera; all-ones masks so that only the border decides.  Device u / v vs host: count and largest ulp distance"""
    total, total_diff, worst_all, px_all, flips_all = 0, 0, 0.0, 0.0, 0
    for cam in _grid_cameras():
        w, h = cam["width"], cam["height"]
        step = max(w, h) / 240.0
        us, vs = np.meshgrid(np.arange(0.75, w - 0.5, step), np.arange(0.75, h - 0.5, step))
        rays = np.array([api.img_to_world(cam, float(u), float(v)) for u, v in zip(us.ravel(), vs.ravel())])
        pos = np.concatenate([rays * 0.7, rays * 13.3, -rays * 2.1])
        n = len(pos)
        nrm = np.tile([0.0, 0.0, 1.0], (n, 1))
        args = (np.eye(4)[None], np.eye(4)[None], [cam], np.ones((1, h, w), np.uint8), pos, nrm,
                np.full(n, 1e-3), np.full(n, 1e3), E.SF12)
        o = oa.project_mappoints(*args)
        g = api.project_mappoints(*args)
        huv = np.stack([o[2], o[3]], axis=-1)
        need = (o[0] == 0) & (g[0] == 1)                       # host out, device in: the host u / v, for the flip check
        for i in np.flatnonzero(need[:, 0]):
            huv[i, 0] = api.world_to_img(cam, *pos[i])
        n_diff, worst, worst_px, flips, bad = compare(o, g, huv)
        assert not bad, f"{cam['width']}x{cam['height']}: in_view differs without a differing projection: {bad[:5]}"
        print(f"\ncamera {w}x{h} u0 {cam['u0']:.1f}: {int(o[0].sum())} of {n} in view, {n_diff} with device u/v != host, "
              f"max {worst:.0f} ulp, {worst_px:.2e} px, {flips} in_view flips")
        total += int(o[0].sum()); total_diff += n_diff; flips_all += flips
        worst_all, px_all = max(worst_all, worst), max(px_all, worst_px)
    print(f"\nall cameras: {total} projections, {total_diff} differ ({100.0 * total_diff / total:.3f} %), max {worst_all:.0f} ulp, "
          f"{px_all:.2e} px, {flips_all} in_view flips")
    assert worst_all <= MAX_ULPS_GRID and total > 500_000


# ---- the motion-model search at the same edges ---------------------------------------------------------------------------------
def _motion_scene(api, rng, th):
    """cameras: Lafida 0 with its mask, and with an all-ones mask; map points: the border / mask / tie points of the identity-pose
    edge scenes; one last-frame keypoint per map point (its camera, a random octave), and per point eight current keypoints on the
    float32 extremes of its window (th * sf[octave] about the host projection) and one float beyond: the ones beyond carry the
    closer descriptors, so a window that takes one in changes the match"""
    from test_window_edges_cpu import _f32_boundary
    scs = [E.scenes()["lafida0/identity"], E.scenes()["lafida0_open/identity"]]
    cams = [scs[0].cams[0], scs[1].cams[0]]
    rig = api.Rig(cams)
    dim = 32
    world, last, cur = [], [[], []], [[], []]
    for c, sc in enumerate(scs):
        pos = sc.arrays()[0]
        for i, L in enumerate(sc.labels):
            if not L.startswith(("border", "mask")):
                continue
            u, v, _ = rig.world_to_cam(c, pos[i])
            if not rig.in_mirror_mask(c, u, v):
                continue
            p = len(world)
            world.append(pos[i])
            oct_ = int(rng.integers(0, 8)) if rng.random() < 0.6 else 0
            base = rng.integers(0, 256, dim).astype(np.uint8)
            last[c].append((p, oct_, base))
            r = th * float(E.SF12[oct_])
            for sign in (-1, 1):
                ix, ox = _f32_boundary(u, r, sign)
                iy, oy = _f32_boundary(v, r, sign)
                for (kx, ky), dist in (((ix, v), 20), ((u, iy), 22), ((ox, v), 4), ((u, oy), 6)):
                    cur[c].append((float(kx), float(ky), oct_, _flip(rng, base, dist + int(rng.integers(0, 2)))))
    sf = E.SF12

    def frame(rows, key):
        per = []
        for c in range(2):
            k = np.zeros(len(rows[c]), api.KEYPOINT_DTYPE)
            if key == "last":
                k["x"], k["y"] = 300.0, 200.0
                k["octave"] = [o for _, o, _ in rows[c]]
                d = np.array([b for _, _, b in rows[c]], np.uint8).reshape(-1, dim)
            else:
                k["x"] = [r[0] for r in rows[c]]; k["y"] = [r[1] for r in rows[c]]; k["octave"] = [r[2] for r in rows[c]]
                d = np.array([r[3] for r in rows[c]], np.uint8).reshape(-1, dim)
            k["size"] = 31.0
            per.append((k, d, None))
        return api.Frame.from_cameras(per, [(754, 480)] * 2, sf)
    Fl, Fc = frame(last, "last"), frame(cur, "cur")
    mp_last = np.array([p for c in range(2) for p, _, _ in last[c]], np.int32)
    return rig, Fl, Fc, np.array(world), mp_last


def _flip(rng, d, nbits):
    out = d.copy()
    for b in rng.choice(8 * len(d), nbits, replace=False):
        out[b // 8] ^= 1 << (b % 8)
    return out


@pytest.mark.parametrize("th", [1.0, 3.0])
def test_motion_model_search_at_the_edges(api, oa, th):
    from test_search_projection_last_device_gpu import _device_last
    rng = np.random.default_rng(int(th * 10))
    rig, Fl, Fc, world, mp_last = _motion_scene(api, rng, th)
    m = api.cORBmatcher(0.8, False, 32, False)
    bad = np.zeros(len(world), np.uint8)
    mp_cur = np.full(len(Fc.keys), -1, np.int32)
    hn, hout = m.SearchByProjectionLastRig(Fc, rig, mp_cur, Fl, mp_last, None, world, bad, th)
    on, oout = m.SearchByProjectionLastRig(Fc, rig, mp_cur, Fl, mp_last, None, world, bad, th, _sw=oa.search_windows)
    assert hn == on and np.array_equal(hout, oout)
    # the device centres: frustum_kernel runs the same cam_project_in_mask as pl_project_kernel
    n = len(world)
    div = set()
    for c in range(2):
        pts = mp_last[Fl.key_cam == c]
        g = api.project_mappoints(rig.MtMc_inv[c:c + 1], rig.MtMc[c:c + 1], [rig.cams[c]], rig.masks[c][None], world[pts],
                                  np.tile([0.0, 0.0, 1.0], (len(pts), 1)), np.zeros(len(pts)), np.full(len(pts), np.inf), E.SF12)
        for j, p in enumerate(pts):
            u, v, _ = rig.world_to_cam(c, world[p])
            host_in = rig.in_mirror_mask(c, u, v)
            if bool(g[0][j, 0]) != host_in or (host_in and (g[2][j, 0] != u or g[3][j, 0] != v)):
                div.add(int(p))
    gn, gout, status, _ = _device_last(api, m, Fc, Fl, rig, mp_cur, mp_last, None, world, bad, th)
    assert status == api.MCS_OK
    keep = ~np.isin(hout, list(div)) & ~np.isin(gout, list(div))
    print(f"\nth {th}: {n} map points, {len(Fc.keys)} current keypoints, {hn} host matches, {gn} device matches, "
          f"{len(div)} queries whose device centre differs from the host's")
    assert np.array_equal(gout[keep], hout[keep])
    if not div:
        assert gn == hn and np.array_equal(gout, hout)
    assert hn > 20
