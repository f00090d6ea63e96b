"""Seeded scenes for the matcher's searches, with the host routes and the reference calls the CPU and GPU tests compare on them."""
import numpy as np

from device_frames import BIG_ID, SIZES, counts, flip, flip_bits, on_device, pack_frames, to_slots, widen


# ---- scenes with 3-D map points for the projection-based searches ---------------------------------------------------------------
def make_scene(api, oa, cams, frame, seed, npts=500, pose_noise=0.0):
    """A key frame = `frame` on a 3-camera rig, and map points that really project near its keypoints: each point sits on the
    bearing ray of a keypoint at a random depth; descriptor = that keypoint's with a few flipped bits."""
    rng = np.random.default_rng(seed)
    rig = rig_of(api, cams, [0, 0, 0])
    M_c, M_t = rig.M_c, rig.M_t
    rays, _, _ = oa.frame_prepare(frame.keys, frame.key_cam, cams)
    src = rng.choice(len(frame.keys), npts, replace=False)
    depth = rng.uniform(2.0, 6.0, npts)
    world = np.zeros((npts, 3))
    for i, k in enumerate(src):
        pc = np.append(rays[k] * depth[i], 1.0)
        world[i] = api._mm(rig.MtMc[int(frame.key_cam[k])], pc)[:3] + rng.normal(0, pose_noise, 3)
    desc = flip_bits(rng, frame.desc[src], 30)
    dmask = frame.dmask[src].copy()
    bad = (rng.random(npts) < 0.05).astype(np.uint8)
    min_d, max_d = depth * rng.uniform(0.5, 0.9, npts), depth * rng.uniform(1.2, 3.0, npts)
    return dict(rig=rig, M_c=M_c, M_t=M_t, rays=rays, src=src, world=world, desc=desc, dmask=dmask, bad=bad, min_d=min_d, max_d=max_d)


def fuse_scene(api, oa, cams, KF, variant, seed=5):
    """the scene of test_ref_match_cpu.py::test_fuse_equals_reference; variant 0 adds a current key frame: a second rig pose a few
    centimetres away whose keypoints carry the query points (their rays are the bearing rays of the points seen from it)"""
    sc = make_scene(api, oa, cams, KF, 11 + variant)
    rng = np.random.default_rng(seed)
    n = len(sc["world"])
    kf_mp = np.full(len(KF.keys), -1, np.int32)
    occupied = rng.choice(len(KF.keys), len(KF.keys) // 3, replace=False)
    extra_bad = (rng.random(len(occupied)) < 0.1).astype(np.uint8)
    kf_mp[occupied] = n + np.arange(len(occupied))
    bad = np.concatenate([sc["bad"], extra_bad])
    in_kf = np.concatenate([(rng.random(n) < 0.1), np.ones(len(occupied), bool)])
    pad = lambda a, fill=0.0: np.concatenate([a, np.full((len(occupied),) + a.shape[1:], fill, a.dtype)])  # noqa: E731
    s = dict(sc=sc, n=n, kf_mp=kf_mp, occupied=occupied, bad=bad, in_kf=in_kf, points=np.arange(n, dtype=np.int32),
             world=pad(sc["world"]), min_d=pad(sc["min_d"], 1.0), max_d=pad(sc["max_d"], 2.0), desc=pad(sc["desc"]), dmask=pad(sc["dmask"]),
             Scw=None, cur=None)
    if variant == 2:
        Scw = api.inv_rigid(sc["M_t"]).copy()
        Scw[:3, :3] *= 1.3
        Scw[:3, 3] *= 1.3
        s["Scw"] = Scw
    if variant == 0:
        # curKF: the same keypoints on a rig moved by a few cm; keypoint j of curKF carries points[j] (one key frame of map points
        # per keypoint, as vpMapPointMatches of curKF).  Rays: the point's bearing from the moved rig, jittered so that the
        # epipolar check both passes and fails among the occupied hits.
        M_t2 = sc["M_t"].copy()
        M_t2[:3, 3] += [0.03, -0.01, 0.02]
        cur_rig = api.Rig(cams, sc["M_c"], M_t2)
        rays = np.zeros((n, 3))
        for j in range(n):
            c = int(KF.key_cam[sc["src"][j]])
            pc = api._mm(cur_rig.MtMc_inv[c], np.append(sc["world"][j], 1.0))[:3]
            r = pc / np.linalg.norm(pc) + rng.normal(0, 0.08 if j % 2 else 0.0005, 3)
            rays[j] = r / np.linalg.norm(r)
        key_cam = np.asarray(KF.key_cam[sc["src"]], np.int32)
        s["cur"] = dict(rig=cur_rig, M_t=M_t2, rays=rays, key_cam=key_cam)
    return s


def reference_ops(api, rm, cams, KF, s, variant, masks):
    sc = s["sc"]
    table = rm.MPTable(3, s["desc"], dmask=s["dmask"], bad=s["bad"], world_pos=s["world"], min_dist=s["min_d"], max_dist=s["max_d"],
                       obs_kf=np.where(s["in_kf"], 0, -1).astype(np.int32), obs_idx=np.zeros(len(s["bad"]), np.int32))
    kfr = rm.KF(KF, cams, M_c=sc["M_c"], M_t=sc["M_t"], mp=s["kf_mp"], rays=sc["rays"])
    cur = None
    if variant == 0:
        Fc = api.Frame(KF.keys[sc["src"]], s["cur"]["key_cam"], KF.desc[sc["src"]], KF.dmask[sc["src"]], SIZES, KF.scale_factors)
        cur = rm.KF(Fc, cams, M_c=sc["M_c"], M_t=s["cur"]["M_t"], mp=s["points"], rays=s["cur"]["rays"])
    return rm.fuse(variant, kfr, table, s["points"], 2.5, 0.6, masks, CurK=cur, Scw=s["Scw"])


def host_fuse(api, m, KF, s, variant, _sw=None, **kw):
    sc = s["sc"]
    cur = s["cur"] or {}
    return m.Fuse(KF, sc["rig"], s["kf_mp"], s["points"], s["world"], s["min_d"], s["max_d"], s["bad"], s["in_kf"], s["desc"], s["dmask"],
                  th=2.5, variant=variant, Scw=s["Scw"], cur_rays=cur.get("rays"), kf_rays=sc["rays"], cur_rig=cur.get("rig"), _sw=_sw, **kw)


def second_view(api, KF, seed):
    """another key frame over the same keypoints: positions jittered by up to half a pixel, a few descriptor bits flipped"""
    rng = np.random.default_rng(seed)
    keys = KF.keys.copy()
    keys["x"] += rng.uniform(-0.5, 0.5, len(keys)).astype(np.float32)
    keys["y"] += rng.uniform(-0.5, 0.5, len(keys)).astype(np.float32)
    return api.Frame(keys, KF.key_cam.copy(), flip_bits(rng, KF.desc, 3), KF.dmask.copy(), list(zip(KF.cam_w, KF.cam_h)), KF.scale_factors)


def sim3_scene(api, oa, cams, KF1, seed=51, s12=1.01):
    """SearchBySim3 between KF1 and a second view KF2 of its keypoints from a rig pose a few centimetres away.  KF1 carries map points
    0..299 on its keypoints' rays, KF2 points 300..599 a few millimetres from them with descriptor variants of their own; a few
    bad points; the Sim3 is the true relative pose with s12 != 1.  Ten KF1 keypoints are matched beforehand to KF2 points whose
    keypoint in KF2 (obs_idx) is then vbAlreadyMatched2."""
    sc1 = make_scene(api, oa, cams, KF1, seed, npts=300)
    KF2 = second_view(api, KF1, seed + 1)
    rng = np.random.default_rng(seed + 2)
    M_t2 = sc1["M_t"].copy()
    M_t2[:3, 3] += [0.012, -0.008, 0.006]
    a = 0.002
    Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1.0]])
    M_t2[:3, :3] = api._mm(Rz, M_t2[:3, :3])
    rig2 = api.Rig(cams, sc1["M_c"], M_t2)
    world2 = sc1["world"] + rng.normal(0, 0.003, sc1["world"].shape)
    world = np.concatenate([sc1["world"], world2])
    desc = np.concatenate([sc1["desc"], flip_bits(rng, KF2.desc[sc1["src"]], 30)])
    dmask = np.concatenate([sc1["dmask"], KF2.dmask[sc1["src"]]])
    bad = np.concatenate([sc1["bad"], np.roll(sc1["bad"], 7)])
    # distance ranges whose predicted level is the point's keypoint octave + 1 (ratio 1.1 * scale factor): the window's levels
    # {l - 1, l} keep the keypoint, so that most queries find it
    cam = KF1.key_cam[sc1["src"]]
    depth = np.array([np.linalg.norm(api._mm(sc1["rig"].MtMc_inv[int(c)], np.append(x, 1.0))[:3]) for c, x in zip(cam, sc1["world"])])
    min1 = depth / (1.1 * np.asarray(KF1.scale_factors)[KF1.keys["octave"][sc1["src"]]])
    min_d = np.concatenate([min1, min1])
    max_d = min_d * 12.0
    mp1 = np.full(len(KF1.keys), -1, np.int32); mp1[sc1["src"]] = np.arange(300)
    mp2 = np.full(len(KF2.keys), -1, np.int32); mp2[sc1["src"]] = 300 + np.arange(300)
    T12 = api._mm(api.inv_rigid(sc1["M_t"]), M_t2)                 # KF2's rig frame -> KF1's: T1w * Tw2
    pre = np.full(len(KF1.keys), -1, np.int32)
    some = rng.choice(sc1["src"], 10, replace=False)
    pre[some] = 300 + rng.choice(300, 10, replace=False)
    obs_idx = np.concatenate([sc1["src"], sc1["src"]]).astype(np.int32)
    return dict(KF1=KF1, KF2=KF2, rig1=sc1["rig"], rig2=rig2, M_c=sc1["M_c"], M_t1=sc1["M_t"], M_t2=M_t2, world=world, desc=desc,
                dmask=dmask, bad=bad, min_d=min_d, max_d=max_d, mp1=mp1, mp2=mp2, s12=s12, R12=T12[:3, :3].copy(), t12=T12[:3, 3].copy(),
                pre=pre, obs_idx=obs_idx)


def reference_sim3(rm, cams, s, th, masks):
    obs_kf = np.concatenate([np.zeros(300, np.int32), np.ones(300, np.int32)])
    table = rm.MPTable(3, s["desc"], dmask=s["dmask"], bad=s["bad"], world_pos=s["world"], min_dist=s["min_d"], max_dist=s["max_d"],
                       obs_kf=obs_kf, obs_idx=s["obs_idx"])
    k1 = rm.KF(s["KF1"], cams, M_c=s["M_c"], M_t=s["M_t1"], mp=s["mp1"])
    k2 = rm.KF(s["KF2"], cams, M_c=s["M_c"], M_t=s["M_t2"], mp=s["mp2"])
    return rm.search_by_sim3(k1, k2, table, s["s12"], s["R12"], s["t12"], th, s["pre"], 0.6, masks)


def host_sim3(m, s, th, _sw=None, **kw):
    return m.SearchBySim3(s["KF1"], s["rig1"], s["mp1"], s["KF2"], s["rig2"], s["mp2"], s["world"], s["min_d"], s["max_d"], s["bad"],
                          s["desc"], s["dmask"], s["s12"], s["R12"], s["t12"], th, matches12=kw.get("pre", s["pre"]),
                          obs_idx2=s["obs_idx"], _sw=_sw)


def scw_scene(api, oa, cams, F, seed=33, cam0_only=True, scale=1.25):
    """SearchByProjection(pKF, Scw, vpPoints, vpMatched, th): loop points on the key frame's rays (entry i of vpPoints projects near
    keypoint src[i]), some NULL and some bad; vpMatched holds taken keypoints, some of them holding points of the list (already found).
    cam0_only: the key frame keeps camera 0's keypoints alone, where the reference's descriptor reads stay defined (contiguous id ==
    row)."""
    if cam0_only:
        sel = np.flatnonzero(F.key_cam == 0)
        KF = api.Frame(F.keys[sel], F.key_cam[sel], F.desc[sel], F.dmask[sel], SIZES, F.scale_factors)
    else:
        KF = F
    n_keys = len(KF.keys)
    sc = make_scene(api, oa, cams, KF, seed, npts=min(n_keys - 5, 400))
    n = len(sc["world"])
    rng = np.random.default_rng(seed + 1)
    points = np.arange(n, dtype=np.int32)
    points[rng.random(n) < 0.05] = -1
    matched = np.full(n_keys, -1, np.int32)
    taken = rng.choice(n_keys, 40, replace=False)
    matched[taken] = rng.choice(n, 40, replace=False)                # points of the list, now already found
    Scw = api.inv_rigid(sc["M_t"]).copy()
    Scw[:3, :3] *= scale
    Scw[:3, 3] *= scale
    return dict(KF=KF, sc=sc, rig=sc["rig"], M_c=sc["M_c"], M_t=sc["M_t"], world=sc["world"], desc=sc["desc"], dmask=sc["dmask"], bad=sc["bad"],
                min_d=sc["min_d"], max_d=sc["max_d"], points=points, matched=matched, Scw=Scw)


def reference_scw(rm, cams, s, masks):
    table = rm.MPTable(3, s["desc"], dmask=s["dmask"], bad=s["bad"], world_pos=s["world"], min_dist=s["min_d"], max_dist=s["max_d"])
    return rm.search_by_projection_scw(rm.KF(s["KF"], cams, M_c=s["M_c"], M_t=s["M_t"]), table, s["Scw"], s["points"], s["matched"], 10,
                                       0.6, masks)


def host_scw(m, s, _sw=None, **kw):
    return m.SearchByProjectionKFScw(s["KF"], s["rig"], s["Scw"], kw.get("points", s["points"]), kw.get("matched", s["matched"]), s["world"],
                                     s["min_d"], s["max_d"], kw.get("bad", s["bad"]), s["desc"], s["dmask"], th=kw.get("th", 10), _sw=_sw)


def max_count(s):
    """the most keypoints a camera of the scene's frames holds"""
    return max(max(counts(F)) for F in [s["KF1"]] + s["cands"])


def bow_kf_scene(api, frames, n_kf, seed=5, dim=32):
    """KF1 = the first frame, about 60 % of its keypoints carrying map points 0 ..; candidate k a variant of either frame (a few bits
    flipped per descriptor, more for later candidates) carrying points of its own; about 5 % of all points bad."""
    F1, F2 = frames
    rng = np.random.default_rng(seed)
    KF1 = widen(api, F1, dim)
    n1 = len(F1.keys)
    mp1 = np.where(rng.random(n1) < 0.6, np.arange(n1), -1).astype(np.int32)
    cands, mps, off = [], [], n1
    for k in range(n_kf):
        B = F2 if k % 2 else F1
        F = api.Frame(B.keys, B.key_cam, flip_bits(rng, B.desc, 2 + k % 6), B.dmask, list(zip(B.cam_w, B.cam_h)), B.scale_factors)
        cands.append(widen(api, F, dim))
        n = len(B.keys)
        mps.append(np.where(rng.random(n) < 0.6, off + np.arange(n), -1).astype(np.int32))
        off += n
    bad = (rng.random(off) < 0.05).astype(np.uint8)
    return dict(KF1=KF1, mp1=mp1, cands=cands, mps=mps, bad=bad, n_points=off)


def host_bow_kf(api, m, s, cap, layout="single", device="cpu", _bf=None, cands=None):
    """SearchByBoWKeyFramesHost on the scene -> (matches12, match_slot, nmatches, status)"""
    idx = range(len(s["cands"])) if cands is None else cands
    packs = pack_frames([s["KF1"]] + [s["cands"][k] for k in idx], cap, layout=layout, device=device)
    kfs = [(packs[1 + i], to_slots(api, s["cands"][k], s["mps"][k], cap, BIG_ID, device)) for i, k in enumerate(idx)]
    return m.SearchByBoWKeyFramesHost(packs[0], to_slots(api, s["KF1"], s["mp1"], cap, BIG_ID, device), kfs, len(s["KF1"].cam_w), cap,
                                      s["n_points"], on_device(s["bad"], device), _bf=_bf)


def reference_bow_kf(rm, cams, s, k, nnratio, masks):
    """the reference's SearchByBoW(KF1, KF_k): (nmatches, map-point id per KF1 keypoint in contiguous order)"""
    table = rm.MPTable(3, np.zeros((s["n_points"], 32), np.uint8), bad=s["bad"])
    return rm.search_by_bow_kfkf(rm.KF(s["KF1"], cams, mp=s["mp1"]), rm.KF(s["cands"][k], cams, mp=s["mps"][k]), table, nnratio, masks)


def parity_scene(api, oa, cams, frames, seed=61):
    """the scene of test_ref_match_cpu.py::test_projection_searches_between_frames_equal_reference"""
    F1, F2 = frames
    sc = make_scene(api, oa, cams, F1, seed, npts=600)
    n = 600
    mp1 = np.full(len(F1.keys), -1, np.int32); mp1[sc["src"]] = np.arange(n)
    mp1[sc["src"][5]] = mp1[sc["src"][4]]                       # one map point on two last-frame keypoints: searched twice
    rng = np.random.default_rng(9)
    M_t2 = sc["M_t"].copy()
    M_t2[:3, 3] += [0.004, -0.003, 0.002]
    rig2 = api.Rig(cams, sc["M_c"], M_t2)
    mp2 = np.full(len(F2.keys), -1, np.int32)
    mp2[rng.choice(len(F2.keys), 80, replace=False)] = rng.choice(n, 80, replace=False)      # pre-assigned current keypoints
    outlier = (rng.random(len(F1.keys)) < 0.1).astype(np.uint8)
    return dict(sc=sc, F1=F1, F2=F2, mp1=mp1, mp2=mp2, rig2=rig2, M_t2=M_t2, outlier=outlier)


def host_window_search(m, F1, F2, mp1, bad, window, lo, hi, sw=None):
    """cORBmatcher.WindowSearch with its vnMatches21 mapped to map-point ids through mp1 -> (nmatches, cur_mp)"""
    valid1 = (mp1 >= 0) & (np.asarray(bad)[np.maximum(mp1, 0)] == 0)
    n, v21 = m.WindowSearch(F1, F2, window, valid1, lo, hi, _sw=sw)
    return n, np.where(v21 >= 0, mp1[np.maximum(v21, 0)], -1).astype(np.int32)


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
    dc = np.stack([flip(rng, base, d) for d in rng.permutation(CHAIN_DISTS)])
    e = np.zeros(0, api.KEYPOINT_DTYPE), np.zeros((0, dim), np.uint8), None
    sf = np.cumprod([1.0] + [1.2000000476837158] * 7)
    Fl = api.Frame.from_cameras([(kl, np.tile(base, (n_last, 1)), None), e, e], SIZES, sf)
    Fc = api.Frame.from_cameras([(kc, dc, None), e, e], SIZES, sf)
    return Fc, Fl, rig, world, np.arange(n_last, dtype=np.int32)


def rig_of(api, cams, shift):
    """make_scene's 3-camera rig at a pose moved by `shift` metres"""
    nc = 3
    M_c = np.tile(np.eye(4), (nc, 1, 1))
    for c in range(nc):                                            # cameras looking 120 degrees apart, 10 cm off the rig centre
        a = 2 * np.pi * c / nc
        M_c[c, :3, :3] = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        M_c[c, :3, 3] = [0.1 * np.sin(a), 0.0, 0.1 * np.cos(a)]
    M_t = np.eye(4)
    M_t[:3, 3] = np.array([0.3, -0.2, 0.1]) + np.asarray(shift)
    return api.Rig(cams, M_c, M_t)


def essential(rig1, rig2):
    """Es[i][j] = ComputeE(KF1.Get_MtMc_inv(i), KF2.Get_MtMc(j)) (ref :988-1001)"""
    from multicol_slam_b200 import settings
    return settings.essential_matrices(rig1.MtMc_inv, rig2.MtMc)


def rays_of(api, F, cams):
    """mvKeysRays: ImgToWorld of each keypoint's float position"""
    return np.array([api.img_to_world(cams[int(F.key_cam[i])], float(k["x"]), float(k["y"])) for i, k in enumerate(F.keys)]).reshape(-1, 3)


def tri_scene(api, frames, cams, n_nb, seed=3, dim=32, free=0.5):
    """KF1 = the first frame with about `free` of its keypoints free (id -1) and the others carrying map points; neighbour k a
    variant of either frame (a few bits flipped per descriptor, more for later neighbours) at a pose a few centimetres from KF1's,
    with its own points.  Poses as rigs, for the reference and for E."""
    F1, F2 = frames
    rng = np.random.default_rng(seed)
    n1 = len(F1.keys)
    mp1 = np.where(rng.random(n1) < free, -1, np.arange(n1)).astype(np.int32)
    nbs, mps, rigs, off = [], [], [], n1
    for k in range(n_nb):
        B = F2 if k % 2 else F1
        F = api.Frame(B.keys, B.key_cam, flip_bits(rng, B.desc, 2 + k % 5), B.dmask, list(zip(B.cam_w, B.cam_h)), B.scale_factors)
        nbs.append(widen(api, F, dim))
        n = len(B.keys)
        mps.append(np.where(rng.random(n) < free, -1, off + np.arange(n)).astype(np.int32))
        rigs.append(rig_of(api, cams, rng.uniform(-0.04, 0.04, 3)))
        off += n
    return dict(KF1=widen(api, F1, dim), mp1=mp1, nbs=nbs, mps=mps, rig1=rig_of(api, cams, [0, 0, 0]), rigs=rigs, next_id=off)


def reference_tri(rm, api, s, k, cams, mp1, mp2, masks):
    """the reference's SearchForTriangulationRaw(KF1, KF_k): (nmatches, vMatchedPairs)"""
    r1, r2 = s["rig1"], s["rigs"][k]
    k1 = rm.KF(s["KF1"], cams, M_c=r1.M_c, M_t=r1.M_t, mp=np.where(mp1 == -1, -1, 0).astype(np.int32), rays=rays_of(api, s["KF1"], cams))
    k2 = rm.KF(s["nbs"][k], cams, M_c=r2.M_c, M_t=r2.M_t, mp=np.where(mp2 == -1, -1, 0).astype(np.int32), rays=rays_of(api, s["nbs"][k], cams))
    return rm.search_for_triangulation_raw(k1, k2, rm.MPTable(3, np.zeros((1, 32), np.uint8)), 0.6, masks)


def epipolar_residual(api, r1, r2, E):
    """(nom * nom) / den of CheckDistEpipolarLine (ref src/misc.cpp:53-69), cv::Matx order"""
    nom = float(api._mm(api._mm(r2.reshape(1, 3), E), r1.reshape(3, 1))[0, 0])
    ex1 = api._mm(E, r1.reshape(3, 1)).ravel()
    etx2 = api._mm(E.T.copy(), r2.reshape(3, 1)).ravel()
    den = float(ex1[0] * ex1[0] + ex1[1] * ex1[1] + ex1[2] * ex1[2] + etx2[0] * etx2[0] + etx2[1] * etx2[1] + etx2[2] * etx2[2])
    return (nom * nom) / den
