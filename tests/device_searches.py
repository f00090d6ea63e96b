"""The device searches called on host arrays: pack the frames, stage the inputs, launch, read back in contiguous order."""
import numpy as np

from device_frames import (BIG_ID, FILL, GUARD, INT_MAX, POISON, PREV_FILL, counts, from_slots, on_device, pack_frames, per_cam, reversed_image,
                           sizes, slot_to_contiguous_index, to_slots)


def projection_inputs(api, per_cam, mps, pre=None, layout="single", first_image=2, cap=None):
    """per_cam [(kps, desc, dmask)] -> the device inputs of mcs_search_by_projection_device, frame_mp in slot order"""
    cc = [len(p[0]) for p in per_cam]
    cap = cap or max(cc) + 5
    packed, n_parts, part_images, first = pack_frames([per_cam], cap, layout=layout, first_image=first_image)[0]
    fm = np.full(sum(cc), -1, np.int32) if pre is None else pre
    mdev = api.MapPointsDevice.from_host(mps, packed.device) if isinstance(mps, api.MapPoints) else mps
    return dict(packed=packed, n_parts=n_parts, part_images=part_images, first=first, nc=len(cc), cap=cap, cc=cc,
                fm_t=to_slots(api, cc, fm, cap, FILL), mdev=mdev)


def launch_projection(matcher, d, sizes, sf, th, stream=None):
    return matcher.SearchByProjectionDevice(d["packed"], d["n_parts"], d["part_images"], d["first"], d["nc"], d["cap"], sizes, sf, d["mdev"],
                                            th, d["fm_t"], stream=stream, diag=True)


def device_projection(api, matcher, per_cam, sizes, sf, mps, th, pre=None, layout="single", first_image=2, cap=None):
    """-> (nmatches, contiguous frame_mp, status, diag) of mcs_search_by_projection_device"""
    import torch
    d = projection_inputs(api, per_cam, mps, pre, layout, first_image, cap)
    res = launch_projection(matcher, d, sizes, sf, th)
    torch.cuda.synchronize()
    return collect(api, d, *res)


def collect(api, d, n_t, st_t, fm_t, diag_t=None):
    """-> (nmatches, contiguous frame_mp, status[, diag]), checking that every slot beyond a camera's count still holds FILL"""
    out = int(n_t.item()), from_slots(api, fm_t, d["cc"], d["cap"], FILL), int(st_t.item())
    return out if diag_t is None else out + (diag_t.cpu().numpy(),)


def pack_cur_last(Fc, Fl, layout, cap):
    """-> (cur, last) packed-frame records.  single: each frame in a buffer of its own, with the current frame's first camera
    reversed as decoys, two before and one after the current frame's cameras and one before the last frame's; parts: each frame's
    cameras one-image parts of a buffer of its own, as the allgather leaves them; shared: the last frame's cameras, then the
    current frame's, as images of one buffer"""
    if layout == "single":
        decoy = reversed_image(per_cam(Fc)[0])
        return pack_frames([Fc], cap, first_image=2)[0], pack_frames([Fl], cap, after=0, decoy=decoy)[0]
    if layout == "parts":
        return tuple(pack_frames([Fc, Fl], cap, layout="separate"))
    last, cur = pack_frames([Fl, Fc], cap, layout="joint")
    return cur, last


def cur_last_inputs(api, Fc, Fl, mp_last, layout, cap, last_keys):
    """the inputs of every current / last frame search: both frames packed and the last frame's map points in slot order.
    last_keys replaces the last frame's packed keypoints (the host composition keeps Fl's)."""
    cc, cl = counts(Fc), counts(Fl)
    cap = cap or max(cc + cl) + 5
    if last_keys is not None:
        Fl = api.Frame(last_keys, Fl.key_cam, Fl.desc, Fl.dmask, list(zip(Fl.cam_w, Fl.cam_h)), Fl.scale_factors)
    cur, last = pack_cur_last(Fc, Fl, layout, cap)
    return dict(cur=cur, last=last, cap=cap, cc=cc, last_mp_t=to_slots(api, cl, mp_last, cap, BIG_ID))


def device_last(api, m, Fc, Fl, rig_cur, mp_cur, mp_last, outlier, world, bad, th, layout="single", cap=None, stream=None,
                last_keys=None, run=True):
    """mcs_search_by_projection_last_device on host arrays -> (nmatches, contiguous cur_mp, status, diag)"""
    import torch
    d = cur_last_inputs(api, Fc, Fl, mp_last, layout, cap, last_keys)
    cl = counts(Fl)
    d.update(masks_t=on_device(np.stack(rig_cur.masks)),
             outlier_t=None if outlier is None else to_slots(api, cl, outlier, d["cap"], 1, dtype=np.uint8),
             world_t=on_device(np.asarray(world, np.float64).reshape(-1, 3)), bad_t=None if bad is None else on_device(np.asarray(bad, np.uint8)),
             cur_mp_t=to_slots(api, d["cc"], mp_cur, d["cap"], FILL))
    if not run:
        return d
    res = launch_last(m, d, rig_cur, Fc.scale_factors, th, stream)
    torch.cuda.synchronize()
    return collect(api, d, *res)


def launch_last(m, d, rig_cur, sf, th, stream=None):
    return m.SearchByProjectionLastDevice(d["cur"], d["last"], d["cap"], rig_cur, d["masks_t"], sf, d["last_mp_t"], d["world_t"], th,
                                          d["cur_mp_t"], bad_t=d["bad_t"], last_outlier_t=d["outlier_t"], stream=stream, diag=True)


def device_ws(api, m, Fc, Fl, mp_last, bad, window, lo=0, hi=INT_MAX, layout="single", cap=None, stream=None, last_keys=None, run=True,
              seed=5):
    """mcs_window_search_device on host arrays -> (nmatches, contiguous cur_mp, status, diag).  cur_mp starts from arbitrary ids: the
    call must overwrite every slot below each camera's count and leave the others (FILL) alone."""
    import torch
    d = cur_last_inputs(api, Fc, Fl, mp_last, layout, cap, last_keys)
    junk = np.random.default_rng(seed).integers(-1, 600, len(Fc.keys)).astype(np.int32)
    d.update(sizes=sizes(Fc), bad_t=on_device(np.asarray(bad, np.uint8)), cur_mp_t=to_slots(api, d["cc"], junk, d["cap"], FILL), window=window,
             lo=lo, hi=hi)
    if not run:
        return d
    res = launch_ws(m, d, stream)
    torch.cuda.synchronize()
    return collect(api, d, *res)


def launch_ws(m, d, stream=None):
    return m.WindowSearchDevice(d["cur"], d["last"], d["cap"], d["sizes"], d["last_mp_t"], d["window"], d["cur_mp_t"], min_level=d["lo"],
                                max_level=d["hi"], bad_t=d["bad_t"], stream=stream, diag=True)


def device_search_frames(api, m, Fc, Fl, rig_cur, mp_cur, mp_last, world, bad, window, layout="single", cap=None, stream=None, last_keys=None,
                         run=True):
    """mcs_search_by_projection_frames_device on host arrays -> (nmatches, contiguous cur_mp, status, diag)"""
    import torch
    d = cur_last_inputs(api, Fc, Fl, mp_last, layout, cap, last_keys)
    d.update(rig=rig_cur, window=window, masks_t=on_device(np.stack(rig_cur.masks)), world_t=on_device(np.asarray(world, np.float64).reshape(-1, 3)),
             bad_t=None if bad is None else on_device(np.asarray(bad, np.uint8)), cur_mp_t=to_slots(api, d["cc"], mp_cur, d["cap"], FILL))
    if not run:
        return d
    res = launch_frames(m, d, stream)
    torch.cuda.synchronize()
    return collect(api, d, *res)


def launch_frames(m, d, stream=None):
    return m.SearchByProjectionFramesDevice(d["cur"], d["last"], d["cap"], d["rig"], d["masks_t"], d["last_mp_t"], d["world_t"], d["window"],
                                            d["cur_mp_t"], bad_t=d["bad_t"], stream=stream, diag=True)


def prev_slots(prev, counts, cap):
    out = np.full((len(counts), cap, 2), PREV_FILL)
    o = 0
    for c, n in enumerate(counts):
        out[c, :n] = prev[o:o + n]
        o += n
    return out.reshape(-1)


def init_inputs(api, F1, F2, prev, layout="single", cap=None, seed=3):
    c1, c2 = counts(F1), counts(F2)
    cap = cap or max(c1 + c2) + 5
    f2, f1 = pack_cur_last(F2, F1, layout, cap)
    junk = np.random.default_rng(seed).integers(-1, 600, len(F1.keys)).astype(np.int32)
    return dict(f1=f1, f2=f2, cap=cap, c1=c1, c2=c2, sizes=sizes(F1), prev_t=on_device(prev_slots(np.asarray(prev, np.float64), c1, cap)),
                m12_t=to_slots(api, c1, junk, cap, FILL))


def launch_init(m, d, window, stream=None):
    return m.SearchForInitializationDevice(d["f1"], d["f2"], d["cap"], d["sizes"], d["prev_t"], window, d["m12_t"], stream=stream, diag=True)


def collect_init(api, d, n_t, m12_t, diag_t):
    """-> (nmatches, contiguous matches12 as contiguous F2 indices, contiguous prev [n1, 2], diag), checking the untouched slots"""
    cap, c1, c2 = d["cap"], d["c1"], d["c2"]
    m = from_slots(api, m12_t, c1, cap, FILL)
    p = d["prev_t"].cpu().numpy().reshape(len(c1), cap, 2)
    assert all(np.all(p[c, n:] == PREV_FILL) for c, n in enumerate(c1))
    m12 = np.full(len(m), -1, np.int32)
    m12[m >= 0] = slot_to_contiguous_index(m[m >= 0], c2, cap)
    prev = np.concatenate([p[c, :c1[c]] for c in range(len(c1))])
    return int(n_t.item()), m12, prev, diag_t.cpu().numpy()


def device_init(api, m, F1, F2, prev, window, layout="single", cap=None):
    import torch
    d = init_inputs(api, F1, F2, prev, layout, cap)
    res = launch_init(m, d, window)
    torch.cuda.synchronize()
    return collect_init(api, d, *res)


def host_init(m, F1, F2, prev, window):
    p = np.array(prev, np.float64, copy=True)
    n, m12 = m.SearchForInitialization(F1, F2, p, window)
    return n, m12, p


def dev_map(s, bad=None, desc=None):
    """the scene's map points on the device"""
    return dict(world_t=on_device(np.asarray(s["world"], np.float64)), min_t=on_device(np.asarray(s["min_d"], np.float64)),
                max_t=on_device(np.asarray(s["max_d"], np.float64)), desc_t=on_device(s["desc"] if desc is None else desc),
                dmask_t=on_device(s["dmask"]), bad_t=None if bad is None else on_device(np.asarray(bad, np.uint8)))


def fuse_pose(rig, variant, Scw):
    """(MtMc_inv, ow) of the pose a variant projects with"""
    from multicol_slam_b200.api import _sim3_rig
    r = rig if variant != 2 else _sim3_rig(rig, Scw)
    return r.MtMc_inv, r.M_t[:3, 3].copy()


def fuse_device(api, m, KFs, rigs, mps, points, dm, cap, layout, variant, Scw=None, th=2.5, max_hits=None, stream=None, sf=None):
    """FuseDevice over the key frames -> (hits [n, 3] numpy, n_hits, status, out tensors)"""
    import torch
    packed = pack_frames(KFs, cap, layout=layout)
    kfs = [(packed[k], mps[k]) + fuse_pose(rigs[k], variant, Scw) for k in range(len(KFs))]
    out = m.FuseDevice(kfs, on_device(np.asarray(points, np.int32)), cap, rigs[0].cams, on_device(np.stack(rigs[0].masks)),
                       KFs[0].scale_factors if sf is None else sf, dm["world_t"], dm["min_t"], dm["max_t"], dm["desc_t"], dm["dmask_t"],
                       bad_t=dm["bad_t"], variant=variant, th=th, max_hits=max_hits, stream=stream)
    torch.cuda.synchronize()
    n = int(out[1].item())
    return out[0].cpu().numpy()[:n], n, int(out[2].item()), out


def fuse_replay(m, KF, s, variant, hits, cap, k=0, **kw):
    sc, cur = s["sc"], s["cur"] or {}
    rows = hits[hits[:, 0] == k][:, 1:]
    return m.FuseReplay(KF, sc["rig"], s["kf_mp"], s["points"], rows, cap, s["world"], s["min_d"], s["max_d"], s["bad"], s["in_kf"], s["desc"],
                        s["dmask"], th=2.5, variant=variant, Scw=s["Scw"], cur_rays=cur.get("rays"), kf_rays=sc["rays"], cur_rig=cur.get("rig"),
                        **kw)


def fuse_targets(api, cams, sc, n_kf, seed):
    """n_kf poses of the key frame's rig around the scene's, a few centimetres apart"""
    rng = np.random.default_rng(seed)
    rigs = []
    for _ in range(n_kf):
        M_t = sc["M_t"].copy()
        M_t[:3, 3] += rng.normal(0, 0.02, 3)
        rigs.append(api.Rig(cams, sc["M_c"], M_t))
    return rigs


def device_scw(api, m, s, cap, layout, points=None, matched=None, th=10, stream=None):
    """SearchByProjectionKFScwDevice on the scene -> (nmatches, status, vpMatched in contiguous order, diag)"""
    import torch
    KF = s["KF"]
    (kf,) = pack_frames([KF], cap, layout=layout)
    dm = dev_map(s, bad=s["bad"])
    pts = s["points"] if points is None else points
    matched_t = to_slots(api, KF, s["matched"] if matched is None else matched, cap, GUARD)
    n, st, out, diag = m.SearchByProjectionKFScwDevice(kf, cap, s["rig"], s["Scw"], on_device(np.stack(s["rig"].masks)), KF.scale_factors,
                                                       on_device(np.asarray(pts, np.int32)), dm["world_t"], dm["min_t"], dm["max_t"],
                                                       dm["desc_t"], dm["dmask_t"], th, matched_t, bad_t=dm["bad_t"], stream=stream, diag=True)
    torch.cuda.synchronize()
    return int(n.item()), int(st.item()), from_slots(api, out, counts(KF), cap, GUARD), diag.cpu().numpy()


def tri_inputs(api, KF1, KF2, mp1, mp2, cams, cap, layout="single", same=False):
    """freshly packed frames, map-point rows with -1 (free) past the counts and poisoned outputs, all on the device:
    (kf1, mp1_t, kf2, mp2_t, out)"""
    import torch
    packs = pack_frames([KF1] if same else [KF1, KF2], cap, layout=layout)
    mp1_t = to_slots(api, KF1, mp1, cap, -1)
    mp2_t = mp1_t if same else to_slots(api, KF2, mp2, cap, -1)
    out = (torch.full((1,), -3, dtype=torch.int32, device="cuda"), torch.full((len(cams) * cap,), POISON, dtype=torch.int32, device="cuda"),
           torch.full((2,), -3, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    return packs[0], mp1_t, packs[0 if same else 1], mp2_t, out


def device_tri(api, m, KF1, KF2, mp1, mp2, cams, cap, E, layout="single", epi=1e-2, same=False):
    """-> (nmatches, matches12, diag) of the device call, on the host"""
    p1, mp1_t, p2, mp2_t, out = tri_inputs(api, KF1, KF2, mp1, mp2, cams, cap, layout, same)
    r = m.SearchForTriangulationRawDevice(p1, mp1_t, p2, mp2_t, cams, cap, E, epi, out=out, diag=True)
    return int(r[0].item()), r[1].cpu().numpy(), r[2].cpu().numpy()


def host_tri(api, m, KF1, KF2, mp1, mp2, cams, cap, E, epi=1e-2, oa=None):
    packs = pack_frames([KF1, KF2], cap, device="cpu")
    return m.SearchForTriangulationRawHost(packs[0], to_slots(api, KF1, mp1, cap, BIG_ID, "cpu"), packs[1], to_slots(api, KF2, mp2, cap, BIG_ID, "cpu"),
                                           cams, cap, E, epi, _st=None if oa is None else oa.search_for_triangulation)


def assert_same_tri(api, KF1, dev, host, cap):
    """nmatches and every slot below KF1's counts equal; every slot at or beyond a count still poisoned"""
    assert dev[0] == host[0]
    n = counts(KF1)
    assert np.array_equal(from_slots(api, dev[1], n, cap, POISON), api.slots_to_contiguous(host[1], n, cap))
