"""Frames and rigs for the matcher's GPU tests."""
import numpy as np


def make_frames(api, oa, cams, seeds, nf=600, masks=True):
    from multicol_slam_b200 import synth
    ex = api.mdBRIEFextractorOct(nfeatures=nf, do_dBrief=True, learnMasks=masks)
    per = []
    for c, s in enumerate(seeds):
        per.append(ex(synth.frame(cams[c], s), synth.mirror_mask(cams[c]), cams[c]))
    sf = [ex.info.scale_factor[l] for l in range(8)]
    return api.Frame.from_cameras(per, [(754, 480)] * len(seeds), sf)


def random_rig(rng, n_cams):
    """MtMc[c] = [R t; 0 1] with random rotations looking roughly outwards, and the rigid inverse (cConverter::invMat)."""
    mtmc, inv = np.zeros((n_cams, 4, 4)), np.zeros((n_cams, 4, 4))
    for c in range(n_cams):
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        if np.linalg.det(q) < 0:
            q[:, 0] = -q[:, 0]
        t = rng.normal(0, 0.2, 3)
        mtmc[c, :3, :3], mtmc[c, :3, 3], mtmc[c, 3, 3] = q, t, 1.0
        inv[c, :3, :3], inv[c, :3, 3], inv[c, 3, 3] = q.T, -(q.T @ t), 1.0
    return mtmc, inv
