"""The extractor against the CPU oracle image by image, and the adversarial images built on K1's tiles and FAST cells."""
import math

import numpy as np

MODES = {"orb": dict(do_dbrief=False, learn_masks=False), "dbrief": dict(do_dbrief=True, learn_masks=False),
         "mdbrief": dict(do_dbrief=True, learn_masks=True)}
EDGE = 25
MIN_B = EDGE - 3
TILE_W, TILE_H, WARPS = 64, 32, 8          # K1 tile and warps per CTA; warp w collects tile rows w, w + 8, w + 16, w + 24


def axis_cells(n, x_axis):
    """FAST cell index of every pixel along one axis of a level (-1 outside every cell) and the cell size, with the formulas of
    oracle/pyref.py detect_level: minB = 22, nCols = int(width / 30), wCell = ceil(width / nCols); a cell is skipped when it starts
    6 (columns) or 3 (rows) px before maxB, and cv::FAST reports nothing in the 3 px frame of the cell's image."""
    max_b = n - EDGE + 3
    size = max_b - MIN_B
    ncell = int(size / 30.0)
    wc = int(math.ceil(size / ncell))
    out = np.full(n, -1, np.int64)
    for j in range(ncell):
        ini = MIN_B + j * wc
        if ini >= max_b - (6 if x_axis else 3):
            continue
        out[ini + 3:min(ini + wc + 6, max_b) - 3] = j
    return out, wc


def cams_for(cams, w, h):
    """the three Lafida cameras at size w x h, full masks (Camera.mirrorMask: 0)"""
    from multicol_slam_b200 import synth
    out = []
    for c in cams:
        c = dict(c) if (w, h) == (c["width"], c["height"]) else synth.scaled_cam(c, w, h)
        c["mirror_mask"] = 0
        out.append(c)
    return out


def run_batch(api, oa, imgs, masks, cams, coi, nf, mode, levels=True, **kw):
    """extract_batch against the oracle image by image; returns the oracle's (keypoints, level-0 raw corners) per image"""
    m = MODES[mode]
    ex = api.mdBRIEFextractorOct(nfeatures=nf, do_dBrief=m["do_dbrief"], learnMasks=m["learn_masks"], **kw)
    okw = {"fast_threshold": kw.get("fastThreshold", 20), "nlevels": kw.get("nlevels", 8)}
    oe = oa.OracleExtractor(nfeatures=nf, **m, **okw)
    kps, desc, dmask, counts = ex.extract_batch(np.ascontiguousarray(imgs), np.ascontiguousarray(masks), cams, coi)
    out = []
    for i, c in enumerate(coi):
        ok, od, om = oe.extract(imgs[i], masks[c], cams[c])
        if levels:
            for l in range(ex.GetLevels()):
                assert np.array_equal(ex.debug_read(l, 0, i), oe.debug_read(l, 0)), f"image {i}: pyramid level {l}"
                assert np.array_equal(ex.debug_read(l, 1, i), oe.debug_read(l, 1)) or not np.any(ok["octave"] == l), \
                    f"image {i}: blurred level {l}"
                assert np.array_equal(ex.debug_read(l, 2, i), oe.debug_read(l, 2)), f"image {i}: mask level {l}"
                assert np.array_equal(ex.debug_read(l, 3, i), oe.debug_read(l, 3)), f"image {i}: raw corners level {l}"
        n = counts[i]
        k = kps[i, :n]
        assert n == len(ok), f"image {i}: {n} keypoints, oracle {len(ok)}"
        for f in ("x", "y", "size", "response", "octave", "class_id"):
            assert np.array_equal(k[f], ok[f]), f"image {i}: keypoint field {f}"
        assert np.array_equal(k["angle"].view(np.uint32), ok["angle"].view(np.uint32)), f"image {i}: IC angle bits"
        assert np.array_equal(desc[i, :n], od), f"image {i}: descriptor bits"
        assert np.array_equal(dmask[i, :n], om), f"image {i}: descriptor mask bits"
        out.append((ok, oe.debug_read(0, 3)))
    return out


def dense_row(w):
    """One row of dots that reaches the per-tile bound on strict per-cell 3x3 maxima in every even K1 tile: each piece of a FAST
    cell inside a tile (a segment) holds dots at every other pixel from its first pixel on, ceil(length / 2) of them.  The per-cell
    NMS treats a neighbour in another cell as 0, so the last pixel of a cell and the first pixel of the next can both be dots, and
    a 64-pixel tile row holds 33 or 34 maxima where its segments have odd lengths.  Where a cell runs across a tile edge, two
    dots would touch inside one cell and suppress each other: the even tile of the two keeps its dot."""
    cx, _ = axis_cells(w, True)
    x = np.arange(w)
    first = (cx >= 0) & np.concatenate([[True], cx[1:] != cx[:-1]])
    seg0 = np.maximum(np.maximum.accumulate(np.where(first, x, 0)), x // TILE_W * TILE_W)
    dot = (cx >= 0) & ((x - seg0) % 2 == 0)
    for x0 in range(TILE_W, w, TILE_W):
        if dot[x0 - 1] and dot[x0] and cx[x0 - 1] == cx[x0]:
            dot[x0 if (x0 // TILE_W) % 2 else x0 - 1] = False
    return dot


def boundary_lattice(w, h, variant=0):
    """Dense rows (dense_row, dots of 255 on black) on the four rows of one K1 warp (w = variant) in every tile.  In the last of
    them one dot makes room for a dot in the row below, which belongs to warp w + 1 of the same tile.  Every dot is an isolated
    FAST corner of score 254, so K2 sees nothing but ties as well."""
    dot = dense_row(w)
    img = np.zeros((h, w), np.uint8)
    img[variant::WARPS][:, dot] = 255
    for y0 in range(0, h, TILE_H):
        y = y0 + 3 * WARPS + variant                          # last row of warp `variant` in this tile
        if y + 1 >= h:
            continue
        for x0 in range(0, w, TILE_W):
            g = np.nonzero(dot[x0 + 30 + 2 * variant:x0 + TILE_W])[0]
            if len(g):
                g = x0 + 30 + 2 * variant + g[0]
                img[y, g] = 0                                 # its neighbours in the row are empty already
                img[y + 1, g] = 255
    return img


def extract_and_compare(api, oa, imgs, masks, cams, coi, nf, mode="mdbrief", ex=None, **kw):
    """extract_batch of imgs (camera coi[i] of cams / masks) against the oracle per image; returns the per-image counts"""
    m = MODES[mode]
    ex = ex or api.mdBRIEFextractorOct(nfeatures=nf, do_dBrief=m["do_dbrief"], learnMasks=m["learn_masks"], **kw)
    okw = {"nlevels": kw["nlevels"]} if "nlevels" in kw else {}
    if "descSize" in kw:
        okw["desc_size"] = kw["descSize"]
    oe = oa.OracleExtractor(nfeatures=nf, **m, **okw)
    kps, desc, dmask, counts = ex.extract_batch(np.stack(imgs), np.stack(masks), cams, coi)
    for i, img in enumerate(imgs):
        ok, od, om = oe.extract(img, masks[coi[i]], cams[coi[i]])
        n = counts[i]
        assert n == len(ok), f"image {i}: {n} keypoints, oracle {len(ok)}"
        assert kps[i, :n].tobytes() == ok.tobytes(), f"image {i}: keypoints"
        assert np.array_equal(desc[i, :n], od), f"image {i}: descriptors"
        assert np.array_equal(dmask[i, :n], om), f"image {i}: descriptor masks"
    return counts
