"""The extractor against the CPU oracle image by image, and the adversarial images built on K1's tiles and FAST cells."""
import math

import numpy as np

from k1_geometry import K1, ROWS_PER_WARP, WARPS, warp_of_row

MODES = {"orb": dict(do_dbrief=False, learn_masks=False), "dbrief": dict(do_dbrief=True, learn_masks=False),
         "mdbrief": dict(do_dbrief=True, learn_masks=True)}
EDGE = 25
MIN_B = EDGE - 3
TILE_W, TILE_H = K1["kTW"], K1["kTH"]      # K1 tile; warp w of its CTA collects tile rows w, w + WARPS, .. (ROWS_PER_WARP rows)


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
    okw = {"fast_threshold": kw.get("fastThreshold", 20), "nlevels": kw.get("nlevels", 8), "scale_factor": kw.get("scaleFactor", 1.2)}
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
    dots would touch inside one cell and suppress each other: the even tile of the two keeps its dot.  An odd tile continues the
    dots of a cell coming from the even tile on its left, so that the even tile's last dot does not get a dot 3 px away on each
    side: with two bright pixels opposite on its FAST circle it would not be a corner."""
    cx, _ = axis_cells(w, True)
    x = np.arange(w)
    first = (cx >= 0) & np.concatenate([[True], cx[1:] != cx[:-1]])
    even0 = (x // TILE_W - (x // TILE_W) % 2) * TILE_W                   # first pixel of the even tile of x's tile pair
    seg0 = np.maximum(np.maximum.accumulate(np.where(first, x, 0)), np.where((x // TILE_W) % 2, even0, x // TILE_W * TILE_W))
    dot = (cx >= 0) & ((x - seg0) % 2 == 0)
    for x0 in range(TILE_W, w, TILE_W):
        if dot[x0 - 1] and dot[x0] and cx[x0 - 1] == cx[x0]:
            dot[x0 if (x0 // TILE_W) % 2 else x0 - 1] = False
    return dot


def tile_dots(w):
    """dots of dense_row(w) in each K1 tile column: the strict maxima one of its rows holds there"""
    return np.add.reduceat(dense_row(w).astype(np.int64), np.arange(0, w, TILE_W))


def boundary_lattice(w, h, variant=0):
    """Dense rows (dense_row, dots of 255 on black) on the ROWS_PER_WARP rows of one K1 warp (v = variant) in every tile.  In the
    last of them one dot makes room for a dot in the row below, which belongs to warp v + 1 of the same tile: the segment of warp
    v holds boundary_lattice_target(w) corners and the next one is not empty.  Every dot is an isolated FAST corner of score 254,
    so K2 sees nothing but ties as well."""
    dot = dense_row(w)
    img = np.zeros((h, w), np.uint8)
    img[variant::WARPS][:, dot] = 255
    for y0 in range(0, h, TILE_H):
        y = y0 + (ROWS_PER_WARP - 1) * WARPS + variant       # last row of warp `variant` in this tile
        if y + 1 >= min(y0 + TILE_H, h):
            continue
        for x0 in range(0, w, TILE_W):
            g = np.nonzero(dot[x0 + 30 + 2 * variant:x0 + TILE_W])[0]
            if len(g):
                g = x0 + 30 + 2 * variant + g[0]
                img[y, g] = 0                                 # its neighbours in the row are empty already
                img[y + 1, g] = 255
    return img


def boundary_lattice_target(w):
    """the fullest warp segment with a non-empty next warp that boundary_lattice reaches at width w: all rows of the warp at the
    most maxima a tile row holds, less the dot moved into the next warp"""
    return ROWS_PER_WARP * int(tile_dots(w).max()) - 1


def warp_fill_lattice(w, h, phase=0):
    """Dense rows on all ROWS_PER_WARP rows of one warp v of each tile row, so that a tile column where a dense row holds 34 maxima
    (four cell pieces of odd length, e.g. cells of 31 px at width 1280) fills warp v's segment to kWarpCorners.  Each tile column
    also gets one dot in warp v + 1, on the first row of a FAST cell whose previous row is one of warp v's: the per-cell NMS counts
    a neighbour in another cell as 0, so that dot is a maximum and costs warp v nothing.  v is chosen per tile row from the cell
    edges it crosses (`phase` picks which), and v < WARPS - 1: an overflow of the last warp's segment would land in the unused
    tail of the pixel tile, where no result shows it."""
    dot = dense_row(w)
    cy, _ = axis_cells(h, False)
    img = np.zeros((h, w), np.uint8)
    for y0 in range(0, h, TILE_H):
        edges = [r for r in range(y0 + 1, min(y0 + TILE_H, h))
                 if cy[r - 1] >= 0 and cy[r] >= 0 and cy[r] != cy[r - 1] and warp_of_row(r - 1)[1] < WARPS - 1]
        if not edges:
            continue
        r = edges[phase % len(edges)]
        img[y0 + warp_of_row(r - 1)[1]:min(y0 + TILE_H, h):WARPS][:, dot] = 255
        for x0 in range(0, w, TILE_W):
            g = np.nonzero(dot[x0:x0 + TILE_W])[0]
            if len(g):
                img[r, x0 + g[len(g) // 2]] = 255
    return img


def warp_segments(raw):
    """raw corners (x, y, score) of a level -> {(tile x, tile y, warp): corners}, the segments K1 collects them in"""
    seg = {}
    for x, y, _ in raw:
        key = (int(x) // TILE_W, *warp_of_row(int(y)))
        seg[key] = seg.get(key, 0) + 1
    return seg


def segments_before_corners(raw):
    """{(tile x, tile y, warp): corners} of the warp segments whose next warp in the same tile holds corners too: where a
    segment that overflowed would overwrite the next one's"""
    seg = warp_segments(raw)
    return {k: v for k, v in seg.items() if seg.get((k[0], k[1], k[2] + 1), 0) > 0}


def fullest_segment(raw):
    """the most corners a K1 warp segment holds while the next warp of its tile holds corners too"""
    return max(segments_before_corners(raw).values(), default=0)


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
