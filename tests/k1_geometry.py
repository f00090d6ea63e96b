"""K1 (pyr_fast_kernel) geometry as the kernel source states it: its tile, warp and staging constants, read from mcs_common.cuh and
pyr_fast_kernel.cu with C integer arithmetic, and the staged source region of every pyramid level as build_geometry (mcs_api.cu)
computes it.  The tests and the image generators built on K1's tiles take the geometry from here, so that they follow the kernel."""
import functools
import pathlib
import re
from typing import NamedTuple

import numpy as np

CSRC = pathlib.Path(__file__).resolve().parents[1] / "multicol_slam_b200" / "csrc"


@functools.lru_cache(maxsize=None)
def _constants():
    common = (CSRC / "mcs_common.cuh").read_text()
    kern = (CSRC / "pyr_fast_kernel.cu").read_text()
    c = {k: int(re.search(rf"\b{k} = (\d+)", common).group(1)) for k in ("kTW", "kTH", "kHalo", "kSrcWB", "kSrcH")}
    for k in ("kThreads", "kScoreS", "kScoreBytes", "kRowSumBytes", "kStagingMin", "kWarpCorners"):
        expr = re.search(rf"constexpr int {k} = ([^;]+);", kern).group(1)
        assert re.fullmatch(r"[\w\s()+*/-]+", expr), (k, expr)
        c[k] = eval(expr.replace("/", "//"), {"__builtins__": {}}, dict(c))
    return tuple(c.items())


def constants():
    """kTW, kTH, kHalo, kSrcWB, kSrcH, kThreads, kWarpCorners and kStagingMin (the least staging the launcher passes: the score
    tile and the packed row sums that reuse the area)"""
    return dict(_constants())


K1 = constants()
WARPS = K1["kThreads"] // 32
ROWS_PER_WARP = K1["kTH"] // WARPS          # warp w of a CTA collects the corners of tile rows w, w + WARPS, ..


def warp_of_row(y):
    """(tile row, warp) of the K1 CTA whose warp collects the corners of level row y"""
    return y // K1["kTH"], (y % K1["kTH"]) % WARPS


def src_offsets(n, sn):
    """source row / column of every output pixel of a level (the host's resize table, float arithmetic as in build_geometry)"""
    scale = 1.0 / (n / sn)
    f = ((np.arange(n) + 0.5) * scale - 0.5).astype(np.float32)
    return np.floor(f).astype(np.int64), scale


class LevelBox(NamedTuple):
    w: int            # level size
    h: int
    box_w: int        # the level's TMA box: the widest and tallest staged source region over its tiles
    box_h: int
    ratio: float      # largest source / level ratio of the two axes
    past: int         # rows the bottom tiles' box reaches past the source level (zero-filled by the tensor map)


def level_boxes(W, H, sf, nlevels):
    """LevelBox of every level above 0 as build_geometry computes it"""
    c = K1
    inv, isf = 1.0 / float(np.float32(sf)), 1.0
    sw, sh, out = W, H, []
    for _ in range(1, nlevels):
        isf *= inv
        w, h = round(W * isf), round(H * isf)
        xofs, sx = src_offsets(w, sw)
        yofs, sy = src_offsets(h, sh)
        assert sx <= 2.08 and sy <= 2.08
        xofs = np.clip(xofs, 0, sw - 1)              # the host clamps columns; rows are clamped where they are used
        bw = bh = 1
        for t in range(0, w, c["kTW"]):
            xa, xb = max(t - c["kHalo"], 0), min(t + c["kTW"] + c["kHalo"], w) - 1
            bw = max(bw, min(xofs[xb] + 1, sw - 1) - (xofs[xa] & ~15) + 1)
        for t in range(0, h, c["kTH"]):
            ya, yb = max(t - c["kHalo"], 0), min(t + c["kTH"] + c["kHalo"], h) - 1
            lo, hi = min(max(yofs[ya], 0), sh - 1), min(max(yofs[yb] + 1, 0), sh - 1)
            bh = max(bh, hi - lo + 1)
        out.append(LevelBox(w, h, (bw + 15) & ~15, bh, max(sx, sy), lo + bh - sh))
        sw, sh = w, h
    return out


def staging_bytes(box_h):
    """dynamic shared memory launch_pyr_fast passes for a level of this box height"""
    return max(box_h * K1["kSrcWB"], K1["kStagingMin"])
