"""K1 (pyr_fast_kernel) collects the strict per-cell 3x3 maxima of FAST scores in fixed buffers: a shared-memory segment of
kWarpCorners slots per warp (a warp owns 8 rows of a 64x64 tile), and a raw corner list of raw_cap entries per level and image.
Both are sized from the FAST cell grid.  The NMS treats a neighbour in another cell as 0 (cv::FAST runs per cell), so two maxima
can touch across a cell edge; inside a cell they cannot.  These checks run the cell grid of every level width and height the
extractor accepts and compare the worst case with the sizes the kernel and the host use."""
import math

import numpy as np

from k1_geometry import ROWS_PER_WARP, constants

EDGE = 25
MIN_B = EDGE - 3
LEVEL_SIZES = range(2 * EDGE + 8, 4096)    # the host refuses levels below 58 px and images of 4096 px or more


def axis_cells(n, x_axis):
    """FAST cell index of every pixel along one axis of a level (-1 outside every cell), None where the host refuses the level
    (oracle/pyref.py detect_level: minB = 22, nCols = int(width / 30), wCell = ceil(width / nCols); a cell is skipped when it starts
    6 (columns) or 3 (rows) px before maxB; cv::FAST reports nothing in the 3 px frame of a cell's image)"""
    max_b = n - EDGE + 3
    size = max_b - MIN_B
    ncell = int(size / 30.0)
    if ncell < 1:
        return None
    wc = int(math.ceil(size / ncell))
    out = np.full(n, -1, np.int64)
    for j in range(ncell):
        ini = MIN_B + j * wc
        if ini >= max_b - (6 if x_axis else 3):
            continue
        out[ini + 3:min(ini + wc + 6, max_b) - 3] = j
    return out


def runs(cell):
    """lengths of the cells along an axis"""
    return np.bincount(cell[cell >= 0])


def tile_row_maxima(cell, tw):
    """most strict per-cell maxima any tw-pixel tile row can hold: a cell's piece inside the tile holds at most every other pixel"""
    x = np.arange(len(cell))
    first = (cell >= 0) & np.concatenate([[True], cell[1:] != cell[:-1]])
    seg0 = np.maximum(np.maximum.accumulate(np.where(first, x, 0)), x // tw * tw)
    slot = ((cell >= 0) & ((x - seg0) % 2 == 0)).astype(np.int64)
    return int(np.add.reduceat(slot, np.arange(0, len(cell), tw)).max())


def test_cells_are_at_least_30_px_wide():
    """the premise of the segment size: with cells of 30 px or more a 64-pixel row meets at most four cells"""
    for n in LEVEL_SIZES:
        cell = axis_cells(n, True)
        if cell is not None:
            r = runs(cell)
            assert r[:-1].min(initial=30) >= 30, n           # only the last cell can be cut short by the border


def test_warp_segment_holds_the_worst_tile_rows():
    c = constants()
    worst = 0
    for n in LEVEL_SIZES:
        cell = axis_cells(n, True)
        if cell is None:
            continue
        m = tile_row_maxima(cell, c["kTW"])
        assert ROWS_PER_WARP * m <= c["kWarpCorners"], f"level width {n}: {ROWS_PER_WARP} rows of {m} maxima"
        worst = max(worst, m)
    assert worst == c["kTW"] // 2 + 2                                   # the bound is reached: it is not loose
    assert ROWS_PER_WARP * worst > ROWS_PER_WARP * (c["kTW"] // 2)      # one maximum per pixel pair would not be enough


def raw_cap(w, h):
    """the raw corner capacity of a level as build_geometry (mcs_api.cu) computes it: per axis the sum of ceil(cell length / 2)"""
    cx, cy = axis_cells(w, True), axis_cells(h, False)
    return int(((runs(cx) + 1) // 2).sum() * ((runs(cy) + 1) // 2).sum())


def test_raw_capacity_holds_every_strict_maximum():
    """every cell holds at most ceil(w_c / 2) * ceil(h_c / 2) strict maxima (one per 2x2 block); raw_cap must hold the sum over
    the cells.  The old capacity, one maximum per 2x2 block of the whole detection area, falls short as soon as cells have odd
    sides: checked over every level size, with the sum taken cell by cell"""
    short = 0
    for w in LEVEL_SIZES:
        cx = axis_cells(w, True)
        if cx is None:
            continue
        for h in (w, 480, 720, 1080):
            if h not in LEVEL_SIZES or axis_cells(h, False) is None:
                continue
            rw, rh = runs(cx), runs(axis_cells(h, False))
            per_cell = int(np.outer((rw + 1) // 2, (rh + 1) // 2).sum())
            assert per_cell <= raw_cap(w, h), (w, h)
            short += per_cell > ((w - 2 * EDGE + 1) // 2 + 1) * ((h - 2 * EDGE + 1) // 2 + 1)
    assert short > 0
    assert raw_cap(754, 480) == 78045
