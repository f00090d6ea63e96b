"""K1 (pyr_fast_kernel) stages the source region of each 64x64 tile (72x72 with its ring) in shared memory sized per level: box_h
rows of kSrcWB bytes, at most kSrcH rows.  build_geometry (mcs_api.cu) takes the widest and tallest region over a level's tiles as
the level's TMA box and refuses a level whose box exceeds kSrcWB x kSrcH.  These checks recompute the boxes the way the host does
(OpenCV INTER_LINEAR source offsets) for the shipped and tested geometries and for scale factors up to 2, so that none of them is
refused, and check that the config-2 levels (scale 1.2) stage few enough rows for five CTAs per SM."""
import math

import numpy as np
import pytest

from k1_geometry import constants, level_boxes


GEOMETRIES = [(754, 480, 1.2, 8), (1280, 720, 1.2, 8), (1920, 1080, 1.2, 8), (333, 211, 1.2, 4), (754, 480, 1.5, 5),
              (754, 480, 2.0, 3), (754, 480, 1.1, 8), (754, 480, 1.33, 6), (705, 577, 1.2, 8), (833, 383, 1.2, 8), (420, 269, 1.2, 8),
              (1001, 997, 2.0, 4), (999, 963, 2.0, 4), (754, 480, 1.385, 6)]


@pytest.mark.parametrize("W,H,sf,nl", GEOMETRIES)
def test_tested_geometries_fit_the_staging(W, H, sf, nl):
    c = constants()
    for w, h, bw, bh, *_ in level_boxes(W, H, sf, nl):
        assert bw <= c["kSrcWB"] and bh <= c["kSrcH"], (w, h, bw, bh)


def test_scale_factors_up_to_2_fit_the_staging():
    """the bound the host's scale check (source / level ratio <= 2.08) stands for: every ratio it accepts fits kSrcWB x kSrcH"""
    c = constants()
    worst = 0
    for sf in np.linspace(1.05, 2.0, 20):
        for W, H in ((754, 480), (1280, 720), (1001, 997)):
            nl = max(2, min(8, int(math.log(min(W, H) / 80) / math.log(sf)) + 1))
            for w, h, bw, bh, *_ in level_boxes(W, H, float(sf), nl):
                assert bw <= c["kSrcWB"] and bh <= c["kSrcH"], (sf, W, H, w, h, bw, bh)
                worst = max(worst, bh)
    assert worst > c["kSrcH"] - 8                  # scale 2 comes close to the buffer: kSrcH is not loose


def test_config2_levels_stage_few_rows():
    """scale 1.2: 72 * 1.2 + 3 rows, 15.7 KB, below the 17.3 KB that the score tile and the row sums take from the staging area
    after the resize.  With 23 KB of pixel tiles and tables that is 41 KB per CTA, five 256-thread CTAs per SM"""
    c = constants()
    boxes = level_boxes(754, 480, 1.2, 8)
    assert max(b.box_h for b in boxes) <= 90
    assert max(b.box_h for b in boxes) * c["kSrcWB"] <= c["kStagingMin"]
