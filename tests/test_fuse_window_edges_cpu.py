"""CPU: Fuse's window decisions on scenes built at their edges (tests/fuse_window_scenes.py), for all three overloads:
Fuse(pKF, curKF, ., th) and Fuse(pKF, Scw, ., th) keep the best candidate (ref :1265, :1570), Fuse(pKF, ., th) the first one
in visiting order (:1420).  The scenes put keypoints on and one float beyond a window's radius, on exact cell-range bounds,
at the corner of two cells whose visiting order is opposite to their slot order, behind 36 failing items of a crowded cell,
around the l = 0 and top-level filters, past the image's edges, at TH_LOW_ and TH_LOW_ + 1, in windows whose items all fail
the level test and in a camera without keypoints.

Here the scene is checked: every case decides as it was built to, a numpy model of the walk reproduces the host's hits and
gives other hits under each mistake a copy of the walk could make, and the host Fuse (over the oracle's window search) gives
the reference's own map mutations (replayed from tests/golden/ref_tape_fuse_window_edges_cpu.*, see oracle/ref_tape.py).
tests/test_fuse_window_edges_gpu.py runs the device on the same scenes."""
from collections import Counter

import numpy as np
import pytest

from device_frames import taped_rm
from fuse_window_scenes import (BEST_MUTATIONS, EDGES, EMPTY_CAM, FIRST_MUTATIONS, N_KF, N_NOKEYS, PLAN, _grid, cameras, designed, host_best,
                                model_best, scene, thresholds, windows)
from search_scenes import host_fuse, reference_ops

rm = taped_rm("fuse_window_edges_cpu")


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_scene_reaches_every_case(api, oa, variant):
    """each kind is built the stated number of times, and each window decides for the keypoint it was built around (or for
    none), on the oracle's window search and on the model; the model's grid is the oracle's"""
    KFs, ss = scene(api, oa, variant)
    m = api.cORBmatcher(0.6, False, 32, False)
    seen = Counter()
    for k, (KF, s) in enumerate(zip(KFs, ss)):
        _, start, items = oa.frame_prepare(KF.keys, KF.key_cam, cameras())
        cells = _grid(KF)
        flat = [cells.get((c, ix, iy), []) for c in range(len(KF.cam_w)) for ix in range(64) for iy in range(48)]
        assert np.array_equal(np.diff(start), [len(v) for v in flat]) and items.tolist() == [j for v in flat for j in v]
        assert (KF.key_cam == EMPTY_CAM).sum() == 0
        hb = host_best(api, m, KF, s, variant, _sw=oa.search_windows)
        assert np.array_equal(model_best(api, KF, s, variant, m.TH_LOW_, False), hb)
        for kind, i, c, want in designed(api, KF, s, variant, k):
            assert hb[i, c] == want, (k, kind, i)
            seen[kind] += 1
        # the crowded cells hold more than 40 items, the first hit among them is item 37
        per_cell = np.diff(start)
        assert per_cell.max() >= 41
    want = {kind: 2 * N_KF * n for kind, n in PLAN.items()}
    want.update({e: 2 * N_KF for e in EDGES}, nokeys=N_KF * N_NOKEYS)
    assert seen == Counter(want)


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_edges_discriminate(api, oa, variant):
    """the model's hits change under each mistake a copy of the walk could make: `>=` in the radius test or the test in float32,
    the cells row by row, ties broken by slot, `< TH_LOW_`, the level filter {l, l + 1}, the first-candidate walk stopping
    after a cell's first 32 items"""
    KFs, ss = scene(api, oa, variant)
    th_low, _ = thresholds(32, False)
    wins = [windows(api, KF, s, variant) for KF, s in zip(KFs, ss)]
    base = [model_best(api, KF, s, variant, th_low, False, win=w) for KF, s, w in zip(KFs, ss, wins)]
    for mut in (FIRST_MUTATIONS if variant == 1 else BEST_MUTATIONS):
        changed = sum(int((model_best(api, KF, s, variant, th_low, False, (mut,), w) != b).sum()) for KF, s, w, b in zip(KFs, ss, wins, base))
        assert changed >= 4, mut


@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("variant", [0, 1, 2])
def test_host_fuse_equals_reference(api, oa, rm, variant, dim, masks):
    """per key frame: the host Fuse over the oracle's window search gives the reference's mutations in order, and its window
    decisions are the model's, at every width with masks on and off"""
    KFs, ss = scene(api, oa, variant, dim, masks)
    m = api.cORBmatcher(0.6, False, dim, masks)
    for k, (KF, s) in enumerate(zip(KFs, ss)):
        rn, rops = reference_ops(api, rm, cameras(), KF, s, variant, masks)
        on, oops, _ = host_fuse(api, m, KF, s, variant, _sw=oa.search_windows)
        assert rn == on and np.array_equal(rops, oops) and len(oops) > 40
        hb = host_best(api, m, KF, s, variant, _sw=oa.search_windows)
        assert np.array_equal(model_best(api, KF, s, variant, m.TH_LOW_, masks), hb)
        assert all(hb[i, c] == want for _, i, c, want in designed(api, KF, s, variant, k))
