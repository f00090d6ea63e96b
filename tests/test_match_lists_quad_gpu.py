"""K-best lists of hamming_stream_kernel / hamming_topk_kernel, which keep one list per query row spread over the four lanes of a
quad and buffer a pair iff its (distance, index) key is below the row's K-th key.  Planted rows: the K-th and (K+1)-th best at
an exact tie in columns of different lanes (columns 8m + 2t, 8m + 2t + 1 belong to lane t), in one 8-column step (merged in the
same fold) and in steps far apart (the later one must be refused at the buffer); 3K exact copies at one distance over every
lane; and bursts of 36 near copies inside one 256-column tile, each closer than the previous, so that more than the quad's
4 x kCandDepth = 28 buffer slots of one row fill between folds.  Compared with numpy (distance, index) order; exact."""
import numpy as np
import pytest

from match_lists import check_stream, pair_dist, ref_lists, stream_lists

pytestmark = pytest.mark.gpu

BURST = 36                      # > 4 * kCandDepth (multicol_slam_b200/csrc/match_kernels.cu)


def planted(rng, dim, masked, K, nq, nd):
    """queries [nq, dim], database [nd, dim] and masks (or None).  Row i % 8 in {0, 4}: K - 1 near copies and a tie at the
    K-th place (same step for i % 8 == 0, steps apart for 4); 1: a burst; 5: 3K exact copies at one distance; others random.
    Planted rows and their copies have all-ones masks, so that the masked distance is the plain popcount."""
    q = rng.integers(0, 256, (nq, dim), dtype=np.uint8)
    d = rng.integers(0, 256, (nd, dim), dtype=np.uint8)
    qm = np.packbits(rng.random((nq, dim * 8)) < 0.6, axis=1, bitorder="little") if masked else None
    dm = np.packbits(rng.random((nd, dim * 8)) < 0.6, axis=1, bitorder="little") if masked else None
    free = np.ones(nd, bool)
    tie_bits = dim

    def copy(i, c, bits):
        free[c] = False
        d[c] = q[i] ^ np.packbits(rng.permutation(dim * 8) < bits, bitorder="little")
        if masked:
            dm[c] = 0xFF

    def free_in(lo, hi):
        return lo + np.flatnonzero(free[lo:hi])

    for i in range(nq):
        kind = i % 8
        if kind not in (0, 1, 4, 5):
            continue
        if masked:
            qm[i] = 0xFF
        if kind == 1:
            tiles = [t0 for t0 in range(0, nd - 255, 256) if len(free_in(t0, t0 + 256)) >= BURST]
            t0 = tiles[int(rng.integers(0, len(tiles)))]
            cols = np.sort(rng.choice(free_in(t0, t0 + 256), BURST, replace=False))
            for j, c in enumerate(cols):                     # each column closer than every earlier one
                copy(i, c, BURST + 4 - j)
        elif kind == 5:
            cols = rng.choice(free_in(0, nd), 3 * K, replace=False)
            copy(i, cols[0], tie_bits)
            for c in cols[1:]:
                free[c] = False
                d[c] = d[cols[0]]
                if masked:
                    dm[c] = dm[cols[0]]
        else:
            for c in rng.choice(free_in(0, nd), K - 1, replace=False):
                copy(i, c, int(rng.integers(0, tie_bits)))
            while True:
                lanes = rng.choice(4, 2, replace=False)
                s1 = int(rng.integers(0, nd // 8 - 1))
                s2 = s1 if kind == 0 else int(rng.integers(s1 + 1, nd // 8))
                c1, c2 = (8 * s + 2 * int(t) + int(rng.integers(0, 2)) for s, t in zip((s1, s2), lanes))
                if c1 != c2 and free[c1] and free[c2]:
                    break
            copy(i, c1, tie_bits)
            free[c2] = False
            d[c2] = d[c1]
            if masked:
                dm[c2] = dm[c1]
    return q, d, qm, dm


@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("K", range(1, 9))
def test_quad_lists_planted(api, dim, masked, K):
    """stream lists (match_stream_device) and top-K lists (hamming_topk_device) of the planted rows equal numpy"""
    import torch
    rng = np.random.default_rng(100 * dim + 10 * masked + K)
    nq, nd = 128, 2048
    q, d, qm, dm = planted(rng, dim, masked, K, nq, nd)
    ri, rd = ref_lists(pair_dist(q, d, qm, dm), K + 1)
    tie = np.arange(nq) % 8
    assert (rd[(tie == 0) | (tie == 4), K - 1] == rd[(tie == 0) | (tie == 4), K]).all()   # the planted ties are at the K-th place

    desc = np.zeros((2, nd, dim), np.uint8)
    desc[0], desc[1, :nq] = d, q
    dmask = None
    if masked:
        dmask = np.zeros_like(desc)
        dmask[0], dmask[1, :nq] = dm, qm
    counts = np.array([nd, nq], np.int32)
    idx, dist = stream_lists(api, desc, dmask, counts, 2, 1, K)
    check_stream(desc, dmask, counts, 1, idx, dist, K)

    dev = torch.device("cuda", 0)
    t = lambda a: None if a is None else torch.from_numpy(a).to(dev)  # noqa: E731
    gi, gd = api.hamming_topk_device(t(q), t(d), K, t(qm), t(dm), None)
    torch.cuda.synchronize(dev)
    assert np.array_equal(gi.cpu().numpy(), ri[:, :K]) and np.array_equal(gd.cpu().numpy(), rd[:, :K])
