"""K-best lists of hamming_stream_kernel / hamming_topk_kernel where the pruning bound shared by the four lanes of a quad and the
buffered insertions could go wrong: the K-th and (K+1)-th best of a row at equal distance in columns that different lanes visit
(columns 8m + 2t, 8m + 2t + 1 belong to lane t), in both index orders, in the same and in different 8-column steps, ties exactly
at the relevance bound, and rows where one lane's partial list fills long before the other three (near neighbours clustered in
one residue class mod 8).  Unbounded lists are compared with numpy (distance, index) order; bounded lists, which only the greedy
matchers consume, through their matches against the oracle's SearchByBoW.  Integer work: every comparison is exact."""
import numpy as np
import pytest

from device_frames import INT_MAX
from match_lists import check_stream, greedy_dist_bound, pair_dist, ref_lists, stream_lists

pytestmark = pytest.mark.gpu

LIST_KS = (1, 4, 5, 8)


def planted(rng, dim, masked, K, nq, nd, tie_bits, low_first_lane):
    """queries [nq, dim] and a database [nd, dim] (masks or None).  Query i gets K - 1 near copies, then one more copy at
    tie_bits flipped bits placed twice (identical descriptor and mask: an exact tie) in columns of two different lanes.  Odd
    queries have both copies in the same 8-column step; even ones in different steps, the lower column in lane low_first_lane
    (0: before the other lane's, 3: after it within a step).  Every fourth query
    also gets 2K copies at tie_bits + 1 .. tie_bits + 2 flipped bits, all in one residue class mod 8 among the first 600
    columns: that lane's list fills first.  Queries with planted exact distances have all-ones masks, so that their masked
    distance is the plain popcount."""
    q = rng.integers(0, 256, (nq, dim), dtype=np.uint8)
    d = rng.integers(0, 256, (nd, dim), dtype=np.uint8)
    qm = np.packbits(rng.random((nq, dim * 8)) < 0.6, axis=1, bitorder="little") if masked else None
    dm = np.packbits(rng.random((nd, dim * 8)) < 0.6, axis=1, bitorder="little") if masked else None
    free = np.ones(nd, bool)

    def take(cols):
        cols = [c for c in cols if free[c]]
        free[cols] = False
        return cols

    def put(cols, i, bits):
        for c in cols:
            d[c] = q[i] ^ np.packbits(rng.permutation(dim * 8) < bits, bitorder="little")
            if masked:
                dm[c] = 0xFF
    for i in range(nq):
        if masked:
            qm[i] = 0xFF
        if i % 4 == 0:                                     # one lane's list fills long before the others
            rho = int(rng.integers(0, 8))
            put(take(list(rng.permutation(np.arange(rho, 600, 8))[:2 * K])), i, tie_bits + 1 + int(rng.integers(0, 2)))
        for c in take(list(rng.choice(np.flatnonzero(free), K - 1, replace=False))):
            put([c], i, int(rng.integers(0, tie_bits)))
        if i % 2:                                          # same step: the lower column is in the lower lane
            lo_lane, hi_lane = sorted(int(x) for x in rng.choice(4, 2, replace=False))
        else:
            lo_lane, hi_lane = low_first_lane, (low_first_lane + 1 + int(rng.integers(0, 3))) % 4
        for _ in range(100):
            step = int(rng.integers(0, nd // 8 - 1))
            other = step if i % 2 else int(rng.integers(step + 1, nd // 8))
            c1, c2 = 8 * step + 2 * lo_lane + int(rng.integers(0, 2)), 8 * other + 2 * hi_lane + int(rng.integers(0, 2))
            if c1 < c2 and c2 < nd and free[c1] and free[c2]:
                break
        else:
            raise AssertionError("no free pair of columns")
        put(take([c1]), i, tie_bits)
        d[c2] = d[c1]
        if masked:
            dm[c2] = dm[c1]
        take([c2])
    return q, d, qm, dm


@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("K", LIST_KS)
def test_stream_lists_planted_ties(api, dim, masked, K):
    """stream lists (4- and 8-entry kernels) with the K-th / (K+1)-th tie across lanes, both index orders"""
    for low_first_lane in (0, 3):
        rng = np.random.default_rng(1000 * dim + 100 * masked + 10 * K + low_first_lane)
        nq, nd = 96, 2000
        q, d, qm, dm = planted(rng, dim, masked, K, nq, nd, dim // 2, low_first_lane)
        cap = nd
        desc = np.zeros((2, cap, dim), np.uint8)
        desc[0], desc[1, :nq] = d, q
        dmask = None
        if masked:
            dmask = np.zeros_like(desc)
            dmask[0], dmask[1, :nq] = dm, qm
        counts = np.array([nd, nq], np.int32)
        idx, dist = stream_lists(api, desc, dmask, counts, 2, 1, K)
        check_stream(desc, dmask, counts, 1, idx, dist, K)
        ri, rd = ref_lists(pair_dist(q, d, qm, dm), K + 1)
        assert (rd[:, K - 1] == rd[:, K]).mean() > 0.9            # the planted ties are the K-th and (K+1)-th best


@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("K", LIST_KS)
def test_topk_lists_planted_ties(api, dim, masked, K):
    """top-K lists over 8 database chunks merged by topk_merge_kernel, host and device entry points, with and without a skip
    mask that removes some of the tie columns"""
    import torch
    rng = np.random.default_rng(2000 * dim + 100 * masked + 10 * K)
    q, d, qm, dm = planted(rng, dim, masked, K, 128, 2048, dim // 2, int(rng.integers(0, 4)))
    dist = pair_dist(q, d, qm, dm)
    skip = (rng.random(len(d)) < 0.05).astype(np.uint8)
    dev = torch.device("cuda", 0)
    t = lambda a: None if a is None else torch.from_numpy(a).to(dev)  # noqa: E731
    for sk in (None, skip):
        ref = dist if sk is None else np.where(sk[None, :] != 0, 1 << 20, dist)
        ri, rd = ref_lists(ref, K)
        ri, rd = np.where(rd >= 1 << 20, -1, ri), np.where(rd >= 1 << 20, INT_MAX, rd)
        idx, dd = api.hamming_topk(q, d, K, qm, dm, db_skip=sk)
        assert np.array_equal(idx, ri) and np.array_equal(dd, rd), (K, sk is None)
        gi, gd = api.hamming_topk_device(t(q), t(d), K, t(qm), t(dm), t(sk))
        torch.cuda.synchronize(dev)
        assert np.array_equal(gi.cpu().numpy(), ri) and np.array_equal(gd.cpu().numpy(), rd), (K, sk is None, "device")


@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masked", [False, True])
def test_bounded_lists_ties_at_bound(api, oa, dim, masked):
    """bounded lists through the greedy matchers (stream: match_stream_greedy_device; key-frame:
    match_bruteforce_device) against the oracle, with the planted ties one below, at and one above the relevance bound of
    (TH_LOW_, 0.9) and (TH_LOW_, 1.0)"""
    import torch
    dev = torch.device("cuda", 0)
    t = lambda a: None if a is None else torch.from_numpy(a).to(dev)  # noqa: E731
    matcher = api.cORBmatcher(0.9, False, dim, masked)
    th = matcher.TH_LOW_
    for nn in (0.9, 1.0):
        bound = greedy_dist_bound(th, nn)
        for k, tie in enumerate((bound - 1, bound, bound + 1, th - 1)):
            if tie >= dim * 4:
                continue
            rng = np.random.default_rng(3000 * dim + 100 * masked + 10 * k + int(nn * 10))
            nq, nd = 96, 2000
            q, d, qm, dm = planted(rng, dim, masked, 8, nq, nd, tie, k % 4)
            desc = np.zeros((2, nd, dim), np.uint8)
            desc[0], desc[1, :nq] = d, q
            dmask = None
            if masked:
                dmask = np.zeros_like(desc)
                dmask[0], dmask[1, :nq] = dm, qm
            m12, nm = api.match_stream_greedy_device(t(desc), t(dmask), t(np.array([nd, nq], np.int32)), 2, 1, th, nn)
            torch.cuda.synchronize(dev)
            on, om = oa.match_bruteforce(q, d, th, nn, qm, dm)
            assert int(nm.cpu()[1]) == on and np.array_equal(m12.cpu().numpy()[1, :nq], om), (nn, tie, "stream")
            n1, m1 = api.match_bruteforce_device(t(q), t(qm), None, t(d), t(dm), None, th, nn)
            assert n1 == on and np.array_equal(m1, om), (nn, tie, "key-frame")
            assert (pair_dist(q, d, qm, dm) == tie).any(axis=1).mean() > 0.9
