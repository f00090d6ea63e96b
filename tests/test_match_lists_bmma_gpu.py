"""K-best lists of the binary tensor-core kernels (hamming_stream_kernel, hamming_topk_kernel) at the edges of their tiling:
query and database counts around the 16x8 fragment and the 256-entry shared-memory tile, all-equal distances (every pair
ties, the list is decided by the index alone and its entries are spread over the four lanes of a quad), and a query that
equals a database row whose mask is all zero (masked distance 0 from both masks' terms).  Compared with numpy; exact."""
import numpy as np
import pytest

from device_frames import INT_MAX
from match_lists import check_stream, pair_dist, ref_lists, stream_lists

pytestmark = pytest.mark.gpu

EDGE_COUNTS = (1, 2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17, 255, 256, 257)


@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("K", [3, 8])
def test_stream_lists_tile_edges(api, dim, masked, K):
    """every (query count, database count) pair of EDGE_COUNTS, on consecutive images of one camera"""
    rng = np.random.default_rng(dim * 10 + masked * 2 + K)
    seq = [n for a in EDGE_COUNTS for n in (a, EDGE_COUNTS[(EDGE_COUNTS.index(a) * 7 + 3) % len(EDGE_COUNTS)])]
    counts = np.array([257] + seq, np.int32)
    cap = 260
    desc = rng.integers(0, 256, (len(counts), cap, dim), dtype=np.uint8)
    dmask = (rng.integers(0, 256, desc.shape, dtype=np.uint8) | rng.integers(0, 256, desc.shape, dtype=np.uint8)) if masked else None
    idx, dist = stream_lists(api, desc, dmask, counts, len(counts), 1, K)
    check_stream(desc, dmask, counts, 1, idx, dist, K)


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("K", [4, 8])
def test_stream_lists_all_ties(api, masked, K):
    """a database of identical descriptors: every distance ties, the lists are the first K slots"""
    rng = np.random.default_rng(7 + masked + K)
    cap, dim = 300, 32
    counts = np.array([299, 300, 17, 257], np.int32)
    desc = rng.integers(0, 256, (4, cap, dim), dtype=np.uint8)
    desc[0] = desc[0, 0]
    desc[2] = desc[2, 0]
    dmask = None
    if masked:
        dmask = rng.integers(0, 256, desc.shape, dtype=np.uint8) | rng.integers(0, 256, desc.shape, dtype=np.uint8)
        dmask[0] = dmask[0, 0]
        dmask[2] = dmask[2, 0]
        desc[1, :, :] = desc[1, 0]                      # and identical queries with identical masks
        dmask[1, :, :] = dmask[1, 0]
    idx, dist = stream_lists(api, desc, dmask, counts, 4, 1, K)
    check_stream(desc, dmask, counts, 1, idx, dist, K)
    assert (idx[1, :300] == np.arange(K)).all() and (idx[3, :257] == np.arange(K)).all()


def test_stream_lists_zero_mask_copy(api):
    """a query equal to a database row whose mask is all zero: masked distance 0, listed first"""
    rng = np.random.default_rng(11)
    cap, dim = 64, 32
    counts = np.array([40, 40], np.int32)
    desc = rng.integers(0, 256, (2, cap, dim), dtype=np.uint8)
    dmask = rng.integers(0, 256, desc.shape, dtype=np.uint8) | rng.integers(0, 256, desc.shape, dtype=np.uint8)
    dmask[0, 13] = 0
    desc[1, 5] = desc[0, 13]
    idx, dist = stream_lists(api, desc, dmask, counts, 2, 1, 4)
    check_stream(desc, dmask, counts, 1, idx, dist, 4)
    assert idx[1, 5, 0] == 13 and dist[1, 5, 0] == 0


@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masked", [False, True])
def test_topk_tile_edges(api, dim, masked):
    """host and device top-K entry points at query and database counts around the fragment and tile edges, with a skip mask"""
    import torch
    rng = np.random.default_rng(dim + 100 * masked)
    dev = torch.device("cuda", 0)
    for nq, nd in [(1, 1), (9, 15), (16, 16), (17, 17), (255, 256), (257, 255), (8, 257), (256, 9)]:
        q = rng.integers(0, 256, (nq, dim), dtype=np.uint8)
        d = rng.integers(0, 256, (nd, dim), dtype=np.uint8)
        d[nd // 2] = q[0]
        qm = (rng.integers(0, 256, q.shape, dtype=np.uint8) | rng.integers(0, 256, q.shape, dtype=np.uint8)) if masked else None
        dm = (rng.integers(0, 256, d.shape, dtype=np.uint8) | rng.integers(0, 256, d.shape, dtype=np.uint8)) if masked else None
        if masked:
            dm[nd // 2] = 0
        skip = (rng.random(nd) < 0.2).astype(np.uint8)
        skip[nd // 2] = 0
        dist = pair_dist(q, d, qm, dm)
        for K, sk in ((5, None), (8, skip)):
            ref = dist if sk is None else np.where(sk[None, :] != 0, 1 << 20, dist)
            ri, rd = ref_lists(ref, K)
            cut = rd >= (1 << 20)
            ri, rd = np.where(cut, -1, ri), np.where(cut, INT_MAX, rd)
            idx, dd = api.hamming_topk(q, d, K, qm, dm, db_skip=sk)
            assert np.array_equal(idx, ri) and np.array_equal(dd, rd), (nq, nd, K)
            t = lambda a: None if a is None else torch.from_numpy(a).to(dev)
            gi, gd = api.hamming_topk_device(t(q), t(d), K, t(qm), t(dm), t(sk))
            torch.cuda.synchronize()
            assert np.array_equal(gi.cpu().numpy(), ri) and np.array_equal(gd.cpu().numpy(), rd), (nq, nd, K, "device")
        assert idx[0, 0] == nd // 2 or dist[0, idx[0, 0]] == 0


def test_topk_all_ties(api):
    """every database entry identical: the lists are the first K indices, across database splits"""
    rng = np.random.default_rng(5)
    q = rng.integers(0, 256, (130, 32), dtype=np.uint8)
    d = np.broadcast_to(rng.integers(0, 256, (1, 32), dtype=np.uint8), (3000, 32)).copy()
    idx, dd = api.hamming_topk(q, d, 8)
    assert (idx == np.arange(8)).all()
    assert np.array_equal(dd, np.broadcast_to(pair_dist(q, d[:1])[:, :1], (130, 8)))
