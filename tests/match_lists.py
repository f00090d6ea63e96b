"""Plain-numpy K-best lists and the stream matcher's list read-back, for the list kernels' GPU tests."""
import numpy as np

from device_frames import INT_MAX


def pair_dist(q, d, qm=None, dm=None):
    """[nq, nd] distances: popcount of q ^ d, or the masked form (popc(x & qm) + popc(x & dm)) // 2 summed over the descriptor"""
    q64 = np.ascontiguousarray(q).view(np.uint64)
    d64 = np.ascontiguousarray(d).view(np.uint64)
    out = np.zeros((len(q), len(d)), np.int64)
    for r0 in range(0, len(q), 256):
        x = q64[r0:r0 + 256, None, :] ^ d64[None, :, :]
        if qm is None:
            out[r0:r0 + 256] = np.bitwise_count(x).sum(axis=2, dtype=np.int64)
        else:
            a = np.bitwise_count(x & np.ascontiguousarray(qm).view(np.uint64)[r0:r0 + 256, None, :]).sum(axis=2, dtype=np.int64)
            b = np.bitwise_count(x & np.ascontiguousarray(dm).view(np.uint64)[None, :, :]).sum(axis=2, dtype=np.int64)
            out[r0:r0 + 256] = (a + b) // 2
    return out


def ref_lists(dist, K):
    """the K best (index, distance) of every row ordered by (distance, index), padded with (-1, INT_MAX)"""
    order = np.argsort(dist, axis=1, kind="stable")[:, :K]
    idx = np.full((dist.shape[0], K), -1, np.int32)
    dd = np.full((dist.shape[0], K), INT_MAX, np.int32)
    idx[:, :order.shape[1]] = order
    dd[:, :order.shape[1]] = np.take_along_axis(dist, order, axis=1)
    return idx, dd


def greedy_dist_bound(th_low, nnratio):
    """mirror of greedy_dist_bound (multicol_slam_b200/csrc/kernels.h): lists of the greedy matchers stop below this distance"""
    if th_low <= 0:
        return 0
    b = th_low
    while b < (1 << 20) and not (th_low - 1 < nnratio * b):
        b += 1
    return b


def stream_lists(api, desc, dmask, counts, n_frames, n_cams, K):
    import torch
    dev = torch.device("cuda", 0)
    idx, dist = api.match_stream_device(torch.from_numpy(desc).to(dev), None if dmask is None else torch.from_numpy(dmask).to(dev),
                                        torch.from_numpy(counts).to(dev), n_frames, n_cams, K=K)
    torch.cuda.synchronize()
    return idx.cpu().numpy(), dist.cpu().numpy()


def check_stream(desc, dmask, counts, n_cams, idx, dist, K):
    cap = desc.shape[1]
    for b in range(len(counts)):
        if b < n_cams or counts[b] == 0:
            assert (idx[b] == -1).all() and (dist[b] == INT_MAX).all(), b
            continue
        nq, nd = counts[b], counts[b - n_cams]
        if nd == 0:
            ri, rd = np.full((nq, K), -1, np.int32), np.full((nq, K), INT_MAX, np.int32)
        else:
            qm = None if dmask is None else dmask[b, :nq]
            dm = None if dmask is None else dmask[b - n_cams, :nd]
            ri, rd = ref_lists(pair_dist(desc[b, :nq], desc[b - n_cams, :nd], qm, dm), K)
        assert np.array_equal(idx[b, :nq], ri) and np.array_equal(dist[b, :nq], rd), (b, nq, nd)
        assert (idx[b, nq:cap] == -1).all() and (dist[b, nq:cap] == INT_MAX).all(), b
