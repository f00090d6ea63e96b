"""Every matcher kernel instantiation the launchers can pick, against plain references.

- Stream matcher: the K-best list kernel (hamming_stream_kernel, 4- and 8-entry lists) and the greedy acceptance on both replay
  paths (stream_replay_smem_kernel for one wave of images whose database fits in shared memory, stream_replay_kernel otherwise)
  at 16-, 32- and 64-byte descriptors, with and without masks.
- Key-frame brute force (bruteforce_replay_kernel) at 16 and 64 bytes, with and without cooperative helper CTAs, and the limit
  of its database size.
- Top-K (hamming_topk_kernel) with 5..7 entries, a skip mask and the database split over many CTAs.
- The host stream pipeline (extract + match in chunks of frames) across its chunk boundaries.

Lists are compared with numpy all-pairs distances ordered by (distance, index); matches with the oracle's SearchByBoW(KF1, KF2).
Integer work: every comparison is exact."""
import math
import re

import numpy as np
import pytest

from device_frames import INT_MAX
from match_lists import greedy_dist_bound, pair_dist, ref_lists

pytestmark = pytest.mark.gpu


def bounded(idx, dist, bound):
    """lists cut at the relevance bound: entries at distance >= bound become (-1, INT_MAX)"""
    cut = dist >= bound
    return np.where(cut, -1, idx), np.where(cut, INT_MAX, dist)


def replay_uses_smem(n_images, sms, capacity, dim, masked, K):
    """launch_stream_replay's choice (multicol_slam_b200/csrc/match_kernels.cu:800-807): stream_replay_smem_kernel when the
    launch holds no more images than the device has SMs and the previous image's descriptors (and masks) fit in 200 KB beside
    the walk, stream_replay_kernel otherwise"""
    smem = 64 * K * 4 + (capacity + 31) // 32 * 4
    return n_images <= sms and smem + capacity * dim * (2 if masked else 1) + 16 <= 200 * 1024


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def flip_bits(rng, src, max_rate):
    """near copies: every row gets each bit flipped with its own probability in [0, max_rate)"""
    n, dim = src.shape
    rate = rng.uniform(0, max_rate, (n, 1))
    return src ^ np.packbits(rng.random((n, dim * 8)) < rate, axis=1, bitorder="little")


def edge_counts(rng, n_frames, n_cams, capacity):
    """per-image descriptor counts: frame 0 full, then 0 (no queries against frame 0, no database for frame 2), 1, 31, 32, 33
    and capacity on the images after frame 0, the rest random"""
    c = rng.integers(capacity // 2, capacity + 1, n_frames * n_cams).astype(np.int32)
    c[0] = capacity
    edges = [0, 1, 31, 32, 33, capacity]
    n = min(len(edges), len(c) - n_cams)
    c[n_cams:n_cams + n] = edges[:n]
    c[-1] = capacity
    return c


def clustered_stream(rng, n_frames, n_cams, capacity, dim, counts):
    """descriptor slots [B, capacity, dim] (and masks) with dozens of near-duplicates per query, so that K-best lists run out
    and the acceptance kernels rescan.  Slots past an image's count hold a cluster centre: a kernel reading past the count
    would find it.  Image i's first query is an exact copy of its database's first and last entries (masks included): a
    best == second tie, which the ratio test must reject."""
    B = n_frames * n_cams
    centres = rng.integers(0, 256, (12, dim), dtype=np.uint8)
    desc = np.broadcast_to(centres[0], (B, capacity, dim)).copy()
    dmask = np.full((B, capacity, dim), 0xFF, np.uint8)
    for b in range(B):
        n = counts[b]
        which = rng.choice(13, n, p=[0.09] * 8 + [0.025] * 4 + [0.18])
        base = np.where((which < 12)[:, None], centres[np.minimum(which, 11)], rng.integers(0, 256, (n, dim), dtype=np.uint8))
        desc[b, :n] = flip_bits(rng, base, 14 / 256)
        dmask[b, :n] = rng.integers(0, 256, (n, dim), dtype=np.uint8) | rng.integers(0, 256, (n, dim), dtype=np.uint8)
    ties = []
    for b in range(n_cams, B):
        nd = counts[b - n_cams]
        if counts[b] >= 1 and nd >= 2:
            desc[b - n_cams, nd - 1], dmask[b - n_cams, nd - 1] = desc[b - n_cams, 0], dmask[b - n_cams, 0]
            desc[b, 0] = desc[b - n_cams, 0]
            ties.append(b)
    return desc, dmask, ties


# (descriptor bytes, masks, capacity, replay path).  "global" launches hold more images than the device has SMs; the 2016-slot
# 64-byte masked case (mdBRIEF descSize=64 at 2000 features) takes stream_replay_kernel by size alone.
STREAM_CASES = ([(dim, m, 700, "smem") for dim in (16, 32, 64) for m in (False, True)]
                + [(dim, m, 600, "global") for dim in (16, 32, 64) for m in (False, True)]
                + [(32, True, 2016, "smem"), (64, True, 2016, "global")])
LIST_KS = (1, 4, 5, 8)          # both list instantiations (4 and 8 entries), full and partial


def stream_shape(path, capacity):
    """(n_frames, n_cams) of a stream case"""
    if path == "global" and capacity < 1000:
        nc = 4
        return sm_count() // nc + 2, nc
    return (4, 3) if path == "smem" else (2, 3)


def make_stream_case(dim, masked, capacity, path, seed):
    rng = np.random.default_rng(seed)
    F, nc = stream_shape(path, capacity)
    counts = edge_counts(rng, F, nc, capacity)
    desc, dmask, ties = clustered_stream(rng, F, nc, capacity, dim, counts)
    return F, nc, counts, desc, dmask if masked else None, ties


def stream_thresholds(api, dim, masked):
    """(th_low, nnratio) pairs: the matcher's own, one whose bound excludes nothing, a tight one, one that accepts nothing, and
    ratio 1.0 where the planted best == second ties must be rejected"""
    th = api.cORBmatcher(0.9, False, dim, masked).TH_LOW_
    return [(th, 0.9), (dim * 8 + 1, 0.99), (1, 0.5), (0, 0.9), (th, 1.0)]


@pytest.mark.parametrize("dim,masked,capacity,path", STREAM_CASES,
                         ids=[f"d{d}-{'m' if m else 'u'}-cap{c}-{p}" for d, m, c, p in STREAM_CASES])
def test_stream_matcher_variants(api, oa, dim, masked, capacity, path):
    """match_stream_device lists equal numpy for K = 1, 4, 5, 8; match_stream_replay_device over each of them and
    match_stream_greedy_device equal the oracle's SearchByBoW(image, image - n_cams) for five threshold settings"""
    import torch
    F, nc, counts, desc, dmask, ties = make_stream_case(dim, masked, capacity, path, seed=dim * 7 + masked + capacity)
    B = F * nc
    sms = sm_count()
    for K in LIST_KS + (8,):        # the greedy matcher's lists are 8 long
        assert replay_uses_smem(B, sms, capacity, dim, masked, K) == (path == "smem")
    dev = torch.device("cuda", 0)
    d_t, c_t = torch.from_numpy(desc).to(dev), torch.from_numpy(counts).to(dev)
    m_t = torch.from_numpy(dmask).to(dev) if masked else None
    lists = {K: api.match_stream_device(d_t, m_t, c_t, F, nc, K=K) for K in LIST_KS}
    torch.cuda.synchronize(dev)
    host = {K: (i.cpu().numpy(), d.cpu().numpy()) for K, (i, d) in lists.items()}
    for img in range(B):
        n = counts[img]
        for K in LIST_KS:
            gi, gd = host[K]
            if img < nc:
                assert np.all(gi[img] == -1) and np.all(gd[img] == INT_MAX), (img, K)
                continue
            assert np.all(gi[img, n:] == -1) and np.all(gd[img, n:] == INT_MAX), (img, K)
        if img < nc:
            continue
        nd = counts[img - nc]
        dist = pair_dist(desc[img, :n], desc[img - nc, :nd], None if dmask is None else dmask[img, :n],
                         None if dmask is None else dmask[img - nc, :nd])
        ri, rd = ref_lists(dist, 8)
        for K in LIST_KS:
            gi, gd = host[K]
            assert np.array_equal(gi[img, :n], ri[:, :K]) and np.array_equal(gd[img, :n], rd[:, :K]), (img, K)

    accepted = 0
    for th, nn in stream_thresholds(api, dim, masked):
        m12, nm = api.match_stream_greedy_device(d_t, m_t, c_t, F, nc, th, nn)
        replays = {K: api.match_stream_replay_device(*lists[K], c_t, d_t, m_t, F, nc, th, nn) for K in LIST_KS}
        torch.cuda.synchronize(dev)
        runs = [("greedy", m12.cpu().numpy(), nm.cpu().numpy(), None)]
        runs += [(f"replay K={K}", r[0].cpu().numpy(), r[1].cpu().numpy(), r[2].cpu().numpy()) for K, r in replays.items()]
        for img in range(B):
            n = counts[img]
            if img < nc:
                on, om = 0, np.full(n, -1, np.int32)      # frame 0 has no predecessor
            else:
                nd = counts[img - nc]
                on, om = oa.match_bruteforce(desc[img, :n], desc[img - nc, :nd], th, nn, None if dmask is None else dmask[img, :n],
                                             None if dmask is None else dmask[img - nc, :nd])
            for what, gm, gn, redo in runs:
                assert gn[img] == on and np.array_equal(gm[img, :n], om), (th, nn, img, what)
                assert np.all(gm[img, n:] == -1), (th, nn, img, what)
                if redo is not None:
                    assert redo[img] == 0
        for b in ties:                           # best == second: never accepted while nnratio <= 1
            assert runs[0][1][b, 0] == -1, (th, nn, b)
        if th == 0:
            assert runs[0][2].sum() == 0
        accepted += int(runs[0][2].sum())
    assert accepted > 10 * (B - nc) and len(ties) >= 2


@pytest.mark.parametrize("nd", [5000, 40000])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("dim", [16, 64])
def test_keyframe_bruteforce_widths(api, oa, dim, masked, nd):
    """SearchByBoW (host entry), match_bruteforce_device per query set and match_bruteforce_batch_device over 3 sets, at 16 and
    64 bytes, against the oracle per set.  nd = 5000 walks in one CTA per set; nd >= 32768 adds cooperative helper CTAs to every
    rescan (match_kernels.cu launch_bruteforce_replay).  Clusters of near-identical queries against 12 near copies of each
    cluster centre use up the 8-entry lists, so that the acceptance kernel rescans."""
    import torch
    rng = np.random.default_rng(dim + 3 * masked + nd)
    nseg, ncl, per_cl = 3, 60, 6
    centres = rng.integers(0, 256, (ncl, dim), dtype=np.uint8)
    db = rng.integers(0, 256, (nd, dim), dtype=np.uint8)
    db[rng.choice(nd, ncl * 12, replace=False)] = flip_bits(rng, np.repeat(centres, 12, axis=0), 8 / 256)
    dbm = np.packbits(rng.random((nd, dim * 8)) < 0.9, axis=1, bitorder="little")
    q = np.concatenate([flip_bits(rng, np.repeat(centres, per_cl, axis=0)[rng.permutation(ncl * per_cl)], 6 / 256)
                        for _ in range(nseg)])
    qm = np.packbits(rng.random((len(q), dim * 8)) < 0.9, axis=1, bitorder="little")
    if not masked:
        qm = dbm = None
    valid1 = (rng.random(len(q)) < 0.93).astype(np.uint8)
    valid2 = (rng.random(nd) < 0.97).astype(np.uint8)
    seg = np.arange(nseg + 1) * (ncl * per_cl)
    dev = torch.device("cuda", 0)
    t = lambda a: None if a is None else torch.from_numpy(a).to(dev)  # noqa: E731
    for nn in (0.9, 1.01):                       # 1.01: cluster members keep taking entries, many rescans
        matcher = api.cORBmatcher(nn, False, dim, masked)
        th = matcher.TH_LOW_
        n_all, m_all = matcher.SearchByBoW(q, db, qm, dbm, valid1, valid2)
        on_all, om_all = oa.match_bruteforce(q, db, th, nn, qm, dbm, valid1, valid2)
        assert n_all == on_all and np.array_equal(m_all, om_all), nn
        nms, m12 = api.match_bruteforce_batch_device(t(q), t(qm), valid1, seg, t(db), t(dbm), valid2, th, nn)
        for s in range(nseg):
            sl = slice(seg[s], seg[s + 1])
            on, om = oa.match_bruteforce(q[sl], db, th, nn, None if qm is None else qm[sl], dbm, valid1[sl], valid2)
            n1, m1 = api.match_bruteforce_device(t(q[sl]), t(None if qm is None else qm[sl]), valid1[sl], t(db), t(dbm), valid2, th, nn)
            assert n1 == on == nms[s] and np.array_equal(m1, om) and np.array_equal(m12[sl], om), (nn, s)
            if nn > 1:
                assert on > 0.5 * valid1[sl].sum()


@pytest.mark.parametrize("K", [5, 7])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("dim", [16, 64])
def test_topk_long_lists_skip_device(api, dim, masked, K):
    """hamming_topk (host) and hamming_topk_device with 5..7-entry lists (the 8-entry kernel), a skip mask, and 100 queries: the
    5000-entry database is split over 20 CTAs whose partial lists are merged.  Exact copies of a query sit in different splits:
    equal distances keep the lower index; a skipped copy never appears."""
    import torch
    rng = np.random.default_rng(100 * dim + 10 * K + masked)
    nq, nd = 100, 5000
    q = rng.integers(0, 256, (nq, dim), dtype=np.uint8)
    d = rng.integers(0, 256, (nd, dim), dtype=np.uint8)
    src = rng.integers(0, nq, 600)
    src[src == 3] = 4                            # only the planted copies are at distance 0 from query 3
    d[rng.choice(nd, 600, replace=False)] = flip_bits(rng, q[src], 20 / 256)   # close neighbours
    copies = [10, 1300, 2600, 4999]
    d[copies] = q[3]
    skip = (rng.random(nd) < 0.1).astype(np.uint8)
    skip[copies] = [0, 1, 0, 0]
    qm = dm = None
    if masked:
        qm = rng.integers(0, 256, (nq, dim), dtype=np.uint8) | rng.integers(0, 256, (nq, dim), dtype=np.uint8)
        dm = rng.integers(0, 256, (nd, dim), dtype=np.uint8) | rng.integers(0, 256, (nd, dim), dtype=np.uint8)
    dist = pair_dist(q, d, qm, dm)
    dist[:, skip != 0] = 1 << 30
    ri, rd = ref_lists(dist, K)
    ri, rd = np.where(rd >= 1 << 30, -1, ri), np.where(rd >= 1 << 30, INT_MAX, rd)
    idx, dd = api.hamming_topk(q, d, K, qm, dm, db_skip=skip)
    assert np.array_equal(idx, ri) and np.array_equal(dd, rd)
    assert list(idx[3, :3]) == [10, 2600, 4999] and list(dd[3, :3]) == [0, 0, 0]
    dev = torch.device("cuda", 0)
    t = lambda a: None if a is None else torch.from_numpy(a).to(dev)  # noqa: E731
    gi, gd = api.hamming_topk_device(t(q), t(d), K, t(qm), t(dm), t(skip))
    torch.cuda.synchronize(dev)
    assert np.array_equal(gi.cpu().numpy(), ri) and np.array_equal(gd.cpu().numpy(), rd)


def chunk_starts(n_frames):
    """first frame of every chunk of the host stream pipeline (multicol_slam_b200/csrc/mcs_api.cu extract_match_stream_impl)"""
    if n_frames >= 32:
        first = max(4, n_frames // 16)
        each = (n_frames - first + 2) // 3
        return sorted({0, first, min(first + each, n_frames), min(first + 2 * each, n_frames)} - {n_frames})
    nc = min(max(n_frames // 8, 1), 4)
    each = (n_frames + nc - 1) // nc
    return sorted({min(c * each, n_frames) for c in range(nc)} - {n_frames})


# (frames, cameras (None: enough for more images than SMs), learnMasks, descSize, K)
PIPELINE_CASES = [(16, 3, True, 32, 5), (33, 2, False, 16, 3), (15, None, True, 64, 2)]


@pytest.mark.parametrize("n_frames,n_cams,masks,desc_size,K", PIPELINE_CASES,
                         ids=[f"f{f}-c{c or 'many'}-{'m' if m else 'u'}-d{d}" for f, c, m, d, _ in PIPELINE_CASES])
def test_extract_match_stream_chunks(api, oa, cams, n_frames, n_cams, masks, desc_size, K):
    """extract_match_stream plain and packed + greedy, over several chunks of frames (the first frame of a chunk is matched
    against the last frame of the previous chunk) or one chunk with more images than SMs: extraction identical to extract_batch
    (and to the oracle next to every chunk boundary), lists equal numpy, greedy-mode lists equal the plain lists cut at the
    relevance bound, greedy matches equal the oracle's SearchByBoW per pair, and the packed buffer holds the host outputs."""
    import torch
    from multicol_slam_b200 import rig, synth
    if n_cams is None:
        n_cams = math.ceil((sm_count() + 1) / n_frames)
    starts = chunk_starts(n_frames)
    if n_frames == 16:
        assert starts == [0, 8]
    if n_frames == 33:
        assert starts == [0, 4, 14, 24]
    F, nc, B = n_frames, n_cams, n_frames * n_cams
    if len(starts) == 1:
        assert B > sm_count()
    cam_s = [synth.scaled_cam(cams[c % 3], 333, 211) for c in range(nc)]
    imgs = np.ascontiguousarray(np.stack([synth.texture_stream(cam_s[c], F, seed=90 + c) for c in range(nc)], axis=1))
    mk = np.stack([synth.mirror_mask(c) for c in cam_s])
    ex = api.mdBRIEFextractorOct(nfeatures=300, nlevels=4, do_dBrief=True, learnMasks=masks, descSize=desc_size)
    cap, ds = ex.capacity, desc_size
    matcher = api.cORBmatcher(0.9, False, ds, masks)
    th, nn = matcher.TH_LOW_, 0.9
    r = ex.extract_match_stream(imgs, mk, cam_s, K=K)
    packed = torch.zeros(rig.packed_layout(B, cap, ds)[1], dtype=torch.uint8, device=torch.device("cuda", 0))
    g = ex.extract_match_stream(imgs, mk, cam_s, K=K, packed_t=packed, greedy=(th, nn))
    kps, desc, dmask, counts = ex.extract_batch(imgs.reshape(B, *imgs.shape[2:]), mk, cam_s, np.tile(np.arange(nc), F))
    assert np.array_equal(r["counts"], counts) and np.array_equal(g["counts"], counts)
    per_img = rig.unpack(packed.cpu().numpy(), B, cap, ds)
    for i in range(B):
        n = counts[i]
        for o in (r, g):
            assert o["kps"][i, :n].tobytes() == kps[i, :n].tobytes() and np.array_equal(o["desc"][i, :n], desc[i, :n]), i
            if masks:
                assert np.array_equal(o["dmask"][i, :n], dmask[i, :n]), i
        assert per_img[i][0].tobytes() == kps[i, :n].tobytes() and np.array_equal(per_img[i][1], desc[i, :n]), i
        if masks:
            assert np.array_equal(per_img[i][2], dmask[i, :n]), i
    oe = oa.OracleExtractor(nfeatures=300, nlevels=4, do_dbrief=True, learn_masks=masks, desc_size=ds)
    for s in starts[1:]:
        for f in (s - 1, s):
            for c in range(nc):
                i = f * nc + c
                ok, od, om = oe.extract(imgs[f, c], mk[c], cam_s[c])
                assert counts[i] == len(ok) and kps[i, :counts[i]].tobytes() == ok.tobytes() and np.array_equal(desc[i, :counts[i]], od)
                if masks:
                    assert np.array_equal(dmask[i, :counts[i]], om)

    bound = greedy_dist_bound(th, nn)
    assert np.all(g["redo"] == 0)
    cut = False
    for i in range(B):
        n = counts[i]
        if i < nc:
            for o in (r, g):
                assert np.all(o["match_idx"][i] == -1) and np.all(o["match_dist"][i] == INT_MAX)
            assert g["nmatches"][i] == 0 and np.all(g["matches12"][i] == -1)
            continue
        nd = counts[i - nc]
        qm, dm = (dmask[i, :n], dmask[i - nc, :nd]) if masks else (None, None)
        ri, rd = ref_lists(pair_dist(desc[i, :n], desc[i - nc, :nd], qm, dm), K)
        assert np.array_equal(r["match_idx"][i, :n], ri) and np.array_equal(r["match_dist"][i, :n], rd), i
        bi, bd = bounded(ri, rd, bound)
        cut |= bool((bi != ri).any())
        assert np.array_equal(g["match_idx"][i, :n], bi) and np.array_equal(g["match_dist"][i, :n], bd), i
        assert np.all(r["match_idx"][i, n:] == -1) and np.all(g["match_idx"][i, n:] == -1)
        on, om = oa.match_bruteforce(desc[i, :n], desc[i - nc, :nd], th, nn, qm, dm)
        assert g["nmatches"][i] == on and np.array_equal(g["matches12"][i, :n], om), i
        assert np.all(g["matches12"][i, n:] == -1)
    assert g["nmatches"].sum() > 3 * (B - nc) and cut          # the bound does cut list entries


_KERNEL = re.compile(r"(\w+_kernel)<(\d+), (true|false)(?:, (\d+))?>")


def test_every_matcher_instantiation_launched(api):
    """torch.profiler over one short run of the cases above (no reference work): every instantiation of the stream list kernel,
    both stream replay kernels and the key-frame acceptance kernel was launched, i.e. the cases reach every variant"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda", 0)
    t = lambda a: None if a is None else torch.from_numpy(a).to(dev)  # noqa: E731
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for dim, masked, capacity, path in STREAM_CASES:
            F, nc, counts, desc, dmask, _ = make_stream_case(dim, masked, capacity, path, seed=1)
            d_t, m_t, c_t = t(desc), t(dmask), t(counts)
            for K in LIST_KS:
                api.match_stream_device(d_t, m_t, c_t, F, nc, K=K)
            api.match_stream_greedy_device(d_t, m_t, c_t, F, nc, 20, 0.9)
        rng = np.random.default_rng(0)
        for dim in (16, 32, 64):
            for masked in (False, True):
                for nd in (5000, 40000):
                    q, d = rng.integers(0, 256, (300, dim), dtype=np.uint8), rng.integers(0, 256, (nd, dim), dtype=np.uint8)
                    d[:300] = q
                    qm, dm = (q | 0x5A, d | 0xA5) if masked else (None, None)
                    api.match_bruteforce_device(t(q), t(qm), None, t(d), t(dm), None, dim * 2, 0.9)
        torch.cuda.synchronize(dev)
    seen = set()
    for e in prof.key_averages():
        m = _KERNEL.search(e.key)
        if m:
            seen.add((m.group(1), int(m.group(2)), m.group(3) == "true", int(m.group(4)) if m.group(4) else None))
    want = set()
    for w in (4, 8, 16):
        for masked in (False, True):
            want |= {("stream_replay_kernel", w, masked, None), ("stream_replay_smem_kernel", w, masked, None),
                     ("bruteforce_replay_kernel", w, masked, None)}
            want |= {("hamming_stream_kernel", w, masked, kt) for kt in (4, 8)}
    missing = sorted(want - seen)
    assert not missing, f"never launched: {missing}"


BF_MAX_ND = 1_622_016      # kernels.h bruteforce_max_nd(8): 200 KB of shared memory minus the list chunk, one bit per entry


def test_keyframe_database_size_limit(api, oa):
    """The largest key-frame database the brute-force entry points take matches the oracle (planted queries, one of them on the
    last entry); one entry more is refused as unsupported by all three entry points, and the next call works again"""
    import torch
    rng = np.random.default_rng(17)
    dim = 32
    d = rng.integers(0, 256, (BF_MAX_ND + 1, dim), dtype=np.uint8)
    targets = np.array([0, 31, 777_777, 1_000_003, BF_MAX_ND - 33, BF_MAX_ND - 1])
    q = flip_bits(rng, d[targets], 6 / 256)
    valid2 = np.ones(BF_MAX_ND, np.uint8)
    valid2[targets[2]] = 0                       # this query's planted entry is not usable
    dev = torch.device("cuda", 0)
    q_t, d_t = torch.from_numpy(q).to(dev), torch.from_numpy(d).to(dev)
    on, om = oa.match_bruteforce(q, d[:BF_MAX_ND], 64, 0.9, None, None, None, valid2)
    assert on == len(targets) - 1 and np.array_equal(om[[0, 1, 3, 4, 5]], targets[[0, 1, 3, 4, 5]])

    def at_limit():
        n, m12 = api.match_bruteforce_device(q_t, None, None, d_t[:BF_MAX_ND], None, valid2, 64, 0.9)
        assert n == on and np.array_equal(m12, om)
    at_limit()
    matcher = api.cORBmatcher(0.9, False, dim, False)
    calls = [lambda: api.match_bruteforce_device(q_t, None, None, d_t, None, None, 64, 0.9),
             lambda: api.match_bruteforce_batch_device(q_t, None, None, [0, 3, len(q)], d_t, None, None, 64, 0.9),
             lambda: matcher.SearchByBoW(q, d)]
    for call in calls:
        with pytest.raises(api.McsError) as err:
            call()
        assert err.value.code == api.MCS_ERR_UNSUPPORTED and str(BF_MAX_ND) in str(err.value)
    at_limit()
