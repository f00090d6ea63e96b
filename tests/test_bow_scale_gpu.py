"""GPU: the bag of words on a full-size vocabulary (tests/bow_scale.py: k = 10, L = 6, 1 064 066 nodes and 956 865 words), where the
device code runs paths the small vocabulary never reaches:
  - bv_tile_emit_kernel adds up the tiles before its own with a strided loop, which goes round more than once past 256 tiles of
    2 048 ids, and the word array runs out of tiles before the node array does;
  - bv_normalize_kernel sums the BowVector in chunks of 2 048 words;
  - bs_search_kernel's grid stops at 16 384 blocks (131 072 warps) and the (key frame, node) items beyond it are strided;
  - node ids pass 2^20 and word ids 2^16.
Each test asserts from the shapes and outputs that its limit is crossed.  Host entry points, mcs_bow_vectors_device and
mcs_search_by_bow_device against the CPU oracle (which tests/test_bow_scale_cpu.py pins to the reference's own DBoW2 on the same
seeded tree and frames), the host route and, where oracle/_ref travelled, the reference's SearchByBoW(KF, F).  Bit for bit."""
import ctypes as C

import numpy as np
import pytest

import bow_scale
from bow_device import TAIL_WORDS, VEC_FILL, call, check, device_bow_search, frame_of, host_bow_search, pack_bow_frames, same, split
from device_frames import SIZES, on_device, rm, slot_to_contiguous_index, to_slots  # noqa: F401  (rm: a fixture)

pytestmark = pytest.mark.gpu
TILE, NORM_CHUNK, GRID_WARPS = 2048, 2048, 16384 * 256 // 32


@pytest.fixture(scope="module")
def voc():
    return bow_scale.vocabulary()


@pytest.fixture(scope="module")
def v(api, voc):
    """the tree on the device, uploaded once for the module (scoring L1, weighting TF-IDF)"""
    return api.ORBVocabulary(voc)


@pytest.fixture(scope="module")
def o(oa, voc):
    return oa.OracleVocabulary(voc)


def tiles(n):
    return (n + TILE - 1) // TILE


def test_tile_counts_and_level_nodes(v, voc):
    tn, tw = tiles(len(voc["parent"])), tiles(len(voc["word_node"]))
    print(f"\nnode tiles {tn}, word tiles {tw}")
    assert tn > 256 and tw > 256 and tw < tn              # a strided prefix in both arrays; word blocks idle past tile tw
    for levelsup in range(8):
        assert v.level_nodes(levelsup) == bow_scale.numpy_level_nodes(voc, levelsup), levelsup
    assert v.level_nodes(0) == v.size() == len(voc["word_node"]) and v.level_nodes(6) == v.level_nodes(7) == 1


def test_host_entry_points(v, o, voc):
    """mcs_bow_transform / mcs_bow_vectors / mcs_bow_score against the oracle, on the frames the CPU file pins to the reference"""
    frames = dict(spread=bow_scale.spread(voc, 6000, 1), clustered=bow_scale.clustered(voc, 1500, 2), stopped=bow_scale.stopped(voc, 2000, 3))
    for name, d in frames.items():
        for levelsup in range(8) if name == "spread" else (0, 4):
            bw, bv, fv = v.transform(d, levelsup)
            A = o.transform(d, levelsup)
            assert all(np.array_equal(x, y) for x, y in zip((bw, bv) + fv, A)), (name, levelsup)
            assert all(np.array_equal(x, y) for x, y in zip(v.transform_features(d, levelsup), o.transform_features(d, levelsup)))
            if name == "spread" and levelsup == 0:
                assert len(bw) > 2 * NORM_CHUNK and fv[0].max() >= 2**20 and bw.max() >= 2**16
    a, b = v.transform(frames["spread"][:3000], 0), v.transform(frames["spread"][1500:], 0)
    assert v.score(a[:2], b[:2]) == o.score(a[0], a[1], b[0], b[1])


@pytest.mark.parametrize("n_cams,cap,layout", [(4, 2048, "single"), (4, 2048, "shared"), (3, 2600, "parts")])
def test_device_vectors_at_every_levelsup(api, v, o, voc, n_cams, cap, layout):
    counts = [cap - 7 * c for c in range(n_cams)]
    desc = bow_scale.spread(voc, sum(counts), 10 + n_cams)
    other = split(bow_scale.clustered(voc, 100 * n_cams, 3), [100] * n_cams)         # frame 0 of the shared buffer
    packed = pack_bow_frames([other, split(desc, counts)], cap, 32, layout)[1]
    seen = dict(nb=0, node=0, word=0)
    for levelsup in range(8):
        H = call(api, v, packed, counts, cap, levelsup)
        nb, nf = check(api, H, v, desc, counts, cap, levelsup, o)
        seen = dict(nb=max(seen["nb"], nb), node=max(seen["node"], int(H["fv_nodes"][:nf].max())),
                    word=max(seen["word"], int(H["bow_words"][:nb].max())))
        assert nf <= v.level_nodes(levelsup)
    print(f"\n{n_cams} cameras x {cap}: largest n_bow {seen['nb']}, largest node id {seen['node']}, largest word id {seen['word']}")
    assert seen["nb"] > 2 * NORM_CHUNK                          # the norm runs three chunks or more
    assert seen["node"] >= 2**20 and seen["word"] >= 2**16 and seen["word"] >= 256 * TILE       # ids in tiles past the 256th


@pytest.mark.parametrize("scoring", range(6))
def test_device_vectors_every_scoring_and_weighting(api, oa, voc, scoring):
    counts = [2048, 2040, 2030, 2020]
    desc = bow_scale.spread(voc, sum(counts), 30 + scoring)
    packed = pack_bow_frames([split(desc, counts)], 2048, 32, "parts")[0]
    for weighting in range(4):
        vs, os_ = api.ORBVocabulary(voc, scoring, weighting), oa.OracleVocabulary(voc, scoring, weighting)
        for levelsup in (0, 4):
            nb, _ = check(api, call(api, vs, packed, counts, 2048, levelsup), vs, desc, counts, 2048, levelsup, os_)
            assert nb > 2 * NORM_CHUNK
        del vs, os_


def test_device_vectors_clustered_and_stopped(api, v, o, voc):
    counts = [1500, 1200, 1400]
    for desc in (bow_scale.clustered(voc, sum(counts), 40), bow_scale.stopped(voc, sum(counts), 41)):
        packed = pack_bow_frames([split(desc, counts)], 1500, 32, "single")[0]
        for levelsup in (0, 2, 4):
            check(api, call(api, v, packed, counts, 1500, levelsup), v, desc, counts, 1500, levelsup, o)


@pytest.mark.parametrize("levelsup", [0, 1])
def test_max_nodes_one_short_at_full_size(api, v, voc, levelsup):
    counts = [2048, 2048, 2048]
    desc = bow_scale.spread(voc, sum(counts), 50)
    packed = pack_bow_frames([split(desc, counts)], 2048, 32, "single")[0]
    bw, bv, (fn, fo, ff) = v.transform(desc, levelsup)
    short = len(fn) - 1
    assert fn[-1] >= (2**20 if levelsup == 0 else 100000)
    H = call(api, v, packed, counts, 2048, levelsup, max_nodes=short)                # the guard words are checked inside
    assert H["status"][0] == api.MCS_ERR_CAPACITY and H["n_fv"][0] == short
    assert np.array_equal(H["fv_nodes"][:short], fn[:short]) and np.array_equal(H["fv_offsets"][:short + 1], fo[:short + 1])
    assert np.array_equal(slot_to_contiguous_index(H["fv_features"][:fo[short]], counts, 2048), ff[:fo[short]])
    assert np.all(H["fv_features"][fo[short]:3 * 2048] == VEC_FILL)
    assert np.array_equal(H["bow_words"][:len(bw)], bw) and np.array_equal(H["bow_values"][:len(bw)], bv)


@pytest.mark.parametrize("dim", [16, 64])
def test_other_widths_are_refused(api, v, voc, dim):
    import torch
    from multicol_slam_b200.ctypes_defs import PackedFrame
    counts = [500, 400, 300]
    d = bow_scale.other_width(voc, sum(counts), 60, dim)
    packed = pack_bow_frames([split(d, counts)], 512, dim, "single")[0]
    out = [torch.full((3 * 512 + TAIL_WORDS,), VEC_FILL, dtype=torch.float64 if k == 5 else torch.int32, device="cuda") for k in range(8)]
    fr = PackedFrame(packed[0].data_ptr(), *packed[1:4])
    rc = api.lib().mcs_bow_vectors_device(v._h, C.byref(fr), 3, 512, dim, 4, 200, None, None, None,
                                          *(C.c_void_p(t.data_ptr()) for t in out), None)
    assert rc == api.MCS_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert all(bool((t == VEC_FILL).all()) for t in out)
    with pytest.raises(ValueError):
        v.transform(d, 4)


# ---- SearchByBoW(KF_i, F) for 44 key frames ----
N_KF, CAP = 44, 2100


@pytest.fixture(scope="module")
def reloc(voc):
    """a current frame and 44 key frames seen around the same scene: each key frame holds most of the scene's descriptors with a few
    bits flipped, plus some of its own; map points on ~70 % of its keypoints, 5 % of them bad.  Random masks.  Key frames 0-21 in
    buffers of their own, 22-43 and the current frame in one shared buffer"""
    rng = np.random.default_rng(70)
    scene = bow_scale.spread(voc, 6500, 71)
    n_points = 20000
    bad = (rng.random(n_points) < 0.05).astype(np.uint8)

    def frame(n, own, mp):
        near = bow_scale.flip(rng, scene[rng.choice(len(scene), n - own, replace=False)], 4)
        d = np.concatenate([near, bow_scale.spread(voc, own, int(rng.integers(1 << 30)))])
        d = d[rng.permutation(n)]
        c = [n // 3, n // 3, n - 2 * (n // 3)]
        per = split(d, c)
        for p in per:
            p[2][:] = rng.integers(0, 256, p[2].shape, dtype=np.uint8) | rng.integers(0, 256, p[2].shape, dtype=np.uint8)
        m = np.where(rng.random(n) < 0.7, rng.integers(0, n_points, n), -1) if mp else None
        return per, m

    cur = frame(6000, 300, False)
    kfs = [frame(int(rng.integers(4500, 6200)), int(rng.integers(200, 1500)), True) for _ in range(N_KF)]
    half = N_KF // 2
    packed = pack_bow_frames([p for p, _ in kfs[:half]], CAP, 32, "single") + pack_bow_frames([p for p, _ in kfs[half:]] + [cur[0]], CAP, 32, "shared")
    assert packed[half][0].data_ptr() == packed[-1][0].data_ptr() != packed[0][0].data_ptr()
    return dict(kfs=kfs, cur=cur, packed=packed, n_points=n_points, bad=bad)


@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("levelsup", [0, 1, 2, 4])
def test_search_many_key_frames(api, oa, rm, cams, v, reloc, levelsup, masks):
    frames = [p for p, _ in reloc["kfs"]] + [reloc["cur"][0]]
    bows = [v.transform_device(p, 3, CAP, levelsup) for p in reloc["packed"]]
    hosts = []
    for b, per in zip(bows, frames):                               # the device containers equal the host route's
        desc = np.concatenate([p[1] for p in per])
        bw, bv, fv = v.transform(desc, levelsup)
        db = b.host()
        assert int(b.status.item()) == 0 and np.array_equal(db[0], bw) and np.array_equal(db[1], bv) and np.array_equal(db[2][0], fv[0])
        assert np.array_equal(db[2][1], fv[1]) and np.array_equal(slot_to_contiguous_index(db[2][2], [len(p[0]) for p in per], CAP), fv[2])
        hosts.append(fv)
    kfs = [frame_of(per, fv, mp) for (per, mp), fv in zip(reloc["kfs"], hosts)]
    cur = frame_of(reloc["cur"][0], hosts[-1])
    max_nodes = v.level_nodes(levelsup)
    items = N_KF * max_nodes
    print(f"\nlevelsup {levelsup}: n_kf * max_nodes = {items} ({'strided' if items > GRID_WARPS else 'one pass'})")
    if levelsup <= 2:
        assert items > GRID_WARPS
    m = api.cORBmatcher(0.9, False, 32, masks)
    n_points, bad = reloc["n_points"], reloc["bad"]
    res, status = device_bow_search(api, m, kfs, cur, n_points, bad, cap=CAP, bows=bows)
    assert status == api.MCS_OK
    total = 0
    for k, (kf, r) in enumerate(zip(kfs, res)):
        h = host_bow_search(api, m, kf, cur, n_points, bad)
        assert same(r, h), k
        total += r[0]
        if k % 11 == 0:
            assert same(h, host_bow_search(api, m, kf, cur, n_points, bad, oa.search_by_bow)), k
        if rm and k % 11 == 0 and levelsup == 4:
            sf = [1.2 ** lv for lv in range(8)]
            F1, F2 = (api.Frame.from_cameras(f["per"], SIZES, sf) for f in (kf, cur))
            table = rm.MPTable(3, np.zeros((n_points, 32), np.uint8), bad=bad)
            rn, rout = rm.search_by_bow_kff(rm.KF(F1, cams[:3], mp=kf["mp"], featvec=kf["fv"]), rm.KF(F2, cams[:3], featvec=cur["fv"]), table, 0.9,
                                            masks)
            assert rn == r[0] and np.array_equal(rout, r[2]), k
    assert min(r[0] for r in res) > 50 and total > 100 * N_KF


@pytest.mark.parametrize("masks", [False, True])
def test_full_chain_on_a_config3_rig(api, v, masks):
    """config 3 (four 1280x720 cameras, 2000 features): two stream frames extracted into one packed buffer, mcs_bow_vectors_device on
    each with the full-size vocabulary, the search -- equal to the host chain (D2H of the features, mcs_bow_vectors,
    mcs_search_by_bow)"""
    import torch
    import bench
    from multicol_slam_b200 import rig
    cfg = bench.CONFIGS[3]
    cams = bench.rig_cams(cfg)
    nc, W, H = len(cams), cfg["w"], cfg["h"]
    ex = api.mdBRIEFextractorOct(nfeatures=cfg["nfeatures"], nlevels=bench.NLEVELS, do_dBrief=True, learnMasks=True)
    cap = ex.capacity
    imgs = bench.make_stream(cams, list(range(nc)), 2, 1000)
    pitch = (W + 63) // 64 * 64
    dev_images = torch.zeros((2 * nc, H, pitch), dtype=torch.uint8, device="cuda")
    dev_images[:, :, :W] = on_device(imgs.reshape(2 * nc, H, W))
    from multicol_slam_b200 import synth
    packed = torch.zeros(rig.packed_layout(2 * nc, cap, 32)[1], dtype=torch.uint8, device="cuda")
    views = ex.extract_batch_packed_device(dev_images, np.stack([synth.mirror_mask(c) for c in cams]), cams, list(range(nc)) * 2, packed, width=W)
    torch.cuda.synchronize()
    counts = views["counts"].cpu().numpy()
    D = [np.concatenate([views["desc"][nc * f + c, :counts[nc * f + c]].cpu().numpy() for c in range(nc)]) for f in range(2)]
    M = [np.concatenate([views["dmask"][nc * f + c, :counts[nc * f + c]].cpu().numpy() for c in range(nc)]) for f in range(2)]
    rng = np.random.default_rng(3)
    mp = np.where(rng.random(len(D[0])) < 0.7, np.arange(len(D[0])), -1).astype(np.int32)
    mp_t = to_slots(api, counts[:nc], mp, cap, -1)
    mt = api.cORBmatcher(0.9, False, 32, masks)
    for levelsup in (4, 0):
        bows = [v.transform_device((packed, 1, 2 * nc, nc * f), nc, cap, levelsup) for f in range(2)]
        mmp, msl, nm, st = mt.SearchByBoWDevice([(bows[0], mp_t)], bows[1], len(D[0]))
        torch.cuda.synchronize()
        fv = [v.transform(D[f], levelsup)[2] for f in range(2)]
        n_h, m_h = mt.SearchByBoWFrame(D[0], fv[0], D[1], fv[1], M[0] if masks else None, M[1] if masks else None, (mp >= 0).astype(np.uint8))
        assert int(st.item()) == api.MCS_OK and int(nm[0].item()) == n_h and n_h > 100, (levelsup, n_h)
        sl = api.slots_to_contiguous(msl[0].cpu().numpy(), counts[nc:], cap)
        assert np.array_equal(np.where(sl >= 0, slot_to_contiguous_index(np.maximum(sl, 0), counts[:nc], cap), -1), m_h)
        assert np.array_equal(api.slots_to_contiguous(mmp[0].cpu().numpy(), counts[nc:], cap), np.where(m_h >= 0, mp[np.maximum(m_h, 0)], -1))
        for f in range(2):
            bw, bv, (fn, fo, ff) = bows[f].host()
            hw, hv, _ = v.transform(D[f], levelsup)
            assert np.array_equal(bw, hw) and np.array_equal(bv, hv) and np.array_equal(fn, fv[f][0]) and np.array_equal(fo, fv[f][1])
            assert np.array_equal(slot_to_contiguous_index(ff, counts[nc * f:nc * f + nc], cap), fv[f][2])
