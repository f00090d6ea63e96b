"""GPU: SearchByBoW(KF_i, F) for a batch of key frames on the device (mcs_search_by_bow_device), against mcs_search_by_bow run per
key frame on the host copies, the CPU oracle and, where oracle/_ref travelled, the reference's own SearchByBoW(KF, F).  Every frame
comes from a packed feature buffer; slots are compared after the slot -> contiguous conversion.  Integer work: bit-exact."""
import numpy as np
import pytest

from bow_device import GOLD, LAYOUTS, device_bow_search, frame_of, host_bow_search, same, split
from device_frames import SIZES, on_device, rm, slot_to_contiguous_index, to_slots  # noqa: F401  (rm: a fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def voc():
    return np.load(GOLD / "voc_small_9_6.npz")


@pytest.fixture(scope="module")
def scene(api, cams, voc):
    """four consecutive 3-camera frames of the sliding-texture stream from the device extractor, their host FeatureVectors, and map
    points on ~70 % of every frame's keypoints: some bad, one id beyond the table in frame 3"""
    from multicol_slam_b200 import synth
    ex = api.mdBRIEFextractorOct(nfeatures=600, do_dBrief=True, learnMasks=True)
    imgs = [synth.texture_stream(cams[c], 4, seed=4 + c) for c in range(3)]
    v = api.ORBVocabulary(voc)
    rng = np.random.default_rng(2)
    n_points = 900
    bad = (rng.random(n_points) < 0.1).astype(np.uint8)
    frames = []
    for f in range(4):
        per = [ex(imgs[c][f], synth.mirror_mask(cams[c]), cams[c]) for c in range(3)]
        desc = np.concatenate([p[1] for p in per])
        mp = np.where(rng.random(len(desc)) < 0.7, rng.integers(0, n_points, len(desc)), -1)
        frames.append(frame_of(per, v.transform(desc)[2], mp))
    sf = [float(ex.info.scale_factor[l]) for l in range(8)]
    return dict(frames=frames, n_points=n_points, bad=bad, voc=v, sf=sf)


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("masks", [False, True])
def test_parity_with_host_oracle_and_reference(api, oa, rm, cams, scene, masks, layout):
    fr, n_points, bad = scene["frames"], scene["n_points"], scene["bad"]
    m = api.cORBmatcher(0.9, False, 32, masks)
    kfs, cur = [fr[0], fr[2]], fr[1]
    res, status = device_bow_search(api, m, kfs, cur, n_points, bad, layout)
    assert status == api.MCS_OK
    for kf, r in zip(kfs, res):
        h = host_bow_search(api, m, kf, cur, n_points, bad)
        assert same(r, h) and same(h, host_bow_search(api, m, kf, cur, n_points, bad, oa.search_by_bow))
        assert r[0] > 60 and (r[1] >= 0).sum() == r[0] and np.all(kf["mp"][r[1][r[1] >= 0]] >= 0)
        if rm:
            F1, F2 = (api.Frame.from_cameras(f["per"], SIZES, scene["sf"]) for f in (kf, cur))
            table = rm.MPTable(3, np.zeros((n_points, 32), np.uint8), bad=bad)
            rn, rout = rm.search_by_bow_kff(rm.KF(F1, cams, mp=kf["mp"], featvec=kf["fv"]), rm.KF(F2, cams, featvec=cur["fv"]), table, 0.9, masks)
            assert rm.thresholds(32, masks)[1] == m.TH_LOW_ and rn == r[0] and np.array_equal(rout, r[2])     # vpMapPointMatches: map-point ids


def test_batches_equal_single_calls_and_no_state_leaks(api, scene):
    fr, n_points, bad = scene["frames"], scene["n_points"], scene["bad"]
    m = api.cORBmatcher(0.9, False, 32, True)
    cur = fr[1]
    eight = [fr[0], fr[2], fr[3], fr[0], fr[2], fr[1], fr[3], fr[0]]          # repeated key frames, and the current frame itself
    for kfs in (eight[:1], eight[:2], eight):
        res, status = device_bow_search(api, m, kfs, cur, n_points, None, "shared" if len(kfs) == 2 else "single")
        assert status == api.MCS_OK
        for k, kf in enumerate(kfs):
            one, st1 = device_bow_search(api, m, [kf], cur, n_points, None)
            assert st1 == api.MCS_OK and same(res[k], one[0]) and same(res[k], host_bow_search(api, m, kf, cur, n_points, None))
    assert same(res[0], res[3]) and same(res[0], res[7]) and same(res[1], res[4]) and same(res[2], res[6])
    assert res[5][0] > 0.6 * (cur["mp"] >= 0).sum()                            # the frame against itself
    # n_kf = 0 is a successful no-op
    assert api.lib().mcs_search_by_bow_device(None, 0, None, 3, 700, 32, 81, 10, None, 64, 0.9, 1, None, None, None, None, None) == 0


def test_map_point_ids_bad_points_and_status(api, scene):
    fr, n_points, bad = scene["frames"], scene["n_points"], scene["bad"]
    m = api.cORBmatcher(0.9, False, 32, False)
    kf, cur = dict(fr[3]), fr[2]
    with_bad, st = device_bow_search(api, m, [kf], cur, n_points, bad)
    without, st2 = device_bow_search(api, m, [kf], cur, n_points, None)
    assert st == st2 == api.MCS_OK
    assert same(with_bad[0], host_bow_search(api, m, kf, cur, n_points, bad)) and same(without[0], host_bow_search(api, m, kf, cur, n_points, None))
    assert without[0][0] > with_bad[0][0] and np.all(bad[with_bad[0][2][with_bad[0][2] >= 0]] == 0)
    # an id beyond the table: status raised, only that keypoint dropped
    good = without[0][1][without[0][1] >= 0]
    kf["mp"] = kf["mp"].copy()
    kf["mp"][good[3]] = n_points + 5
    res, st = device_bow_search(api, m, [fr[0], kf], cur, n_points, None)
    assert st == api.MCS_ERR_INVALID and good[3] not in res[1][1]
    assert same(res[1], host_bow_search(api, m, kf, cur, n_points, None)) and same(res[0], host_bow_search(api, m, fr[0], cur, n_points, None))


def built(rng, dim, n_kf_pts, n_cur_pts, nodes_kf, nodes_cur, flips):
    """hand-built frames at any descriptor width: the current frame's descriptors are the key frame's with a few bits flipped, and
    both feature vectors put keypoint i into node `nodes[i % len(nodes)]`"""
    def fv_of(node_of, all_nodes):
        nodes = np.array(sorted(all_nodes), np.int32)
        lists = [rng.permutation(np.flatnonzero(node_of == nd)) for nd in nodes]
        return nodes, np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32), np.concatenate(lists).astype(np.int32)
    d1 = rng.integers(0, 256, (n_kf_pts, dim), dtype=np.uint8)
    src = rng.integers(0, n_kf_pts, n_cur_pts)
    d2 = d1[src].copy()
    for i in range(n_cur_pts):
        for b in rng.integers(0, dim * 8, rng.integers(0, flips + 1)):
            d2[i, b // 8] ^= 1 << (b % 8)
    n1 = np.asarray(nodes_kf)[np.arange(n_kf_pts) % len(nodes_kf)]
    n2 = n1[src].copy()
    stray = rng.random(n_cur_pts) < 0.1
    n2[stray] = np.asarray(nodes_cur)[rng.integers(0, len(nodes_cur), stray.sum())]
    only_kf = sorted(set(nodes_kf) - set(nodes_cur))
    n2[np.isin(n2, only_kf)] = sorted(set(nodes_cur) - set(nodes_kf))[0]       # a node of the key frame alone stays its alone
    c1, c2 = [n_kf_pts // 2, 0, n_kf_pts - n_kf_pts // 2], [n_cur_pts // 3, n_cur_pts // 3, n_cur_pts - 2 * (n_cur_pts // 3)]
    p1, p2 = split(d1, c1), split(d2, c2)
    for p in p1 + p2:
        p[2][:] = rng.integers(0, 256, p[2].shape, dtype=np.uint8) | rng.integers(0, 256, p[2].shape, dtype=np.uint8)
    mp = np.where(rng.random(n_kf_pts) < 0.8, np.arange(n_kf_pts), -1)
    return frame_of(p1, fv_of(n1, set(nodes_kf) | {1000}), mp), frame_of(p2, fv_of(n2, set(nodes_cur) | set(n2.tolist()) | {2000}))


@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("dim", [16, 32, 64])
def test_descriptor_widths_with_hand_built_feature_vectors(api, oa, dim, masks):
    """nodes 1000 / 2000 have empty lists; node 7 is in the key frame only, node 9 in the current frame only"""
    rng = np.random.default_rng(dim + masks)
    kf, cur = built(rng, dim, 900, 1100, [3, 5, 7, 11, 40], [3, 5, 9, 11, 40], 4 * dim // 16)
    assert 7 not in cur["fv"][0] and 9 not in kf["fv"][0]
    m = api.cORBmatcher(0.8, False, dim, masks)
    for layout in ("single", "parts"):
        res, st = device_bow_search(api, m, [kf, kf], cur, 900, None, layout)
        h = host_bow_search(api, m, kf, cur, 900, None)
        assert st == api.MCS_OK and same(res[0], h) and same(res[1], h) and same(h, host_bow_search(api, m, kf, cur, 900, None, oa.search_by_bow))
        assert h[0] > 100


def bits(n, dim=32):
    d = np.zeros(dim, np.uint8)
    for b in range(n):
        d[b // 8] |= 1 << (b % 8)
    return d


def edge_case(api, m, q_descs, c_descs, expect):
    """one node; key-frame keypoints q_descs in list order against candidates c_descs -> match_of_f must equal `expect`"""
    from multicol_slam_b200.ctypes_defs import KEYPOINT_DTYPE
    per = lambda ds: [(np.zeros(len(ds), KEYPOINT_DTYPE), np.stack(ds), np.full((len(ds), 32), 255, np.uint8))]  # noqa: E731
    kf = frame_of(per(q_descs), ([4], [0, len(q_descs)], np.arange(len(q_descs))), np.arange(len(q_descs)) + 10)
    cur = frame_of(per(c_descs), ([4], [0, len(c_descs)], np.arange(len(c_descs))))
    res, st = device_bow_search(api, m, [kf], cur, 100, None)
    assert st == api.MCS_OK and same(res[0], host_bow_search(api, m, kf, cur, 100, None))
    assert list(res[0][1]) == expect, (list(res[0][1]), expect)


def test_decision_edges(api):
    z = bits(0)
    m = api.cORBmatcher(0.9, False, 32, False)
    assert m.TH_LOW_ == 64
    edge_case(api, m, [z], [bits(64)], [0])                    # best == th_low is accepted, a lone candidate has second = INT_MAX
    edge_case(api, m, [z], [bits(65)], [-1])                   # th_low + 1 is not
    h = api.cORBmatcher(0.5, False, 32, False)
    edge_case(api, h, [z], [bits(10), bits(20)], [-1, -1])     # 10 < 0.5 * 20 is false: strict
    edge_case(api, h, [z], [bits(20), bits(10)], [-1, -1])
    edge_case(api, h, [z], [bits(10), bits(21)], [0, -1])
    edge_case(api, h, [z], [bits(21), bits(10)], [-1, 0])
    flipped = bits(10)[::-1].copy()                            # another descriptor at distance 10
    edge_case(api, h, [z], [bits(10), flipped], [-1, -1])      # a tie: the ratio fails for nnratio < 1
    edge_case(api, api.cORBmatcher(1.5, False, 32, False), [z], [flipped, bits(10)], [0, -1])   # ... and the first in list order is best
    # the first keypoint takes candidate 0; the second one's best (candidate 0, distance 2) is gone: it sees candidate 1 alone and
    # takes it, which it would not have done with candidate 0 still free
    edge_case(api, h, [z, bits(2)], [z, bits(30)], [0, 1])
    edge_case(api, h, [bits(2)], [z, bits(30)], [0, -1])
    edge_case(api, h, [z, bits(30)], [bits(1), bits(29), bits(31)], [0, -1, -1])     # 1 vs 1: a tie between the two left
    # more candidates than one pass of the warp, the best at the far end
    far = [bits(40)] * 70 + [bits(3)]
    edge_case(api, h, [z], far, [-1] * 70 + [0])


def test_one_big_node_and_disjoint_vectors(api, oa):
    from multicol_slam_b200.ctypes_defs import KEYPOINT_DTYPE
    rng = np.random.default_rng(9)
    n = 3400
    d1 = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    d2 = d1[rng.permutation(n)].copy()
    d2 ^= (rng.integers(0, 256, d2.shape, dtype=np.uint8) & rng.integers(0, 256, d2.shape, dtype=np.uint8) & rng.integers(0, 256, d2.shape, dtype=np.uint8))
    kf = frame_of(split(d1, [1700, 1700]), ([17], [0, n], np.arange(n)), np.arange(n))
    cur = frame_of(split(d2, [3000, 400]), ([3, 17], [0, 0, n], rng.permutation(n)))
    m = api.cORBmatcher(0.8, False, 32, False)
    res, st = device_bow_search(api, m, [kf], cur, n, None)
    h = host_bow_search(api, m, kf, cur, n, None)
    assert st == api.MCS_OK and same(res[0], h) and same(h, host_bow_search(api, m, kf, cur, n, None, oa.search_by_bow)) and h[0] > 3000
    # disjoint vectors: no match, both outputs all -1
    other = frame_of(cur["per"], ([3, 18], [0, 0, n], cur["fv"][2]))
    res, st = device_bow_search(api, m, [kf], other, n, None)
    assert st == api.MCS_OK and res[0][0] == 0 and np.all(res[0][1] == -1) and np.all(res[0][2] == -1)
    assert KEYPOINT_DTYPE.itemsize == 28


@pytest.mark.parametrize("masks", [False, True])
def test_full_chain_from_the_device_extractor(api, voc, cams, masks):
    """two texture-stream frames extracted into one packed buffer, mcs_bow_vectors_device on each, the search -- equal to the host
    chain (D2H of the features, mcs_bow_vectors, mcs_search_by_bow); queued on a stream that is busy with earlier work"""
    import torch
    from multicol_slam_b200 import rig, synth
    ex = api.mdBRIEFextractorOct(nfeatures=1500, do_dBrief=True, learnMasks=True)
    cap = ex.capacity
    imgs = np.stack([synth.texture_stream(cams[c], 2, seed=4 + c) for c in range(3)], axis=1)          # [2, 3, H, W]
    H, W = imgs.shape[2:]
    pitch = (W + 63) // 64 * 64
    dev_images = torch.zeros((6, H, pitch), dtype=torch.uint8, device="cuda")
    dev_images[:, :, :W] = on_device(imgs.reshape(6, H, W))
    masks_np = np.stack([synth.mirror_mask(c) for c in cams[:3]])
    packed = torch.zeros(rig.packed_layout(6, cap, 32)[1], dtype=torch.uint8, device="cuda")
    views = ex.extract_batch_packed_device(dev_images, masks_np, cams[:3], [0, 1, 2] * 2, packed, width=W)
    torch.cuda.synchronize()
    counts = views["counts"].cpu().numpy()
    v = api.ORBVocabulary(voc)
    s = torch.cuda.Stream()
    a = torch.randn(4096, 4096, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        for _ in range(10):
            a = a @ a * 1e-3
    bows = [v.transform_device((packed, 1, 6, 3 * f), 3, cap, stream=s) for f in range(2)]
    rng = np.random.default_rng(2)
    D = [np.concatenate([views["desc"][3 * f + c, :counts[3 * f + c]].cpu().numpy() for c in range(3)]) for f in range(2)]
    M = [np.concatenate([views["dmask"][3 * f + c, :counts[3 * f + c]].cpu().numpy() for c in range(3)]) for f in range(2)]
    mp = np.where(rng.random(len(D[0])) < 0.7, np.arange(len(D[0])), -1).astype(np.int32)
    mp_t = to_slots(api, counts[:3], mp, cap, -1)
    mt = api.cORBmatcher(0.9, False, 32, masks)
    torch.cuda.current_stream().synchronize()
    mmp, msl, nm, st = mt.SearchByBoWDevice([(bows[0], mp_t)], bows[1], len(D[0]), stream=s)
    torch.cuda.synchronize()
    fv = [v.transform(D[f])[2] for f in range(2)]
    n_h, m_h = mt.SearchByBoWFrame(D[0], fv[0], D[1], fv[1], M[0] if masks else None, M[1] if masks else None, (mp >= 0).astype(np.uint8))
    assert int(st.item()) == api.MCS_OK and int(nm[0].item()) == n_h and n_h > 100
    sl = api.slots_to_contiguous(msl[0].cpu().numpy(), counts[3:], cap)
    assert np.array_equal(np.where(sl >= 0, slot_to_contiguous_index(np.maximum(sl, 0), counts[:3], cap), -1), m_h)
    assert np.array_equal(api.slots_to_contiguous(mmp[0].cpu().numpy(), counts[3:], cap), np.where(m_h >= 0, mp[np.maximum(m_h, 0)], -1))
    for f in range(2):
        bw, bv, (fn, fo, ff) = bows[f].host()
        hw, hv, _ = v.transform(D[f])
        assert np.array_equal(bw, hw) and np.array_equal(bv, hv) and np.array_equal(fn, fv[f][0]) and np.array_equal(fo, fv[f][1])
        assert np.array_equal(slot_to_contiguous_index(ff, counts[3 * f:3 * f + 3], cap), fv[f][2])
