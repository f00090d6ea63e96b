"""GPU: ComputeBoW on a frame that stays in its packed feature buffer (mcs_bow_vectors_device) against mcs_bow_vectors /
mcs_bow_transform on the concatenated host copy of the same descriptors, the CPU oracle vocabulary and the stored outputs of the
reference's own DBoW2.  Ids and feature lists bit-exact, weights and values == (same double operation order).  Feature indices of
the device call are slots c * capacity + j; they are compared after the slot -> contiguous conversion."""
import ctypes as C
import sys

import numpy as np
import pytest

from bow_device import GOLD, LAYOUTS, VEC_FILL, call, check, pack_bow_frames, split
from device_frames import slot_to_contiguous_index

pytestmark = pytest.mark.gpu
sys.path.insert(0, str(GOLD))


@pytest.fixture(scope="module")
def voc():
    return np.load(GOLD / "voc_small_9_6.npz")


def toy_tree(seed=5, k=40):
    """k = 40 children under the root (more than one pass of the 16-lane group), three leaves under each, duplicate children"""
    rng = np.random.default_rng(seed)
    parent = np.concatenate([[0], np.zeros(k, np.int32), np.repeat(np.arange(1, k + 1), 3)]).astype(np.int32)
    n = len(parent)
    desc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    desc[7] = desc[3]; desc[k + 5] = desc[k + 4]
    leaf = np.ones(n, bool); leaf[parent[1:]] = False; leaf[0] = False
    return dict(k=k, L=2, scoring=0, weighting=0, parent=parent, weight=np.where(leaf, rng.random(n) + 0.1, 0.0), desc=desc,
                word_node=np.nonzero(leaf)[0].astype(np.int32))


def numpy_level_nodes(v, levelsup):
    parent = np.asarray(v["parent"]); n = len(parent)
    depth = np.zeros(n, np.int64)
    for i in np.argsort(parent, kind="stable"):          # not assumed topological: walk up instead
        a, d = i, 0
        while a != 0:
            a = parent[a]; d += 1
        depth[i] = d
    leaf = np.zeros(n, bool); leaf[np.asarray(v["word_node"])] = True
    level = max(int(v["L"]) - levelsup, 0)
    return int((depth == level).sum() + (leaf & (depth < level)).sum())


@pytest.fixture(scope="module")
def extracted(api, cams):
    """a 3-camera frame from the device extractor"""
    from multicol_slam_b200 import synth
    ex = api.mdBRIEFextractorOct(nfeatures=1200, do_dBrief=True, learnMasks=True)
    return [ex(synth.frame(cams[c], 3 * 16 + c), synth.mirror_mask(cams[c]), cams[c]) for c in range(3)]


def test_level_nodes(api, voc):
    v = api.ORBVocabulary(voc)
    for levelsup in (4, 1, 0, 6, 8):
        assert v.level_nodes(levelsup) == numpy_level_nodes(voc, levelsup), levelsup
    assert v.level_nodes(4) <= 81 and v.level_nodes(6) == v.level_nodes(8) == 1 and v.level_nodes(0) == v.size()
    toy = toy_tree()
    tv = api.ORBVocabulary(toy)
    for levelsup in (1, 0, 2, 3):
        assert tv.level_nodes(levelsup) == numpy_level_nodes(toy, levelsup)
    assert tv.level_nodes(1) == 40 and tv.level_nodes(0) == 120
    n = C.c_int32(0)
    assert api.lib().mcs_vocabulary_level_nodes(None, 4, C.byref(n)) == api.MCS_ERR_INVALID
    assert api.lib().mcs_vocabulary_level_nodes(v._h, 4, None) == api.MCS_ERR_INVALID


@pytest.mark.parametrize("layout", LAYOUTS)
def test_extracted_frame_in_every_buffer_shape(api, oa, voc, extracted, layout):
    counts = [len(p[0]) for p in extracted]
    cap = max(counts) + 7
    desc = np.concatenate([p[1] for p in extracted])
    assert len(desc) > 2500
    other = [(k[: len(k) // 2], d[: len(k) // 2], m[: len(k) // 2]) for k, d, m in extracted]       # frame 0 of the shared buffer
    packed = pack_bow_frames([other, extracted], cap, 32, layout)[1]
    assert layout != "shared" or packed[3] == 3
    v, o = api.ORBVocabulary(voc), oa.OracleVocabulary(voc)
    for levelsup in (4, 0):
        nb, nf = check(api, call(api, v, packed, counts, cap, levelsup), v, desc, counts, cap, levelsup, o)
        assert nb > 500 and nf > (20 if levelsup else 500)
    # the Python mirror returns the same containers
    b = v.transform_device(packed, 3, cap, 4, per_slot=True)
    bw, bv, (fn, fo, ff) = b.host()
    hw, hv, (hn, ho, hf) = v.transform(desc, 4)
    assert np.array_equal(bw, hw) and np.array_equal(bv, hv) and np.array_equal(fn, hn) and np.array_equal(fo, ho)
    assert np.array_equal(slot_to_contiguous_index(ff, counts, cap), hf) and int(b.status.item()) == 0
    assert b.max_nodes == v.level_nodes(4) and b.node is not None


@pytest.mark.parametrize("scoring,weighting", [(0, 0), (1, 1), (2, 2), (3, 3), (4, 0), (5, 1), (5, 3)])
def test_scoring_and_weighting(api, oa, voc, scoring, weighting):
    from make_bow_golden import descriptors
    v, o = api.ORBVocabulary(voc, scoring, weighting), oa.OracleVocabulary(voc, scoring, weighting)
    desc = descriptors(voc, 3000, 40 + scoring)
    counts = [1100, 900, 1000]
    packed = pack_bow_frames([split(desc, counts)], 1101, 32, "single")[0]
    for levelsup in (4, 1, 0, 6, 8):
        check(api, call(api, v, packed, counts, 1101, levelsup), v, desc, counts, 1101, levelsup, o)


def test_empty_camera_empty_frame_one_keypoint(api, oa, voc):
    from make_bow_golden import descriptors
    v, o = api.ORBVocabulary(voc), oa.OracleVocabulary(voc)
    desc = descriptors(voc, 700, 3)
    for layout in LAYOUTS:
        for counts, d in (([400, 0, 300], desc), ([0, 0, 0], desc[:0]), ([0, 1, 0], desc[5:6]), ([0, 0, 700], desc)):
            per = split(d, counts)
            full = split(desc, [300, 200, 200])                          # the neighbour frame of the shared buffer is not empty
            packed = pack_bow_frames([full, per], 420 if counts[2] != 700 else 700, 32, layout)[1]
            cap = 420 if counts[2] != 700 else 700
            H = call(api, v, packed, counts, cap, 4)
            nb, nf = check(api, H, v, d, counts, cap, 4, o if len(d) else None)
            if not len(d):
                assert nb == 0 and nf == 0 and H["fv_offsets"][0] == 0
            if len(d) == 1:
                assert nb == 1 and nf == 1 and list(H["fv_offsets"][:2]) == [0, 1] and H["fv_features"][0] == cap


@pytest.mark.parametrize("scoring,weighting", [(0, 0), (1, 1), (5, 0), (0, 2)])
def test_identical_descriptors_and_stopped_words(api, oa, voc, scoring, weighting):
    """every descriptor identical: one node, one word, its weight added n - 1 times one after another (not w * n); and a vocabulary
    half of whose words are stopped (weight 0): their features are in neither vector"""
    from make_bow_golden import descriptors
    v, o = api.ORBVocabulary(voc, scoring, weighting), oa.OracleVocabulary(voc, scoring, weighting)
    one = descriptors(voc, 1, 11)
    desc = np.repeat(one, 2500, axis=0)
    counts = [1000, 700, 800]
    packed = pack_bow_frames([split(desc, counts)], 1000, 32, "parts")[0]
    for levelsup in (4, 0):
        H = call(api, v, packed, counts, 1000, levelsup)
        assert check(api, H, v, desc, counts, 1000, levelsup, o) == (1, 1)
        assert np.array_equal(slot_to_contiguous_index(H["fv_features"][:2500], counts, 1000), np.arange(2500))
    stopped = {k: voc[k].copy() for k in voc.files}
    wn = stopped["word_node"]
    stopped["weight"][wn[::2]] = 0.0
    vs, os_ = api.ORBVocabulary(stopped, scoring, weighting), oa.OracleVocabulary(stopped, scoring, weighting)
    desc = descriptors(voc, 2500, 12)
    packed = pack_bow_frames([split(desc, counts)], 1000, 32, "single")[0]
    for levelsup in (4, 0):
        H = call(api, vs, packed, counts, 1000, levelsup)
        check(api, H, vs, desc, counts, 1000, levelsup, os_)
        n_live = int(H["fv_offsets"][H["n_fv"][0]])
        assert 500 < n_live < 2000 and np.all(H["weight"][:3000][H["weight"][:3000] != VEC_FILL] >= 0)


def test_wide_toy_tree(api, oa):
    toy = toy_tree()
    tv, to = api.ORBVocabulary(toy), oa.OracleVocabulary(toy)
    rng = np.random.default_rng(6)
    n = len(toy["parent"])
    q = np.concatenate([toy["desc"][rng.integers(1, n, 300)], rng.integers(0, 256, (300, 32), dtype=np.uint8)]).astype(np.uint8)
    counts = [250, 150, 200]
    packed = pack_bow_frames([split(q, counts)], 256, 32, "single")[0]
    for levelsup in (1, 0, 2):
        check(api, call(api, tv, packed, counts, 256, levelsup), tv, q, counts, 256, levelsup, to)


def test_max_nodes_too_small(api, voc):
    from make_bow_golden import descriptors
    v = api.ORBVocabulary(voc)
    desc = descriptors(voc, 3000, 21)
    counts = [1000, 1000, 1000]
    packed = pack_bow_frames([split(desc, counts)], 1024, 32, "single")[0]
    bw, bv, (fn, fo, ff) = v.transform(desc, 4)
    for short in (len(fn) - 1, 1):
        H = call(api, v, packed, counts, 1024, 4, max_nodes=short)              # the guard words are checked inside
        assert H["status"][0] == api.MCS_ERR_CAPACITY and H["n_fv"][0] == short
        # the nodes that fit are complete; the BowVector does not depend on max_nodes
        assert np.array_equal(H["fv_nodes"][:short], fn[:short]) and np.array_equal(H["fv_offsets"][:short + 1], fo[:short + 1])
        assert np.array_equal(slot_to_contiguous_index(H["fv_features"][:fo[short]], counts, 1024), ff[:fo[short]])
        assert np.all(H["fv_features"][fo[short]:3 * 1024] == VEC_FILL)
        assert np.array_equal(H["bow_words"][:len(bw)], bw) and np.array_equal(H["bow_values"][:len(bw)], bv)
    H = call(api, v, packed, counts, 1024, 4, max_nodes=len(fn))
    assert H["status"][0] == 0 and H["n_fv"][0] == len(fn)


def test_busy_stream(api, voc, extracted):
    """the call is queued behind earlier work of its stream and gives the same result"""
    import torch
    counts = [len(p[0]) for p in extracted]
    cap = max(counts)
    desc = np.concatenate([p[1] for p in extracted])
    packed = pack_bow_frames([extracted], cap, 32, "single")[0]
    v = api.ORBVocabulary(voc)
    s = torch.cuda.Stream()
    a = torch.randn(4096, 4096, device="cuda")
    with torch.cuda.stream(s):
        for _ in range(10):
            a = a @ a * 1e-3
    check(api, call(api, v, packed, counts, cap, 4, stream=s), v, desc, counts, cap, 4)


def test_reference_golden_through_the_packed_buffer(api, voc):
    """the stored outputs of the reference's own DBoW2, the stored descriptors placed in a packed buffer"""
    g = np.load(GOLD / "bow_small_voc.npz")
    for ci in range(int(g["n_cases"][0])):
        sc, wg, levelsup, n, _ = (int(x) for x in g[f"c{ci}_cfg"])
        v = api.ORBVocabulary(voc, sc, wg)
        d = g[f"c{ci}_desc"]
        counts = [n // 3, n - n // 3 - n // 4, n // 4]
        cap = max(counts) + 3
        H = call(api, v, pack_bow_frames([split(d, counts)], cap, 32, "parts")[0], counts, cap, levelsup)
        nb, nf = int(H["n_bow"][0]), int(H["n_fv"][0])
        assert np.array_equal(H["bow_words"][:nb], g[f"c{ci}_bow_words"]) and np.array_equal(H["bow_values"][:nb], g[f"c{ci}_bow_values"])
        assert np.array_equal(H["fv_nodes"][:nf], g[f"c{ci}_fv_nodes"]) and np.array_equal(H["fv_offsets"][:nf + 1], g[f"c{ci}_fv_off"])
        assert np.array_equal(slot_to_contiguous_index(H["fv_features"][:H["fv_offsets"][nf]], counts, cap), g[f"c{ci}_fv_feat"])
        live = np.concatenate([np.arange(c * cap, c * cap + k) for c, k in enumerate(counts)])
        assert np.array_equal(H["word"][live], g[f"c{ci}_word"]) and np.array_equal(H["weight"][live], g[f"c{ci}_weight"])


def test_refusals_that_need_a_vocabulary(api, voc, extracted):
    counts = [len(p[0]) for p in extracted]
    cap = max(counts)
    packed = pack_bow_frames([extracted], cap, 32, "single")[0]
    v = api.ORBVocabulary(voc)
    with pytest.raises(api.McsError) as e:
        v.transform_device((packed[0], 1, 5, 3), 3, cap)                   # first_image + n_cams beyond the buffer's images
    assert e.value.code == api.MCS_ERR_INVALID
    with pytest.raises(api.McsError) as e:
        v.transform_device(packed, 3, cap, max_nodes=0)
    assert e.value.code == api.MCS_ERR_INVALID
