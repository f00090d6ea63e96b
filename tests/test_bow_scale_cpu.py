"""Bag of words on a full-size vocabulary (tests/bow_scale.py: k = 10, L = 6, 1 064 066 nodes and 956 865 words), CPU side: the
oracle's restatement of DBoW2 (oracle/mcs_oracle.cpp) against the reference's own TemplatedVocabulary::transform / score loading
the same tree from DBoW2's text layout.  Every levelsup from 0 to 7 and every scoring x weighting; ids, values and the
FeatureVector bit for bit (the values are doubles made in the same operation order).  The reference's results are recorded to
tests/golden/ref_tape_bow_scale_cpu.* (MCS_RECORD_REF_TAPE=1 next to the built reference) and replayed everywhere else."""
import pathlib
import sys
import tempfile

import numpy as np
import pytest

import bow_scale

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
import ref_tape  # noqa: E402


@pytest.fixture(scope="module")
def voc():
    return bow_scale.vocabulary()


@pytest.fixture(scope="module")
def ref(voc):
    """the reference's DBoW2 on the same tree: the text file exists only while recording; its name carries the tree's digest, which
    the tape checks on replay"""
    ra = ref_tape.module("ref_dbow2_api", "bow_scale_cpu", 0)
    with tempfile.TemporaryDirectory() as d:
        path = pathlib.Path(d) / f"voc_k10_L6_{bow_scale.tree_crc(voc):08x}.txt"
        if ref_tape.RECORD:
            bow_scale.write_text(voc, path)
        yield ra.RefVocabulary(path)


@pytest.fixture(scope="module")
def frames(voc):
    return dict(spread=bow_scale.spread(voc, 6000, 1), clustered=bow_scale.clustered(voc, 1500, 2),
                stopped=bow_scale.stopped(voc, 2000, 3))


def test_tree_shape(voc):
    parent, depth, wn = voc["parent"], voc["depth"], voc["word_node"]
    n = len(parent)
    assert n > 2**20 + 10000 and len(wn) > 2**19 and (n + 2047) // 2048 > 256 and (len(wn) + 2047) // 2048 < (n + 2047) // 2048
    assert np.all(parent[1:] < np.arange(1, n)) and depth.max() == 6
    children = np.bincount(parent[1:], minlength=n)
    leaf = children == 0; leaf[0] = False
    assert np.array_equal(np.flatnonzero(leaf), wn) and children.max() == 10
    assert ((children > 0) & (children < 10)).sum() > 1000 and (leaf & (depth < 6)).sum() > 100       # irregular
    assert (voc["weight"][wn] == 0).sum() > 10000 and (voc["weight"][~leaf] == 0).all() and (voc["weight"] >= 0).all()
    dup = np.all(voc["desc"][2:] == voc["desc"][1:-1], axis=1) & (parent[2:] == parent[1:-1])      # a sibling's exact copy
    assert dup.sum() > 1000
    assert bow_scale.tree_crc(bow_scale.vocabulary()) == bow_scale.tree_crc(voc)                     # the seed decides the tree


def test_level_nodes_walk_the_parents(voc):
    """numpy_level_nodes (depths made while building) against depths found by walking up from every node"""
    parent = voc["parent"]
    depth, a = np.zeros(len(parent), np.int64), np.arange(len(parent))
    while np.any(a != 0):
        depth += a != 0
        a = parent[a]
    assert np.array_equal(depth, voc["depth"])
    got = [bow_scale.numpy_level_nodes(voc, s) for s in range(8)]
    assert got[0] == len(voc["word_node"]) and got[6] == got[7] == 1 and got[1] > 90000 and got[2] > 9000


def test_frames_reach_the_shapes(oa, voc, frames):
    o = oa.OracleVocabulary(voc)
    nb = {k: len(o.transform(d, 0)[0]) for k, d in frames.items()}
    assert nb["spread"] > 4096 and nb["clustered"] <= 12
    w, wt, _ = o.transform_features(frames["stopped"], 4)
    assert (wt == 0).mean() > 0.4 and len(np.unique(w)) > 1000


def deep(o, voc, d, levelsup):
    """the descriptors whose leaf lies at depth L - levelsup or deeper.  For a leaf above that depth the reference never writes the
    node id (its caller's uninitialised variable reaches the FeatureVector); the oracle and the library put the leaf itself there"""
    w = o.transform_features(d, 0)[0]
    return d[voc["depth"][voc["word_node"][w]] >= int(voc["L"]) - levelsup]


def same_as_reference(o, ref, voc, d, levelsup, what):
    """the BowVector of the whole frame, and both vectors of its deep part, bit for bit"""
    A, B = o.transform(d, levelsup), ref.transform(d, levelsup)
    dd = deep(o, voc, d, levelsup)
    if len(dd) == len(d):
        assert all(ref_tape.same(x, y) for x, y in zip(A, B)), what
        return
    assert ref_tape.same(A[0], B[0]) and ref_tape.same(A[1], B[1]), what
    assert all(ref_tape.same(x, y) for x, y in zip(o.transform(dd, levelsup), ref.transform(dd, levelsup))), what


def test_shallow_leaves_keep_their_own_node(oa, voc, frames):
    o = oa.OracleVocabulary(voc)
    d = frames["spread"]
    w, _, _ = o.transform_features(d, 0)
    leaf = voc["word_node"][w]
    for levelsup in (0, 1):
        shallow = voc["depth"][leaf] < int(voc["L"]) - levelsup
        assert shallow.sum() > 0 and len(deep(o, voc, d, levelsup)) == len(d) - shallow.sum()
        _, _, nd = o.transform_features(d, levelsup)
        assert np.array_equal(nd[shallow], leaf[shallow]) and np.all(voc["depth"][nd[~shallow]] == int(voc["L"]) - levelsup)


@pytest.mark.parametrize("scoring", range(6))
def test_oracle_matches_reference(oa, voc, ref, frames, scoring):
    for weighting in range(4):
        o = oa.OracleVocabulary(voc, scoring, weighting)
        ref.set_types(scoring, weighting)
        for levelsup in range(8):
            same_as_reference(o, ref, voc, frames["spread"], levelsup, (scoring, weighting, levelsup))
        for name in ("clustered", "stopped"):
            for levelsup in (0, 4):
                same_as_reference(o, ref, voc, frames[name], levelsup, (name, scoring, weighting, levelsup))
        a, b = o.transform(frames["spread"][:3000], 0), o.transform(frames["spread"][1500:], 0)
        assert o.score(a[0], a[1], b[0], b[1]) == ref.score(a[0], a[1], b[0], b[1])
        c = o.transform(frames["clustered"], 2)
        assert o.score(c[0], c[1], c[0], c[1]) == ref.score(c[0], c[1], c[0], c[1])


def test_words_match_reference(oa, voc, ref):
    o = oa.OracleVocabulary(voc)
    ref.set_types(0, 0)
    d = np.concatenate([bow_scale.spread(voc, 3000, 7), bow_scale.stopped(voc, 1000, 8)])
    w, wt, _ = o.transform_features(d, 4)
    rw, rwt = ref.words(d)
    assert ref_tape.same(w, rw) and ref_tape.same(wt, rwt)
    assert ref.size() == len(voc["word_node"])
