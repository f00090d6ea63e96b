"""A full-size bag-of-words vocabulary and frames to run through it, generated from a seed (nothing of it is stored).

vocabulary(seed) is a k = 10, L = 6 tree (1 064 066 nodes and 956 865 words at the default seed), the size DBoW2 vocabularies
are trained at, in the layout api.ORBVocabulary and oracle_api.OracleVocabulary take.  It is built level by level, each child's
descriptor being its parent's with a few bits flipped, so a descriptor made from a leaf by a few flips descends to that leaf or a
near one (with independent random descriptors every query would end in a handful of words).  It is irregular the way k-means trees are: some
nodes have fewer than k children, some leaves sit above level L, some siblings are exact duplicates (the descent's first-minimum
rule decides between them) and some words are stopped (weight 0).  Node ids are breadth-first, so a parent's id is below its
children's and a leaf's word id is its rank among the leaves in id order, as DBoW2's text loader numbers them.

write_text() writes it in DBoW2's text layout for the reference's own loader; the frame generators below make descriptor sets
that spread over many words, cluster into a few, hit stopped words, or have rows of another width."""
import pathlib
import zlib

import numpy as np

K, L = 10, 6
FLIPS = [0, 128, 36, 22, 13, 8, 5]          # bits flipped from parent to child at each depth (depth 1: independent random rows)


def flip(rng, rows, nbits):
    """rows (n, 32) with up to nbits random bits flipped in each (a bit drawn twice flips once)"""
    n = len(rows)
    if nbits >= 256:
        return rng.integers(0, 256, (n, 32), dtype=np.uint8)
    mask = np.zeros((n, 256), np.uint8)
    mask[np.arange(n)[:, None], rng.integers(0, 256, (n, nbits))] = 1
    return rows ^ np.packbits(mask, axis=1, bitorder="little")


def vocabulary(seed=2026, scoring=0, weighting=0):
    rng = np.random.default_rng(seed)
    parent, desc, depth = [np.zeros(1, np.int32)], [np.zeros((1, 32), np.uint8)], [np.zeros(1, np.int32)]
    level, first = np.zeros(1, np.int64), 0                  # ids of the nodes at the current depth
    for d in range(1, L + 1):
        nc = np.full(len(level), K)
        if d > 1:
            few = rng.random(len(level)) < 0.015             # fewer than k children
            nc[few] = rng.integers(1, K, few.sum())
        if d > 2:
            nc[rng.random(len(level)) < 0.003] = 0           # a leaf above level L
        par = np.repeat(level, nc)
        cd = flip(rng, desc[-1][par - first], FLIPS[d])
        pos = np.arange(len(par)) - np.repeat(np.cumsum(nc) - nc, nc)              # position among the siblings
        dup = (pos > 0) & (rng.random(len(par)) < 0.01)
        cd[dup] = cd[np.flatnonzero(dup) - 1]                # an exact duplicate of the sibling before it
        first = sum(len(p) for p in parent)
        parent.append(par.astype(np.int32)); desc.append(cd); depth.append(np.full(len(par), d, np.int32))
        level = first + np.arange(len(par))
    parent, desc, depth = np.concatenate(parent), np.concatenate(desc), np.concatenate(depth)
    n = len(parent)
    leaf = np.ones(n, bool); leaf[parent[1:]] = False; leaf[0] = False
    word_node = np.flatnonzero(leaf).astype(np.int32)
    weight = np.zeros(n)
    weight[word_node] = np.log(1e5 / rng.integers(1, 20000, len(word_node)))      # IDF-like: log(N / N_i) > 0
    weight[word_node[rng.random(len(word_node)) < 0.04]] = 0.0                     # stopped words
    return dict(k=K, L=L, scoring=scoring, weighting=weighting, parent=parent, weight=weight, desc=desc, word_node=word_node,
                depth=depth)


def tree_crc(v):
    """a short digest of the tree, for a file name that changes when the tree does"""
    c = 0
    for key in ("parent", "weight", "desc", "word_node"):
        c = zlib.crc32(np.ascontiguousarray(v[key]).tobytes(), c)
    return c


def write_text(v, path):
    """DBoW2's text layout (TemplatedVocabulary::loadFromTextFile): 'k L scoring weighting', then per node in id order
    'parent isLeaf d0..d31 weight'.  No newline after the last line: the loader would read an empty one as another node."""
    n = len(v["parent"])
    leaf = np.zeros(n, bool); leaf[v["word_node"]] = True
    cols = [v["parent"][1:].astype(str), leaf[1:].astype(int).astype(str)]
    cols += [v["desc"][1:, b].astype(str) for b in range(32)]
    cols.append(np.array([repr(float(w)) for w in v["weight"][1:]]))
    body = cols[0]
    for c in cols[1:]:
        body = np.char.add(np.char.add(body, " "), c)
    head = "%d %d %d %d" % (v["k"], v["L"], v["scoring"], v["weighting"])
    pathlib.Path(path).write_text("\n".join([head] + body.tolist()))


def numpy_level_nodes(v, levelsup):
    """the most node ids a FeatureVector can hold: the nodes at depth L - levelsup and the leaves above it"""
    level = max(int(v["L"]) - levelsup, 0)
    leaf = np.zeros(len(v["parent"]), bool); leaf[v["word_node"]] = True
    return int((v["depth"] == level).sum() + (leaf & (v["depth"] < level)).sum())


def spread(v, n, seed, flips=2):
    """n descriptors, each a few bits from a different random leaf, one in fifty from a leaf above level L: thousands of distinct
    words"""
    rng = np.random.default_rng(seed)
    wn = v["word_node"]
    leaves = wn[rng.choice(len(wn), n, replace=False)]
    shallow = wn[v["depth"][wn] < v["L"]]
    leaves[::50] = shallow[rng.integers(0, len(shallow), len(leaves[::50]))]
    return flip(rng, v["desc"][leaves], flips)


def clustered(v, n, seed, n_words=6, flips=2):
    """n descriptors around a handful of leaves"""
    rng = np.random.default_rng(seed)
    wn = v["word_node"]
    return flip(rng, v["desc"][wn[rng.choice(len(wn), n_words, replace=False)][rng.integers(0, n_words, n)]], flips)


def stopped(v, n, seed, share=0.5):
    """about `share` of the descriptors sit exactly on a stopped word's leaf, the rest are spread"""
    rng = np.random.default_rng(seed)
    wn = v["word_node"]
    st = wn[v["weight"][wn] == 0]
    d = spread(v, n, seed + 1)
    on = rng.random(n) < share
    d[on] = v["desc"][st[rng.integers(0, len(st), on.sum())]]
    return d


def other_width(v, n, seed, dim):
    """rows of dim bytes (16 or 64): the first 32 bytes (or half of one) of spread descriptors"""
    d = spread(v, n, seed)
    return np.ascontiguousarray(np.concatenate([d, d[::-1]], axis=1)[:, :dim])
