"""K2 (octree_kernel, the device DistributeOctTree) works in fixed buffers: a node table per image and level, sel_cap selected slots
per level, and the output capacity of mcs_extractor_info, which is fixed at mcs_extractor_create before the image size is known.

DistributeOctTree (ref src/mdBRIEFextractorOct.cpp:625-874) starts from nIni = cvRound((maxX - minX) / (maxY - minY)) roots, and its
first pass divides every root holding more than one corner into up to 4 nodes, whatever the level's quota N.  Every later pass
starts below N and adds at most 3 nodes per division, so it stops below N + 3.  A level therefore holds up to max(4 nIni, N + 2)
nodes and returns that many keypoints; on wide images with small budgets the first pass alone exceeds the quota.  These checks plan
every geometry the extractor accepts (mcs_extractor_octree_plan, host only) and compare the sizes with those bounds, check the
bounds against the reference's own per-level counts, and check the oracle restatement against the reference fixtures of those
edges, including the geometries the extractor refuses."""
import glob
import json
import math
import pathlib
import re

import numpy as np
import pytest

GOLD = pathlib.Path(__file__).resolve().parent / "golden"
CSRC = pathlib.Path(__file__).resolve().parents[1] / "multicol_slam_b200" / "csrc"
FIXTURES = sorted(glob.glob(str(GOLD / "ref_octree_*.npz")))
EDGE = 25
TOO_WIDE = "image too wide for nfeatures: the octree can return more keypoints than the capacity"
# what the extractor says about each fixture's geometry before any launch; every other fixture is extracted
REFUSED = {
    "wide_4095x600_orb100": TOO_WIDE,
    "wide_3000x400_orb200": TOO_WIDE,
    "wide_3000x400_mdbrief100": TOO_WIDE,
    "wide_1500x200_l4_orb40": TOO_WIDE,
    "wide_4095x244_l7_orb100": TOO_WIDE,
    "one_level_4095x600_orb10": TOO_WIDE,
    "wide_2000x250_orb50": "level too small for the 30 px cell grid",     # level 7 is 70 px high: no row of 30 px cells
}
# the extractor's refusals of a geometry for reasons other than the octree
OTHER_REFUSALS = {"pyramid level smaller than 58 px", "level too small for the 30 px cell grid", "FAST cells narrower than 30 px",
                  "portrait images narrower than half their height"}
# (scale factor, levels): the shipped 1.2 / 8, and the corners the other fixtures use
PYRAMIDS = [(1.2, 8), (1.2, 4), (1.2, 1), (1.1, 8), (1.3, 6), (1.5, 5), (2.0, 3)]


def k_max_nodes():
    return int(re.search(r"constexpr int kMaxNodes = (\d+);", (CSRC / "mcs_common.cuh").read_text()).group(1))


def quotas(nf, sf, L):
    """mnFeaturesPerLevel and the inverse scale factors as mcs_extractor_create computes them (ref :151-179)"""
    sfd = float(np.float32(sf))
    isf = [1.0]
    for _ in range(1, L):
        isf.append(isf[-1] * (1.0 / sfd))
    factor = 1.0 / sfd
    nd = nf * (1 - factor) / (1 - math.pow(factor, L))
    q = []
    for _ in range(L - 1):
        q.append(round(nd))           # cvRound: ties to even, as Python's round
        nd *= factor
    q.append(max(nf - sum(q), 0))
    return q, isf


def roots(W, H, isf):
    """nIni of every level (ref :640): maxX - minX = w - 2 (EDGE - 3), level sizes cvRound(W / scale)"""
    out = []
    for s in isf:
        w, h = round(W * s), round(H * s)
        out.append(round((w - 2 * (EDGE - 3)) / (h - 2 * (EDGE - 3))))
    return out


def worst_case(nf, sf, L, W, H):
    """(most nodes a level's list holds, most keypoints per level) by the DistributeOctTree rules"""
    q, isf = quotas(nf, sf, L)
    n = roots(W, H, isf)
    return q, n, [max(4 * r, a + 2) for a, r in zip(q, n)]


def largest_nfeatures(api, sf, L):
    """the largest budget mcs_extractor_create accepts: the top quota + 8 must fit kMaxNodes"""
    lo, hi = 1, 1 << 16
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if api.octree_plan(754, 480, nfeatures=mid, scale_factor=sf, nlevels=L)[0] == api.MCS_ERR_UNSUPPORTED and \
                "node table" in api.lib().mcs_last_error().decode():
            hi = mid - 1
        else:
            lo = mid
    return lo


def sizes(sf, L):
    """image sizes up to 4095 whose top level is at least 58 px high: every width with the lowest heights (the widest levels), and
    the usual heights"""
    h_min = next(h for h in range(58, 4096) if round(h * float(np.float32(sf)) ** -(L - 1)) >= 2 * EDGE + 8)
    hs = sorted({h_min, h_min + 1, int(h_min * 1.3), 2 * h_min, 480, 720, 1080} & set(range(h_min, 4096)))
    ws = sorted(set(range(h_min, 4096, 61)) | {4095})
    return [(w, h) for h in hs for w in ws]


@pytest.mark.parametrize("sf,L", PYRAMIDS)
def test_octree_buffers_cover_every_accepted_geometry(api, sf, L):
    kmax = k_max_nodes()
    nf_max = largest_nfeatures(api, sf, L)
    assert quotas(nf_max, sf, L)[0][0] + 8 <= kmax < quotas(nf_max + 1, sf, L)[0][0] + 8
    accepted = refused = over_quota = 0
    for nf in sorted({1, 8, 50, 100, 400, 1000, nf_max}):
        for W, H in sizes(sf, L):
            rc, node_table, n_ini, sel_cap, cap = api.octree_plan(W, H, nfeatures=nf, scale_factor=sf, nlevels=L)
            msg = api.lib().mcs_last_error().decode()
            q, n, most = worst_case(nf, sf, L, W, H)
            assert cap == sum(max(a + 2, 16) for a in q)
            if rc and msg != TOO_WIDE:
                assert rc == api.MCS_ERR_UNSUPPORTED and msg in OTHER_REFUSALS, (W, H, nf, msg)
                continue
            assert n_ini.tolist() == n, (W, H, nf)
            if rc:
                assert sum(most) > cap, (W, H, nf)
                refused += 1
                continue
            accepted += 1
            over_quota += any(r > a + 2 for a, r in zip(q, most))
            assert sum(most) <= cap, (W, H, nf)
            assert node_table % 32 == 0 and max(max(a + 8, 4 * r) for a, r in zip(q, n)) <= node_table <= kmax, (W, H, nf)
            assert all(s >= m for s, m in zip(sel_cap, most)), (W, H, nf)
    # both outcomes occur, and some accepted geometries return more keypoints than quota + 2 on a level
    assert accepted and refused and over_quota, (accepted, refused, over_quota)


def test_plan_of_the_benchmark_geometries_is_unchanged(api):
    """754x480 and 1920x1080 (BASELINE.json configs 2 and 4) have nIni <= 2: the node table stays max(quota) + 8 rounded up to 32"""
    for W, H, nf in [(754, 480, 2000), (1920, 1080, 4000), (1280, 720, 2000)]:
        rc, node_table, n_ini, sel_cap, cap = api.octree_plan(W, H, nfeatures=nf)
        q, _ = quotas(nf, 1.2, 8)
        assert rc == api.MCS_OK and max(n_ini) <= 2
        assert node_table == (max(q) + 8 + 31) // 32 * 32 and cap == sum(q) + 16
        assert sel_cap.tolist() == [a + 3 for a in q]


def load(path):
    from multicol_slam_b200 import synth
    g = np.load(path)
    cam = json.loads(bytes(g["cam_json"]).decode())
    kw = json.loads(bytes(g["params_json"]).decode())
    img = synth.frame(cam, int(g["seed"]))
    assert zlib_crc(img) == int(g["image_crc"]), "synthetic image generator changed"
    return pathlib.Path(path).stem[len("ref_octree_"):], g, cam, kw, img


def zlib_crc(a):
    import zlib
    return zlib.crc32(np.ascontiguousarray(a).tobytes())


def test_fixture_set_covers_the_edges():
    """wide images refused and accepted, zero quotas, one-level pyramids at the node-table limit, mdBRIEF with masks"""
    names = {pathlib.Path(p).stem[len("ref_octree_"):] for p in FIXTURES}
    assert set(REFUSED) < names
    kmax = k_max_nodes()
    seen = dict(over_quota=0, zero_quota=0, node_limit=0, wide_masked=0, roots_over_32=0)
    for path in FIXTURES:
        name, g, cam, kw, _ = load(path)
        L = kw.get("nlevels", 8)
        q, n, most = worst_case(kw["nfeatures"], kw.get("scale_factor", 1.2), L, cam["width"], cam["height"])
        per_level = g["per_level"].tolist()
        seen["over_quota"] += name not in REFUSED and any(c > a + 2 for a, c in zip(q, per_level))
        seen["zero_quota"] += q[-1] == 0 and per_level[-1] > 0
        seen["node_limit"] += L == 1 and q[0] + 8 == kmax and per_level[0] == q[0] + 2
        seen["wide_masked"] += kw.get("learn_masks", False) and cam.get("mirror_mask", 1) == 1 and max(n) > 2
        seen["roots_over_32"] += name in REFUSED and max(n) > 32
    assert all(seen.values()), seen


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: pathlib.Path(p).stem[len("ref_octree_"):])
def test_reference_counts_within_the_bound(api, path):
    """the reference's own per-level counts never exceed max(4 nIni, quota + 2), and the refusals are exactly the fixtures whose
    bound sums above the capacity (or whose levels the extractor cannot grid)"""
    name, g, cam, kw, _ = load(path)
    L = kw.get("nlevels", 8)
    q, n, most = worst_case(kw["nfeatures"], kw.get("scale_factor", 1.2), L, cam["width"], cam["height"])
    per_level = g["per_level"].tolist()
    assert all(c <= m for c, m in zip(per_level, most)), (per_level, most)
    rc, _, n_ini, _, cap = api.octree_plan(cam["width"], cam["height"], **kw)
    assert (rc, api.lib().mcs_last_error().decode() if rc else None) == \
        ((api.MCS_ERR_UNSUPPORTED, REFUSED[name]) if name in REFUSED else (api.MCS_OK, None))
    if REFUSED.get(name) == TOO_WIDE:
        assert sum(per_level) > cap or sum(most) > cap
    if name == "wide_4095x600_orb100":          # the bound is reached: the first pass alone gives 4 nIni on every level
        assert per_level == [4 * r for r in n]


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: pathlib.Path(p).stem[len("ref_octree_"):])
def test_oracle_equals_reference_octree_fixture(oa, path):
    """the oracle restatement keeps the extractor's capacity rule: bit for bit on the accepted geometries (keypoints, descriptors,
    masks, pyramid and mask levels), the same refusal before any work on the wide ones"""
    name, g, cam, kw, img = load(path)
    from multicol_slam_b200 import synth
    e = oa.OracleExtractor(**kw)
    if name in REFUSED:
        with pytest.raises(RuntimeError, match="failed -2"):          # MCS_ERR_UNSUPPORTED
            e.extract(img, synth.mirror_mask(cam), cam)
        return
    k, d, m = e.extract(img, synth.mirror_mask(cam), cam)
    assert len(k) == int(g["n"])
    assert zlib_crc(k) == int(g["kps_crc"]) and zlib_crc(d) == int(g["desc_crc"]) and zlib_crc(m) == int(g["dmask_crc"])
    if "kps" in g.files:
        assert k.tobytes() == g["kps"].tobytes() and np.array_equal(d, g["desc"]) and np.array_equal(m, g["dmask"])
    for l in range(kw.get("nlevels", 8)):
        lvl = e.debug_read(l, 1) if int(g["per_level"][l]) else e.debug_read(l, 0)
        assert zlib_crc(lvl) == int(g["level_after_crc"][l]), f"pyramid level {l}"
        assert zlib_crc(e.debug_read(l, 2)) == int(g["mask_level_crc"][l]), f"mask level {l}"
