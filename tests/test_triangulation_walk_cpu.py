"""CPU: the plain-Python model of the device SearchForTriangulationRaw (tests/triangulation_model.py) against the sequential loop on
every planted scene -- the oracle's search, the Python restatement and the reference's own SearchForTriangulationRaw (recorded in
tests/golden/ref_tape_triangulation_walk_cpu.*) -- each scene class reaching the decision edge it is built for, and each rule
mutant of the model told apart from the sequential loop by some scene, in its matches or in its rescans."""
import numpy as np
import pytest

import triangulation_model as tm
from device_frames import counts, taped_rm
from search_scenes import reference_tri

SPECS = tm.catalogue()
_cache = {}
rm = taped_rm("triangulation_walk_cpu")


def scene(api, oa, cams, spec):
    if spec not in _cache:
        s = tm.make(api, oa, cams, spec)
        _cache[spec] = (s, tm.predict(oa, s))
    return _cache[spec]


def oracle(oa, s):
    """oracle_api.search_for_triangulation on the scene -> (nmatches, contiguous matches12)"""
    F1, F2, mk = s["KF1"], s["nbs"][0], (lambda F: F.dmask if s["masked"] else None)
    return oa.search_for_triangulation(F1.desc, mk(F1), F1.key_cam, (s["mp1"] == -1).astype(np.uint8), s["rays1"], F2.desc, mk(F2),
                                       F2.key_cam, (s["mps"][0] == -1).astype(np.uint8), s["rays2"], s["E"], s["th_low"], s["epi"])


@pytest.mark.parametrize("spec", SPECS, ids=[tm.spec_id(s) for s in SPECS])
def test_model_equals_the_sequential_loop(api, oa, rm, cams, spec):
    import pyref_match
    s, p = scene(api, oa, cams, spec)
    on, om12 = oracle(oa, s)
    assert p["n"] == on and np.array_equal(p["m12"], om12)
    F1, F2, mk = s["KF1"], s["nbs"][0], (lambda F: F.dmask if s["masked"] else None)
    if len(F2.keys) < 5000:                                              # the Python loop: not over a 65535-row camera
        pn, pm12 = pyref_match.search_for_triangulation(F1.desc, mk(F1), F1.key_cam, s["mp1"] == -1, s["rays1"], F2.desc, mk(F2),
                                                        F2.key_cam, s["mps"][0] == -1, s["rays2"], s["E"], s["th_low"], s["epi"])
        assert pn == p["n"] and np.array_equal(pm12, p["m12"])
    if s["epi"] == 1e-2:                                                 # the reference's threshold (ref :1085)
        assert rm.thresholds(s["dim"], s["masked"])[1] == s["th_low"]
        rn, rpairs = reference_tri(rm, api, s, 0, cams, s["mp1"], s["mps"][0], s["masked"])
        hit = np.flatnonzero(p["m12"] >= 0)
        assert rn == p["n"] and np.array_equal(rpairs, np.stack([hit, p["m12"][hit]], 1).astype(np.int32).reshape(-1, 2))
    assert p["diag"][0] == int((s["mp1"] == -1).sum())


def _runs(api, oa, cams, cls):
    out = [(spec,) + scene(api, oa, cams, spec) for spec in SPECS if spec[0] == cls]
    assert out
    return out


def test_window_edge(api, oa, cams):
    """the winner behind a taken and a failing entry at wd == 2 * best is accepted, at 2 * best + 1 rejected, from the list and in
    a rescan that must skip a taken row"""
    for spec, s, p in _runs(api, oa, cams, "window"):
        eq = spec[3] == "eq"
        r0, r1, r2 = (p["record"][c][-1] for c in range(3))
        assert r0["rule"] == ("list_win" if eq else "list_window_reject") and r0["wpos"] == 2, r0
        assert r0["wd"] == 2 * r0["best"] + (0 if eq else 1) and p["lists"][0][-1][0][0] in {r["win"] for r in p["record"][0][:-1]}
        assert r2["rule"] == r0["rule"] and r2["wpos"] == 1 and r2["wd"] == r0["wd"]
        assert r1["rule"] == ("rescan_no_pass_win" if eq else "rescan_no_pass_none"), r1
        assert r1["rescan_wd"] == 2 * r1["rescan_best"] + (0 if eq else 1) and r1["n_listed"] == tm.K


def test_list_length(api, oa, cams):
    """7 candidates: the short list decides; 8: a rescan when dK <= 2 * best (== and <), none when dK > 2 * best; 9: the ninth,
    tied with dK at a larger index, is the one that passes and only a rescan finds it"""
    want = {"7": ["list_short_none"] * 3, "8": ["rescan_no_pass_none", "list_dK_none", "rescan_no_pass_none"],
            "9": ["rescan_no_pass_win"] * 3}
    for spec, s, p in _runs(api, oa, cams, "length"):
        n = int(spec[3])
        recs = [p["record"][c][0] for c in range(3)]
        assert [r["rule"] for r in recs] == want[spec[3]], recs
        assert all(r["n_cand"] == n and r["n_listed"] == min(n, tm.K) for r in recs)
        if n == 8:
            assert [np.sign(r["dK"] - 2 * r["best"]) for r in recs] == [0, 1, -1]
        if n == 9:
            for c, r in enumerate(recs):
                assert r["rescan_wd"] == r["dK"] and r["win"] > p["lists"][c][0][-1][0] and r["rescan_wd"] <= 2 * r["best"]
        assert all(p["record"][c][1]["rule"] == "list_short_none" and p["record"][c][1]["n_listed"] == 0 for c in range(3))


def test_exhausted_lists(api, oa, cams):
    """chains of >= 9 identical queries: from the ninth on every listed entry is taken and the camera is rescanned, with and without
    a winner"""
    for spec, s, p in _runs(api, oa, cams, "chains"):
        for c in range(3):
            rules = [r["rule"] for r in p["record"][c]]
            assert len(rules) >= 9 and rules[:tm.K] == ["list_win"] * tm.K, (tm.spec_id(spec), rules)
            assert all(r.startswith("rescan_no_open") for r in rules[tm.K:]), (tm.spec_id(spec), rules)
        rules = [r["rule"] for rc in p["record"] for r in rc]
        assert rules.count("rescan_no_open_win") >= 3 and rules.count("rescan_no_open_none") >= 3


def test_th_low_edge(api, oa, cams):
    """a candidate at th_low is listed and taken; one at th_low + 1 is never listed and never taken, even by a rescan whose window
    2 * best reaches past th_low"""
    for spec, s, p in _runs(api, oa, cams, "th_low"):
        th = s["th_low"]
        for c in range(3):
            at, over, scan = p["record"][c]
            assert at["rule"] == "list_win" and at["wd"] == th
            assert over["rule"] == "list_short_none" and over["n_listed"] == 0
            assert 2 * scan["best"] > th and scan["rule"] == ("rescan_no_pass_win" if spec[3] == "in" else "rescan_no_pass_none")
            if spec[3] == "in":
                assert scan["rescan_wd"] == th


def test_ties_across_chunks_and_scan_warps(api, oa, cams):
    """equal-distance candidates straddle a database chunk boundary of seg_lists_kernel and are taken in index order; equal-distance
    candidates held by different scanning warps of a rescan are taken in index order"""
    (spec, s, p), = _runs(api, oa, cams, "ties")
    chunk, splits = tm.chunk_of(s["cap"], 3)
    rows = s["tie_rows"]
    assert splits >= 2 and rows[0] < chunk <= rows[-1]
    wins0 = [r["win"] for r in p["record"][0]]
    assert wins0 == rows + [-1]
    assert [r["rule"] for r in p["record"][0]][tm.K:] == ["rescan_no_open_win"] * 2 + ["rescan_no_open_none"]
    wins1 = [r["win"] for r in p["record"][1]]
    assert wins1 == s["warp_rows"] + [-1] and all(r["rule"].startswith("rescan_no_pass") for r in p["record"][1])
    assert len({tm.scan_warp(j) for j in s["warp_rows"]}) >= 3


def test_epipolar_threshold_in_the_rescan(api, oa, cams):
    """epi_thresh == the residual of a pair only a rescan reaches rejects it; the next double accepts it"""
    for spec, s, p in _runs(api, oa, cams, "epi"):
        r = p["record"][0][0]
        assert r["n_listed"] == tm.K
        if spec[3] == "at":
            assert r["rule"] == "rescan_no_pass_none"
        else:
            assert r["rule"] == "rescan_no_pass_win" and r["win"] == s["near_row"]
    eps = sorted(s["epi"] for _, s, _ in _runs(api, oa, cams, "epi"))
    assert eps[1] == np.nextafter(eps[0], np.inf)


def test_walk_and_list_blocks(api, oa, cams):
    """query counts at the walk's 32-query chunks and the lists' 128-row blocks, rescans at t = 31 and the next chunk's t = 0; a
    camera with queries and no free KF2 row, one with no query"""
    seen = set()
    for spec, s, p in _runs(api, oa, cams, "blocks"):
        for c, n in enumerate(s["n_queries"]):
            rec = p["record"][c]
            assert len(rec) == n
            seen.add(n)
            if spec[3] == "edge" and c == 1:
                assert all(r["rule"] == "list_short_none" and r["n_listed"] == 0 for r in rec)
                continue
            for t in (31, 32, 63, 64, 127, 128):
                if t < n:
                    assert rec[t]["rule"] == "rescan_no_pass_win", (tm.spec_id(spec), c, t)
    assert {31, 32, 33, 65, 127, 128, 129, 0} <= seen


def test_capacity_bound(api, oa, cams):
    """a camera with count == capacity == 65535 free KF2 rows: a winner at compact index 65534 from the list, and one in the last
    stride of tr_scan from a rescan, both in the last database chunk"""
    (spec, s, p), = _runs(api, oa, cams, "capacity")
    assert counts(s["nbs"][0])[0] == s["cap"] == tm.CAPACITY and (s["mps"][0] == -1).all()
    chunk, splits = tm.chunk_of(s["cap"], 3)
    by_win = {r["win"]: r for r in p["record"][0]}
    assert by_win[tm.CAPACITY - 1]["rule"] == "list_win"
    assert by_win[s["scan_row"]]["rule"] == "rescan_no_pass_win"
    assert s["scan_row"] >= tm.CAPACITY - tm.CAPACITY % tm.SCAN_THREADS and -(-tm.CAPACITY // tm.SCAN_THREADS) == 293
    assert min(s["scan_row"], tm.CAPACITY - 1) >= (splits - 1) * chunk and splits >= 2


def test_rule_mutants_are_caught(api, oa, cams):
    """each rule mutant of the model gives other matches than the sequential loop, or other rescans than the model, on some scene"""
    caught = {}
    for mut in tm.MUTANTS:
        for spec in SPECS:
            s, p = scene(api, oa, cams, spec)
            q = tm.predict(oa, s, mut)
            if q["n"] != p["n"] or not np.array_equal(q["m12"], p["m12"]) or q["diag"] != p["diag"]:
                caught[mut] = tm.spec_id(spec)
                break
    assert set(caught) == set(tm.MUTANTS), sorted(set(tm.MUTANTS) - set(caught))
