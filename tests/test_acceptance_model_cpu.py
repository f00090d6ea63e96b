"""CPU: the plain-Python model of the device searches' ordered acceptance (tests/acceptance_model.py) against the oracle's
sequential entry points on every generated contention scene, and each scene class reaching the edge it is built for: the rounds
the fixpoint needs and where the walk starts, windows of exactly 8 and 9 candidates, decisions that oscillate between rounds,
exact ratio ties and threshold edges, and SearchForInitialization's evictions and equal-distance skips."""
import numpy as np
import pytest

import acceptance_model as am


def _cap():
    import multicol_slam_b200.api as api
    return api.lib().mcs_search_by_projection_max_rounds()


SPECS = am.catalogue(_cap())


@pytest.mark.parametrize("spec", SPECS, ids=[am.spec_id(s) for s in SPECS])
def test_model_equals_the_sequential_loop(api, oa, spec):
    m, s = am.make(api, spec)
    p = am.predict(api, oa, m, s)
    on, oout = p["oracle"][:2]
    assert p["n"] == on and np.array_equal(p["out"], oout)
    if s["kind"] == "init":
        assert p["prev"].tobytes() == p["oracle"][2].tobytes()
    assert p["n"] > 0


def _class_runs(api, oa, cls):
    out = []
    for spec in SPECS:
        if spec[0] == cls:
            m, s = am.make(api, spec)
            out.append((spec, m, s, am.predict(api, oa, m, s)))
    assert out
    return out


def test_depth_scenes_converge_at_the_cap_edges(api, oa):
    cap = _cap()
    for n_chain in (cap - 2, cap - 1):                   # cap - 1 and cap rounds: the rounds settle every query, no walk
        for spec, m, s, p in _class_runs(api, oa, f"depth{n_chain}"):
            assert p["diag"][0] == n_chain + 1 and p["diag"][1] == -1, am.spec_id(spec)
    for wm in (0, 1, 31):                                # cap + 1 rounds needed: the walk starts at that residue of a ballot window
        for spec, m, s, p in _class_runs(api, oa, f"depth{cap}_s{wm}"):
            assert p["diag"][0] == cap and p["diag"][1] % 32 == wm and p["diag"][1] > cap, am.spec_id(spec)
            qs = p["R"]["queries"]
            assert {q.cam for q in qs[:p["diag"][1]]} == {0, 1}               # the chain's queries interleave with camera 1's
            assert qs[p["diag"][1]].cam == 0


def test_oscillation_scenes_flip_decisions_back(api, oa):
    counts = [am.oscillating(p["R"]) for _, _, _, p in _class_runs(api, oa, "oscillation")]
    assert min(counts) >= 1, counts


def test_dense_scenes_tie_and_contend(api, oa):
    for spec, m, s, p in _class_runs(api, oa, "dense"):
        qs = p["R"]["queries"]
        assert len(qs) >= 50 and max(len(q.dists) for q in qs) >= 20, am.spec_id(spec)
        assert sum(len(set(q.dists)) < len(q.dists) for q in qs) >= len(qs) // 4, am.spec_id(spec)     # equal distances
        if s["kind"] != "init":
            assert p["diag"][0] >= 5, am.spec_id(spec)
        if s["kind"] in ("local", "window", "frames"):     # the ratio rules: decisions flip back between rounds
            assert am.oscillating(p["R"]) >= 1, am.spec_id(spec)


@pytest.mark.parametrize("n_cand", [8, 9])
def test_list_edge_windows(api, oa, n_cand):
    for mode in ("entry", "queries"):
        for spec, m, s, p in _class_runs(api, oa, f"list{n_cand}_{mode}"):
            qs = p["R"]["queries"]
            assert all(len(q.dists) == n_cand for q in qs), am.spec_id(spec)
            if n_cand == 9:                                # the 8th and 9th keys at one distance, for each group's base query
                ties = sum(q.keys()[7] >> 16 == q.keys()[8] >> 16 for q in qs)
                assert ties == len(qs) if mode == "entry" else ties >= len(qs) // 8, am.spec_id(spec)
            if mode == "entry":                            # every listed keypoint but one taken on entry
                taken = set(np.flatnonzero((s["pre"] if s["kind"] == "local" else s["mp_cur"]) >= 0).tolist())
                assert all(sum(sl in taken for sl in q.slots) == n_cand - 1 for q in qs), am.spec_id(spec)
            else:
                assert p["diag"][0] == 3, am.spec_id(spec)   # the copies take their keypoints in round 0, the query moves in round 1


def test_rule_edge_pairs(api, oa):
    hit_ratio = hit_th = 0
    for spec, m, s, p in [r for nn in (0.6, 0.75, 0.8, 0.9) for r in _class_runs(api, oa, f"rule{nn}")]:
        th = m.TH_LOW_ if s["kind"] == "init" else m.TH_HIGH_
        for q in p["R"]["queries"]:
            d = sorted(q.dists)
            if len(d) == 2 and float(d[1]) * m.mfNNratio == d[0]:
                hit_ratio += 1
            if len(d) == 1 and d[0] in (th, th + 1):
                hit_th += 1
    assert hit_ratio >= 40 and hit_th >= 40


def test_eviction_scenes_evict_and_skip_equal_distances(api, oa):
    for spec, m, s, p in _class_runs(api, oa, "evictions"):
        ev, ties = am.evicted(p["R"]["queries"], m.TH_LOW_, m.mfNNratio, 3)
        assert ev >= 3 and ties >= 3 and p["diag"][1] >= 0, am.spec_id(spec)

