"""GPU: map initialisation's search on the device, SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, window)
(mcs_search_for_initialization_device) and FirstInitialization's seed of vbPrevMatched (mcs_search_for_initialization_seed_device),
against the host entry point cORBmatcher.SearchForInitialization, the CPU oracle and, where oracle/_ref travelled, the reference's
own method.  Both frames come from packed feature buffers in every layout.  nmatches, matches12 after the slot -> contiguous
conversion and prev are compared bit for bit; the slots beyond each camera's count must come back untouched."""
import numpy as np
import pytest

from device_frames import PREV_FILL, SIZES, flip, keep_cameras, rm  # noqa: F401  (rm: a fixture)
from device_searches import collect_init, device_init, host_init, init_inputs, launch_init

pytestmark = pytest.mark.gpu


def init_frames(api, cams, masks, n=2, nfeatures=800):
    """n consecutive 3-camera frames of the sliding-texture stream through the tracker's initialisation extractor settings"""
    from multicol_slam_b200 import synth
    ex = api.mdBRIEFextractorOct(nfeatures=nfeatures, fastThreshold=5, do_dBrief=True, learnMasks=masks)
    sf = [ex.info.scale_factor[l] for l in range(8)]
    streams = [synth.texture_stream(cams[c], n, seed=40 + c) for c in range(3)]
    return [api.Frame.from_cameras([ex(streams[c][t], synth.mirror_mask(cams[c]), cams[c]) for c in range(3)], SIZES, sf)
            for t in range(n)]


def _same(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2].tobytes() == b[2].tobytes()


def _kp_prev(F):
    return np.stack([F.keys["x"], F.keys["y"]], axis=1).astype(np.float64)


@pytest.mark.parametrize("layout", ["single", "parts", "shared"])
@pytest.mark.parametrize("masks", [False, True])
def test_parity_with_host_oracle_and_reference(api, oa, rm, cams, masks, layout):
    F1, F2 = init_frames(api, cams, masks)
    m = api.cORBmatcher(0.9, False, 32, masks)
    prev = _kp_prev(F1)
    h = host_init(m, F1, F2, prev, 50)
    o = oa.search_for_initialization(F1, F2, prev, 50, 0.9, m.TH_LOW_, masks)
    assert _same(h, o) and h[0] > 200
    if rm:
        assert _same(h, rm.search_for_initialization(rm.KF(F1, cams), rm.KF(F2, cams), prev, 50, 0.9, masks))
    gn, gm, gp, diag = device_init(api, m, F1, F2, prev, 50, layout)
    assert _same(h, (gn, gm, gp)) and diag[0] == len(F1.keys)


def test_seed_and_chained_frames(api, cams):
    """FirstInitialization's seed, then the initial frame against four successive frames with prev carried on the device"""
    import torch
    fr = init_frames(api, cams, True, n=5)
    F1 = fr[0]
    m = api.cORBmatcher(0.9, False, 32, True)
    d = init_inputs(api, F1, fr[1], np.zeros((len(F1.keys), 2)))
    m.SearchForInitializationSeedDevice(d["f1"], 3, d["cap"], d["prev_t"])
    torch.cuda.synchronize()
    p = d["prev_t"].cpu().numpy().reshape(3, d["cap"], 2)
    seeded = np.concatenate([p[c, :d["c1"][c]] for c in range(3)])
    assert seeded.tobytes() == _kp_prev(F1).tobytes() and np.all(np.concatenate([p[c, d["c1"][c]:] for c in range(3)]) == PREV_FILL)
    hp = _kp_prev(F1)
    for F2 in fr[1:]:
        h = host_init(m, F1, F2, hp, 50)
        hp = h[2]
        # the same packed F1 and prev tensor every call; F2 packed anew
        d2 = init_inputs(api, F1, F2, np.zeros((len(F1.keys), 2)), cap=d["cap"])
        d2["f1"], d2["prev_t"] = d["f1"], d["prev_t"]
        res = launch_init(m, d2, 50)
        torch.cuda.synchronize()
        g = collect_init(api, d2, *res)
        assert _same(h, g[:3]) and h[0] > 100


@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("dim", [16, 64])
def test_descriptor_sizes(api, oa, cams, dim, masks):
    from multicol_slam_b200 import synth
    ex = oa.OracleExtractor(nfeatures=400, fast_threshold=5, do_dbrief=True, learn_masks=True, desc_size=dim)
    streams = [synth.texture_stream(cams[c], 2, seed=60 + c) for c in range(3)]
    sf = [float(ex.info.scale_factor[l]) for l in range(8)]
    F1, F2 = [api.Frame.from_cameras([ex.extract(streams[c][t], synth.mirror_mask(cams[c]), cams[c]) for c in range(3)], SIZES, sf)
              for t in range(2)]
    assert F1.desc.shape[1] == dim
    m = api.cORBmatcher(0.9, False, dim, masks)
    prev = _kp_prev(F1)
    h = host_init(m, F1, F2, prev, 50)
    assert _same(h, oa.search_for_initialization(F1, F2, prev, 50, 0.9, m.TH_LOW_, masks)) and h[0] > 50
    for layout in ("single", "parts"):
        assert _same(h, device_init(api, m, F1, F2, prev, 50, layout)[:3])


def _frame(api, per_cam0, dim=32):
    """camera 0 holds (kps, desc); cameras 1 and 2 are empty"""
    e = np.zeros(0, api.KEYPOINT_DTYPE), np.zeros((0, dim), np.uint8), None
    k, dsc = per_cam0
    return api.Frame.from_cameras([(k, dsc, None), e, e], SIZES, np.cumprod([1.0] + [1.2000000476837158] * 7))


def _kps(api, xy):
    k = np.zeros(len(xy), api.KEYPOINT_DTYPE)
    k["x"], k["y"] = np.asarray(xy, np.float64).T
    return k


def displacement_scene(api, rng, dim=32):
    """F1 queries and F2 keypoints of camera 0 for the acceptance's edges (no masks: TH_LOW_ = 2 * dim = 64, nnratio 0.9).  Each
    group sits at its own spot, more than two windows (10 px) away from the others.  -> (F1, F2, expected matches12)"""
    q_xy, q_d, t_xy, t_d, expect = [], [], [], [], []

    def target(xy, d):
        t_xy.append(xy); t_d.append(d)
        return len(t_xy) - 1

    def query(xy, d, exp):
        q_xy.append(xy); q_d.append(d); expect.append(exp)
    # an eviction chain: twelve queries, each taking the one keypoint from the one before with a strictly smaller distance; the last
    # keeps it.  Then one at the owner's distance (d == MD: skipped, nothing left) and one above it.
    base = rng.integers(0, 256, dim).astype(np.uint8)
    t0 = target((100.0, 100.0), base)
    chain = [62, 58, 51, 47, 40, 33, 29, 22, 17, 11, 6, 2]
    for i, d in enumerate(chain):
        query((100.0 + 0.5 * i, 100.0), flip(rng, base, d), t0 if i == len(chain) - 1 else -1)
    query((101.0, 101.0), flip(rng, base, 2), -1)
    query((101.0, 100.5), flip(rng, base, 3), -1)
    query((101.0, 99.0), flip(rng, base, 1), t0)         # ... and one below it takes it again
    expect[len(chain) - 1] = -1
    # d0 == th_low accepted, th_low + 1 rejected (one candidate each: second = INT_MAX)
    b1, b2 = (rng.integers(0, 256, dim).astype(np.uint8) for _ in range(2))
    t1 = target((200.0, 100.0), b1)
    query((200.0, 100.0), flip(rng, b1, 2 * dim), t1)
    target((300.0, 100.0), b2)
    query((300.0, 100.0), flip(rng, b2, 2 * dim + 1), -1)
    # an exact ratio tie: 9 against 10 at 0.9 (9 < 9.0 fails)
    b3 = rng.integers(0, 256, dim).astype(np.uint8)
    q3 = flip(rng, b3, 0)
    target((400.0, 100.0), flip(rng, b3, 9)); target((402.0, 101.0), flip(rng, b3, 10))
    query((401.0, 100.0), q3, -1)
    assert 9 >= 10 * 0.9
    # rescans: ten candidates at distances 1..10 from a query; seven earlier queries take the seven best with distance 0, so the
    # query's list of 8 holds one free entry and its window is scanned again: 8 against 9 passes (8 < 8.1)
    b4 = rng.integers(0, 256, dim).astype(np.uint8)
    cands = [flip(rng, b4, d) for d in range(1, 11)]
    ids = [target((500.0 + 1.5 * (i % 5), 100.0 + 2.0 * (i // 5)), cands[i]) for i in range(10)]
    for i in range(7):
        query((503.0, 101.0), cands[i], ids[i])
    query((503.0, 101.0), b4, ids[7])
    q = _kps(api, q_xy)
    t = _kps(api, t_xy)
    return _frame(api, (q, np.stack(q_d))), _frame(api, (t, np.stack(t_d))), np.asarray(expect, np.int32)


def test_displacement_edges(api, oa, rm, cams):
    F1, F2, expect = displacement_scene(api, np.random.default_rng(11))
    m = api.cORBmatcher(0.9, False, 32, False)
    prev = _kp_prev(F1)
    h = host_init(m, F1, F2, prev, 10)
    assert _same(h, oa.search_for_initialization(F1, F2, prev, 10, 0.9, m.TH_LOW_, False))
    if rm:
        assert _same(h, rm.search_for_initialization(rm.KF(F1, cams), rm.KF(F2, cams), prev, 10, 0.9, False))
    assert np.array_equal(h[1], expect) and h[0] == int((expect >= 0).sum())
    for layout in ("single", "parts", "shared"):
        gn, gm, gp, diag = device_init(api, m, F1, F2, prev, 10, layout)
        assert _same(h, (gn, gm, gp)) and diag[1] > 0        # the rescan group rescanned


@pytest.mark.parametrize("cap", [24000, 30000])
def test_large_capacities(api, oa, cams, cap):
    """capacities whose MD needs more than the default 48 KB of shared memory with the walk's static lists: 24 000 (MD alone is
    under 48 KB) and 30 000 (MD alone is over)"""
    F1, F2, expect = displacement_scene(api, np.random.default_rng(11))
    m = api.cORBmatcher(0.9, False, 32, False)
    prev = _kp_prev(F1)
    h = host_init(m, F1, F2, prev, 10)
    assert np.array_equal(h[1], expect)
    for layout in ("single", "parts"):
        assert _same(h, device_init(api, m, F1, F2, prev, 10, layout, cap=cap)[:3])
    F1, F2 = init_frames(api, cams, True)
    m = api.cORBmatcher(0.9, False, 32, True)
    prev = _kp_prev(F1)
    h = host_init(m, F1, F2, prev, 50)
    assert h[0] > 200 and _same(h, device_init(api, m, F1, F2, prev, 50, "shared", cap=cap)[:3])


def test_equal_distances_earlier_visit_wins(api, oa):
    """two candidates at one distance; at nnratio 1.2 the best is accepted, and it must be the one visited first: keypoint 1, in a
    grid cell to the left of keypoint 0's"""
    rng = np.random.default_rng(5)
    base = rng.integers(0, 256, 32).astype(np.uint8)
    F2 = _frame(api, (_kps(api, [(318.0, 200.0), (290.0, 200.0)]), np.stack([flip(rng, base, 5), flip(rng, base, 5)])))
    F1 = _frame(api, (_kps(api, [(304.0, 200.0)]), base[None, :].copy()))
    m = api.cORBmatcher(1.2, False, 32, False)
    prev = _kp_prev(F1)
    h = host_init(m, F1, F2, prev, 20)
    assert _same(h, oa.search_for_initialization(F1, F2, prev, 20, 1.2, m.TH_LOW_, False)) and h[1][0] == 1
    assert _same(h, device_init(api, m, F1, F2, prev, 20)[:3])


def test_shapes(api, oa, cams):
    F1, F2 = init_frames(api, cams, True)
    m = api.cORBmatcher(0.9, False, 32, True)
    sub = lambda F, keep: keep_cameras(api, F, keep)[0]  # noqa: E731
    # empty cameras in either frame
    for A, B in ((sub(F1, [0, 2]), F2), (F1, sub(F2, [1])), (sub(F1, [1]), sub(F2, [0, 1]))):
        prev = _kp_prev(A)
        h = host_init(m, A, B, prev, 50)
        assert _same(h, device_init(api, m, A, B, prev, 50, "parts")[:3])
    # centres outside the image and at negative coordinates
    prev = _kp_prev(F1)
    rng = np.random.default_rng(9)
    i = rng.choice(len(prev), 60, replace=False)
    prev[i[:20]] = -rng.uniform(1, 80, (20, 2))
    prev[i[20:40], 0] += 760.0
    prev[i[40:], 1] = -prev[i[40:], 1] + 5.0
    h = host_init(m, F1, F2, prev, 50)
    assert _same(h, device_init(api, m, F1, F2, prev, 50)[:3])
    # window 0: only keypoints exactly at the centre (F1 against itself)
    prev = _kp_prev(F1)
    h = host_init(m, F1, F1, prev, 0)
    assert h[0] > 100 and _same(h, device_init(api, m, F1, F1, prev, 0)[:3])
    # a 200-px window: hundreds of candidates per query
    h = host_init(m, F1, F2, prev, 200)
    g = device_init(api, m, F1, F2, prev, 200, "shared")
    assert _same(h, g[:3])


def test_call_does_not_wait_for_the_stream(api, cams):
    import torch
    F1, F2 = init_frames(api, cams, True)
    m = api.cORBmatcher(0.9, False, 32, True)
    prev = _kp_prev(F1)
    h = host_init(m, F1, F2, prev, 50)
    d = init_inputs(api, F1, F2, prev)
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda._sleep(400_000_000)                  # a few hundred milliseconds of work ahead of the call
        res = launch_init(m, d, 50, stream=st)
        busy = st.query()
    assert busy is False
    st.synchronize()
    assert _same(h, collect_init(api, d, *res)[:3])
