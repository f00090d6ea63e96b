"""GPU: local mapping's device SearchForTriangulationRaw (mcs_search_for_triangulation_device) equals the host route
(cORBmatcher.SearchForTriangulationRawHost: read back, slots_to_contiguous, host rays, mcs_search_for_triangulation) bit for bit --
matches12 row and nmatches -- which the CPU tests pin to the reference's own SearchForTriangulationRaw: at 16-, 32- and 64-byte
descriptors with and without masks, in the three packed layouts, on a scene whose lists cannot decide some queries (rescans) and
one where they decide all, at the empty-camera / no-query / all-free / full-capacity / KF1 == KF2 edges, on a busy stream and the
NULL stream, and along CreateNewMapPoints' sequence of five neighbours with the new points written on the device.  Slots at or
beyond a camera's count hold free ids (-1) and a poisoned output, and must stay unread and unwritten.  One test pins the epipolar
test's arithmetic: the threshold equal to a pair's residual rejects it on both routes, the next double accepts it."""
import numpy as np
import pytest

from device_frames import counts, flip_bits, frames, keep_cameras, pack_frames, to_slots  # noqa: F401  (frames: a fixture)
from device_searches import assert_same_tri, device_tri, host_tri, tri_inputs
from search_scenes import epipolar_residual, essential, rig_of, tri_scene

pytestmark = pytest.mark.gpu


def compare(api, m, s, k, cams, cap, mp1=None, mp2=None, layout="single", epi=1e-2, oa=None):
    mp1 = s["mp1"] if mp1 is None else mp1
    mp2 = s["mps"][k] if mp2 is None else mp2
    E = essential(s["rig1"], s["rigs"][k])
    dev = device_tri(api, m, s["KF1"], s["nbs"][k], mp1, mp2, cams, cap, E, layout, epi)
    host = host_tri(api, m, s["KF1"], s["nbs"][k], mp1, mp2, cams, cap, E, epi)
    assert_same_tri(api, s["KF1"], dev, host, cap)
    if oa is not None:
        ho = host_tri(api, m, s["KF1"], s["nbs"][k], mp1, mp2, cams, cap, E, epi, oa)
        assert host[0] == ho[0] and np.array_equal(host[1], ho[1])
    free1 = int((np.asarray(mp1) == -1).sum())
    assert dev[2][0] == free1                                          # diag: the queries
    return dev


def cap_of(s):
    return max(max(counts(F)) for F in [s["KF1"]] + s["nbs"])


@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masked", [False, True])
def test_widths_and_masks(api, oa, frames, cams, dim, masked):
    s = tri_scene(api, frames, cams, 2, seed=20 + dim, dim=dim)
    m = api.cORBmatcher(0.6, False, dim, masked)
    cap = cap_of(s) + 5
    for k in range(2):
        n = compare(api, m, s, k, cams, cap, oa=oa)[0]
        assert n > 20


@pytest.mark.parametrize("layout", ["single", "parts", "joint"])
def test_layouts(api, frames, cams, layout):
    s = tri_scene(api, frames, cams, 2, seed=31)
    m = api.cORBmatcher(0.6, False, 32, True)
    cap = cap_of(s) + 2
    for k in range(2):
        assert compare(api, m, s, k, cams, cap, layout=layout)[0] > 20


def paging_scene(api, frames, cams, dim, seed):
    """test_search_for_triangulation_paging's construction on a tri_scene: 40 free same-camera near copies of two free KF1
    queries in the neighbour, so that their lists are full of candidates an epipolar test may reject"""
    s = tri_scene(api, frames, cams, 1, seed=seed, dim=dim)
    rng = np.random.default_rng(seed)
    KF1, F2 = s["KF1"], s["nbs"][0]
    d2 = F2.desc.copy()
    free1 = np.flatnonzero(s["mp1"] == -1)
    for q, at in ((free1[3], 0), (free1[4], 40)):
        same_cam = np.flatnonzero(F2.key_cam == KF1.key_cam[q])[at:at + 40]
        d2[same_cam] = KF1.desc[q]
        d2[same_cam, 1] ^= rng.integers(0, 4, len(same_cam)).astype(np.uint8)
        s["mps"][0][same_cam] = -1
    s["nbs"][0] = api.Frame(F2.keys, F2.key_cam, d2, F2.dmask, list(zip(F2.cam_w, F2.cam_h)), F2.scale_factors)
    return s


@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masked", [False, True])
def test_rescans(api, frames, cams, dim, masked):
    """the paging scene: some decisions rescan the camera's database.  A scene where a query has at most a few candidates, at a
    threshold every pair passes: no list is ever full, so the lists decide every query."""
    s = paging_scene(api, frames, cams, dim, seed=40 + dim)
    m = api.cORBmatcher(0.6, False, dim, masked)
    cap = cap_of(s) + 1
    rescans = 0
    for epi in (1e-2, 1e-4, 1e-6, 1e300):
        rescans += compare(api, m, s, 0, cams, cap, epi=epi)[2][1]
    assert rescans > 0
    sparse = tri_scene(api, frames, cams, 1, seed=40 + dim, dim=dim)
    rng = np.random.default_rng(dim)
    KF1 = sparse["KF1"]                                                 # (neighbour 0 has KF1's keypoints)
    d1 = rng.integers(0, 256, KF1.desc.shape, dtype=np.uint8)           # random rows: unrelated pairs lie far beyond th_low
    d2 = flip_bits(rng, d1, 2)                                        # the neighbour: each row a near copy of KF1's
    full = np.full(KF1.desc.shape, 255, np.uint8)
    sizes = list(zip(KF1.cam_w, KF1.cam_h))
    sparse["KF1"] = api.Frame(KF1.keys, KF1.key_cam, d1, full, sizes, KF1.scale_factors)
    sparse["nbs"][0] = api.Frame(KF1.keys, KF1.key_cam, d2, full, sizes, KF1.scale_factors)
    n, _, diag = compare(api, m, sparse, 0, cams, cap_of(sparse) + 1, epi=1e300)
    assert n > 50 and diag[1] == 0


def test_edges(api, frames, cams):
    """an empty camera on either side, a camera without a free query, every slot free, a camera's count == capacity"""
    m = api.cORBmatcher(0.6, False, 32, True)
    s = tri_scene(api, frames, cams, 2, seed=50)
    cap = max(counts(s["KF1"]))                                       # a camera's count == capacity, in both frames
    assert counts(s["nbs"][0]) == counts(s["KF1"])
    compare(api, m, s, 0, cams, cap)
    # camera 1 of KF1 empty, camera 2 of the neighbour empty
    (K1, k1), (K2, k2) = keep_cameras(api, s["KF1"], [0, 2]), keep_cameras(api, s["nbs"][0], [0, 1])
    e = dict(s, KF1=K1, mp1=s["mp1"][k1], nbs=[K2], mps=[s["mps"][0][k2]])
    assert counts(e["KF1"])[1] == 0 and counts(e["nbs"][0])[2] == 0
    assert compare(api, m, e, 0, cams, cap)[0] > 10
    # no free query in camera 0
    mp1 = s["mp1"].copy()
    mp1[(s["KF1"].key_cam == 0) & (mp1 == -1)] = 123456
    n0, m12, _ = compare(api, m, s, 0, cams, cap, mp1=mp1)
    assert n0 > 10 and (m12[:counts(s["KF1"])[0]] == -1).all()
    # every slot free
    allfree1, allfree2 = np.full(len(s["KF1"].keys), -1, np.int32), np.full(len(s["nbs"][0].keys), -1, np.int32)
    assert compare(api, m, s, 0, cams, cap, mp1=allfree1, mp2=allfree2)[0] > 50


def test_kf1_is_kf2(api, frames, cams):
    """KF1 searched against itself, one buffer and one map-point row for both"""
    m = api.cORBmatcher(0.6, False, 32, True)
    s = tri_scene(api, frames, cams, 1, seed=60)
    cap = cap_of(s) + 4
    E = essential(s["rig1"], rig_of(api, cams, [0.03, 0.0, 0.01]))
    dev = device_tri(api, m, s["KF1"], s["KF1"], s["mp1"], s["mp1"], cams, cap, E, same=True)
    host = host_tri(api, m, s["KF1"], s["KF1"], s["mp1"], s["mp1"], cams, cap, E)
    assert_same_tri(api, s["KF1"], dev, host, cap)
    assert dev[0] > 50


def test_busy_and_null_stream(api, frames, cams):
    """queued behind long matrix products on a side stream, and on the NULL stream (the call synchronises)"""
    import torch
    m = api.cORBmatcher(0.6, False, 32, True)
    s = tri_scene(api, frames, cams, 1, seed=70)
    cap = cap_of(s) + 3
    E = essential(s["rig1"], s["rigs"][0])
    args = (s["KF1"], s["nbs"][0], s["mp1"], s["mps"][0], cams, cap)
    host = host_tri(api, m, *args, E)
    p1, mp1_t, p2, mp2_t, out = tri_inputs(api, *args)
    side = torch.cuda.Stream()
    a = torch.randn(8192, 8192, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        for _ in range(4):
            a = a @ a * 1e-4
    n_t, m12_t, d_t = m.SearchForTriangulationRawDevice(p1, mp1_t, p2, mp2_t, cams, cap, E, stream=side, out=out, diag=True)
    side.synchronize()
    assert_same_tri(api, s["KF1"], (int(n_t.item()), m12_t.cpu().numpy(), d_t.cpu().numpy()), host, cap)
    assert torch.cuda.current_stream().cuda_stream == 0                  # stream=None passes the NULL stream
    p1, mp1_t, p2, mp2_t, out = tri_inputs(api, *args)
    n_t, m12_t = m.SearchForTriangulationRawDevice(p1, mp1_t, p2, mp2_t, cams, cap, E, out=out)
    assert_same_tri(api, s["KF1"], (int(n_t.item()), m12_t.cpu().numpy(), None), host, cap)


@pytest.mark.parametrize("masked", [False, True])
def test_neighbour_sequence_on_device(api, frames, cams, masked):
    """CreateNewMapPoints over five neighbours: after each device search a seeded stand-in for the triangulation checks writes new
    ids into KF1's and the neighbour's rows on the device; every step equals the host route from the rows as they stand"""
    import torch
    s = tri_scene(api, frames, cams, 5, seed=11)
    m = api.cORBmatcher(0.6, False, 32, masked)
    cap = cap_of(s) + 3
    packs = pack_frames([s["KF1"]] + s["nbs"], cap, layout="joint")
    mp1_t = to_slots(api, s["KF1"], s["mp1"], cap, -1)
    gen = torch.Generator(device="cuda").manual_seed(5)
    next_id = s["next_id"]
    for k in range(5):
        mp2_t = to_slots(api, s["nbs"][k], s["mps"][k], cap, -1)
        E = essential(s["rig1"], s["rigs"][k])
        mp1_now = api.slots_to_contiguous(mp1_t.cpu().numpy(), counts(s["KF1"]), cap)
        host = host_tri(api, m, s["KF1"], s["nbs"][k], mp1_now, s["mps"][k], cams, cap, E)
        n_t, m12_t = m.SearchForTriangulationRawDevice(packs[0], mp1_t, packs[1 + k], mp2_t, cams, cap, E)
        m12 = m12_t.cpu().numpy()
        assert int(n_t.item()) == host[0] > 10
        n1 = counts(s["KF1"])
        assert np.array_equal(api.slots_to_contiguous(m12, n1, cap), api.slots_to_contiguous(host[1], n1, cap)), k
        # the stand-in, on the device: about 70 % of the pairs become points with new ids
        keep = (m12_t >= 0) & (torch.rand(m12_t.shape, generator=gen, device="cuda") < 0.7)
        ids = next_id + torch.cumsum(keep.to(torch.int32), 0, dtype=torch.int32) - 1
        mp1_t[keep] = ids[keep]
        mp2_t[m12_t[keep].long()] = ids[keep]
        next_id += int(keep.sum().item())
    # KF1's row went from searches to the next: later searches see fewer queries than the entry state has
    assert int((mp1_t.cpu().numpy() == -1).sum()) < int((to_slots(api, s["KF1"], s["mp1"], cap, 0, "cpu").numpy() == -1).sum())


def test_epipolar_threshold_edge(api, cams):
    """one free query and its one candidate (equal descriptors, camera 0): epi_thresh = the host's residual of the pair rejects it
    on both routes (the test is strict), nextafter(residual, inf) accepts it on both"""
    keys = np.zeros(2, api.KEYPOINT_DTYPE)
    keys["x"], keys["y"] = [400.25, 431.5], [300.75, 287.0]
    rng = np.random.default_rng(80)
    d = rng.integers(0, 256, (1, 32), dtype=np.uint8)
    mk = np.full((1, 32), 255, np.uint8)
    sizes, sf = [(754, 480)] * 3, [1.2 ** i for i in range(8)]
    KF1 = api.Frame(keys[:1], np.zeros(1, np.int32), d, mk, sizes, sf)
    KF2 = api.Frame(keys[1:], np.zeros(1, np.int32), d, mk, sizes, sf)
    E = essential(rig_of(api, cams, [0, 0, 0]), rig_of(api, cams, [0.03, -0.01, 0.02]))
    r1 = np.array(api.img_to_world(cams[0], float(keys["x"][0]), float(keys["y"][0])))
    r2 = np.array(api.img_to_world(cams[0], float(keys["x"][1]), float(keys["y"][1])))
    res = epipolar_residual(api, r1, r2, E[0, 0])
    assert res > 0
    m = api.cORBmatcher(0.6, False, 32, True)
    mp = np.array([-1], np.int32)
    for thr, want in ((res, 0), (float(np.nextafter(res, np.inf)), 1)):
        host = host_tri(api, m, KF1, KF2, mp, mp, cams, 4, E, thr)
        dev = device_tri(api, m, KF1, KF2, mp, mp, cams, 4, E, epi=thr)
        assert host[0] == want and dev[0] == want, (thr, host[0], dev[0])
        assert_same_tri(api, KF1, dev, host, 4)
