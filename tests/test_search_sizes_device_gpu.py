"""GPU: the device searches' query build past one pass of its scan.  ps_count_kernel counts the valid entries of each block of
2048 (kQbTile), ps_scan_kernel scans those counts in one CTA of 1024 threads, 1024 blocks per pass with a carry between passes,
and ps_fill_kernel / fu_entry_kernel place each query at its scanned offset; Fuse scans its hits the same way.  The calls here
run 1024 blocks less one entry, 1024 full blocks, 1025 blocks, three and five passes, and the 2^24 - 1 entries the C ABI
accepts, with empty and full blocks on both sides of each pass boundary.  SearchByProjection is compared bit for bit with the
host route (C++ window search and host replay) and with the same search split into calls of under 2^21 entries; Fuse with the
same key frames split into calls of under 2^21 entries and with the host Fuse on a key frame past the boundary.  A numpy model of
the count / scan / fill gives the query count each call must report, so a lost or shifted carry fails with its own message.

Scenes keep the acceptance's dependency chains short (each window holds one or two keypoints of a pair), so the fixpoint
rounds settle the queries and the single-warp walk has little to do; each call prints its rounds, walk start and rescans."""
import time

import numpy as np
import pytest

from device_frames import counts, frames  # noqa: F401  (frames: a fixture)
from device_searches import dev_map, device_projection, device_scw, fuse_device, fuse_replay, fuse_targets, launch_projection, projection_inputs
from search_scenes import fuse_scene, host_fuse, host_scw

TILE = 2048                 # entries per count / fill block (kQbTile)
PASS = 1024 * TILE          # entries one pass of the single-CTA scan covers: 2^21
BOUND = 1 << 24             # the first entry count the C ABI refuses
W, H, DIM = 640, 480, 32
PX, PY = 38, 38             # keypoint pairs per camera: a 38 x 38 lattice
NPAIR = PX * PY
QUERY_BYTES = 40 + 4 * 8 + 4 * 8 + 4 + 8        # front-end scratch per entry: query, list keys and slots, count, decisions
ENTRY_BYTES = 1 + 4 + 3 * 8                     # in_view, level, proj_x, proj_y, view_cos


def scan_model(valid):
    """count / scan of a validity vector in numpy, as the device runs it: per-block counts of TILE entries and their exclusive
    scan, offsets[b] = the first query index of block b's entries, offsets[-1] = the query count.  -> (counts, offsets)"""
    valid = np.asarray(valid, bool)
    nb = -(-len(valid) // TILE)
    counts = np.add.reduceat(valid.astype(np.int64), np.arange(nb) * TILE) if nb else np.zeros(0, np.int64)
    return counts, np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)


def _query_count_message(nq, offsets):
    return (f"the device built {nq} queries, the count / scan model {offsets[-1]} (blocks past 1024 start at query "
            f"{offsets[min(1024, len(offsets) - 1)]})")


def test_scan_model_matches_a_plain_enumeration():
    """the model itself, across pass boundaries: block b's offset is the number of valid entries before its first entry"""
    rng = np.random.default_rng(0)
    for n in (0, 1, TILE - 1, TILE + 1, 3 * TILE + 5, PASS + 3 * TILE + 1):
        valid = rng.random(n) < 0.4
        counts, offsets = scan_model(valid)
        assert len(counts) == -(-n // TILE) and offsets[-1] == valid.sum()
        starts = np.arange(len(counts)) * TILE
        assert np.array_equal(offsets[:-1], np.concatenate([[0], np.cumsum(valid)])[starts])


def _fits(nbytes, what):
    """skip when the call's device memory would not fit in what the shared device has free"""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if nbytes > 0.8 * free:
        pytest.skip(f"{what} needs about {nbytes / 2**30:.1f} GiB of device memory; {free / 2**30:.1f} GiB are free")


def _pattern(n, rng):
    """which of n entries are valid: a random density per block, with every 11th block empty and every 13th full, and around each
    pass boundary e (1024, 2048, ... blocks) blocks e - 2 and e + 1 empty, e - 1 and e full"""
    nb = -(-n // TILE)
    dens = rng.uniform(0.05, 0.7, nb)
    b = np.arange(nb)
    dens[b % 11 == 3] = 0.0
    dens[b % 13 == 5] = 1.0
    for e in range(1024, nb + 1, 1024):
        for off, d in ((-2, 0.0), (-1, 1.0), (0, 1.0), (1, 0.0)):
            if 0 <= e + off < nb:
                dens[e + off] = d
    return rng.random(n) < np.repeat(dens, TILE)[:n]


def _noise(rng, n, p):
    """n descriptor xor masks, each bit set with probability p (drawn from a pool of 4096)"""
    pool = np.packbits(rng.random((4096, 8 * DIM)) < p, axis=1)
    return pool[rng.integers(0, len(pool), n)]


def _projection_scene(api, n_entries, nc, seed):
    """n_entries = n_points * nc (map point outer, camera inner).  Every camera holds a lattice of keypoint pairs A (even) and B
    = A + 7 px (odd), all on octave 0, B's descriptor A's with about 20 bits flipped.  Point i aims at a pair of camera i % nc
    near its place in the order, so each pair is wanted by queries of one stretch of the order, on both sides of every pass
    boundary: a window around A (r = 2.5), around B, or around both (r = 4.0, the descriptor near one of them, so that the other
    is the fallback when it is taken).  Its other cameras' entries are random windows.  Validity follows _pattern; a point whose
    entries are all invalid is bad or out of view."""
    rng = np.random.default_rng(seed)
    n = n_entries // nc
    assert n * nc == n_entries
    ix, iy = np.meshgrid(np.arange(PX), np.arange(PY), indexing="ij")
    ax, ay = 16.0 + 16 * ix.ravel(), 14.0 + 12 * iy.ravel()
    per, kdesc = [], np.zeros((nc, 2 * NPAIR, DIM), np.uint8)
    for c in range(nc):
        k = np.zeros(2 * NPAIR, api.KEYPOINT_DTYPE)
        k["x"][0::2], k["y"][0::2], k["x"][1::2], k["y"][1::2] = ax, ay, ax + 7.0, ay
        kdesc[c, 0::2] = rng.integers(0, 256, (NPAIR, DIM), dtype=np.uint8)
        kdesc[c, 1::2] = kdesc[c, 0::2] ^ _noise(rng, NPAIR, 0.08)
        per.append((k, kdesc[c], None))
    valid = _pattern(n_entries, rng).reshape(n, nc)
    dead = ~valid.any(1)
    bad = (dead & (rng.random(n) < 0.5)).astype(np.uint8)
    in_view = valid.astype(np.uint8)
    in_view[bad != 0] = rng.random((int(bad.sum()), nc)) < 0.5
    px, py = rng.uniform(0, W, (n, nc)), rng.uniform(0, H, (n, nc))
    level = rng.integers(0, 3, (n, nc)).astype(np.int32)
    vc = rng.uniform(0.99, 1.0, (n, nc))
    i = np.arange(n)
    c = i % nc
    pair = np.minimum(NPAIR - 1, i * NPAIR // n + rng.integers(0, 2, n))
    kind = rng.integers(0, 3, n)                       # 0: A alone, 1: B alone, 2: both
    px[i, c] = ax[pair] + np.choose(kind, [0.0, 7.0, 3.5]) + rng.uniform(-0.3, 0.3, n)
    py[i, c] = ay[pair] + rng.uniform(-0.5, 0.5, n)
    level[i, c] = 0
    vc[i, c] = np.where(kind == 2, 0.99, 0.999)
    target = 2 * pair + np.where(kind == 1, 1, np.where(kind == 2, rng.integers(0, 2, n), 0))
    desc = kdesc[c, target] ^ _noise(rng, n, 0.03)
    sf = np.cumprod([1.0] + [1.2000000476837158] * 7)
    F = api.Frame.from_cameras(per, [(W, H)] * nc, sf)
    mps = api.MapPoints(bad, in_view, level, px, py, vc, desc, None)
    return F, per, mps, (in_view != 0) & (bad[:, None] == 0)


def _report(label, n_entries, nq, diag, t):
    print(f"\n{label}: {n_entries} entries, {-(-n_entries // TILE)} blocks, {nq} queries; rounds {diag[0]}, walk from query "
          f"{diag[1]}, rescans {diag[3]}; {t:.1f} s")


# (n_points * n_cams): 1024 blocks less one entry, 1024 full blocks, 1025 blocks, three passes (the last partial), five passes
SIZES = [(PASS - 1, 7), (PASS, 4), (PASS + 1, 3), (2 * PASS + 17, 3), (5 * 1_678_000, 5)]


@pytest.mark.gpu
@pytest.mark.parametrize("n_entries,nc", SIZES, ids=["pass-1", "pass", "pass+1", "3-passes", "5-passes"])
def test_search_by_projection_past_one_scan_pass(api, n_entries, nc):
    """mcs_search_by_projection_device == mcs_search_by_projection (host route) bit for bit, and its query count == the model's"""
    _fits(n_entries * (ENTRY_BYTES + QUERY_BYTES) + (n_entries // nc) * (DIM + 1), f"{n_entries} entries")
    t0 = time.time()
    F, per, mps, valid = _projection_scene(api, n_entries, nc, seed=n_entries % 1000)
    counts, offsets = scan_model(valid.reshape(-1))
    nb = len(counts)
    for e in range(1024, nb + 1, 1024):           # the scene has what it is meant to have at every pass boundary
        full = lambda b: min(TILE, n_entries - b * TILE)  # noqa: E731
        assert counts[e - 2] == 0 and counts[e - 1] == full(e - 1) and (e == nb or counts[e] == full(e))
    m = api.cORBmatcher(0.8, False, DIM, False)
    hn, hfmp = m.SearchByProjection(F, mps, 1.0)
    gn, gfmp, status, diag = device_projection(api, m, per, [(W, H)] * len(per), F.scale_factors, mps, 1.0, layout="parts")
    _report("SearchByProjection", n_entries, int(diag[2]), diag, time.time() - t0)
    assert status == api.MCS_OK
    assert diag[2] == offsets[-1], _query_count_message(diag[2], offsets)
    assert gn == hn and np.array_equal(gfmp, hfmp)
    # real work next to the first pass boundary: points whose entries lie in the 64 blocks before entry 2^21 matched, and in the
    # 64 blocks after it where the call has them
    e = hfmp[hfmp >= 0].astype(np.int64) * nc
    assert ((e >= PASS - 64 * TILE) & (e < PASS)).sum() > 20
    if n_entries >= PASS + 64 * TILE:
        assert ((e >= PASS) & (e < PASS + 64 * TILE)).sum() > 20


def _split_search(api, m, per, sf, mps, chunk):
    """the same search as calls over consecutive map points of at most `chunk` points, each starting from the frame_mp the
    previous one left (the acceptance is sequential in point order, so this is the one-call result); a call's tags are its own
    point indices, so the new ones are shifted back to the whole map's"""
    import torch
    n = len(mps.bad)
    d = projection_inputs(api, per, api.MapPoints(mps.bad[:1], mps.in_view[:1], mps.level[:1], mps.proj_x[:1], mps.proj_y[:1], mps.view_cos[:1],
                                           mps.desc[:1]), layout="parts")
    full = api.MapPointsDevice.from_host(mps, d["packed"].device)
    total, worst = 0, 0
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        d["mdev"] = api.MapPointsDevice(full.bad[a:b], full.in_view[a:b], full.level[a:b], full.proj_x[a:b], full.proj_y[a:b],
                                        full.view_cos[a:b], full.desc[a:b])
        before = d["fm_t"].clone()
        n_t, st_t, fm_t, diag_t = launch_projection(m, d, [(W, H)] * len(per), sf, 1.0)
        torch.cuda.synchronize()
        assert int(st_t.item()) == api.MCS_OK
        new = fm_t != before
        fm_t[new] += a
        total += int(n_t.item())
        worst = max(worst, int(diag_t[0].item()))
    return total, api.slots_to_contiguous(d["fm_t"].cpu().numpy(), d["cc"], d["cap"]), worst


@pytest.mark.gpu
def test_search_by_projection_at_the_bound(api):
    """2^24 - 1 entries: accepted, and equal to the same search in calls of under 2^21 entries; 2^24 entries: refused before any
    launch, with every output untouched"""
    import torch
    nc = 5
    n_entries = BOUND - 1                     # 3 * 5 * 17 * 257 * 257
    _fits(n_entries * (2 * ENTRY_BYTES + QUERY_BYTES) + (n_entries // nc) * 2 * (DIM + 1), f"{n_entries} entries")
    t0 = time.time()
    F, per, mps, valid = _projection_scene(api, n_entries, nc, seed=24)
    m = api.cORBmatcher(0.8, False, DIM, False)
    gn, gfmp, status, diag = device_projection(api, m, per, [(W, H)] * len(per), F.scale_factors, mps, 1.0, layout="parts")
    _report("SearchByProjection at the bound", n_entries, int(diag[2]), diag, time.time() - t0)
    offsets = scan_model(valid.reshape(-1))[1]
    assert status == api.MCS_OK and diag[2] == offsets[-1], _query_count_message(diag[2], offsets)
    sn, sfmp, _ = _split_search(api, m, per, F.scale_factors, mps, (PASS - 1) // nc)
    assert gn == sn > 1000 and np.array_equal(gfmp, sfmp)
    # one entry more: refused by the 2^24 bound before any launch.  The map-point arrays are real (about 0.6 GiB), every entry
    # in view, so that a call that went ahead would read memory it owns and fail on the comparison below, not fault.
    nc4, npts = 4, BOUND // 4
    dev = torch.device("cuda")
    _fits(npts * (nc4 * ENTRY_BYTES + DIM), f"{BOUND} entries")
    z = lambda dt, *s: torch.zeros(s, dtype=dt, device=dev)  # noqa: E731
    mdev = api.MapPointsDevice(None, torch.ones((npts, nc4), dtype=torch.uint8, device=dev), z(torch.int32, npts, nc4),
                               *(z(torch.float64, npts, nc4) for _ in range(3)), z(torch.uint8, npts, DIM))
    assert mdev.view().n_points * nc4 == BOUND
    d = projection_inputs(api, per[:1] * nc4, mdev, layout="parts")
    out = tuple(torch.full((k,), -777, dtype=torch.int32, device=dev) for k in (1, 1, 4))
    before = d["fm_t"].clone()
    with pytest.raises(api.McsError, match=r"more than 2\^24 - 1 \(map point, camera\) entries") as err:
        m.SearchByProjectionDevice(d["packed"], d["n_parts"], d["part_images"], d["first"], d["nc"], d["cap"], [(W, H)] * nc4,
                                   F.scale_factors, mdev, 1.0, d["fm_t"], out=out, diag=True)
    torch.cuda.synchronize()
    assert err.value.code == api.MCS_ERR_UNSUPPORTED
    assert all(bool((o == -777).all()) for o in out) and torch.equal(d["fm_t"], before)


# ---- Fuse ---------------------------------------------------------------------------------------------------------------------
def _entries(hits, n_q, nc, cap):
    """a hit row (k, q, slot)'s maker entry (k * n_q + q) * n_cams + camera"""
    return (hits[:, 0].astype(np.int64) * n_q + hits[:, 1]) * nc + hits[:, 2] // cap


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [0, 1, 2])
def test_fuse_past_one_scan_pass(api, oa, frames, cams, variant):
    """mcs_fuse_device over more than 2^21 entries and more than 2^21 hits (so the hit scan's blocks past 1024 hold hits) ==
    the same key frames in calls of under 2^21 entries each, hit for hit; the hits come in maker order, as the model's fill
    places them; and a key frame whose entries lie past entry 2^21 replays to the host Fuse's ops"""
    KF = frames[0]
    s = fuse_scene(api, oa, cams, KF, variant)
    nc = len(cams)
    m = api.cORBmatcher(0.6, False, 32, True)
    cap = max(counts(KF)) + 3
    dm = dev_map(s)
    # one key frame at the scene's pose: its hits pick the queries.  Every query with a hit and every fourth without one, repeated,
    # so that more than an eighth of the entries hit and the hits outgrow one scan pass below the 2^24 entry bound.
    h1, n1, st1, _ = fuse_device(api, m, [KF], [s["sc"]["rig"]], [None], s["points"], dm, cap, "single", variant, Scw=s["Scw"])
    assert st1 == api.MCS_OK and n1 > 50
    hit_q = np.unique(h1[:, 1])
    base = np.union1d(hit_q, np.setdiff1d(np.arange(len(s["points"])), hit_q)[::4])
    reps = 48
    n_q = reps * len(base)
    per_kf = n_q * nc
    n_kf = min((BOUND - 1) // per_kf, int(1.3 * PASS / (reps * n1)) + 1)
    assert n_kf * per_kf > PASS
    _fits(n_kf * per_kf * (33 + QUERY_BYTES + 12), f"{n_kf * per_kf} Fuse entries")
    kstar = PASS // per_kf + 1                    # its entries all lie past entry 2^21
    assert kstar < n_kf
    rigs = fuse_targets(api, cams, s["sc"], n_kf, 21)
    rigs[kstar] = s["sc"]["rig"]
    pts = np.tile(s["points"][base], reps).astype(np.int32)
    t0 = time.time()
    hits, n, status, _ = fuse_device(api, m, [KF] * n_kf, rigs, [None] * n_kf, pts, dm, cap, "parts", variant, Scw=s["Scw"])
    t_batch = time.time() - t0
    assert status == api.MCS_OK
    e = _entries(hits, n_q, nc, cap)
    if not np.all(np.diff(e) > 0):
        o = int(np.argmin(np.diff(e) > 0))
        pytest.fail(f"hit rows out of maker order: row {o + 1} of {n} holds entry {e[o + 1]} (block {e[o + 1] // TILE}, scan pass "
                    f"{e[o + 1] // PASS + 1}) after entry {e[o]}; the fill places every row after the rows of all earlier entries")
    assert n > PASS, f"{n} hits: the hit scan does not reach past block 1024"
    step = (PASS - 1) // per_kf
    sep, total = [], 0
    for a in range(0, n_kf, step):
        b = min(n_kf, a + step)
        h, nn, st, _ = fuse_device(api, m, [KF] * (b - a), rigs[a:b], [None] * (b - a), pts, dm, cap, "parts", variant, Scw=s["Scw"])
        assert st == api.MCS_OK
        h = h.copy()
        h[:, 0] += a
        sep.append(h)
        total += nn
    sep = np.concatenate(sep)
    print(f"\nFuse variant {variant}: {n_kf} key frames x {n_q} queries x {nc} cameras = {n_kf * per_kf} entries, {n} hits; "
          f"one call {t_batch:.1f} s, {time.time() - t0:.1f} s with the split calls")
    assert n == total == len(sep), f"n_hits {n}, the split calls' hits {total}"
    assert np.array_equal(hits, sep)
    # the key frame past the boundary, replayed, == the host Fuse on the same queries
    sk = dict(s, points=pts)
    if variant == 0:
        sk["cur"] = dict(s["cur"], rays=np.tile(s["cur"]["rays"][base], (reps, 1)))
    hn, hops, hmp = host_fuse(api, m, KF, sk, variant)
    dn, dops, dmp = fuse_replay(m, KF, sk, variant, hits, cap, k=kstar)
    assert dn == hn and np.array_equal(dops, hops) and np.array_equal(dmp, hmp) and len(hops) > 50
    # and that key frame's hits == the single-key-frame call's, replica by replica
    mine = hits[hits[:, 0] == kstar][:, 1:]
    one = np.stack([np.searchsorted(base, h1[:, 1]), h1[:, 2]], 1)
    assert np.array_equal(mine, np.concatenate([one + [r * len(base), 0] for r in range(reps)]))


# ---- SearchByProjection(KF, Scw) ----------------------------------------------------------------------------------------------
SCW_CAMS, SCW_KEYS = 40, 60_000         # 2.4 M keypoints: entry i of vpPoints is searched in the camera of contiguous keypoint i


def _scw_scene(api, cams, seed=7):
    """A key frame of SCW_CAMS copies of one camera at the origin (Scw = identity), SCW_KEYS keypoints each, and n_q = every
    keypoint's entry.  Most entries are NULL; the real ones are a dense run around entry 2^21 and a sparse spread over the rest
    (camera 0 densest).  A real entry i is a point on the ray of a pixel in the mirror mask of keypoint i's camera, 2 to 8 m
    away, with keypoint i next to that pixel on octave 0 and the point's descriptor that keypoint's with a few bits flipped; its
    distance range puts it on level 1.  The other keypoints lie anywhere on octave 7, outside every window's levels.  Some real
    points are bad, some already found (vpMatched holds them).  The reference reads candidate descriptors at the contiguous id
    as a row of the query's camera, so only camera 0's queries can match; past entry 2^21 the queries are built, searched and
    matched against nothing, and a misplaced one shows as a camera 0 query overwritten or as a wrong query count."""
    rng = np.random.default_rng(seed)
    cam = cams[0]
    nc, nk = SCW_CAMS, SCW_KEYS
    n = nc * nk
    rig = api.Rig([cam] * nc)
    mask = rig.masks[0]
    keys = np.zeros(n, api.KEYPOINT_DTYPE)
    keys["x"] = rng.uniform(0, cam["width"] - 1, n)
    keys["y"] = rng.uniform(0, cam["height"] - 1, n)
    keys["octave"] = 7
    key_cam = np.repeat(np.arange(nc, dtype=np.int32), nk)
    kdesc = rng.integers(0, 256, (n, DIM), dtype=np.uint8)
    real = rng.random(n) < np.where(key_cam == 0, 0.3, 0.01)
    real[PASS - 3 * TILE:PASS + 3 * TILE] = rng.random(6 * TILE) < 0.9
    real[0] = True
    idx = np.flatnonzero(real)
    vy, vx = np.nonzero(mask[8:-8, 8:-8])
    pick = rng.integers(0, len(vx), len(idx))
    u, v = vx[pick] + 8 + rng.uniform(-0.5, 0.5, len(idx)), vy[pick] + 8 + rng.uniform(-0.5, 0.5, len(idx))
    world = np.zeros((len(idx), 3))
    for k, (uu, vv) in enumerate(zip(u, v)):
        r = np.asarray(api.img_to_world(cam, float(uu), float(vv)))
        world[k] = r / np.linalg.norm(r) * rng.uniform(2.0, 8.0)
    keys["x"][idx] = u + rng.uniform(-1.5, 1.5, len(idx))
    keys["y"][idx] = v + rng.uniform(-1.5, 1.5, len(idx))
    keys["octave"][idx] = 0
    d = np.linalg.norm(world, axis=1)
    points = np.full(n, -1, np.int32)
    points[idx] = np.arange(len(idx), dtype=np.int32)
    desc = kdesc[idx] ^ _noise(rng, len(idx), 0.03)
    bad = (rng.random(len(idx)) < 0.05).astype(np.uint8)
    matched = np.full(n, -1, np.int32)
    found = rng.choice(np.flatnonzero(key_cam[idx] == 0), 300, replace=False)
    matched[rng.choice(np.flatnonzero(~real[:nk]), 300, replace=False)] = found      # free keypoints of camera 0 hold them
    sf = np.cumprod([1.0] + [1.2000000476837158] * 7)
    KF = api.Frame(keys, key_cam, kdesc, None, [(cam["width"], cam["height"])] * nc, sf)
    return dict(KF=KF, rig=rig, Scw=np.eye(4), world=world, min_d=d / 1.1, max_d=d * 2.0, desc=desc,
                dmask=np.zeros_like(desc), bad=bad, points=points, matched=matched)


@pytest.mark.gpu
def test_search_by_projection_scw_past_one_scan_pass(api, cams):
    """mcs_search_by_projection_scw_device with n_q = 2.4 M entries (1172 blocks) == its host mirror, bit for bit, and its query
    count == the model's over the entries the host projection passes"""
    n = SCW_CAMS * SCW_KEYS
    _fits(n * (QUERY_BYTES + 4 * 8 + 2 * 28 + 2 * DIM + 16), f"{n} Scw entries")
    t0 = time.time()
    s = _scw_scene(api, cams)
    m = api.cORBmatcher(0.6, False, DIM, False)
    hn, hm = host_scw(m, s)
    # the entries the host projection passes: not NULL, bad or already found, in the mask and in the distance range
    live = np.flatnonzero(s["points"] >= 0)
    p = s["points"][live]
    keep = (s["bad"][p] == 0) & ~np.isin(p, s["matched"][s["matched"] >= 0])
    live, p = live[keep], p[keep]
    _, ok, _ = api._project(api._sim3_rig(s["rig"], s["Scw"]), s["KF"].scale_factors, s["world"], s["min_d"], s["max_d"], p,
                            s["KF"].key_cam[live][:, None], float_dist=False)
    valid = np.zeros(n, bool)
    valid[live[ok[:, 0] != 0]] = True
    counts, offsets = scan_model(valid)
    assert counts[1024:].sum() > TILE and counts[1022:1026].min() > 0.5 * TILE
    dn, st, dmatched, diag = device_scw(api, m, s, SCW_KEYS + 3, "parts")
    _report("SearchByProjection(KF, Scw)", n, int(diag[2]), diag, time.time() - t0)
    assert st == api.MCS_OK
    assert diag[2] == offsets[-1], _query_count_message(diag[2], offsets)
    assert dn == hn > 1000 and np.array_equal(dmatched, hm)
