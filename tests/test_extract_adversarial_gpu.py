"""GPU parity of the front of the extractor (K1 pyr_fast_kernel, K2 octree_kernel) on adversarial images: dense dot lattices that
put strict per-cell maxima on both sides of FAST cell boundaries, lattices of equal responses, contrasts at the FAST threshold,
saturated patterns, symmetric blobs and striped masks.  Natural-looking frames never come near these cases: corners there are
sparse, responses spread out, and no 64-pixel tile row holds more than a handful of maxima.

Every case compares every stage with the CPU oracle bit for bit (levels, blurred levels, masks, raw corners, keypoints including the
IC angle bits, descriptors and descriptor masks); extract_batch raises on any capacity status of the kernels.  Each family also
checks on the oracle's output that its images reach the edge they are built for, so that a change of a generator cannot quietly
turn a case into an easy one."""
import numpy as np
import pytest

from extract_cases import axis_cells, boundary_lattice, boundary_lattice_target, cams_for, fullest_segment, run_batch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", ["orb", "dbrief", "mdbrief"])
@pytest.mark.parametrize("nlevels", [1, 8])
@pytest.mark.parametrize("w,h", [(754, 480), (1280, 720), (764, 480), (641, 479)])
def test_dense_lattice_cell_boundaries(api, oa, cams, w, h, nlevels, mode):
    cs = cams_for(cams, w, h)
    imgs = np.stack([boundary_lattice(w, h, v) for v in range(3)])
    masks = np.stack([np.ones((h, w), np.uint8)] * 3)
    res = run_batch(api, oa, imgs, masks, cs, [0, 1, 2], 2000 if w > 1000 else 1000, mode, nlevels=nlevels)
    for i, (_, raw) in enumerate(res):
        assert fullest_segment(raw) == boundary_lattice_target(w), f"image {i}: fullest warp segment before a non-empty one"


def test_dense_lattice_device_unaligned(api, oa, cams):
    """the same lattices from a tight 754-byte-stride device batch: K1 stages such rows byte by byte instead of by TMA"""
    import torch
    w, h = 754, 480
    cs = cams_for(cams, w, h)
    imgs = np.stack([boundary_lattice(w, h, v) for v in range(3)])
    masks = np.stack([np.ones((h, w), np.uint8)] * 3)
    ex = api.mdBRIEFextractorOct(nfeatures=1000, do_dBrief=True, learnMasks=True)
    oe = oa.OracleExtractor(nfeatures=1000, do_dbrief=True, learn_masks=True)
    dev = torch.device("cuda", 0)
    tight = torch.from_numpy(imgs).to(dev)
    st = torch.cuda.Stream(dev)
    with torch.cuda.stream(st):
        out = ex.extract_batch_device(tight, masks, cs, [0, 1, 2], stream=st)
    ex.check_status(st)
    counts = out["counts"].cpu().numpy()
    kps = out["kps"].cpu().numpy().view(api.KEYPOINT_DTYPE).reshape(3, -1)
    for i in range(3):
        ok, od, om = oe.extract(imgs[i], masks[i], cs[i])
        assert fullest_segment(oe.debug_read(0, 3)) == boundary_lattice_target(w)
        assert np.array_equal(ex.debug_read(0, 3, i), oe.debug_read(0, 3)), f"image {i}: raw corners level 0"
        n = counts[i]
        assert n == len(ok) and kps[i, :n].tobytes() == ok.tobytes()
        assert np.array_equal(out["desc"][i, :n].cpu().numpy(), od)
        assert np.array_equal(out["dmask"][i, :n].cpu().numpy(), om)


# ---- 2. all-equal responses ------------------------------------------------------------------------------------------------------
def dot_lattice(w, h, period, ox, oy, value=255, background=0):
    img = np.full((h, w), background, np.uint8)
    img[oy::period, ox::period] = value
    return img


@pytest.mark.parametrize("nf", [300, 1000, 2000])
def test_equal_responses(api, oa, cams, nf):
    """Isolated identical dots: every dot is a corner of score 254.  Periods 4, 5 and 7 do not divide the tile or cell sizes, so the
    lattice phase differs from tile to tile and cell to cell; every "first maximum in reference order" choice of K2 and every
    "largest first, later created first" order of its pass B is decided by a tie."""
    w, h = 754, 480
    cs = cams_for(cams, w, h)
    imgs = np.stack([dot_lattice(w, h, 4, 1, 2), dot_lattice(w, h, 5, 3, 0), dot_lattice(w, h, 7, 2, 5)])
    masks = np.stack([np.ones((h, w), np.uint8)] * 3)
    res = run_batch(api, oa, imgs, masks, cs, [0, 1, 2], nf, "orb")
    for ok, raw in res:
        assert len(raw) > 2 * nf and np.all(raw[:, 2] == 254)
        assert np.all(ok["response"][ok["octave"] == 0] == 254)


# ---- 3. FAST threshold edge ------------------------------------------------------------------------------------------------------
def threshold_dots(w, h, th, spacing=9):
    """Bright and dark dots on mid-grey whose contrast cycles through th, th + 1, th + 2 -> (image, {(x, y): contrast})"""
    img = np.full((h, w), 128, np.uint8)
    dots = {}
    k = 0
    for y in range(4, h - 4, spacing):
        for x in range(4 + (y // spacing) % 3, w - 4, spacing):
            c = th + k % 3
            img[y, x] = 128 + c if (k // 3) % 2 == 0 else 128 - c
            dots[(x, y)] = c
            k += 1
    return img, dots


@pytest.mark.parametrize("th", [20, 5])
def test_fast_threshold_edge(api, oa, cams, th):
    """A pixel is a corner iff its FAST margin exceeds the threshold, with score = margin - 1: dots of contrast th never appear,
    th + 1 appear with response th, th + 2 with response th + 1"""
    w, h = 754, 480
    cs = cams_for(cams, w, h)
    img, dots = threshold_dots(w, h, th)
    imgs = np.stack([img, img[:, ::-1], 255 - img])
    masks = np.stack([np.ones((h, w), np.uint8)] * 3)
    res = run_batch(api, oa, imgs, masks, cs, [0, 1, 2], 1000, "dbrief", fastThreshold=th)
    cx, _ = axis_cells(w, True)
    cy, _ = axis_cells(h, False)
    want = {(x, y, c - 1) for (x, y), c in dots.items() if c > th and cx[x] >= 0 and cy[y] >= 0}
    got = {tuple(int(v) for v in r) for r in res[0][1]}
    assert got == want
    assert {th, th + 1} <= {int(r[2]) for r in res[0][1]}


# ---- 4. saturation ---------------------------------------------------------------------------------------------------------------
def saturated_images(w, h):
    """0/255 checkerboards of square sizes 1..6 and uniform binary noise: FAST margins of 255, 5x5 blur sums of 6375, saturated
    bilinear resizes on every level"""
    y, x = np.mgrid[0:h, 0:w]
    out = [(((x // s) + (y // s)) % 2 * 255).astype(np.uint8) for s in range(1, 7)]
    out.append((np.random.default_rng(7).integers(0, 2, (h, w)) * 255).astype(np.uint8))
    return np.stack(out)


@pytest.mark.parametrize("w,h", [(754, 480), (641, 479)])
def test_saturated_patterns(api, oa, cams, w, h):
    cs = cams_for(cams, w, h)
    imgs = saturated_images(w, h)
    masks = np.stack([np.ones((h, w), np.uint8)] * 3)
    res = run_batch(api, oa, imgs, masks, cs, [i % 3 for i in range(len(imgs))], 1000, "mdbrief")
    assert any(np.any(raw[:, 2] == 254) for _, raw in res)                # margin 255 reached


# ---- 5. symmetric blobs ----------------------------------------------------------------------------------------------------------
BLOBS = [
    [],                                        # lone dot: both moments 0 -> fastAtan2(0, 0)
    [(8, 0, 255)], [(0, 8, 255)], [(-8, 0, 255)], [(0, -8, 255)],              # on an axis: 0, 90, 180, 270 degrees
    [(8, 5, 255), (-8, -5, 255)],              # point-symmetric: both moments 0
    [(6, 6, 255), (6, -6, 255)],               # symmetric about the x axis: m01 = 0
    [(6, 6, 255), (-6, 6, 255)],               # symmetric about the y axis: m10 = 0
    [(8, 0, 255), (0, -1, 1)],                 # just below 360
    [(8, 0, 255), (0, 1, 1)],                  # just above 0
    [(6, 6, 255)],                             # diagonal
]


def blob_image(w, h, shift=0, spacing=37):
    img = np.zeros((h, w), np.uint8)
    k = shift
    for y in range(30, h - 30, spacing):
        for x in range(30, w - 30, spacing):
            img[y, x] = 255
            for dx, dy, v in BLOBS[k % len(BLOBS)]:
                img[y + dy, x + dx] = v
            k += 1
    return img


@pytest.mark.parametrize("mode", ["orb", "mdbrief"])
def test_symmetric_blobs(api, oa, cams, mode):
    """IC moments exactly zero or on an axis: fastAtan2(0, 0), angles of exactly 0 / 90 / 180 / 270, wrap-around near 360, and the
    mdBRIEF +-20 degree mask patterns around them"""
    w, h = 754, 480
    cs = cams_for(cams, w, h)
    imgs = np.stack([blob_image(w, h, s) for s in range(3)])
    masks = np.stack([np.ones((h, w), np.uint8)] * 3)
    res = run_batch(api, oa, imgs, masks, cs, [0, 1, 2], 3000, mode)
    ang =np.concatenate([ok["angle"][ok["octave"] == 0] for ok, _ in res])
    for a in (0.0, 90.0, 180.0, 270.0):
        assert np.any(ang == np.float32(a)), f"no keypoint at exactly {a} degrees"
    assert np.any(ang > 359.0) and np.any((ang > 0.0) & (ang < 1.0))


# ---- 6. mask stripes -------------------------------------------------------------------------------------------------------------
def stripe_masks(w, h):
    """1-pixel alternating columns, alternating rows, and holes on the cell boundaries: every K1 tile lies on the mask border"""
    y, x = np.mgrid[0:h, 0:w]
    cols = ((x % 2) * 255).astype(np.uint8)
    rows = ((y % 2 == 0) * 255).astype(np.uint8)
    cx, _ = axis_cells(w, True)
    cy, _ = axis_cells(h, False)
    holes = np.full((h, w), 255, np.uint8)
    bx = np.nonzero((cx[1:] != cx[:-1]) & (cx[1:] >= 0) & (cx[:-1] >= 0))[0]      # last column of a cell
    by = np.nonzero((cy[1:] != cy[:-1]) & (cy[1:] >= 0) & (cy[:-1] >= 0))[0]
    holes[1::2, :][:, bx] = 0
    holes[::2, :][:, bx + 1] = 0
    holes[by, :] = np.where(x[0] % 3 == 0, 0, 255)
    for yy in by:
        for xx in bx:
            holes[yy - 2:yy + 3, xx - 2:xx + 3] = 0
    return np.stack([cols, rows, holes])


def test_mask_stripes(api, oa, cams):
    w, h = 754, 480
    cs = cams_for(cams, w, h)
    imgs = np.stack([boundary_lattice(w, h, v) for v in (0, 1, 2, 0, 1, 2)])
    masks = stripe_masks(w, h)
    res = run_batch(api, oa, imgs, masks, cs, [0, 1, 2, 1, 2, 0], 1000, "mdbrief")
    for i, (_, raw) in enumerate(res):                                # every mask keeps some corners and drops others
        assert 0 < len(raw) < np.count_nonzero(imgs[i]) * 0.95, f"image {i}: {len(raw)} corners"
