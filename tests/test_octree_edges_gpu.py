"""GPU parity at DistributeOctTree's edges (tests/golden/ref_octree_*.npz, written from the reference's own extractor): wide images
with small budgets, where the first pass of the octree returns up to 4 nIni keypoints per level whatever the quota; zero quotas;
one-level pyramids at the node-table limit.  Every accepted fixture is compared bit for bit (keypoints including the IC angle bits,
per-level counts, descriptors, descriptor masks, pyramid and mask levels) through mcs_extract, the graph-replayed mcs_extract_batch
and mcs_extract_batch_packed_device, in a multi-camera batch next to another camera's frame (checked against the oracle).  Every
refused fixture is checked as that refusal, made before any kernel writes an output."""
import numpy as np
import pytest
from test_octree_bounds_cpu import FIXTURES, REFUSED, load, zlib_crc

pytestmark = pytest.mark.gpu
KW = {"nfeatures": "nfeatures", "scale_factor": "scaleFactor", "nlevels": "nlevels", "fast_threshold": "fastThreshold",
      "do_dbrief": "do_dBrief", "learn_masks": "learnMasks", "desc_size": "descSize"}
IDS = [p.rsplit("ref_octree_", 1)[1][:-4] for p in FIXTURES]


def extractor(api, kw):
    return api.mdBRIEFextractorOct(**{KW[k]: v for k, v in kw.items()})


def same_keypoints(k, d, m, ek, ed, em, what):
    assert len(k) == len(ek), f"{what}: {len(k)} keypoints, expected {len(ek)}"
    for f in ("x", "y", "size", "response", "octave", "class_id"):
        assert np.array_equal(k[f], ek[f]), f"{what}: keypoint field {f}"
    assert np.array_equal(k["angle"].view(np.uint32), ek["angle"].view(np.uint32)), f"{what}: IC angle bits"
    assert np.array_equal(d, ed), f"{what}: descriptor bits"
    assert np.array_equal(m, em), f"{what}: descriptor mask bits"


def check_fixture(g, k, d, m, L, what):
    assert [int((k["octave"] == l).sum()) for l in range(L)] == g["per_level"].tolist(), f"{what}: keypoints per level"
    if "kps" in g.files:
        same_keypoints(k, d, m, g["kps"], g["desc"], g["dmask"], what)
    assert (len(k), zlib_crc(k), zlib_crc(d), zlib_crc(m)) == (int(g["n"]), int(g["kps_crc"]), int(g["desc_crc"]), int(g["dmask_crc"])), what


def second_camera(cam, seed):
    """a Lafida camera of another calibration at the fixture's size, with its mirror mask, and a frame of it: the batch's normal image"""
    from multicol_slam_b200 import synth
    for c in synth.lafida_cams()[::-1]:
        other = dict(c) if (c["width"], c["height"]) == (cam["width"], cam["height"]) else synth.scaled_cam(c, cam["width"], cam["height"])
        if other["u0"] != cam["u0"] or other["pol"] != cam["pol"]:
            return other, synth.frame(other, seed + 1000)
    raise AssertionError("no second calibration")


@pytest.mark.parametrize("path", FIXTURES, ids=IDS)
def test_extract_equals_reference(api, path):
    """mcs_extract (operator()) on one image"""
    name, g, cam, kw, img = load(path)
    ex = extractor(api, kw)
    if name in REFUSED:
        with pytest.raises(api.McsError) as e:
            ex(img, api.mirror_mask(cam), cam)
        assert (e.value.code, api.lib().mcs_last_error().decode()) == (api.MCS_ERR_UNSUPPORTED, REFUSED[name])
        return
    k, d, m = ex(img, api.mirror_mask(cam), cam)
    check_fixture(g, k, d, m, ex.GetLevels(), name)
    for l in range(ex.GetLevels()):
        lvl = ex.debug_read(l, 1) if int(g["per_level"][l]) else ex.debug_read(l, 0)
        assert zlib_crc(lvl) == int(g["level_after_crc"][l]), f"pyramid level {l}"
        assert zlib_crc(ex.debug_read(l, 2)) == int(g["mask_level_crc"][l]), f"mask level {l}"


@pytest.mark.parametrize("path", FIXTURES, ids=IDS)
def test_batches_equal_reference(api, oa, path):
    """[fixture image (camera A), a frame of camera B with its mirror mask, fixture image again] through mcs_extract_batch twice
    (the second call replays the cached CUDA graph) and mcs_extract_batch_packed_device; camera B's frame against the oracle.
    A refused geometry leaves the caller's buffers as they were."""
    import torch
    name, g, cam, kw, img = load(path)
    other, oimg = second_camera(cam, int(g["seed"]))
    imgs = np.stack([img, oimg, img])
    masks = np.stack([api.mirror_mask(cam), api.mirror_mask(other)])
    coi = [0, 1, 0]
    ex = extractor(api, kw)
    dev = torch.device("cuda", 0)
    from multicol_slam_b200 import rig
    packed = torch.full((rig.packed_layout(3, ex.capacity, ex.GetDescriptorSize())[1],), 0xAB, dtype=torch.uint8, device=dev)
    if name in REFUSED:
        for call in (lambda: ex.extract_batch(imgs, masks, [cam, other], coi),
                     lambda: ex.extract_batch_packed_device(torch.from_numpy(imgs).to(dev), masks, [cam, other], coi, packed)):
            with pytest.raises(api.McsError) as e:
                call()
            assert (e.value.code, api.lib().mcs_last_error().decode()) == (api.MCS_ERR_UNSUPPORTED, REFUSED[name])
        torch.cuda.synchronize()
        assert bool((packed == 0xAB).all()), "a refused call wrote into the feature buffer"
        ex.check_status()
        return
    ok, od, om = oa.OracleExtractor(**kw).extract(oimg, masks[1], other)
    L = ex.GetLevels()
    replays = ex.graph_replays()
    for rep in range(2):
        kps, desc, dmask, counts = ex.extract_batch(imgs, masks, [cam, other], coi)
        for i in (0, 2):
            n = counts[i]
            check_fixture(g, kps[i, :n], desc[i, :n], dmask[i, :n], L, f"{name} batch call {rep} image {i}")
        same_keypoints(kps[1, :counts[1]], desc[1, :counts[1]], dmask[1, :counts[1]], ok, od, om, f"{name} batch call {rep} camera B")
    assert ex.graph_replays() == replays + 1
    st = torch.cuda.Stream(dev)
    with torch.cuda.stream(st):
        v = ex.extract_batch_packed_device(torch.from_numpy(imgs).to(dev), masks, [cam, other], coi, packed, stream=st)
    ex.check_status(st)
    counts = v["counts"].cpu().numpy()
    kps = v["kps"].cpu().numpy().view(api.KEYPOINT_DTYPE).reshape(3, -1)
    desc, dmask = v["desc"].cpu().numpy(), v["dmask"].cpu().numpy()
    for i in (0, 2):
        n = counts[i]
        check_fixture(g, kps[i, :n], desc[i, :n], dmask[i, :n], L, f"{name} packed image {i}")
    n = counts[1]
    same_keypoints(kps[1, :n], desc[1, :n], dmask[1, :n], ok, od, om, f"{name} packed camera B")


def test_refusal_leaves_the_extractor_usable(api):
    """an extractor that refused a geometry (too wide for its budget, or a top level without a cell grid) extracts its previous
    geometry as before: a refusal must not leave a half rewritten geometry behind the previous size's cache key"""
    from multicol_slam_b200 import synth
    refused = [load(p) for p in FIXTURES if p.endswith(("_wide_4095x600_orb100.npz", "_wide_2000x250_orb50.npz"))]
    assert len(refused) == 2
    ex = extractor(api, refused[0][3])
    cams = synth.lafida_cams()[:2]
    masks = np.stack([api.mirror_mask(c) for c in cams])
    imgs = np.stack([synth.frame(cams[0], 5), synth.frame(cams[1], 6)])
    first = ex(imgs[0], masks[0], cams[0])
    batch = ex.extract_batch(imgs, masks, cams, [0, 1])
    assert batch[3][0] == len(first[0]) and batch[0][0, :batch[3][0]].tobytes() == first[0].tobytes()
    for _, _, cam, _, img in refused:
        with pytest.raises(api.McsError) as e:
            ex(img, api.mirror_mask(cam), cam)
        assert e.value.code == api.MCS_ERR_UNSUPPORTED
        again = ex(imgs[0], masks[0], cams[0])
        for a, b in zip(first, again):
            assert a.tobytes() == b.tobytes()
        with pytest.raises(api.McsError):
            ex(img, api.mirror_mask(cam), cam)
        for a, b in zip(batch, ex.extract_batch(imgs, masks, cams, [0, 1])):
            assert np.array_equal(a, b)
