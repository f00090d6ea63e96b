"""GPU: every argument refusal of the six extract entry points and of the three stream matchers -- its code and its message -- on a
live extractor, and what a refused call leaves behind: the next valid call returns what a fresh extractor returns, and the cached
per-frame graph is still replayed.  The null-extractor refusals need no device: tests/test_extract_arguments_cpu.py."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NULL_ARG = "null argument"
GEOMETRY = "bad image geometry"
CAPACITY = "capacity below mcs_extractor_info.capacity"
NO_DMASK = "dmask buffer required when learn_masks is set"
N_CAMS = "n_cams must be in [1,64]"
COI = "cam_of_image out of range"


def _refused(api, rc, code, msg):
    assert (rc, api.lib().mcs_last_error().decode()) == (code, msg)


class Scene:
    """one extractor that has cached its per-frame graph, the inputs of that call, and what a fresh extractor returns for them"""

    def __init__(self, api, cams):
        from multicol_slam_b200 import synth
        make = lambda: api.mdBRIEFextractorOct(nfeatures=400, do_dBrief=True, learnMasks=True)  # noqa: E731
        self.api, self.cams = api, cams
        self.masks = np.stack([api.mirror_mask(c) for c in cams])
        self.H, self.W = self.masks.shape[1:]
        self.images = np.stack([synth.frame(cams[i % len(cams)], 50 + i) for i in range(17)])
        self.coi = np.arange(17, dtype=np.int32) % len(cams)
        self.ocs = (api.Ocam * len(cams))(*[api.as_ocam(c) for c in cams])
        self.ref = make().extract_batch(self.images[:2], self.masks, cams, self.coi[:2])
        self.ex = make()
        self.cap = self.ex.capacity
        # the largest buffers first (17 images: the eager path), so that no refused call below has to grow one
        self.ex.extract_batch(self.images, self.masks, cams, self.coi)
        assert self._valid() == 0             # records the graph
        self.replays = self.ex.graph_replays()

    def _valid(self):
        got = self.ex.extract_batch(self.images[:2], self.masks, self.cams, self.coi[:2])
        for a, b in zip(got, self.ref):
            assert a.tobytes() == b.tobytes()
        return self.ex.graph_replays()

    def rerecord(self):
        """the per-frame call after a valid call of another entry point, which changed the shared inputs: recorded anew"""
        assert self._valid() == self.replays

    def still_valid(self):
        """the next per-frame call returns the fresh extractor's features, replayed from the cached graph"""
        n = self._valid()
        assert n == self.replays + 1
        self.replays = n


@pytest.fixture(scope="module")
def scene(api, cams):
    return Scene(api, cams)


def _outputs(n, cap, ds=32, K=None):
    from multicol_slam_b200.ctypes_defs import KEYPOINT_DTYPE
    out = dict(kps=np.zeros((n, cap), KEYPOINT_DTYPE), desc=np.zeros((n, cap, ds), np.uint8), dmask=np.zeros((n, cap, ds), np.uint8),
               counts=np.zeros(n, np.int32))
    if K:
        out.update(idx=np.zeros((n, cap, K), np.int32), dist=np.zeros((n, cap, K), np.int32), m12=np.zeros((n, cap), np.int32),
                   nm=np.zeros(n, np.int32), redo=np.zeros(n, np.int32))
    return out


def test_extract_refusals(api, scene):
    """mcs_extract: a missing mask or camera model; the batch checks it reaches with one image of camera 0"""
    s, p = scene, api._p
    o = _outputs(1, s.cap)
    img, n = s.images[0], C.c_int32(0)

    def call(image=p(img), w=s.W, h=s.H, stride=s.W, mask=p(s.masks[0]), cam=C.byref(s.ocs[0]), dmask=p(o["dmask"]), cap=s.cap,
             n_out=C.byref(n)):
        return api.lib().mcs_extract(s.ex._h, image, w, h, stride, mask, s.W, cam, p(o["kps"]), p(o["desc"]), dmask, cap, n_out)
    _refused(api, call(n_out=None), api.MCS_ERR_INVALID, NULL_ARG)
    assert call(image=None) == api.MCS_OK                     # an empty image: silent return
    s.still_valid()
    for kw in (dict(mask=None), dict(cam=None)):
        _refused(api, call(**kw), api.MCS_ERR_INVALID, "a mask and a camera model are mandatory (ref :913-917 throws on an empty mask)")
        s.still_valid()
    for kw in (dict(h=0), dict(stride=s.W - 1)):
        _refused(api, call(**kw), api.MCS_ERR_INVALID, GEOMETRY)
        s.still_valid()
    # a width of 0 (mask_stride != width) repacks the mask into an empty buffer, which the batch call refuses as missing
    _refused(api, call(w=0), api.MCS_ERR_INVALID, NULL_ARG)
    s.still_valid()
    _refused(api, call(cap=s.cap - 1), api.MCS_ERR_CAPACITY, CAPACITY)
    s.still_valid()
    _refused(api, call(dmask=None), api.MCS_ERR_INVALID, NO_DMASK)
    s.still_valid()


@pytest.mark.parametrize("n", [2, 17], ids=["graph", "eager"])
def test_extract_batch_refusals(api, scene, n):
    """mcs_extract_batch on its per-frame (graph) path and on its eager path"""
    s, p = scene, api._p
    o = _outputs(n, s.cap)

    def call(n_images=n, w=s.W, h=s.H, stride=s.W, n_cams=len(s.cams), coi=None, cap=s.cap, null=()):
        args = dict(images=p(s.images[:n]), masks=p(s.masks), cams=s.ocs, coi=p(s.coi[:n] if coi is None else coi), kps=p(o["kps"]),
                    desc=p(o["desc"]), dmask=p(o["dmask"]), counts=p(o["counts"]))
        a = {k: None if k in null else v for k, v in args.items()}
        return api.lib().mcs_extract_batch(s.ex._h, n_images, a["images"], w, h, stride, a["masks"], a["cams"], n_cams, a["coi"], a["kps"],
                                           a["desc"], a["dmask"], a["counts"], cap)
    for name in ("images", "masks", "cams", "coi", "kps", "desc", "counts"):
        _refused(api, call(null=(name,)), api.MCS_ERR_INVALID, NULL_ARG)
        s.still_valid()
    for kw in (dict(n_images=0), dict(w=0), dict(h=0), dict(stride=s.W - 1)):
        _refused(api, call(**kw), api.MCS_ERR_INVALID, GEOMETRY)
        s.still_valid()
    _refused(api, call(cap=s.cap - 1), api.MCS_ERR_CAPACITY, CAPACITY)
    s.still_valid()
    _refused(api, call(null=("dmask",)), api.MCS_ERR_INVALID, NO_DMASK)
    s.still_valid()
    for nc in (0, 65):
        _refused(api, call(n_cams=nc), api.MCS_ERR_INVALID, N_CAMS)
        s.still_valid()
    for bad in (-1, len(s.cams)):
        coi = s.coi[:n].copy()
        coi[n - 1] = bad
        _refused(api, call(coi=coi), api.MCS_ERR_INVALID, COI)
        s.still_valid()


@pytest.mark.parametrize("packed", [False, True], ids=["batch_device", "batch_packed_device"])
def test_extract_batch_device_refusals(api, scene, packed):
    """mcs_extract_batch_device and mcs_extract_batch_packed_device, on a caller stream and on the extractor's own"""
    import torch
    from multicol_slam_b200 import rig
    s, p, n = scene, api._p, 2
    dev = torch.device("cuda", 0)
    images_t = torch.from_numpy(s.images[:n]).to(dev)
    buf = torch.zeros(rig.packed_layout(n, s.cap, 32)[1], dtype=torch.uint8, device=dev)
    v = s.ex.packed_views(buf, n)
    stream = torch.cuda.Stream(dev)

    def call(n_images=n, w=s.W, h=s.H, stride=s.W, n_cams=len(s.cams), coi=None, cap=s.cap, null=(), st=None):
        args = dict(images=api._dptr(images_t), masks=p(s.masks), cams=s.ocs, coi=p(s.coi[:n] if coi is None else coi), packed=api._dptr(buf),
                    **{k: api._dptr(v[k]) for k in ("kps", "desc", "dmask", "counts")})
        a = {k: None if k in null else x for k, x in args.items()}
        if packed:
            return api.lib().mcs_extract_batch_packed_device(s.ex._h, n_images, a["images"], w, h, stride, a["masks"], a["cams"], n_cams, a["coi"],
                                                             a["packed"], cap, st)
        return api.lib().mcs_extract_batch_device(s.ex._h, n_images, a["images"], w, h, stride, a["masks"], a["cams"], n_cams, a["coi"],
                                                  a["kps"], a["desc"], a["dmask"], a["counts"], cap, st)
    nulls = ("packed", "images", "masks", "cams", "coi") if packed else ("images", "masks", "cams", "coi", "kps", "desc", "counts")
    for st in (None, C.c_void_p(stream.cuda_stream)):
        for name in nulls:
            _refused(api, call(null=(name,), st=st), api.MCS_ERR_INVALID, NULL_ARG)
            s.still_valid()
        for kw in (dict(n_images=0), dict(w=0), dict(h=0), dict(stride=s.W - 1)):
            _refused(api, call(st=st, **kw), api.MCS_ERR_INVALID, GEOMETRY)
            s.still_valid()
        _refused(api, call(cap=s.cap - 1, st=st), api.MCS_ERR_CAPACITY, CAPACITY)
        s.still_valid()
        if not packed:                          # the packed buffer always has a mask section
            _refused(api, call(null=("dmask",), st=st), api.MCS_ERR_INVALID, NO_DMASK)
            s.still_valid()
        for nc in (0, 65):
            _refused(api, call(n_cams=nc, st=st), api.MCS_ERR_INVALID, N_CAMS)
            s.still_valid()
        for bad in (-1, len(s.cams)):
            _refused(api, call(coi=np.array([0, bad], np.int32), st=st), api.MCS_ERR_INVALID, COI)
            s.still_valid()
    torch.cuda.synchronize(dev)
    # the device path after all refusals: the fresh extractor's features
    assert call() == api.MCS_OK
    torch.cuda.synchronize(dev)
    kps, desc, dmask, counts = s.ref
    assert np.array_equal(v["counts"].cpu().numpy(), counts)
    for i in range(n):
        c = counts[i]
        assert v["kps"][i, :c].cpu().numpy().tobytes() == kps[i, :c].tobytes()
        assert np.array_equal(v["desc"][i, :c].cpu().numpy(), desc[i, :c]) and np.array_equal(v["dmask"][i, :c].cpu().numpy(), dmask[i, :c])
    s.rerecord()


def _stream_call(api, s, ex, o, packed_t=None, n_frames=2, n_cams=None, w=None, h=None, stride=None, cap=None, K=2, null=(), greedy=False,
                 images=None, masks=None, ocs=None):
    p = api._p
    n_cams = len(s.cams) if n_cams is None else n_cams
    args = dict(images=p(s.images[:6] if images is None else images), masks=p(s.masks if masks is None else masks),
                cams=s.ocs if ocs is None else ocs, **{k: p(o[k]) for k in o})
    a = {k: None if k in null else x for k, x in args.items()}
    geo = (s.W if w is None else w, s.H if h is None else h, s.W if stride is None else stride)
    head = (ex._h, n_frames, n_cams, a["images"], *geo, a["masks"], a["cams"], a["kps"], a["desc"], a["dmask"], a["counts"],
            s.cap if cap is None else cap, K, a["idx"], a["dist"])
    if packed_t is None and not greedy:
        return api.lib().mcs_extract_match_stream(*head)
    return api.lib().mcs_extract_match_stream_packed(*head, api._dptr(packed_t), 64 if greedy else 0, C.c_double(0.75 if greedy else 0.0),
                                                     a["m12"] if greedy else None, a["nm"] if greedy else None, a["redo"] if greedy else None)


@pytest.mark.parametrize("form", ["plain", "packed", "greedy"])
def test_extract_match_stream_refusals(api, scene, form):
    """mcs_extract_match_stream and mcs_extract_match_stream_packed (plain, packed buffer, greedy acceptance): 2 frames x 3 cameras"""
    import torch
    from multicol_slam_b200 import rig
    s = scene
    o = _outputs(6, s.cap, K=2)
    packed_t = None
    if form != "plain":
        packed_t = torch.zeros(rig.packed_layout(6, s.cap, 32)[1], dtype=torch.uint8, device=torch.device("cuda", 0))
    call = lambda **kw: _stream_call(api, s, s.ex, o, packed_t=packed_t, greedy=form == "greedy", **kw)  # noqa: E731
    for name in ("images", "masks", "cams", "kps", "desc", "counts", "idx", "dist"):
        _refused(api, call(null=(name,)), api.MCS_ERR_INVALID, NULL_ARG)
        s.still_valid()
    for kw in (dict(n_frames=0), dict(n_cams=0), dict(w=0), dict(h=0), dict(stride=s.W - 1)):
        _refused(api, call(**kw), api.MCS_ERR_INVALID, GEOMETRY)
        s.still_valid()
    _refused(api, call(cap=s.cap - 1), api.MCS_ERR_CAPACITY, CAPACITY)
    s.still_valid()
    _refused(api, call(null=("dmask",)), api.MCS_ERR_INVALID, NO_DMASK)
    s.still_valid()
    for K in (0, 9):
        _refused(api, call(K=K), api.MCS_ERR_INVALID, "K must be 1..8")
        s.still_valid()
    if form == "greedy":
        for name in ("nm", "redo"):
            _refused(api, call(null=(name,)), api.MCS_ERR_INVALID, "the greedy acceptance needs all three outputs")
            s.still_valid()
    # a valid stream call returns the fresh extractor's features for the first frame
    assert call() == api.MCS_OK
    kps, desc, dmask, counts = s.ref
    assert np.array_equal(o["counts"][:2], counts) and o["kps"][:2].tobytes() == kps.tobytes()
    s.rerecord()


def test_extract_match_stream_camera_count(api, scene):
    """n_cams above 64 in the stream calls: refused before anything is uploaded; the extractor then extracts as a fresh one.  One
    frame of 65 cameras, on an extractor of its own (the refusal sits after the per-call inputs are read)"""
    s = scene
    ex = api.mdBRIEFextractorOct(nfeatures=400, do_dBrief=True, learnMasks=True)
    n = 65
    images = np.stack([s.images[i % 3] for i in range(n)])
    masks = np.stack([s.masks[i % 3] for i in range(n)])
    ocs = (api.Ocam * n)(*[s.ocs[i % 3] for i in range(n)])
    o = _outputs(n, s.cap, K=2)
    _refused(api, _stream_call(api, s, ex, o, n_frames=1, n_cams=n, images=images, masks=masks, ocs=ocs), api.MCS_ERR_INVALID, N_CAMS)
    got = ex.extract_batch(s.images[:2], s.masks, s.cams, s.coi[:2])
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, s.ref))


def test_match_stream_refusals(api):
    """mcs_match_stream_device, mcs_match_stream_greedy_device and mcs_match_stream_replay_device: every refusal, then one valid
    call of each that gives what it gave before the refusals"""
    import torch
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(3)
    F, Cn, cap, dim, K = 2, 3, 64, 32, 2
    desc = torch.randint(0, 256, (F * Cn, cap, dim), dtype=torch.uint8, generator=g).to(dev)
    dmask = torch.randint(0, 256, (F * Cn, cap, dim), dtype=torch.uint8, generator=g).to(dev)
    counts = torch.full((F * Cn,), cap, dtype=torch.int32, device=dev)
    idx, dist = torch.zeros((F * Cn, cap, K), dtype=torch.int32, device=dev), torch.zeros((F * Cn, cap, K), dtype=torch.int32, device=dev)
    m12, nm, redo = (torch.zeros((F * Cn, cap), dtype=torch.int32, device=dev), torch.zeros(F * Cn, dtype=torch.int32, device=dev),
                     torch.zeros(F * Cn, dtype=torch.int32, device=dev))
    d = api._dptr
    L = api.lib()
    bad_sizes = [dict(F=0), dict(Cn=0), dict(cap=0)]

    def lists(F=F, Cn=Cn, cap=cap, dim=dim, K=K, null=()):
        a = {k: None if k in null else d(t) for k, t in dict(desc=desc, counts=counts, idx=idx, dist=dist).items()}
        return L.mcs_match_stream_device(a["desc"], d(dmask), a["counts"], F, Cn, cap, dim, K, a["idx"], a["dist"], None)

    def greedy(F=F, Cn=Cn, cap=cap, dim=dim, null=()):
        a = {k: None if k in null else d(t) for k, t in dict(desc=desc, counts=counts, m12=m12, nm=nm).items()}
        return L.mcs_match_stream_greedy_device(a["desc"], d(dmask), a["counts"], F, Cn, cap, dim, 64, C.c_double(0.75), a["m12"], a["nm"], None)

    def replay(F=F, Cn=Cn, cap=cap, dim=dim, K=K, null=()):
        a = {k: None if k in null else d(t) for k, t in dict(idx=idx, dist=dist, counts=counts, desc=desc, m12=m12, nm=nm, redo=redo).items()}
        return L.mcs_match_stream_replay_device(a["idx"], a["dist"], a["counts"], a["desc"], d(dmask), F, Cn, cap, dim, K, 64, C.c_double(0.75),
                                                a["m12"], a["nm"], a["redo"], None)
    assert lists() == 0 and replay() == 0
    torch.cuda.synchronize(dev)
    ref_lists, ref_replay = (idx.clone(), dist.clone()), (m12.clone(), nm.clone())
    assert greedy() == 0
    torch.cuda.synchronize(dev)
    ref_greedy = (m12.clone(), nm.clone())
    for name in ("desc", "counts", "idx", "dist"):
        _refused(api, lists(null=(name,)), api.MCS_ERR_INVALID, NULL_ARG)
    for kw in bad_sizes + [dict(K=0), dict(K=9)]:
        _refused(api, lists(**kw), api.MCS_ERR_INVALID, "bad sizes (K must be 1..8)")
    for name in ("desc", "counts", "m12", "nm"):
        _refused(api, greedy(null=(name,)), api.MCS_ERR_INVALID, NULL_ARG)
    for kw in bad_sizes + [dict(cap=65536)]:
        _refused(api, greedy(**kw), api.MCS_ERR_INVALID, "bad sizes (capacity must be 1..65535)")
    for name in ("idx", "dist", "counts", "desc", "m12", "nm", "redo"):
        _refused(api, replay(null=(name,)), api.MCS_ERR_INVALID, NULL_ARG)
    for kw in bad_sizes + [dict(cap=65536), dict(K=0), dict(K=9)]:
        _refused(api, replay(**kw), api.MCS_ERR_INVALID, "bad sizes (K must be 1..8)")
    for f in (lists, greedy, replay):
        for dd in (0, 24, 128):
            _refused(api, f(dim=dd), api.MCS_ERR_INVALID, "dim must be 16, 32 or 64")
    assert greedy() == 0
    torch.cuda.synchronize(dev)
    assert torch.equal(m12, ref_greedy[0]) and torch.equal(nm, ref_greedy[1])
    assert lists() == 0 and replay() == 0
    torch.cuda.synchronize(dev)
    assert torch.equal(idx, ref_lists[0]) and torch.equal(dist, ref_lists[1])
    assert torch.equal(m12, ref_replay[0]) and torch.equal(nm, ref_replay[1])
