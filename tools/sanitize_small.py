"""Small end-to-end invocation for compute-sanitizer (racecheck / initcheck / synccheck are slow: one image, few features)."""
import sys, pathlib
ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "oracle"))
import numpy as np
import multicol_slam_b200.api as api
from multicol_slam_b200 import synth
import oracle_api as oa
cams = synth.lafida_cams()
cam = synth.scaled_cam(cams[0], 333, 211)
img, mask = synth.frame(cam, 5), synth.mirror_mask(cam)
ex = api.mdBRIEFextractorOct(nfeatures=300, nlevels=4, do_dBrief=True, learnMasks=True)
k, d, m = ex(img, mask, cam)
ok, od, om = oa.OracleExtractor(nfeatures=300, nlevels=4, do_dbrief=True, learn_masks=True).extract(img, mask, cam)
assert k.tobytes() == ok.tobytes() and np.array_equal(d, od) and np.array_equal(m, om)
idx, dist = api.hamming_topk(d, d[::-1].copy(), 2, m, m[::-1].copy())
F = api.Frame.from_cameras([(k, d, m)], [(333, 211)], [ex.info.scale_factor[l] for l in range(4)])
prev = np.stack([k["x"], k["y"]], 1).astype(np.float64)
n, m12 = api.cORBmatcher(0.9, False, 32, True).SearchForInitialization(F, F, prev, 30)
# relocalisation's bag-of-words step on the device: the frame packed twice (key frame and current frame of one buffer), ComputeBoW
# on each (the segment placement), then the search of the frame against itself (the taken flags inside a warp)
import torch
from multicol_slam_b200 import rig
cap = len(k) + 3
packed = torch.from_numpy(rig.pack([(k, d, m), (k, d, m)], cap, 32)).cuda()
voc = api.ORBVocabulary(np.load(ROOT / "tests" / "golden" / "voc_small_9_6.npz"))
bows = [voc.transform_device((packed, 1, 2, f), 1, cap) for f in range(2)]
bw, bv, (fn, fo, ff) = bows[1].host()
hw, hv, (hn, ho, hf) = voc.transform(d)
assert np.array_equal(bw, hw) and np.array_equal(bv, hv) and np.array_equal(fn, hn) and np.array_equal(fo, ho) and np.array_equal(ff, hf)
mp_t = torch.arange(cap, dtype=torch.int32, device="cuda")
mt = api.cORBmatcher(0.9, False, 32, True)
mmp, msl, nm, st = mt.SearchByBoWDevice([(bows[0], mp_t)], bows[1], cap)
nh, mh = mt.SearchByBoWFrame(d, (hn, ho, hf), d, (hn, ho, hf), m, m)
assert int(st.item()) == 0 and int(nm[0].item()) == nh and np.array_equal(msl[0, :len(k)].cpu().numpy(), mh)
# map initialisation's search on the device: the seed, then the frame against itself from the packed buffer (the walk's shared state)
prev_t = torch.zeros(cap * 2, dtype=torch.float64, device="cuda")
m12_t = torch.full((cap,), -1, dtype=torch.int32, device="cuda")
mt.SearchForInitializationSeedDevice((packed, 1, 2, 0), 1, cap, prev_t)
ni, _ = mt.SearchForInitializationDevice((packed, 1, 2, 0), (packed, 1, 2, 1), cap, [(333, 211)], prev_t, 30, m12_t)
torch.cuda.synchronize()
assert int(ni.item()) == n and np.array_equal(m12_t[:len(k)].cpu().numpy(), m12)
# Fuse on the device: map points on the bearing rays of the frame's keypoints, the frame packed twice as two target key frames
rg = api.Rig([cam])
rays, _, _ = api.frame_prepare(k, np.zeros(len(k), np.int32), [cam])
world = rays * np.linspace(2.0, 4.0, len(k))[:, None]
lo, hi, pts = np.full(len(k), 1.0), np.full(len(k), 8.0), np.arange(len(k), dtype=np.int32)
kf_mp = np.where(np.arange(len(k)) % 3 == 0, (np.arange(len(k)) + 1) % len(k), -1).astype(np.int32)
fn, fops, _ = mt.Fuse(F, rg, kf_mp, pts, world, lo, hi, np.zeros(len(k), np.uint8), np.zeros(len(k), bool), d, m, th=2.5, variant=2,
                      Scw=api.inv_rigid(rg.M_t))
tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
kft = [((packed, 1, 2, f), None, rg.MtMc_inv, rg.M_t[:3, 3]) for f in range(2)]
hits, nh_t, st_t = mt.FuseDevice(kft, tt(pts), cap, [cam], tt(np.stack(rg.masks)), F.scale_factors, tt(world), tt(lo), tt(hi), tt(d), tt(m),
                                 variant=2, th=2.5)
torch.cuda.synchronize()
h = hits[:int(nh_t.item())].cpu().numpy()
gn, gops, _ = mt.FuseReplay(F, rg, kf_mp, pts, h[h[:, 0] == 0][:, 1:], cap, world, lo, hi, np.zeros(len(k), np.uint8), np.zeros(len(k), bool), d, m,
                            th=2.5, variant=2, Scw=api.inv_rigid(rg.M_t))
assert int(st_t.item()) == 0 and gn == fn and np.array_equal(gops, fops) and len(fops) > 0
assert np.array_equal(h[h[:, 0] == 0][:, 1:], h[h[:, 0] == 1][:, 1:])
print("sanitize_small ok", len(k), n, nh, len(fops))
