"""stage_probe.py -- K1/K2/K3 stage times of one extractor batch (CUDA events inside the library).
python tools/stage_probe.py [frames] [tier_stats]"""
import pathlib
import sys

import numpy as np
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import multicol_slam_b200.api as api  # noqa: E402
from multicol_slam_b200 import rig, synth  # noqa: E402

F = int(sys.argv[1]) if len(sys.argv) > 1 else 64
cams = synth.lafida_cams()
masks = np.stack([synth.mirror_mask(c) for c in cams])
imgs = np.ascontiguousarray(np.stack([synth.texture_stream(cams[c], F, seed=1000 + c) for c in range(3)], axis=1)).reshape(F * 3, 480, 754)
dev = torch.device("cuda", 0)
pitched = torch.zeros((F * 3, 480, 768), dtype=torch.uint8, device=dev)
pitched[:, :, :754] = torch.from_numpy(imgs).to(dev)
ex = api.mdBRIEFextractorOct(nfeatures=2000, do_dBrief=True, learnMasks=True)
packed = torch.zeros(rig.packed_layout(F * 3, ex.capacity, 32)[1], dtype=torch.uint8, device=dev)
coi = np.tile(np.arange(3, dtype=np.int32), F)
st = torch.cuda.Stream(dev)
with torch.cuda.stream(st):
    for _ in range(3):
        ex.extract_batch_packed_device(pitched, masks, cams, coi, packed, stream=st, width=754)
    torch.cuda.synchronize()
    ex.set_profiling(True)
    t = np.zeros(3)
    for _ in range(5):
        ex.extract_batch_packed_device(pitched, masks, cams, coi, packed, stream=st, width=754)
        torch.cuda.synchronize()
        t += np.array(ex.get_timings())
    ex.set_profiling(False)
    if len(sys.argv) > 2:
        ex.tier_stats(True)
        ex.extract_batch_packed_device(pitched, masks, cams, coi, packed, stream=st, width=754)
        torch.cuda.synchronize()
        ts = ex.tier_stats(False)
        print("tiers", ts.tolist(), (ts / ts.sum()).round(4).tolist())
print(f"{F * 3} images: K1 {t[0] / 5:.3f} ms  K2 {t[1] / 5:.3f} ms  K3 {t[2] / 5:.3f} ms")
