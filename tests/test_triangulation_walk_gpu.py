"""GPU: the device SearchForTriangulationRaw (mcs_search_for_triangulation_device) on every planted scene of
tests/triangulation_model.py equals the model -- matches12, nmatches and diag = [queries, rescans] -- and the host route
(SearchForTriangulationRawHost), in the single, parts and joint layouts; slots at or beyond a camera's count stay poisoned.  Classes
1-4 run at 16-, 32- and 64-byte descriptors, masked and not; the rest at 32 bytes, masked.  The CPU tests pin the model to the
sequential loop and to the reference, and show that the scenes tell each rule of the walk apart."""
import numpy as np
import pytest

import triangulation_model as tm
from device_frames import POISON
from device_searches import assert_same_tri, device_tri, host_tri

pytestmark = pytest.mark.gpu
SPECS = tm.catalogue()


@pytest.mark.parametrize("spec", SPECS, ids=[tm.spec_id(s) for s in SPECS])
def test_device_equals_model(api, oa, cams, spec):
    import torch
    s = tm.make(api, oa, cams, spec)
    p = tm.predict(oa, s)
    m = api.cORBmatcher(0.6, False, s["dim"], s["masked"])
    assert m.TH_LOW_ == s["th_low"]
    cap, F1, F2 = s["cap"], s["KF1"], s["nbs"][0]
    if spec[0] in ("ties", "capacity"):                                 # the planted rows straddle / lie in this device's chunks
        chunk, splits = tm.chunk_of(cap, 3, torch.cuda.get_device_properties(0).multi_processor_count)
        rows = s["tie_rows"] if spec[0] == "ties" else [s["scan_row"], tm.CAPACITY - 1]
        assert splits >= 2 and (rows[0] < chunk <= rows[-1] if spec[0] == "ties" else min(rows) >= (splits - 1) * chunk)
    host = host_tri(api, m, F1, F2, s["mp1"], s["mps"][0], cams, cap, s["E"], s["epi"])
    live = np.array([v is not None for v in p["slots"]])
    want = np.where(live, p["slots"], POISON).astype(np.int64)
    assert host[0] == p["n"] and np.array_equal(host[1][live], want[live])
    for layout in ("single", "parts", "joint"):
        dev = device_tri(api, m, F1, F2, s["mp1"], s["mps"][0], cams, cap, s["E"], layout, s["epi"])
        assert_same_tri(api, F1, dev, host, cap)
        assert dev[0] == p["n"] and np.array_equal(dev[1], want), layout
        assert dev[2].tolist() == p["diag"], (layout, dev[2].tolist(), p["diag"])
