"""GPU: the five device searches that decide by ordered acceptance, on every generated contention scene
(tests/acceptance_model.py), against the host entry point (the C++ sequential replay), the oracle and the model of the rounds
and walk.  Results are compared bit for bit, with the slots beyond each camera's count untouched; diag must equal the model's
rounds run, walk start, queries and rescans exactly.  Both packed-buffer layouts of each search are used."""
import numpy as np
import pytest

import acceptance_model as am
from device_frames import per_cam, sizes
from device_searches import device_init, device_last, device_projection, device_search_frames, device_ws, host_init

pytestmark = pytest.mark.gpu


def _cap():
    import multicol_slam_b200.api as api
    return api.lib().mcs_search_by_projection_max_rounds()


SPECS = am.catalogue(_cap())


def _device(api, m, s, layout):
    k = s["kind"]
    if k == "local":
        return device_projection(api, m, per_cam(s["F"]), sizes(s["F"]), s["F"].scale_factors, s["mps"], s["th"], pre=s["pre"].copy(), layout=layout)
    if k == "last":
        return device_last(api, m, s["F"], s["Fl"], s["rig"], s["mp_cur"], s["mp_last"], None, s["world"], s["bad"], s["th"], layout=layout)
    if k == "frames":
        return device_search_frames(api, m, s["F"], s["Fl"], s["rig"], s["mp_cur"], s["mp_last"], s["world"], s["bad"], s["th"], layout=layout)
    return device_ws(api, m, s["F"], s["Fl"], s["mp_last"], s["bad"], s["th"], layout=layout)


@pytest.mark.parametrize("spec", SPECS, ids=[am.spec_id(s) for s in SPECS])
def test_device_equals_host_oracle_and_model(api, oa, spec):
    m, s = am.make(api, spec)
    p = am.predict(api, oa, m, s)
    on, oout = p["oracle"][:2]
    if s["kind"] == "init":
        h = host_init(m, s["F1"], s["F2"], s["prev"], s["window"])
        assert h[0] == on and np.array_equal(h[1], oout) and h[2].tobytes() == p["oracle"][2].tobytes()
        for layout in ("single", "parts"):
            gn, gm, gp, diag = device_init(api, m, s["F1"], s["F2"], s["prev"], s["window"], layout)
            assert gn == h[0] and np.array_equal(gm, h[1]) and gp.tobytes() == h[2].tobytes(), layout
            assert diag.tolist() == p["diag"], layout
        return
    if s["kind"] == "local":
        hn, hout = m.SearchByProjection(s["F"], s["mps"], s["th"], s["pre"].copy())
    else:
        hn, hout = am.host_call(m, s)
    assert hn == on and np.array_equal(hout, oout)
    for layout in ("single", "parts"):
        gn, gout, status, diag = _device(api, m, s, layout)
        assert status == api.MCS_OK and gn == hn and np.array_equal(gout, hout), layout
        assert diag.tolist() == p["diag"], layout
