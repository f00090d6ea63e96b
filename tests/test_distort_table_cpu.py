"""CPU: the per-camera distortion tables behind tiers 1 and 2 of the descriptor kernel (mcs_cam_distort_table, built on the host in
multicol_slam_b200/csrc/describe_kernel.cu: build_distort_lut) checked against the camera model itself, independently of the kernel,
in numpy long double:  R(r) = rho(atan(-z / r)),  rho = the inverse polynomial of cCamModelGeneral_::WorldToImg
(ref src/cam_model_omni.cpp:49-67), z = -a0.  The kernel's rounding decisions rest on these error bounds:
  tier 2   degree-9 polynomial of R on [i - 22.5, i + 22.5]                      |error| < 2e-8 px
  tier 1   s-form  R(i + s) - R(i) = s' q(s'), s' = s / 32                       |error| < 1e-6 px
           m-form  G(c_i + hw_i t) - G(c_i) = t P(t), G(m) = R(sqrt m) / sqrt m  |error| (i + 1) < 1e-6 px
with the float coefficients exactly as the kernel reads them."""
import json
import pathlib

import numpy as np
import pytest

LD = np.longdouble
REACH = 22.5
# fisheye calibrations unlike Lafida's (tests/golden/make_synthetic_cams.py), each meant for one path of the descriptor kernel
SYNTHETIC = {c["name"]: c for c in json.loads((pathlib.Path(__file__).resolve().parent / "golden" / "synthetic_cams.json").read_text())}
LAFIDA_M_START = range(62, 68)        # where the m-form rows start on the three Lafida cameras


def horner(c, x):
    r = np.zeros_like(x)
    for k in range(len(c) - 1, -1, -1):
        r = r * x + LD(c[k])
    return r


def R_exact(cam, r):
    z = -LD(cam["pol"][0])
    return horner([LD(v) for v in cam["inv_pol"]], np.arctan(-z / r))


def floats_of(row, first, count):
    return np.frombuffer(np.ascontiguousarray(row[first:first + (count + 1) // 2]).tobytes(), np.float32)[:count].astype(LD)


def form_start(T, col):
    """first row from which every row but the last has the tier-1 form flagged in column col (17: s-form, 23: m-form)"""
    on = T[:-1, col] == 1.0
    return len(on) - int(np.argmin(on[::-1])) if not on.all() else 0


@pytest.mark.parametrize("which", [0, 1, 2, "hd"] + list(SYNTHETIC))
def test_tables_against_the_camera_model(api, cams, which):
    from multicol_slam_b200 import synth
    cam = synth.scaled_cam(cams[1], 1920, 1080) if which == "hd" else SYNTHETIC[which] if which in SYNTHETIC else cams[which]
    T = api.distort_table(cam)
    n, stride = T.shape
    assert stride == 24 and 200 < n <= 8192
    t = np.linspace(-1, 1, 41).astype(LD) * LD(0.999)
    n2 = n1s = n1m = 0
    for i in list(range(0, 130)) + list(range(130, n, 7)):
        row = T[i]
        lo, hi = max(LD(0), LD(i) - LD(REACH)), LD(i) + LD(REACH)
        if not np.isnan(row[0]):                                   # ---- tier 2
            r = (lo + hi) / 2 + (hi - lo) / 2 * t
            r = r[r > 0]
            tau = r * LD(row[1]) + LD(row[0])
            err = np.abs(horner(row[2:12], tau) - R_exact(cam, r)).max()
            assert err < 2.5e-8, (i, float(err))
            n2 += 1
        if row[17] == 1.0:                                         # ---- tier 1, s-form
            assert i >= 39 and not np.isnan(row[0])
            s = LD(REACH) * t
            s = s[np.abs(s) > 1e-6]
            sp = s / LD(32)
            q = np.concatenate([[LD(row[13])], floats_of(row, 14, 5)])
            err = np.abs(sp * horner(q, sp) - (R_exact(cam, LD(i) + s) - R_exact(cam, np.array([LD(i)]))[0])).max()
            assert abs(float(R_exact(cam, np.array([LD(i)]))[0]) - row[12]) < 1e-12 * max(1.0, abs(row[12]))
            assert err < 1.2e-6, (i, float(err))
            n1s += 1
        if row[23] == 1.0:                                         # ---- tier 1, m-form
            assert row[17] == 1.0 and i > REACH + 1
            c, hw = LD(i) * LD(i) + LD(REACH) ** 2, LD(2 * REACH) * LD(i)
            G = lambda m: R_exact(cam, np.sqrt(m)) / np.sqrt(m)    # noqa: E731
            tt = t[np.abs(t) > 1e-6]
            a = floats_of(row, 19, 8)
            err = np.abs(tt * horner(a, tt) - (G(c + hw * tt) - G(np.array([c]))[0])).max()
            assert abs(float(G(np.array([c]))[0]) - row[18]) < 1e-14
            assert err * (i + 1) < 1.2e-6, (i, float(err * (i + 1)))
            n1m += 1
    # coverage: tier 2 everywhere, tier 1 never below 39
    assert n2 > 100 and n1s > 80 and n1m > 60
    assert not np.isnan(T[:, 0]).any()
    assert not any(T[i, 17] == 1.0 or T[i, 23] == 1.0 for i in range(0, 39))
    if which not in SYNTHETIC:
        # Lafida cameras: the s-form from radius 40..54 on and the m-form from 62..67 on
        assert all(T[i, 17] == 1.0 for i in range(56, n - 1)) and all(T[i, 23] == 1.0 for i in range(72, n - 1))
    elif which in ("equisolid230", "stereographic170"):
        # strong and weak compression move the m-form boundary out of the Lafida range (to 79 and to 39)
        assert form_start(T, 23) not in LAFIDA_M_START and form_start(T, 23) >= form_start(T, 17)
    elif which == "wide1920x1080_195":
        # corner pixels near 90 degrees incidence: the table stops at its cap (keypoints beyond it take the exact path)
        assert n == 8192
    elif which == "narrow1280x720_120":
        assert form_start(T, 23) == 39                      # the m-form from the first tier-1 radius on


def test_table_argument_validation(api, cams):
    import ctypes as C
    lib = api.lib()
    n, row = C.c_int32(0), C.c_int32(0)
    assert lib.mcs_cam_distort_table(None, None, 0, C.byref(n), C.byref(row)) == api.MCS_ERR_INVALID
    oc = api.as_ocam(cams[0])
    assert lib.mcs_cam_distort_table(C.byref(oc), None, 0, None, C.byref(row)) == api.MCS_ERR_INVALID
    assert lib.mcs_cam_distort_table(C.byref(oc), None, 0, C.byref(n), C.byref(row)) == api.MCS_OK and n.value > 200 and row.value == 24
