"""Writes tests/golden/projection_edges_mp200.npz: the projections of the edge scenes of tests/test_projection_edges_cpu.py in
200-bit arithmetic (mpmath), rounded once to double.  tests/test_projection_edges_gpu.py reads them to say how far the host and the
device projections are from the correctly rounded value; mpmath need not be installed where the tests run.

The inputs are the camera-frame points as the kernel computes them in double (the pose product is part of the scene); from there
WorldToImg (ref src/cam_model_omni.cpp:146-161) is evaluated at 200 bits.  The norm == 0 branch is taken where the double
norm is 0, as the code does (x*x + y*y can underflow).  Non-finite inputs give NaN.

    python tests/golden/make_projection_edges_golden.py
"""
import pathlib
import sys

import mpmath
import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def world_to_img_mp(cam, x, y, z):
    if not all(np.isfinite((x, y, z))):
        return np.nan, np.nan
    X, Y, Z = mpmath.mpf(x), mpmath.mpf(y), mpmath.mpf(z)
    norm = mpmath.mpf(1e-14) if np.sqrt(x * x + y * y) == 0.0 else mpmath.sqrt(X * X + Y * Y)
    theta = mpmath.atan(-Z / norm)
    rho = mpmath.mpf(0)
    for c in reversed(cam["inv_pol"]):
        rho = rho * theta + mpmath.mpf(c)
    uu, vv = X / norm * rho, Y / norm * rho
    u = uu * mpmath.mpf(cam["c"]) + vv * mpmath.mpf(cam["d"]) + mpmath.mpf(cam["u0"])
    v = uu * mpmath.mpf(cam["e"]) + vv + mpmath.mpf(cam["v0"])
    return float(u), float(v)


def main():
    import test_projection_edges_cpu as E
    mpmath.mp.prec = 200
    out = {}
    for name, sc in E.scenes().items():
        pos = sc.arrays()[0]
        uv = np.zeros((len(pos), len(sc.cams), 2))
        for i, P in enumerate(pos):
            for c, cam in enumerate(sc.cams):
                uv[i, c] = world_to_img_mp(cam, *(float(t) for t in E.cam_point(sc.inv[c], P)))
        key = name.replace("/", "__")
        out[f"{key}__uv"] = uv
        out[f"{key}__crc"] = np.int64(E.scene_crc(sc))
    np.savez_compressed(E.MP200, **out)
    print(f"wrote {E.MP200} ({len(E.scenes())} scenes)")


if __name__ == "__main__":
    main()
