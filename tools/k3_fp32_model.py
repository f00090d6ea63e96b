"""k3_fp32_model.py -- numpy model of tier 1 of the descriptor kernel (multicol_slam_b200/csrc/describe_kernel.cu): the distorted
BRIEF pattern evaluated in fp32 relative to the keypoint, both forms (s-form: q(s') of 6 coefficients, m-form: P(t) of 8), from
the table rows exactly as mcs_cam_distort_table returns them and with the kernel's choice of form per keypoint.  fp32 arithmetic
WITHOUT fused multiply-add, so the model is pessimistic next to the kernel's fmaf chains.  The error is |fp32 - exact| of the
mean-free projected coordinates, the exact side being WorldToImg in double (ref src/cam_model_omni.cpp:49-67).  The kernel's
guard kT1Guard has to stay well above the worst of it (tests/test_k3_fp32_model_cpu.py).
    python tools/k3_fp32_model.py [keypoints per camera]
prints, for the Lafida cameras and the synthetic ones of tests/golden/synthetic_cams.json, the worst / p99 / median error and the
worst error of the pattern mean (the systematic part the tier-1 repair inherits)."""
import json
import pathlib
import re
import sys

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
f32 = np.float32
T1_SCALE = 32.0             # kT1Scale: s' = s / 32
T1_MIN_RADIUS = 40.0        # kT1MinRadius
REACH = 22.5                # kLutReach


def pattern():
    """learned_pattern_64_ORB, the first 512 points (descSize 32)"""
    txt = re.sub(r"/\*.*?\*/", "", (ROOT / "multicol_slam_b200" / "csrc" / "brief_pairs_64.inc").read_text(), flags=re.S)
    return np.array([int(v) for v in re.findall(r"-?\d+", txt)], np.float64)[:1024].reshape(512, 2)


def horner(c, x):
    r = np.zeros_like(x) if isinstance(x, np.ndarray) else type(x)(0)
    for k in range(len(c) - 1, -1, -1):
        r = r * x + c[k]
    return r


def world_to_img(cam, x, y, z):
    n = np.sqrt(x * x + y * y)
    n = np.where(n == 0, 1e-14, n)
    rho = horner(cam["inv_pol"], np.arctan(-z / n))
    uu, vv = x / n * rho, y / n * rho
    return uu * cam["c"] + vv * cam["d"] + cam["u0"], uu * cam["e"] + vv + cam["v0"]


def undistort(cam, u, v):
    """undistortPointsOcam: the keypoint on the plane z = -a0"""
    inv = cam["c"] - cam["d"] * cam["e"]
    ut, vt = u - cam["u0"], v - cam["v0"]
    x, y = (ut - cam["d"] * vt) / inv, (-cam["e"] * ut + cam["c"] * vt) / inv
    z = -horner(cam["pol"], np.sqrt(x * x + y * y))
    return -x / z * cam["pol"][0], -y / z * cam["pol"][0]


def row_floats(row, first, count):
    return np.frombuffer(np.ascontiguousarray(row[first:first + (count + 1) // 2]).tobytes(), np.float32)[:count]


def keypoint_error(cam, table, kx, ky, angle, pat):
    """(form, worst coordinate error, pattern-mean error) of one keypoint's pattern; form None where the kernel does not take tier 1
    or the tier-1 guard cannot accept the pattern"""
    a0 = cam["pol"][0]
    ukx, uky = undistort(cam, kx, ky)
    rk = np.hypot(ukx, uky)
    if not rk < len(table) - 1 or rk < T1_MIN_RADIUS:
        return None, 0.0, 0.0
    i = int(np.rint(rk))
    row = table[i]
    if row[17] != 1.0:
        return None, 0.0, 0.0
    mform = row[23] == 1.0
    ca, sa = np.cos(angle), np.sin(angle)
    px, py = pat[:, 0], pat[:, 1]
    ue, ve = world_to_img(cam, px * ca - py * sa + ukx, px * sa + py * ca + uky, -a0)
    uk, vk = world_to_img(cam, np.array([ukx]), np.array([uky]), -a0)
    # ---- the kernel's per-keypoint set-up (double) and per-pattern constants ----
    c, d, e = cam["c"], cam["d"], cam["e"]
    nx, ny = f32(2.0 * (ukx * ca + uky * sa)), f32(2.0 * (uky * ca - ukx * sa))
    axx, axy, ayx, ayy = f32(c * ca + d * sa), f32(d * ca - c * sa), f32(e * ca + sa), f32(ca - e * sa)
    auk, avk = f32(c * ukx + d * uky), f32(e * ukx + uky)
    pxf, pyf = px.astype(f32), py.astype(f32)
    n = pxf * nx + (pyf * ny + (pxf * pxf + pyf * pyf))                  # r^2 - r_k^2
    if mform:
        a = row_floats(row, 19, 8)
        inv_hw = 1.0 / (2.0 * REACH * i)
        tk = (rk * rk - (i * i + REACH * REACH)) * inv_hw
        K0 = tk * horner(a.astype(np.float64), tk)
        gkf, K0f = f32(row[18] + K0), f32(K0)
        t = n * f32(inv_hw) + f32(tk)
        dg = t * horner(a, t) - K0f
    else:
        q = row_floats(row, 14, 5)
        s0 = (rk - i) / T1_SCALE
        dRk = s0 * horner(np.concatenate([[row[13]], q.astype(np.float64)]), s0)
        gk = (row[12] + dRk) / rk
        qf = np.concatenate([[f32(row[13] - gk * T1_SCALE)], q]).astype(f32)
        gkf, K0f = f32(gk), f32(dRk - gk * (rk - i))
        r2 = f32(rk * rk) + n
        y = (f32(1) / np.sqrt(r2)).astype(f32)
        z = (f32(1) / (r2 * y + f32(rk))).astype(f32)
        sp = (n * z) * f32(1 / T1_SCALE) + f32(s0)
        dg = (sp * horner(qf, sp) - K0f) * y
    g = gkf + dg
    du = g * (pxf * axx + pyf * axy) + dg * auk
    dv = g * (pxf * ayx + pyf * ayy) + dg * avk
    mu, mv = f32(du.astype(np.float64).mean()), f32(dv.astype(np.float64).mean())
    if max(np.abs(ue - ue.mean()).max(), np.abs(ve - ve.mean()).max()) >= 25.4:
        return None, 0.0, 0.0                  # outside the staged patch: the kernel flags the pattern whatever its rounding
    err = max(np.abs((du - mu).astype(np.float64) - (ue - ue.mean())).max(), np.abs((dv - mv).astype(np.float64) - (ve - ve.mean())).max())
    merr = max(abs(float(mu) - (ue.mean() - uk[0])), abs(float(mv) - (ve.mean() - vk[0])))
    return ("m" if mform else "s"), float(err), float(merr)


def tier1_errors(cam, table, nk=300, seed=0):
    """the model over nk keypoints on the pixels the mirror mask keeps (>= 25 px inside the image), half of them within 80 px of
    the principal point where the s-form serves, at random angles -> (forms, errors, mean errors) of the keypoints that take tier 1"""
    sys.path.insert(0, str(ROOT))
    from multicol_slam_b200 import synth
    rng = np.random.default_rng(seed)
    m = synth.mirror_mask(cam)[25:-25, 25:-25]
    ys, xs = np.nonzero(m)
    near = np.nonzero(np.hypot(xs + 25 - cam["u0"], ys + 25 - cam["v0"]) < 80)[0]
    pat = pattern()
    out = []
    for j in np.concatenate([rng.choice(len(xs), nk - nk // 2, replace=False), rng.choice(near, nk // 2, replace=False)]):
        kx, ky = xs[j] + 25 + rng.uniform(-0.5, 0.5), ys[j] + 25 + rng.uniform(-0.5, 0.5)
        r = keypoint_error(cam, table, kx, ky, rng.uniform(0, 2 * np.pi), pat)
        if r[0] is not None:
            out.append(r)
    forms, errs, merrs = zip(*out) if out else ((), (), ())
    return np.array(forms), np.array(errs), np.array(merrs)


def main(nk):
    sys.path.insert(0, str(ROOT))
    import multicol_slam_b200.api as api
    from multicol_slam_b200 import synth
    cams = [(f"lafida{i}", c) for i, c in enumerate(synth.lafida_cams())]
    cams += [(c["name"], c) for c in json.loads((ROOT / "tests" / "golden" / "synthetic_cams.json").read_text())]
    for name, cam in cams:
        forms, errs, merrs = tier1_errors(cam, api.distort_table(cam), nk, 1)
        print(f"{name:20s} tier-1 keypoints {len(errs)} (m-form {int((forms == 'm').sum())})  max err {errs.max():.2e}  "
              f"p99 {np.percentile(errs, 99):.2e}  median {np.median(errs):.2e}  mean err max {merrs.max():.2e}")


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 400)
