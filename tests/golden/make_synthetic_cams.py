"""make_synthetic_cams.py -- writes tests/golden/synthetic_cams.json: OCamCalib calibrations (5 + 12 coefficients, the format of
multicol_slam_b200/data/lafida_cams.json) of fisheye cameras unlike the Lafida ones, each chosen to drive the descriptor kernel
(K3, describe_kernel.cu) down one path that the Lafida cameras barely reach.   python tests/golden/make_synthetic_cams.py

A camera is an ideal projection rho(phi) (image radius of a ray at incidence phi) fitted the way OCamCalib models it:
  pol     = [a0, 0, a2, a3, a4]: least squares of  pol(rho) = -rho / tan(phi)           (z = -pol(rho), ImgToWorld)
  inv_pol = 12 coefficients:     least squares of  rho(theta), theta = atan(-z / rho) of that same pol   (WorldToImg)
followed by the affine part [c d; e 1] and the principal point.  The tests read the committed JSON and never refit it: lstsq may
differ in the last bits between machines, and every fixture pins the exact coefficients.  The asserts at the end check, with the
camera model and the distortion-table builder of the built library, that each camera reaches the path it is meant for."""
import json
import pathlib
import sys

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[2]
OUT = ROOT / "tests" / "golden" / "synthetic_cams.json"
PROJ = {"equidistant": lambda f, p: f * p, "equisolid": lambda f, p: 2 * f * np.sin(p / 2),
        "stereographic": lambda f, p: 2 * f * np.tan(p / 2)}
PATCH = 25                       # K3 stages the blurred patch ky/kx -25 .. +25 around a keypoint


def fit(proj, f, fov_deg, width=754, height=480, du=0.0, dv=0.0, c=1.0, d=0.0, e=0.0, mirror_mask=1, inv_scale=1.0):
    phi = np.linspace(1e-3, np.radians(fov_deg) / 2, 4000)
    rho = PROJ[proj](f, phi)
    s = rho.max()                                            # fit in rho / s, theta / (pi / 2): well-conditioned Vandermonde
    x = rho / s
    A = np.stack([np.ones_like(x), x ** 2, x ** 3, x ** 4], 1)
    b = np.linalg.lstsq(A, -rho / np.tan(phi), rcond=None)[0]
    pol = [b[0], 0.0, b[1] / s ** 2, b[2] / s ** 3, b[3] / s ** 4]
    z = -(pol[0] + pol[2] * rho ** 2 + pol[3] * rho ** 3 + pol[4] * rho ** 4)
    theta = np.arctan(-z / rho)
    assert np.all(np.diff(theta) > 0), "theta(rho) of the fitted pol is not monotonic"
    t = theta / (np.pi / 2)
    k = np.linalg.lstsq(np.vander(t, 12, increasing=True), rho, rcond=None)[0]
    inv_pol = [inv_scale * k[i] / (np.pi / 2) ** i for i in range(12)]
    return dict(c=c, d=d, e=e, u0=(width - 1) / 2 + 0.3 + du, v0=(height - 1) / 2 + 0.6 + dv, pol=[float(v) for v in pol],
                inv_pol=[float(v) for v in inv_pol], width=width, height=height, mirror_mask=mirror_mask)


CAMS = [
    # a polynomial family other than Lafida's, with a Lafida-like shape
    ("equidistant185", dict(proj="equidistant", f=200, fov_deg=185)),
    # strong compression: the tier-1 forms of the table start at other radii (fitted out to the mirror disc's 266 px)
    ("equisolid230", dict(proj="equisolid", f=160, fov_deg=230)),
    # weak compression: same
    ("stereographic170", dict(proj="stereographic", f=230, fov_deg=170)),
    # an affine part far from the identity and an off-centre principal point, folded into the tier-1 constants
    ("affine185", dict(proj="equidistant", f=200, fov_deg=185, c=1.06, d=0.06, e=-0.05, du=25, dv=-15)),
    # no mirror mask on a 195 deg lens: corner pixels at 90 deg incidence or more, or beyond the table's 8192 rows
    ("wide1920x1080_195", dict(proj="equidistant", f=640, fov_deg=195, width=1920, height=1080, mirror_mask=0)),
    # long undistorted radii: the m-form of tier 1 almost everywhere
    ("narrow1280x720_120", dict(proj="equidistant", f=500, fov_deg=120, width=1280, height=720)),
    # inv_pol 1.3x pol (inconsistent on purpose): magnification > 1 near the centre, pattern offsets beyond the staged patch
    ("magnify130", dict(proj="equidistant", f=200, fov_deg=185, inv_scale=1.3)),
]


def pattern():
    import re
    txt = (ROOT / "multicol_slam_b200" / "csrc" / "brief_pairs_64.inc").read_text()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return np.array([int(v) for v in re.findall(r"-?\d+", txt)], np.float64)[:1024].reshape(512, 2)


def pattern_offsets(api, cam, kx, ky, angle):
    """rotateAndDistortPattern at level 0: the distorted pattern minus its mean, as K3 rounds it (double, reference arithmetic)"""
    x, y, z = api.img_to_world(cam, kx, ky)
    a0 = cam["pol"][0]
    ukx, uky = -x / z * a0, -y / z * a0
    p = pattern()
    ca, sa = np.cos(angle), np.sin(angle)
    uv = np.array([api.world_to_img(cam, px * ca - py * sa + ukx, px * sa + py * ca + uky, -a0) for px, py in p])
    return uv - uv.mean(0)


def tier1_starts(api, cam):
    """first radius from which every table row has the s-form / the m-form of tier 1"""
    T = api.distort_table(cam)
    out = []
    for col in (17, 23):
        on = T[:-1, col] == 1.0
        out.append(int(len(on) - np.argmin(on[::-1])) if not on.all() else 0)
    return out


def check(api, name, cam):
    from multicol_slam_b200 import synth
    mask = synth.mirror_mask(cam)
    ys, xs = np.nonzero(mask)
    rng = np.random.default_rng(0)
    pick = rng.choice(len(xs), 400, replace=False)
    lafida = [tier1_starts(api, c) for c in synth.lafida_cams()]
    if name == "equidistant185":
        worst = 0.0
        for i in pick:
            u, v = api.world_to_img(cam, *api.img_to_world(cam, float(xs[i]), float(ys[i])))
            worst = max(worst, abs(u - xs[i]), abs(v - ys[i]))
        assert worst < 1e-3, worst
    if name in ("equisolid230", "stereographic170"):
        # the s-form can start no lower than radius 39, where Lafida camera 0 starts it too: the m-form boundary has to move
        s, m = tier1_starts(api, cam)
        assert [s, m] not in lafida and not min(l[1] for l in lafida) <= m <= max(l[1] for l in lafida), (s, m, lafida)
    if name == "affine185":
        assert min(abs(cam["c"] - 1), abs(cam["d"]), abs(cam["e"])) >= 0.05
    if name == "wide1920x1080_195":
        n = api.distort_table(cam).shape[0]
        far = 0
        for i in range(0, len(xs), 97):
            x, y, z = api.img_to_world(cam, float(xs[i]), float(ys[i]))
            far += z <= 0 or np.hypot(x / z, y / z) * abs(cam["pol"][0]) >= n - 1
        assert n == 8192 and far > 0, (n, far)
    if name == "magnify130":
        worst = 0.0
        for i in pick[:60]:
            # near the distortion centre the offsets exceed the staged patch; everywhere a keypoint can sit (>= 25 px inside the
            # image) every sample stays inside the image, so the reference reads no byte beyond its 25 px ring
            kx, ky = float(xs[i]), float(ys[i])
            if not (PATCH <= kx < cam["width"] - PATCH and PATCH <= ky < cam["height"] - PATCH):
                continue
            o = np.rint(pattern_offsets(api, cam, kx, ky, rng.uniform(0, 2 * np.pi)))
            assert (kx + o[:, 0] >= 0).all() and (kx + o[:, 0] < cam["width"]).all()
            assert (ky + o[:, 1] >= 0).all() and (ky + o[:, 1] < cam["height"]).all()
        for a in np.linspace(0, np.pi / 2, 7):
            worst = max(worst, np.abs(pattern_offsets(api, cam, cam["u0"] + 5, cam["v0"] + 3, a)).max())
        assert worst > PATCH + 0.5, worst


def main():
    sys.path.insert(0, str(ROOT))
    import multicol_slam_b200.api as api
    cams = []
    for name, spec in CAMS:
        cam = fit(**spec)
        check(api, name, cam)
        cams.append(dict(name=name, **cam))
        print(name, "tier-1 s-form / m-form from radius", tier1_starts(api, cam), "table rows", api.distort_table(cam).shape[0])
    OUT.write_text(json.dumps(cams, indent=1) + "\n")


if __name__ == "__main__":
    main()
