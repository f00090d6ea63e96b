"""CPU: the error budget of tier 1 of the descriptor kernel.  K3 accepts an fp32 pattern when every mean-free coordinate lies more
than kT1Guard from a rounding tie, so kT1Guard has to exceed the worst fp32 error by a clear margin on every camera, not just the
Lafida ones it was measured on.  tools/k3_fp32_model.py models tier 1 without FMA (pessimistic) from the table rows
mcs_cam_distort_table returns, with the kernel's choice of s-form / m-form per keypoint."""
import importlib.util
import json
import pathlib
import re

import pytest

ROOT = pathlib.Path(__file__).resolve().parents[1]
SYNTHETIC = {c["name"]: c for c in json.loads((ROOT / "tests" / "golden" / "synthetic_cams.json").read_text())}


def model():
    spec = importlib.util.spec_from_file_location("k3_fp32_model", ROOT / "tools" / "k3_fp32_model.py")
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def t1_guard():
    src = (ROOT / "multicol_slam_b200" / "csrc" / "describe_kernel.cu").read_text()
    return float(re.search(r"constexpr float kT1Guard = ([0-9.eE+-]+)f;", src).group(1))


@pytest.mark.parametrize("which", [0, 1, 2] + list(SYNTHETIC))
def test_tier1_error_within_the_guard_budget(api, cams, which):
    cam = SYNTHETIC[which] if which in SYNTHETIC else cams[which]
    forms, errs, merrs = model().tier1_errors(cam, api.distort_table(cam), nk=400, seed=1)
    assert len(errs) > 250 and (forms == "m").sum() > 150
    # the design keeps kT1Guard 4x above the worst error.  A camera that magnifies (inv_pol 1.3x pol) scales the coordinates, and
    # with them the fp32 rounding, by up to 1.3: there the margin is 3.9x at worst over 2000 modelled keypoints
    margin = 3.0 if which == "magnify130" else 4.0
    assert errs.max() < t1_guard() / margin, (float(errs.max()), t1_guard())
    # the pattern mean's error is the part the tier-1 repair inherits; kT1RepairGuard (4e-6 px) budgets 1.5e-7 px for it
    assert merrs.max() < 2e-7


def test_model_covers_the_s_form(api, cams):
    forms, errs, _ = model().tier1_errors(cams[0], api.distort_table(cams[0]), nk=400, seed=1)
    assert (forms == "s").sum() > 30
