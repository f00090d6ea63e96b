"""The C++ mirror of the reference interface (include/mcs_shim.hpp): compiles against the C ABI on CPU; on the GPU
the compiled program must reproduce the oracle's descriptors through mdBRIEFextractorOct::operator()."""
import pathlib
import subprocess

import numpy as np
import pytest
import ref_mcs_api          # oracle/, on sys.path through tests/conftest.py (and build())

ROOT = pathlib.Path(__file__).resolve().parents[1]


def build(out_dir):
    """compile tests/cpp/shim_smoke.cpp into out_dir (the checkout itself may be read-only); -> path of the program"""
    exe = pathlib.Path(out_dir) / "shim_smoke"
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-o", str(exe), str(ROOT / "tests/cpp/shim_smoke.cpp"),
                           "-L" + str(ROOT / "multicol_slam_b200"), "-lmcs_b200", "-Wl,-rpath," + str(ROOT / "multicol_slam_b200")])
    return exe


def test_shim_compiles_and_links(api, tmp_path):
    assert build(tmp_path).exists()


def test_shim_opencv_branch_compiles(tmp_path):
    """the -DMCS_WITH_OPENCV branch of include/mcs_shim.hpp (cv::InputArray / cv::OutputArray / std::vector<cv::KeyPoint> overload of
    operator()) against the stand-in OpenCV header the reference-run oracle is built with (oracle/ref_mcs/stub)"""
    src = tmp_path / "cvshim.cpp"
    src.write_text('''#include <opencv2/opencv.hpp>
#include "mcs_shim.hpp"
int use(MultiColSLAM::mdBRIEFextractorOct& ex, const MultiColSLAM::cCamModelGeneral_& cam, const cv::Mat& img, const cv::Mat& mask) {
    std::vector<cv::KeyPoint> kps; cv::Mat d, m;
    ex(img, mask, kps, cam, d, m);            // the reference's call shape (src/cMultiFrame.cpp:138-139)
    return (int)kps.size() + d.rows + m.rows;
}
''')
    subprocess.check_call(["g++", "-std=c++17", "-fsyntax-only", "-DMCS_WITH_OPENCV", "-I" + str(ROOT / "oracle/ref_mcs/stub"),
                           "-I" + str(ROOT / "include"), str(src)])


REF = ref_mcs_api.REFERENCE_DIR
ADAPT = ROOT / "tests" / "cpp" / "adapter_check"


def build_adapter_check():
    """tests/cpp/adapter_check: the reference's own cORBmatcher (objects from `make -C oracle ref`) next to include/mcs_adapters.hpp"""
    obj = ROOT / "oracle" / "_ref" / "obj"
    inc = ["-I" + str(ROOT / "oracle/ref_mcs/stub"), "-I" + str(ROOT / "oracle/ref_mcs/stub/g2o_cfg/a/b"), "-I" + str(ROOT / "oracle/ref_mcs"),
           "-I" + str(REF / "include"), "-I" + str(REF / "ThirdParty/Eigen"), "-I" + str(REF / "ThirdParty/g2o"),
           "-I" + str(REF / "ThirdParty/OpenGV/include"), "-I" + str(REF / "ThirdParty")]
    objs = [str(obj / f) for f in ("cORBmatcher.o", "cam_system_omni.o", "cConverter.o", "cam_model_omni.o", "misc.o", "FeatureVector.o")]
    subprocess.check_call(["g++", "-O1", "-std=c++11", "-w", "-ffp-contract=off", "-include", str(ROOT / "oracle/ref_mcs/stub_slam.h")] + inc +
                          [str(ROOT / "tests/cpp/adapter_check.cpp")] + objs +
                          ["-L" + str(ROOT / "multicol_slam_b200"), "-lmcs_b200", "-Wl,-rpath," + str(ROOT / "multicol_slam_b200"), "-o", str(ADAPT)])


def test_adapters_compile_against_reference_containers(api):
    if not (ref_mcs_api.reference_present() and (ROOT / "oracle" / "_ref" / "obj" / "cORBmatcher.o").exists()):
        pytest.skip("needs a reference checkout (MCS_REFERENCE_DIR) and `make -C oracle ref`")
    build_adapter_check()
    assert ADAPT.exists()


@pytest.mark.gpu
def test_adapters_equal_reference_matcher():
    """C++ drop-in check: the reference's cORBmatcher::SearchByProjection / SearchForInitialization / SearchByBoW(KF,KF) and the
    adapters over the C ABI leave the same reference-shaped containers in the same state (binary built where the reference checkout is readable)"""
    if not ADAPT.exists():
        pytest.skip("tests/cpp/adapter_check was not built (needs a reference checkout, MCS_REFERENCE_DIR)")
    out = subprocess.run([str(ADAPT)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "adapter_check passed" in out.stdout, out.stdout + out.stderr
    assert out.stdout.count(" ok") == 6


@pytest.mark.gpu
def test_shim_extract_and_match(api, oa, cams, tmp_path):
    from multicol_slam_b200 import synth
    exe = build(tmp_path)
    cam = cams[0]
    img, mask = synth.frame(cam, 4), synth.mirror_mask(cam)
    (tmp_path / "i.raw").write_bytes(img.tobytes())
    (tmp_path / "m.raw").write_bytes(mask.tobytes())
    import sys
    sys.path.insert(0, str(ROOT / "tools"))
    from extract_vocabulary import write_text
    voc = np.load(ROOT / "tests" / "golden" / "voc_small_9_6.npz")
    write_text({k: voc[k] for k in voc.files}, tmp_path / "voc.txt")
    out = subprocess.run([str(exe), str(tmp_path / "i.raw"), str(tmp_path / "m.raw"), "754", "480", str(tmp_path / "voc.txt")],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    kv = dict(t.split("=") for t in out.stdout.split()[1:])
    ok, od, om = oa.OracleExtractor(nfeatures=1000, do_dbrief=True, learn_masks=True).extract(img, mask, cam)
    h = 0
    for a, b in zip(od.reshape(-1), om.reshape(-1)):
        h = (h * 1315423911 + int(a) + 7 * int(b)) & 0xFFFFFFFFFFFFFFFF
    assert int(kv["nkp"]) == len(ok) and int(kv["hash"]) == h
    assert kv["same_mask"] == "1" and kv["untouched"] == "1" and kv["levels"] == "8" and kv["ds"] == "32" and kv["d01"] == "1"
    n, m12 = oa.match_bruteforce(od, od ^ np.eye(32, dtype=np.uint8)[np.arange(len(od)) % 32], 32, 0.9, om, om)
    assert int(kv["matches"]) == n and int(kv["self"]) == int((m12 == np.arange(len(od))).sum())
    # bag of words through the C++ ORBVocabulary / SearchByBoW(KF, F)
    other = od ^ np.eye(32, dtype=np.uint8)[np.arange(len(od)) % 32]
    o = oa.OracleVocabulary(voc)
    bw, bv, fn, fo, ff = o.transform(od, 4)
    bw2, bv2, fn2, fo2, ff2 = o.transform(other, 4)
    h = 0
    for k in range(len(fn)):
        h = (h * 1315423911 + int(fn[k])) & 0xFFFFFFFFFFFFFFFF
        for i in ff[fo[k]:fo[k + 1]]:
            h = (h * 1315423911 + int(i)) & 0xFFFFFFFFFFFFFFFF
    for w in bw:
        h = (h * 1315423911 + int(w)) & 0xFFFFFFFFFFFFFFFF
    assert int(kv["bow"]) == len(bw) and int(kv["fvn"]) == len(fn) and int(kv["bowhash"]) == h
    assert float(kv["score"]) == o.score(bw, bv, bw2, bv2)
    nb, _ = oa.search_by_bow(od, om, None, (fn, fo, ff), other, om, (fn2, fo2, ff2), 32, 0.9)
    assert int(kv["bm"]) == nb and nb > 500
