// adapter_check.cpp -- the drop-in claim at the C++ level: the REFERENCE's own cORBmatcher (compiled from
// /root/reference/src/cORBmatcher.cpp, objects under oracle/_ref/obj) and the adapters of include/mcs_adapters.hpp (CUDA path through
// the C ABI) run on the same reference-shaped containers and must leave them in the same state.
// Built by tests/test_shim_cpp.py where /root/reference exists (the binary travels to the GPU box); containers are the data-only
// stand-ins of oracle/ref_mcs/stub_slam.h (force-included), everything else is the reference's code.  TEST INFRASTRUCTURE.
#include "cORBmatcher.h"

#include "../../include/mcs_adapters.hpp"

#include <cstdio>
#include <memory>
#include <random>

using namespace MultiColSLAM;

static cCamModelGeneral_ lafida_cam0() {          // Examples/Lafida/InteriorOrientationFisheye0.yaml, built like src/cSystem.cpp:144-170
    const double a[5] = {-209.200757992065, 0.0, 0.00213741670953883, -4.2203617319086e-06, 1.77146086919594e-08};
    const double pol[12] = {293.667187375663, 149.982043337335, -10.448650568161, 28.2295300683376, 7.13365723186292, 0.056303218962532,
                            10.4144677485333, 0.166354960773665, -5.86858687381081, 1.18165998645705, 3.1108311354746, 0.810799620714366};
    cv::Mat_<double> p = cv::Mat::zeros(5, 1, CV_64F), ip = cv::Mat::zeros(12, 1, CV_64F);
    for (int i = 0; i < 5; ++i) p.at<double>(i, 0) = a[i];
    for (int i = 0; i < 12; ++i) ip.at<double>(i, 0) = pol[i];
    double cde[5] = {0.999626131079017, -0.0034775192597376, 0.00385134991673147, 392.219508388648, 243.494438476351};
    cCamModelGeneral_ cam(cde, p, ip, 754, 480);
    std::vector<cv::Mat> masks;
    CreateMirrorMask(cam, 4, masks);
    cam.SetMirrorMasks(masks);
    return cam;
}

struct Scene {
    std::vector<std::unique_ptr<cMapPoint>> mps;
    std::vector<cMapPoint*> list;
};

static void fill_frame(cMultiFrame& f, std::mt19937& rng, int per_cam, const cMultiFrame* like) {
    const int nc = 3;
    std::vector<cv::Matx44d> Mc(nc, cv::Matx44d::eye());
    std::vector<cCamModelGeneral_> cams(nc, lafida_cam0());
    f.camSystem = cMultiCamSys_(cv::Matx44d::eye(), Mc, cams);
    std::uniform_real_distribution<float> ux(30.f, 720.f), uy(30.f, 450.f), jit(-3.f, 3.f);
    std::uniform_int_distribution<int> lvl(0, 7), byte(0, 255), bit(0, 255), nflip(0, 25);
    f.mDescriptors.resize(nc); f.mDescriptorMasks.resize(nc);
    for (int c = 0; c < nc; ++c) { f.mDescriptors[c] = cv::Mat::zeros(per_cam, 32, CV_8UC1); f.mDescriptorMasks[c] = cv::Mat::zeros(per_cam, 32, CV_8UC1); }
    for (int c = 0; c < nc; ++c)
        for (int r = 0; r < per_cam; ++r) {
            const size_t i = f.mvKeys.size();
            cv::KeyPoint kp;
            if (like) {                                  // the "next frame": the same features moved by a few pixels, a few bits flipped
                kp = like->mvKeys[i];
                kp.pt.x += jit(rng); kp.pt.y += jit(rng);
                std::memcpy(f.mDescriptors[c].ptr<uint8_t>(r), like->mDescriptors[c].ptr<uint8_t>(r), 32);
                for (int k = nflip(rng); k > 0; --k) { const int b = bit(rng); f.mDescriptors[c].ptr<uint8_t>(r)[b >> 3] ^= (uint8_t)(1 << (b & 7)); }
            } else {
                kp = cv::KeyPoint(ux(rng), uy(rng), 32.f, 0.f, 50.f, lvl(rng), -1);
                for (int b = 0; b < 32; ++b) f.mDescriptors[c].ptr<uint8_t>(r)[b] = (uint8_t)byte(rng);
            }
            for (int b = 0; b < 32; ++b) f.mDescriptorMasks[c].ptr<uint8_t>(r)[b] = (uint8_t)(byte(rng) | byte(rng));
            f.mvKeys.push_back(kp);
            f.keypoint_to_cam[i] = c; f.cont_idx_to_local_cam_idx[i] = r;
        }
    f.mvpMapPoints.assign(f.mvKeys.size(), nullptr);
    f.mvbOutlier.assign(f.mvKeys.size(), false);
    f.mnScaleLevels = 8;
    f.mvScaleFactors.resize(8);
    f.mvScaleFactors[0] = 1.0;
    for (int l = 1; l < 8; ++l) f.mvScaleFactors[l] = f.mvScaleFactors[l - 1] * (double)1.2f;
    f.grid.build(f.mvKeys, f.keypoint_to_cam, std::vector<int>(nc, 754), std::vector<int>(nc, 480));
}

static Scene make_points(const cMultiFrame& f, std::mt19937& rng, int n) {
    Scene s;
    std::uniform_int_distribution<int> pick(0, (int)f.mvKeys.size() - 1), bit(0, 255), nflip(0, 35), lv(-1, 1);
    std::normal_distribution<double> noise(0.0, 2.0);
    std::uniform_real_distribution<double> vc(0.99, 1.0), u01(0.0, 1.0);
    for (int i = 0; i < n; ++i) {
        std::unique_ptr<cMapPoint> p(new cMapPoint);
        const int k = pick(rng), c = f.keypoint_to_cam.find(k)->second, r = f.cont_idx_to_local_cam_idx.find(k)->second;
        p->id = i; p->bad = u01(rng) < 0.05;
        p->desc.assign(4, 0); p->dmask.assign(4, 0);
        std::memcpy(p->desc.data(), f.mDescriptors[c].ptr<uint8_t>(r), 32);
        std::memcpy(p->dmask.data(), f.mDescriptorMasks[c].ptr<uint8_t>(r), 32);
        for (int q = nflip(rng); q > 0; --q) { const int b = bit(rng); ((uint8_t*)p->desc.data())[b >> 3] ^= (uint8_t)(1 << (b & 7)); }
        p->mbTrackInView.assign(3, false); p->mnTrackScaleLevel.assign(3, 0); p->mTrackViewCos.assign(3, 0.0);
        p->mTrackProjX.assign(3, 0.0); p->mTrackProjY.assign(3, 0.0);
        p->mbTrackInView[c] = true;
        p->mnTrackScaleLevel[c] = std::min(7, std::max(0, f.mvKeys[k].octave + lv(rng)));
        p->mTrackViewCos[c] = vc(rng);
        p->mTrackProjX[c] = f.mvKeys[k].pt.x + noise(rng); p->mTrackProjY[c] = f.mvKeys[k].pt.y + noise(rng);
        s.list.push_back(p.get());
        s.mps.push_back(std::move(p));
    }
    return s;
}

template <class V> static bool same_ids(const V& a, const V& b) {
    if (a.size() != b.size()) return false;
    for (size_t i = 0; i < a.size(); ++i)
        if ((a[i] ? a[i]->id : -1) != (b[i] ? b[i]->id : -1)) return false;
    return true;
}

int main() {
    if (mcs_device_count() < 1) { std::printf("adapter_check: no sm_90 device\n"); return 3; }
    int fails = 0;
    for (int masks = 0; masks < 2; ++masks) {
        std::mt19937 rng(17 + masks);
        cORBmatcher ref(0.8, checkOrientation, 32, masks != 0);
        // ---- SearchByProjection(F, vpMapPoints, th) ----
        cMultiFrame Fa, Fb;
        fill_frame(Fa, rng, 500, nullptr);
        { std::mt19937 r2(17 + masks); fill_frame(Fb, r2, 500, nullptr); }
        Scene sc = make_points(Fa, rng, 900);
        for (size_t i = 0; i < Fa.mvpMapPoints.size(); i += 11) Fa.mvpMapPoints[i] = Fb.mvpMapPoints[i] = sc.list[0];     // some keypoints taken beforehand
        const int n_ref = ref.SearchByProjection(Fa, sc.list, 3.0);
        const int n_gpu = mcs_adapt::SearchByProjection(Fb, sc.list, 3.0, 0.8, ref.TH_HIGH_, masks != 0);
        const bool ok1 = n_ref == n_gpu && same_ids(Fa.mvpMapPoints, Fb.mvpMapPoints) && n_ref > 100;
        std::printf("masks=%d SearchByProjection ref=%d gpu=%d %s\n", masks, n_ref, n_gpu, ok1 ? "ok" : "MISMATCH");
        fails += !ok1;
        // ---- SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, 50) ----
        cMultiFrame F1, F2;
        { std::mt19937 r3(99 + masks); fill_frame(F1, r3, 400, nullptr); fill_frame(F2, r3, 400, &F1); }
        std::vector<cv::Vec2d> prevA(F1.mvKeys.size()), prevB(F1.mvKeys.size());
        for (size_t i = 0; i < F1.mvKeys.size(); ++i) prevA[i] = prevB[i] = cv::Vec2d(F1.mvKeys[i].pt.x, F1.mvKeys[i].pt.y);
        std::vector<int> m12a, m12b;
        cORBmatcher ref9(0.9, checkOrientation, 32, masks != 0);
        const int i_ref = ref9.SearchForInitialization(F1, F2, prevA, m12a, 50);
        const int i_gpu = mcs_adapt::SearchForInitialization(F1, F2, prevB, m12b, 50, 0.9, ref9.TH_LOW_, masks != 0);
        bool ok2 = i_ref == i_gpu && m12a == m12b && i_ref > 100;
        for (size_t i = 0; ok2 && i < prevA.size(); ++i) ok2 = prevA[i](0) == prevB[i](0) && prevA[i](1) == prevB[i](1);
        std::printf("masks=%d SearchForInitialization ref=%d gpu=%d %s\n", masks, i_ref, i_gpu, ok2 ? "ok" : "MISMATCH");
        fails += !ok2;
        // ---- SearchByBoW(KF1, KF2, vpMatches12): two key frames carrying map points ----
        cMultiKeyFrame K1, K2;
        auto to_kf = [&](const cMultiFrame& f, cMultiKeyFrame& k, Scene& pts, int first_id) {
            k.camSystem = f.camSystem; k.keypoint_to_cam = f.keypoint_to_cam; k.cont_idx_to_local_cam_idx = f.cont_idx_to_local_cam_idx;
            k.mvKeys = f.mvKeys; k.mDescriptors = f.mDescriptors; k.mDescriptorMasks = f.mDescriptorMasks; k.mvScaleFactors = f.mvScaleFactors;
            k.mnScaleLevels = 8; k.grid = f.grid;
            k.mvpMapPoints.assign(f.mvKeys.size(), nullptr);
            for (size_t i = 0; i < f.mvKeys.size(); ++i)
                if (i % 3 != 0) {
                    std::unique_ptr<cMapPoint> p(new cMapPoint);
                    p->id = first_id + (int)i; p->bad = (i % 17 == 0);
                    k.mvpMapPoints[i] = p.get();
                    pts.mps.push_back(std::move(p));
                }
        };
        Scene own;
        to_kf(F1, K1, own, 0); to_kf(F2, K2, own, 100000);
        std::vector<cMapPoint*> va, vb;
        const int b_ref = ref9.SearchByBoW(&K1, &K2, va);
        const int b_gpu = mcs_adapt::SearchByBoW(&K1, &K2, vb, 0.9, ref9.TH_LOW_, masks != 0);
        const bool ok3 = b_ref == b_gpu && same_ids(va, vb) && b_ref > 50;
        std::printf("masks=%d SearchByBoW(KF,KF) ref=%d gpu=%d %s\n", masks, b_ref, b_gpu, ok3 ? "ok" : "MISMATCH");
        fails += !ok3;
    }
    std::printf("adapter_check %s\n", fails ? "FAILED" : "passed");
    return fails ? 1 : 0;
}
