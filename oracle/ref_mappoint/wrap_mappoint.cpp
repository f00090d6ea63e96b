// wrap_mappoint.cpp -- flat C entry point into the reference's own cMapPoint (src/cMapPoint.cpp, compiled where it lies against
// stub_mappoint.h): builds one real cMapPoint over stand-in key frames, calls AddObservation for each listed observation and then
// UpdateNormalAndDepth() and/or ComputeDistinctiveDescriptors(havingMasks), and returns what the device tables hold for the point.
// TEST INFRASTRUCTURE (oracle/ref_mappoint_api.py).
//
// DescriptorDistance64 / DescriptorDistance64Masked are the reference's own, from src/cORBmatcher.cpp as compiled into
// _ref/libmcs_ref.so: that library is opened RTLD_LOCAL and the two functions are called through pointers, so its stand-in
// cMapPoint never meets the real one.
#include <dlfcn.h>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "cMapPoint.h"

namespace {
using D64 = int (*)(const uint64_t*, const uint64_t*, const int&);
using D64M = int (*)(const uint64_t*, const uint64_t*, const uint64_t*, const uint64_t*, const int&);
D64 g_d64 = nullptr;
D64M g_d64m = nullptr;
}  // namespace

namespace MultiColSLAM
{
int DescriptorDistance64(const uint64_t* a, const uint64_t* b, const int& dim) { return g_d64(a, b, dim); }
int DescriptorDistance64Masked(const uint64_t* a, const uint64_t* b, const uint64_t* ma, const uint64_t* mb, const int& dim)
{
	return g_d64m(a, b, ma, mb, dim);
}
}  // namespace MultiColSLAM

using namespace MultiColSLAM;

extern "C" {

// the reference matcher library the distances come from; 0 on success
int refmp_init(const char* libmcs_ref_path) {
    void* h = dlopen(libmcs_ref_path, RTLD_NOW | RTLD_LOCAL);
    if (!h) return -1;
    g_d64 = (D64)dlsym(h, "_ZN12MultiColSLAM20DescriptorDistance64EPKmS1_RKi");
    g_d64m = (D64M)dlsym(h, "_ZN12MultiColSLAM26DescriptorDistance64MaskedEPKmS1_S1_S1_RKi");
    return g_d64 && g_d64m ? 0 : -2;
}

// One map point.  Key frame k: desc / dmask [n_kf][n_cams * capacity][dim] and octave [n_kf][n_cams * capacity] by slot
// c * capacity + j (the slot is the observation index handed to AddObservation, keypoint_to_cam / cont_idx_to_local_cam_idx map it
// to (c, j)), ow [n_kf][3], kf_bad [n_kf].  Observations (obs_kf, obs_slot) [n_obs] in AddObservation order; ref_kf indexes the
// key frames.  Outputs: desc_set (mDescriptor non-empty after the call), out_desc / out_dmask [dim] (mask only when having_masks
// and set), out_nd [5] = GetNormal() (3), GetMinDistanceInvariance(), GetMaxDistanceInvariance(); order [n_kf]: the key-frame
// indices in mObservations iteration order (n_order of them).
int refmp_update(int n_kf, int n_cams, int capacity, int dim, const uint8_t* desc, const uint8_t* dmask, const int* octave,
                 const double* ow, const int* kf_bad, int n_levels, const double* sf, int n_obs, const int* obs_kf, const int* obs_slot,
                 int ref_kf, const double* X, int point_bad, int what, int having_masks, int* desc_set, int* mask_set, uint8_t* out_desc,
                 uint8_t* out_dmask, double* out_nd, int* order, int* n_order) {
    if (!g_d64) return -1;
    const int NS = n_cams * capacity;
    std::vector<std::unique_ptr<cMultiKeyFrame>> kfs;
    for (int k = 0; k < n_kf; ++k) {
        kfs.emplace_back(new cMultiKeyFrame());
        cMultiKeyFrame& f = *kfs.back();
        f.mnId = k;
        f.camSystem.nCams = n_cams;
        f.bad = kf_bad[k] != 0;
        f.masksLearned = having_masks != 0;
        f.ow = cv::Vec3d(ow[3 * k], ow[3 * k + 1], ow[3 * k + 2]);
        f.dim = dim;
        for (int c = 0; c < n_cams; ++c) {
            cv::Mat d(capacity, dim, CV_8UC1), m(capacity, dim, CV_8UC1);
            std::memcpy(d.data, desc + ((size_t)k * NS + (size_t)c * capacity) * dim, (size_t)capacity * dim);
            std::memcpy(m.data, dmask + ((size_t)k * NS + (size_t)c * capacity) * dim, (size_t)capacity * dim);
            f.desc.push_back(d);
            f.dmask.push_back(m);
        }
        f.octave.assign(octave + (size_t)k * NS, octave + (size_t)(k + 1) * NS);
        f.mvScaleFactors.assign(sf, sf + n_levels);
        f.mnScaleLevels = n_levels;
        for (int s = 0; s < NS; ++s) {
            f.keypoint_to_cam[s] = s / capacity;
            f.cont_idx_to_local_cam_idx[s] = s % capacity;
        }
    }
    cMap map;
    cMapPoint mp(cv::Vec3d(X[0], X[1], X[2]), kfs[ref_kf].get(), &map);
    for (int e = 0; e < n_obs; ++e) mp.AddObservation(kfs[obs_kf[e]].get(), (size_t)obs_slot[e]);
    if (point_bad) mp.SetBadFlag();
    if (what & 2) mp.UpdateNormalAndDepth();
    if (what & 1) mp.ComputeDistinctiveDescriptors(having_masks != 0);
    const cv::Mat d = mp.GetDescriptor(), m = mp.GetDescriptorMask();
    *desc_set = !d.empty();
    *mask_set = !m.empty();
    if (*desc_set) std::memcpy(out_desc, d.data, dim);
    if (*mask_set) std::memcpy(out_dmask, m.data, dim);
    const cv::Vec3d n = mp.GetNormal();
    out_nd[0] = n[0]; out_nd[1] = n[1]; out_nd[2] = n[2];
    out_nd[3] = mp.GetMinDistanceInvariance();
    out_nd[4] = mp.GetMaxDistanceInvariance();
    *n_order = 0;
    for (const auto& o : mp.GetObservations())
        order[(*n_order)++] = (int)o.first->mnId;
    return 0;
}

}  // extern "C"
