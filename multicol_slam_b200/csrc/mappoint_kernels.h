// mappoint_kernels.h -- the launcher of mappoint_kernels.cu (cMapPoint::ComputeDistinctiveDescriptors and UpdateNormalAndDepth for
// many map points) as the C-ABI host layer (mcs_mappoint_api.cu) calls it.
#pragma once
#include "kernels.h"

namespace mcs {

struct MpUpdateArgs {
    int n_kf, n_cams, capacity, dim, n_levels, what;
    bool masked;
    const PsCamSlots* slots;              // host [n_kf * n_cams]: camera c of key frame k is slots[k * n_cams + c]
    const int* kf_bad;                    // host [n_kf]
    const double* kf_ow;                  // host [n_kf * 3]
    const double* sf;                     // host [n_levels]
    const int* ids; int n_upd, n_points;  // device from here on
    const int* obs_off; const int* obs_kf; const int* obs_slot;
    const int* ref_kf; const uint8_t* bad; const double* world_pos;
    uint8_t* desc; uint8_t* dmask; double* normal; double* min_dist; double* max_dist;
    int* status;
};

cudaError_t launch_update_mappoints(const MpUpdateArgs& a, cudaStream_t st);

}  // namespace mcs
