// mcs_mappoint_api.cu -- C-ABI host layer of the map-point table update (include/mcs_b200.h, mcs_update_mappoints_device): the
// argument checks, the key frames' packed-buffer slots and the launch of mappoint_kernels.cu.  Nothing is read back.
#include <vector>

#include "api_check.h"
#include "mappoint_kernels.h"
#include "packed_frame.h"

using namespace mcs;

extern "C" {

int mcs_update_mappoints_device(const mcs_mp_keyframe* kfs, int32_t n_kf, int32_t n_cams, int32_t capacity, int32_t dim,
                                int32_t n_levels, const double* scale_factors, int32_t what, int32_t having_masks,
                                const int32_t* point_ids_dev, int32_t n_upd, int32_t n_points, const int32_t* obs_offsets_dev,
                                const int32_t* obs_kf_dev, const int32_t* obs_slot_dev, const int32_t* ref_kf_dev, const uint8_t* bad_dev,
                                const double* world_pos_dev, uint8_t* desc_dev, uint8_t* dmask_dev, double* normal_dev,
                                double* min_dist_dev, double* max_dist_dev, int32_t* status_dev, void* stream) {
    const bool want_desc = (what & MCS_MP_DESCRIPTOR) != 0, want_nd = (what & MCS_MP_NORMAL_DEPTH) != 0;
    if (what < 1 || what > (MCS_MP_DESCRIPTOR | MCS_MP_NORMAL_DEPTH)) return mcs_fail(MCS_ERR_INVALID, "what must select MCS_MP_DESCRIPTOR and/or MCS_MP_NORMAL_DEPTH");
    // point_ids_dev may be NULL only when it has no entry (an empty tensor has no address)
    if (!kfs || !scale_factors || (!point_ids_dev && n_upd > 0) || !obs_offsets_dev || !obs_kf_dev || !obs_slot_dev || !status_dev)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (want_desc && (!desc_dev || (having_masks && !dmask_dev))) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (want_nd && (!ref_kf_dev || !world_pos_dev || !normal_dev || !min_dist_dev || !max_dist_dev))
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (n_kf < 1 || n_upd < 0 || n_points < 0 || n_levels < 1 || n_levels > MCS_MAX_LEVELS) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    for (int k = 0; k < n_kf; ++k)
        if (int rc = check_packed_frames(n_cams, capacity, dim, &kfs[k].frame, nullptr)) return rc;
    if ((long long)n_cams * capacity > INT32_MAX) return mcs_fail(MCS_ERR_UNSUPPORTED, "n_cams * capacity must fit a 32-bit slot");
    std::vector<PsCamSlots> slots;
    std::vector<int> kf_bad(n_kf);
    std::vector<double> kf_ow(3 * (size_t)n_kf);
    for (int k = 0; k < n_kf; ++k) {
        append_slots(slots, kfs[k].frame, n_cams, capacity, dim);
        kf_bad[k] = kfs[k].bad != 0;
        for (int i = 0; i < 3; ++i) kf_ow[3 * k + i] = kfs[k].ow[i];
    }
    MpUpdateArgs a{};
    a.n_kf = n_kf; a.n_cams = n_cams; a.capacity = capacity; a.dim = dim; a.n_levels = n_levels; a.what = what;
    a.masked = want_desc && having_masks != 0;
    a.slots = slots.data(); a.kf_bad = kf_bad.data(); a.kf_ow = kf_ow.data(); a.sf = scale_factors;
    a.ids = point_ids_dev; a.n_upd = n_upd; a.n_points = n_points;
    a.obs_off = obs_offsets_dev; a.obs_kf = obs_kf_dev; a.obs_slot = obs_slot_dev;
    a.ref_kf = ref_kf_dev; a.bad = bad_dev; a.world_pos = world_pos_dev;
    a.desc = desc_dev; a.dmask = a.masked ? dmask_dev : nullptr;
    a.normal = normal_dev; a.min_dist = min_dist_dev; a.max_dist = max_dist_dev; a.status = status_dev;
    cudaStream_t st = (cudaStream_t)stream;
    CUDA_CHECK(launch_update_mappoints(a, st));
    return sync_if_null_stream(stream);
}

}  // extern "C"
