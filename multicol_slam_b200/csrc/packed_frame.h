// packed_frame.h -- packed feature buffers (mcs_packed_layout) as the extractor (mcs_api.cu) writes them, and a frame in them
// (mcs_packed_frame) as the host entry points of the device searches (mcs_match_api.cu) and of the device bag of words
// (mcs_bow_api.cu) read it: the section pointers, and the argument checks the calls share.
#pragma once
#include <vector>
#include "../../include/mcs_b200.h"
#include "api_check.h"
#include "kernels.h"

namespace mcs {

// the features of n images: counts [n], keypoints, descriptors and descriptor masks [n][capacity] (each image's slot row)
struct FeatureView {
    int* counts; mcs_keypoint* kps; uint8_t* desc; uint8_t* dmask;
};

// the four sections of a packed feature buffer of n_images images at `base`
inline FeatureView packed_view(const void* base, int n_images, int capacity, int dim) {
    size_t off[4];
    mcs_packed_layout(n_images, capacity, dim, off);
    uint8_t* b = (uint8_t*)base;
    return FeatureView{(int*)(b + off[0]), (mcs_keypoint*)(b + off[1]), b + off[2], b + off[3]};
}

// `v` from image i on (a NULL dmask stays NULL)
inline FeatureView feature_at(const FeatureView& v, size_t i, int capacity, int dim) {
    const size_t slot = i * capacity;
    return FeatureView{v.counts + i, v.kps + slot, v.desc + slot * dim, v.dmask ? v.dmask + slot * dim : nullptr};
}

// appends the slots of cameras 0 .. n_cams - 1 of a packed frame to `slots`, so that the tables of several frames follow each other:
// camera c = global image first_image + c = image (g mod part_images) of part g / part_images
inline void append_slots(std::vector<PsCamSlots>& slots, const mcs_packed_frame& fr, int n_cams, int capacity, int dim) {
    const size_t part_bytes = mcs_packed_layout(fr.part_images, capacity, dim, nullptr);
    for (int c = 0; c < n_cams; ++c) {
        const int g = fr.first_image + c, p = g / fr.part_images, i = g - p * fr.part_images;
        const FeatureView v = feature_at(packed_view((const uint8_t*)fr.packed_dev + (size_t)p * part_bytes, fr.part_images, capacity, dim),
                                         i, capacity, dim);
        slots.push_back(PsCamSlots{v.counts, v.kps, v.desc, v.dmask});
    }
}

// the slot table of one packed frame
inline std::vector<PsCamSlots> packed_slots(const mcs_packed_frame& fr, int n_cams, int capacity, int dim) {
    std::vector<PsCamSlots> slots;
    append_slots(slots, fr, n_cams, capacity, dim);
    return slots;
}

inline bool packed_frame_ok(const mcs_packed_frame* fr, int n_cams) {
    return fr->packed_dev && fr->n_parts >= 1 && fr->part_images >= 1 && fr->first_image >= 0 &&
           (long long)fr->first_image + n_cams <= (long long)fr->n_parts * fr->part_images;
}

// the arguments of the frame the device searches search, and of the packed feature buffers the images of its cameras come from
// (`last`: the searches between two frames only)
inline int check_packed_frames(int n_cams, int capacity, int dim, const mcs_packed_frame* cur, const mcs_packed_frame* last) {
    if (n_cams < 1) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    if (capacity < 1 || capacity > 65535) return mcs_fail(MCS_ERR_INVALID, "capacity must be 1..65535");
    if (int rc = check_desc_dim(dim)) return rc;
    if (!packed_frame_ok(cur, n_cams)) return mcs_fail(MCS_ERR_INVALID, "current frame: no buffer, or first_image + n_cams exceeds its images");
    if (last && !packed_frame_ok(last, n_cams))
        return mcs_fail(MCS_ERR_INVALID, "last frame: no buffer, or first_image + n_cams exceeds its images");
    return MCS_OK;
}

// every camera's image size positive and, when `equal` (the searches that read the mirror masks as one [n_cams][h][w] array),
// the same for all cameras
inline int check_cam_sizes(int n_cams, const int* w, const int* h, bool equal) {
    for (int c = 0; c < n_cams; ++c) {
        if (w[c] < 1 || h[c] < 1) return mcs_fail(MCS_ERR_INVALID, "camera sizes must be positive");
        if (equal && (w[c] != w[0] || h[c] != h[0])) return mcs_fail(MCS_ERR_UNSUPPORTED, "cameras of different image sizes");
    }
    return MCS_OK;
}

// the device searches keep a query index in 24 bits (the owner words of the ordered acceptance); n is the call's bound on queries
inline int check_query_bound(long long n, const char* msg) {
    return n >= (1LL << 24) ? mcs_fail(MCS_ERR_UNSUPPORTED, msg) : MCS_OK;
}

// the end of an asynchronous entry point: a NULL stream (the legacy default stream) means the caller wants the results on return
inline int sync_if_null_stream(void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (!stream) CUDA_CHECK(cudaStreamSynchronize(st));
    return MCS_OK;
}

}  // namespace mcs
