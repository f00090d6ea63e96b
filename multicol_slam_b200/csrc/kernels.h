// kernels.h -- launchers exported by the .cu files to the C-ABI host layer (mcs_api.cu).
#pragma once
#include <vector>

#include "mcs_common.cuh"

namespace mcs {

struct DescribeArgs {
    const uint8_t* lvl[kMaxLevels];
    const uint8_t* blur[kMaxLevels];
    unsigned long long* tier_stats = nullptr;   // diagnostics (mcs_extractor_tier_stats): patterns decided by tier 1 / 2 / 3 of K3
};

cudaError_t upload_constants(const signed char* pairs, const signed char* du, const signed char* dv);
void launch_pyr_fast(const PyramidGeom& G, int level, int n_images, const uint8_t* src, size_t src_img_bytes,
                     uint8_t* dst, uint8_t* dst_blur, const uint8_t* mask0, int mask_w, size_t mask_bytes,
                     const int* cam_of_image, const uint8_t* tile_flags, uint32_t* raw, int* raw_count, cudaStream_t st);
cudaError_t launch_octree(const PyramidGeom& G, const PyramidGeom* G_dev, int n_images, const uint32_t* raw,
                          const int* raw_count, uint16_t* node_of, uint32_t* sel_xys, int* sel_count, int* status,
                          cudaStream_t st, int level_lo = 0, int level_count = -1);
// per-camera table of R(r) = rho(atan(-z/r)) (describe_kernel.cu): entry i is one degree-9 polynomial in
// tau = r * e[1] + e[0] valid on [max(0, i - 22.5), i + 22.5] -- every pattern point of a keypoint whose undistorted
// radius rounds to i; 12 doubles per entry (tau offset, tau scale, 10 coefficients)
struct DistortLut {
    const double* coef;
    int n;
    double inv_h;
};
void build_distort_lut(const mcs_ocam& cam, std::vector<double>& coef, int& n_out);
cudaError_t launch_describe(const PyramidGeom& G, const PyramidGeom* G_dev, int n_images, const DescribeArgs& args,
                            const mcs_ocam* cams, const DistortLut* luts, const int* cam_of_image, const uint32_t* sel_xys,
                            const int* sel_count, mcs_keypoint* kps, uint8_t* desc, uint8_t* dmask, int* counts, int capacity,
                            cudaStream_t st);

// matching (match_kernels.cu)
cudaError_t launch_hamming_topk(const uint8_t* q, const uint8_t* qmask, int nq, const uint8_t* d, const uint8_t* dmask,
                                int nd, const uint8_t* db_skip, int dim, int K, unsigned bound, int* topk_idx, int* topk_dist,
                                cudaStream_t st);
cudaError_t launch_hamming_stream(const uint8_t* desc, const uint8_t* dmask, const int* counts, int img_lo, int img_count,
                                  int n_cams, int capacity, int dim, int K, unsigned bound, int* out_idx, int* out_dist, cudaStream_t st);
// Relevance bound of the greedy acceptance rule (best1 < th_low && best1 < nnratio * best2, ref src/cORBmatcher.cpp:899-961): the
// smallest distance b >= th_low such that a second-best of b or more passes the ratio test for EVERY admissible best
// (best <= th_low - 1).  A database entry at distance >= b can neither be an accepted best nor make a ratio test fail, so the
// K-best kernels may leave it out of their lists (`bound` argument; 0xFFFFFFFF = keep everything) without changing any decision.
// cudaMallocAsync scratch: by default the device pool hands freed memory back to the driver at the next synchronisation, which
// turns every call's stream-ordered allocation into a real cudaMalloc, which costs several times the kernels of a
// mcs_match_stream_greedy_device call.  Keep freed blocks in the pool.
inline cudaError_t keep_pool_memory() {
    static bool done[64] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess || dev < 0 || dev >= 64 || done[dev]) return e;
    cudaMemPool_t pool;
    e = cudaDeviceGetDefaultMemPool(&pool, dev);
    if (e != cudaSuccess) return e;
    unsigned long long keep = ~0ull;
    e = cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    done[dev] = e == cudaSuccess;
    return e;
}

inline unsigned greedy_dist_bound(int th_low, double nnratio) {
    if (th_low <= 0) return 0u;                      // nothing can be accepted
    long b = th_low;
    while (b < (1L << 20) && !((double)(th_low - 1) < nnratio * (double)b)) ++b;
    return (unsigned)b;
}
cudaError_t launch_stream_replay(const int* list_idx, const int* list_dist, const int* counts, const uint8_t* desc, const uint8_t* dmask,
                                 int dim, int img_lo, int n_images, int n_cams, int capacity, int K, int th_low, double nnratio,
                                 int* matches12, int* nmatches, int* redo, cudaStream_t st);
cudaError_t launch_bruteforce_replay(const int* list_idx, const int* list_dist, int K, const uint8_t* q, const uint8_t* qm, const uint8_t* valid1,
                                     const int* seg, int n_seg, int nq_total, const uint8_t* d, const uint8_t* dm, const uint8_t* valid2, int nd, int dim,
                                     int th_low, double nnratio, int* matches12, int* nmatches, cudaStream_t st);
void launch_repitch(const uint8_t* src, int src_stride, uint8_t* dst, int dst_pitch, int width, size_t rows, cudaStream_t st);
struct WindowFrameDev {
    int n_cams, n_keys, dim;
    const float* kx; const float* ky; const int* koct;      // [n_keys]
    const uint8_t* desc; const uint8_t* dmask;              // [n_keys*dim]
    const int* cell_start;                                  // [n_cams*64*48 + 1] CSR over (cam, ix, iy)
    const int* cell_items;                                  // [n_in_grid] keypoint ids, ascending inside a cell
    const double* winv; const double* hinv;                 // [n_cams]
    // MCS_RULE_SCW only: [n_cams + 1] first contiguous keypoint id of every camera.  When set, candidate `id` of a query of
    // camera c is compared through descriptor row cam_first[c] + id -- the reference indexes camera c's matrix with the
    // contiguous id (src/cORBmatcher.cpp:2367,2372) -- and dropped when that row lies beyond the camera's own rows.
    const int* cam_first = nullptr;
};
cudaError_t launch_window_search(const WindowFrameDev& f, const mcs_window_query* q, int nq, const uint8_t* qdesc,
                                 const uint8_t* qmask, int max_cand, int* cand_idx, int* cand_dist, int* cand_count,
                                 cudaStream_t st);
cudaError_t launch_compact_lists(const int* idx, const int* dist, const int* count, const int* off, int nq, int max_cand, int* oidx, int* odist,
                                 cudaStream_t st);

cudaError_t launch_frame_prepare(const mcs_keypoint* keys, const int* key_cam, int n_keys, const mcs_ocam* cams, int n_cams, float* kx,
                                 float* ky, int* koct, double* rays, int* cell_of, int* cursor, int* cell_start, int* cell_items,
                                 double* winv, double* hinv, cudaStream_t st);
cudaError_t launch_frustum(int n_cams, const double* mtmc_inv, const double* mtmc, const mcs_ocam* cams, const uint8_t* masks,
                           int n_points, const double* pos, const double* nrm, const double* dmin, const double* dmax, const double* sf,
                           int n_levels, uint8_t* in_view, int* level, double* px, double* py, double* vcos, cudaStream_t st);

// ---- bag of words (bow_kernels.cu) ----
// vocabulary tree on the device: CSR children in the reference's order, 32-byte node descriptors as uint4 pairs
struct VocabularyDev {
    const int* child_off;        // [n_nodes + 1]
    const int* child_ids;        // [n_nodes - 1]
    const uint4* desc;           // [2 * n_nodes]
    const int* word_of_node;     // [n_nodes], -1 for inner nodes
    const double* weight;        // [n_nodes]
    int n_nodes, L;
};
cudaError_t launch_bow_descend(const VocabularyDev& v, const uint8_t* desc, int n, int levelsup, int* word, double* weight,
                               int* node, cudaStream_t st);
// one query of the feature-vector guided search: key-frame keypoint `feature` against cand[cand_start .. +cand_count)
struct GroupQuery { int feature, cand_start, cand_count, out_off; };
cudaError_t launch_group_distance(const GroupQuery* queries, int nq, const uint8_t* desc1, const uint8_t* mask1, const uint8_t* desc2,
                                  const uint8_t* mask2, const int* cand, int dim, int* out, cudaStream_t st);

}  // namespace mcs
