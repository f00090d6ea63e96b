// kernels.h -- launchers exported by the .cu files to the C-ABI host layer (mcs_api.cu, mcs_match_api.cu, mcs_bow_api.cu).
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
cudaError_t launch_pyr_fast(const PyramidGeom& G, int level, int n_images, const uint8_t* src, size_t src_img_bytes,
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

// streaming multiprocessors of the current device
inline cudaError_t sm_count(int& n) {
    int dev = 0;
    const cudaError_t e = cudaGetDevice(&dev);
    return e != cudaSuccess ? e : cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
}

// One stream-ordered scratch block cut into pieces, each starting on a 256-byte boundary; a size of 0 gives a zero-length piece.
class StreamScratch {
public:
    // keep_pool_memory(), then one cudaMallocAsync on `st` holding every piece
    cudaError_t alloc(const std::vector<size_t>& sizes, cudaStream_t st) {
        off_.assign(1, 0);
        for (const size_t b : sizes) off_.push_back(off_.back() + ((b + 255) & ~(size_t)255));
        cudaError_t e = keep_pool_memory();
        if (e != cudaSuccess) return e;
        st_ = st;
        return cudaMallocAsync((void**)&base_, off_.back(), st);
    }
    template <class T> T* at(size_t i) const { return (T*)(base_ + off_[i]); }
    // frees the block in stream order, if alloc made one; returns e, or the free's error when e is cudaSuccess
    cudaError_t release(const cudaError_t e) {
        if (!base_) return e;
        const cudaError_t ef = cudaFreeAsync(base_, st_);
        base_ = nullptr;
        return e != cudaSuccess ? e : ef;
    }

private:
    std::vector<size_t> off_;
    uint8_t* base_ = nullptr;
    cudaStream_t st_ = nullptr;
};

// Copies small host data into device memory in stream order through kernel parameters, so that the calling thread never waits
// for the stream (a cudaMemcpyAsync from pageable memory may).  Defined in proj_search_kernels.cu.
cudaError_t stage_to_device(const void* host, size_t bytes, void* dev, cudaStream_t st);

// One small host input of a launcher: n elements at `host`, staged into the launcher's scratch; `dev` receives the device copy.
template <class T> struct HostIn { const T*& dev; const T* host; size_t n; };
template <class T> HostIn<T> host_in(const T*& dev, const T* host, size_t n) { return {dev, host, n}; }

// A launcher's one stream-ordered scratch block: its own pieces first (own[i] is sc.at<T>(i)), then a device copy of every host
// input, staged in stream order.  The caller releases sc, whatever the result.
template <class... T>
cudaError_t open_scratch(StreamScratch& sc, std::vector<size_t> own, cudaStream_t st, const HostIn<T>&... in) {
    size_t i = own.size();
    (own.push_back(sizeof(T) * in.n), ...);
    cudaError_t e = sc.alloc(own, st);
    if (e != cudaSuccess) return e;
    ((in.dev = sc.at<T>(i++)), ...);
    ((e = e == cudaSuccess ? stage_to_device(in.host, sizeof(T) * in.n, (void*)in.dev, st) : e), ...);
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
// Most dynamic shared memory an acceptance kernel is launched with: the stream matcher keeps the previous image resident only
// below it, and the key-frame database is refused above it.
constexpr size_t kReplaySmemMax = 200 * 1024;
// Dynamic shared memory of bruteforce_replay_kernel: the [32][K] list chunk (indices and distances) and the leader's "already
// matched" bitmap of the whole database.  The launcher refuses more than kReplaySmemMax, so the key-frame database holds at
// most bruteforce_max_nd(K) entries.
inline size_t bruteforce_replay_smem(int K, int nd) { return (size_t)64 * K * 4 + (size_t)((nd + 31) / 32) * 4; }
inline int bruteforce_max_nd(int K) { return (int)((kReplaySmemMax - bruteforce_replay_smem(K, 0)) / 4 * 32); }
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
    // contiguous id (src/cORBmatcher.cpp:2367,2372) -- and dropped when that row lies beyond the camera's own rows.  The device
    // search (launch_search_by_projection_scw) reads those rows in its frame view already and uses cam_first only to find
    // contiguous keypoint 0.
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
// skip (may be NULL): [n_points] bytes; the outputs of a flagged point are left untouched
cudaError_t launch_frustum(int n_cams, const double* mtmc_inv, const double* mtmc, const mcs_ocam* cams, const uint8_t* masks,
                           int n_points, const double* pos, const double* nrm, const double* dmin, const double* dmax, const double* sf,
                           int n_levels, uint8_t* in_view, int* level, double* px, double* py, double* vcos, const uint8_t* skip,
                           cudaStream_t st);

// device-resident SearchByProjection (proj_search_kernels.cu)
struct PsCamSlots {                     // camera c of the frame: its image slot inside the packed feature buffer
    const int* count; const mcs_keypoint* kps; const uint8_t* desc; const uint8_t* dmask;
};
struct PsFrameArgs {                    // both searches: the frame searched, the acceptance threshold, the outputs
    int n_cams, capacity, dim, n_levels;
    const PsCamSlots* cams;                                  // host [n_cams] (device pointers inside)
    const int* cam_w; const int* cam_h; const double* sf;    // host; the sizes are read only by searches without camera models
    int th_high; bool masked;
    int* frame_mp; int* nmatches; int* status; int* diag;    // device
};
struct ProjSearchArgs : PsFrameArgs {   // SearchByProjection(F, vpMapPoints, th)
    int n_points;
    const uint8_t* bad; const uint8_t* in_view; const int* level;              // device map-point arrays
    const double* px; const double* py; const double* vcos;
    const uint8_t* mp_desc; const uint8_t* mp_dmask;
    double th, nnratio;
};
cudaError_t launch_search_by_projection(const ProjSearchArgs& a, cudaStream_t st);
// The searches between two frames: the frame searched (PsFrameArgs) is the current one, the queries come from the last frame.
struct PsTwoFrameArgs : PsFrameArgs {
    const PsCamSlots* last;                                  // host [n_cams]: the last frame's image slots
    int n_points;
    const int* last_mp; const uint8_t* bad;                  // device, slot-indexed / [n_points] (bad may be NULL)
    // the current pose, for the searches that project (NULL for WindowSearch)
    const mcs_ocam* models; const double* mtmc_inv;          // host [n_cams], [n_cams * 16]
    const uint8_t* masks;                                    // device [n_cams][h][w] level-0 mirror masks
    const double* world_pos;                                 // device [n_points * 3]
};
struct ProjSearchLastArgs : PsTwoFrameArgs {   // SearchByProjection(CurrentFrame, LastFrame, th)
    const uint8_t* last_outlier;                             // device, slot-indexed (may be NULL)
    double th;
};
cudaError_t launch_search_by_projection_last(const ProjSearchLastArgs& a, cudaStream_t st);
// TrackPreviousFrame's searches, F1 = the last frame, F2 = the frame searched.  Neither reads scale factors (n_levels = 0, sf NULL).
struct WindowSearchDevArgs : PsTwoFrameArgs {   // WindowSearch(F1, F2, window, ., min_level, max_level): frame_mp is an output
    double window, nnratio; int min_level, max_level;
};
cudaError_t launch_window_search_device(const WindowSearchDevArgs& a, cudaStream_t st);
struct SearchFramesDevArgs : PsTwoFrameArgs {   // SearchByProjection(F1, F2, window, .): frame_mp holds F2.mvpMapPoints on entry
    double window, nnratio;
};
cudaError_t launch_search_by_projection_frames(const SearchFramesDevArgs& a, cudaStream_t st);
// SearchForInitialization(F1 = last, F2 = cur, vbPrevMatched, vnMatches12, window): th_high holds TH_LOW_; frame_mp, status,
// last_mp, the map points and the pose are unused (NULL)
struct InitSearchDevArgs : PsTwoFrameArgs {
    double* prev;                                            // device [n_cams * capacity * 2], F1 slot-indexed, in/out
    int* matches12;                                          // device [n_cams * capacity], F1 slot-indexed: the F2 slot or -1
    int window; double nnratio;
};
cudaError_t launch_search_for_initialization(const InitSearchDevArgs& a, cudaStream_t st);
// prev = the position of every F1 keypoint below its camera's count (f1: host [n_cams])
cudaError_t launch_search_for_initialization_seed(const PsCamSlots* f1, int n_cams, int capacity, double* prev, cudaStream_t st);
int proj_search_max_rounds();
// The map points Fuse, SearchBySim3 and SearchByProjection(KF, Scw) project, and the cameras they are projected into.
struct PsMapPoints {
    int n_points;
    const double* world_pos; const double* min_dist; const double* max_dist;   // device [n_points * 3], [n_points], [n_points]
    const uint8_t* desc; const uint8_t* dmask; const uint8_t* bad;             // device (dmask NULL unless masked, bad may be NULL)
    const mcs_ocam* models; const uint8_t* masks;                              // host [cameras], device [cameras][h][w]
};
// The Fuse overloads (mcs_fuse_device) for n_kf key frames in one call: the searched frame (PsFrameArgs) is the n_kf * n_cams
// images of the targets, image k * n_cams + c = camera c of key frame k; th_high holds TH_LOW_; frame_mp and nmatches are unused.
struct FuseDevArgs : PsFrameArgs {
    int n_kf, n_kf_cams, variant, n_q;                        // n_kf_cams: cameras per key frame, the models' count
    const int* const* kf_mp;                                 // host [n_kf]: each key frame's slot-indexed map-point ids (NULL entries)
    const double* mtmc_inv; const double* ow;                // host [n_kf * n_kf_cams * 16], [n_kf * 3]
    const int* query_mp;                                     // device [n_q], -1 = NULL
    PsMapPoints pts;
    double th;
    int* hits; int max_hits; int* n_hits;                    // device [max_hits * 3], [1]
};
cudaError_t launch_fuse_device(const FuseDevArgs& a, cudaStream_t st);
// SearchBySim3(KF1, KF2, .) (mcs_search_by_sim3_device): PsFrameArgs is KF2 (cams) with th_high = TH_HIGH_; nmatches is nFound;
// frame_mp and diag are unused.
struct Sim3SearchDevArgs : PsFrameArgs {
    const PsCamSlots* kf1;                                   // host [n_cams]
    const double* xf;                                        // host [48]: per direction R[9] t[3] sR[9] st[3] (direction 1, then 2)
    const double* mc_inv;                                    // host [n_cams * 16]: invMat(Get_M_c(c))
    double th;
    PsMapPoints pts;
    const int* mp1; const int* mp2;                          // device, slot-indexed
    const uint8_t* already2;                                 // device, KF2 slot-indexed, may be NULL
    int* matches12;                                          // device, KF1 slot-indexed, in/out
};
cudaError_t launch_search_by_sim3(const Sim3SearchDevArgs& a, cudaStream_t st);
// SearchByProjection(pKF, Scw, vpPoints, vpMatched, th) (mcs_search_by_projection_scw_device): PsFrameArgs is the key frame with
// th_high = TH_LOW_ and frame_mp = vpMatched (slot-indexed, in/out).
struct ScwSearchDevArgs : PsFrameArgs {
    const double* mtmc_inv; const double* ow;                // host [n_cams * 16], [3]: the Sim3's rigid pose
    int n_q;
    const int* points;                                       // device [n_q], -1 = NULL
    PsMapPoints pts;
    int th;
};
cudaError_t launch_search_by_projection_scw(const ScwSearchDevArgs& a, cudaStream_t st);

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

// ComputeBoW on a frame in packed feature buffers (mcs_bow_vectors_device): every output in device memory, slot-indexed
struct BowVectorsDevArgs {
    int n_cams, capacity, levelsup, max_nodes;
    int n_words, scoring, weighting;                           // of the vocabulary
    const PsCamSlots* cams;                                    // host [n_cams] (device pointers inside)
    int* word; double* weight; int* node;                      // [n_cams * capacity], each may be NULL
    int* fv_nodes; int* fv_offsets; int* n_fv; int* fv_features;
    int* bow_words; double* bow_values; int* n_bow; int* status;
};
cudaError_t launch_bow_vectors_device(const VocabularyDev& v, const BowVectorsDevArgs& a, cudaStream_t st);

// SearchByBoW(KF_i, F) for a batch of key frames (mcs_search_by_bow_device)
struct BowFrameDev {                                           // the device arrays of one mcs_bow_frame
    const int* fv_nodes; const int* fv_offsets; const int* n_fv; const int* fv_features; const int* mp;
};
struct BowSearchDevArgs {
    int n_kf, n_cams, capacity, dim, max_nodes, n_points, th_low;
    double nnratio; bool masked;
    const PsCamSlots* kf_cams;                                 // host [n_kf * n_cams]
    const PsCamSlots* cur_cams;                                // host [n_cams]
    const BowFrameDev* kfs;                                    // host [n_kf]
    BowFrameDev cur;
    const uint8_t* bad;                                        // device [n_points], may be NULL
    int* match_mp; int* match_slot; int* nmatches; int* status;   // device; match_slot may be NULL
};
cudaError_t launch_search_by_bow_device(const BowSearchDevArgs& a, cudaStream_t st);

// SearchByBoW(KF1, KF_k) for n_kf candidate key frames (mcs_search_by_bow_keyframes_device, match_kernels.cu).  The launcher refuses
// nothing: the host entry point has checked n_cams * capacity <= bruteforce_max_nd(kTopKMax) and n_kf * n_cams * capacity < 2^31.
struct BowKfSearchDevArgs {
    int n_kf, n_cams, capacity, dim, n_points, th_low;
    double nnratio; bool masked;
    const PsCamSlots* cams;                                    // host [(1 + n_kf) * n_cams]: KF1's cameras, then each candidate's
    const int* const* mp;                                      // host [1 + n_kf]: the frames' slot-indexed map-point ids (device)
    const uint8_t* bad;                                        // device [n_points], may be NULL
    int* matches12; int* match_slot; int* nmatches; int* status;   // device; match_slot may be NULL
};
cudaError_t launch_search_by_bow_keyframes(const BowKfSearchDevArgs& a, cudaStream_t st);

// SearchForTriangulationRaw(KF1, KF2) (mcs_search_for_triangulation_device, match_kernels.cu).  The launcher refuses nothing: the host
// entry point has checked capacity <= 65535 and n_cams * capacity < 2^24.
struct TriSearchDevArgs {
    int n_cams, capacity, dim, th_low;
    bool masked; double epi_thresh;
    const PsCamSlots* cams;                                    // host [2 * n_cams]: KF1's cameras, then KF2's
    const int* mp[2];                                          // device, slot-indexed map-point ids of KF1 / KF2 (-1 = free)
    const mcs_ocam* models;                                    // host [n_cams]
    const double* E;                                           // host [n_cams][9]: the diagonal blocks E[c][c]
    int* matches12; int* nmatches; int* diag;                  // device; diag may be NULL
};
cudaError_t launch_search_for_triangulation(const TriSearchDevArgs& a, cudaStream_t st);

}  // namespace mcs
