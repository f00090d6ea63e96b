// proj_search_kernels.cu -- SearchByProjection(F, vpMapPoints, th) (ref src/cORBmatcher.cpp:67-166), the motion-model
// SearchByProjection(CurrentFrame, LastFrame, th) (ref :1990-2118) and TrackPreviousFrame's WindowSearch(F1, F2) (:326-473) and
// SearchByProjection(F1, F2, window) (:476-577) with every input and output resident on the device: the frames come straight from
// packed feature buffers (mcs_packed_layout), the map points from device arrays, and the reference's ordered greedy acceptance
// runs on the device.
//
//   ps_gather_kernel    a frame's keypoints / descriptors / masks in slot order (slot = cam * capacity + j); empty slots get a
//                       position outside every image, so the unchanged frame_prepare_kernel leaves them out of the grid.
//                       <true>: SearchByProjection(KF, Scw)'s descriptor rows, first[cam] + j
//   pl_project_kernel   motion model only: per last-frame slot, its map point projected with the current pose into its camera
//   pw_clear_kernel     WindowSearch only: the searched frame's assignments start free
//   pf_flag / pf_project  SearchByProjection(F1, F2) only: "already found" and first-slot flags per map point, then per
//                       (last-frame slot, camera) the slot's map point projected with the current pose into that camera
//   ps_count / ps_fill  the query array in the reference's order, a count / scan / fill over a query maker: map point outer,
//                       camera inner over in_view and bad (MapPointQueries), last-frame slot order (LastFrameQueries,
//                       WindowQueries), or last-frame slot outer, camera inner (FramesQueries)
//   ps_list_kernel      per query the K smallest (distance, visiting position) keys of its window and the true candidate count
//   ps_round_kernel     one round of the fixpoint iteration of the ordered acceptance (DESIGN.md section 4)
//   ps_walk_kernel      the sequential fallback past the round cap: one warp per camera walks the unsettled queries in order
//                       Both are templates over (rule, width, mask): MCS_RULE_LEVEL_RATIO for the local map, MCS_RULE_BEST for
//                       the motion model, MCS_RULE_RATIO for the previous-frame searches
//   pi_walk_kernel      SearchForInitialization(F1, F2) (:579-726) only: its acceptance can take a keypoint back from an earlier
//                       query, so it runs no rounds; one warp per camera walks the camera's queries in order (InitQueries: one per
//                       F1 slot) and writes matches12 and the survivors' prev.  pi_seed_kernel: FirstInitialization's prev
//   fu_*                the Fuse overloads (:1265, :1420, :1570) for n_kf key frames searched as one frame of n_kf * n_cams
//                       images: membership pre-filter, (key frame, query, camera) projections (ProjectedQueries), a stateless
//                       decision per query (fu_best / fu_first) and the hit rows in the reference's order
//
// No kernel reads anything back to the host: every size that depends on the data (the number of queries, the rounds the
// fixpoint needed, where the walk starts) lives in device memory and the kernels are launched for the upper bound.
#include <algorithm>
#include <climits>
#include <cstring>
#include <type_traits>
#include <vector>

#include "cam_model.cuh"
#include "kernels.h"

namespace mcs {

// ------------------------------------------------------------------------------------------------
// small host inputs, staged through a kernel parameter: a pageable cudaMemcpyAsync may wait for the stream
// ------------------------------------------------------------------------------------------------
namespace {
constexpr int kStageBytes = 3968;
struct StageBlob { unsigned char b[kStageBytes]; };
__global__ void stage_kernel(const StageBlob blob, const int n, unsigned char* __restrict__ dst) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = blob.b[i];
}
}  // namespace

cudaError_t stage_to_device(const void* host, size_t bytes, void* dev, cudaStream_t st) {
    const unsigned char* src = (const unsigned char*)host;
    for (size_t off = 0; off < bytes; off += kStageBytes) {
        const int n = (int)std::min<size_t>(kStageBytes, bytes - off);
        StageBlob blob;
        std::memcpy(blob.b, src + off, n);
        stage_kernel<<<1, 256, 0, st>>>(blob, n, (unsigned char*)dev + off);
    }
    return cudaGetLastError();
}

namespace {

constexpr int kPsK = 8;                      // list length per query
constexpr int kPsRounds = 8;                 // fixpoint rounds before the walk takes over
constexpr unsigned kNoKey = 0xFFFFFFFFu;
constexpr int kNoChange = 0x7F7F7F7F;        // memset(0x7F): no decision changed in that round
constexpr int kQbThreads = 256, kQbPer = 8, kQbTile = kQbThreads * kQbPer;
static_assert(kPsRounds < 255, "round versions live in the top byte of the owner words");

// slot s = c * capacity + j of a frame's slot table lies below camera c's count
__device__ __forceinline__ bool ps_live(const PsCamSlots* cams, const int capacity, const int s) {
    const int c = s / capacity;
    return s - c * capacity < min(*cams[c].count, capacity);
}

// ---- frame view from the packed slots ----
// Slot c * capacity + j carries keypoint j of camera c with the descriptor and mask of row j, or with SCW_ROWS those of row
// first[c] + j (SearchByProjection(KF, Scw) compares candidate idx through GetDescriptorRowPtr(camIdx, idx), idx the contiguous
// id, ref :2367, :2372); a keypoint whose row lies at or beyond the camera's count is left out like an empty slot.
template <bool SCW_ROWS>
__global__ void ps_gather_kernel(const PsCamSlots* __restrict__ cams, const int* __restrict__ first, const int n_cams, const int capacity,
                                 const int dim, const bool masked, mcs_keypoint* __restrict__ keys, int* __restrict__ key_cam,
                                 uint8_t* __restrict__ desc, uint8_t* __restrict__ dmask) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_cams * capacity) return;
    const int c = s / capacity, j = s - c * capacity;
    const PsCamSlots cs = cams[c];
    const int n = min(*cs.count, capacity), row = SCW_ROWS ? first[c] + j : j;
    if (key_cam) key_cam[s] = c;          // NULL: a frame that is only read by slot, never through a grid
    const int v4 = dim / 16;
    if (j < n && (!SCW_ROWS || row < n)) {
        keys[s] = cs.kps[j];
        for (int k = 0; k < v4; ++k) ((uint4*)desc)[(size_t)s * v4 + k] = ((const uint4*)cs.desc)[(size_t)row * v4 + k];
        if (masked)
            for (int k = 0; k < v4; ++k) ((uint4*)dmask)[(size_t)s * v4 + k] = ((const uint4*)cs.dmask)[(size_t)row * v4 + k];
    } else {
        mcs_keypoint e{};
        e.x = e.y = -1.0e6f;                 // PosInGrid falls outside the image: never a candidate
        keys[s] = e;
        for (int k = 0; k < v4; ++k) ((uint4*)desc)[(size_t)s * v4 + k] = make_uint4(0, 0, 0, 0);
        if (masked)
            for (int k = 0; k < v4; ++k) ((uint4*)dmask)[(size_t)s * v4 + k] = make_uint4(0, 0, 0, 0);
    }
}

// ---- motion model: which last-frame slots make a query (ref :1997-2029) ----
// Slot s = c * capacity + j (j < camera c's count) queries when its map point exists, is not bad and s is not an outlier, and the
// point, projected with the current pose into camera c (the keypoint's own camera), falls in c's mirror mask.  A map-point id
// >= n_points or an octave outside [0, n_levels) drops the query and raises status.
struct LastProjArgs {
    const PsCamSlots* cams; int n_cams, capacity, n_levels, n_points;
    const mcs_keypoint* keys;                                  // the last frame in slot order (ps_gather_kernel)
    const int* last_mp; const uint8_t* outlier; const uint8_t* bad; const double* pos;
    const mcs_ocam* models; const double* mtmc_inv; const uint8_t* masks;
};
__global__ void __launch_bounds__(256) pl_project_kernel(const LastProjArgs a, uint8_t* __restrict__ ok, double* __restrict__ u,
                                                         double* __restrict__ v, int* __restrict__ status) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n_cams * a.capacity) return;
    const int c = s / a.capacity;
    ok[s] = 0;
    if (!ps_live(a.cams, a.capacity, s)) return;
    const int i = a.last_mp[s];
    if (i < 0) return;
    if (i >= a.n_points) { *status = MCS_ERR_INVALID; return; }
    if ((a.bad && a.bad[i]) || (a.outlier && a.outlier[s])) return;
    const mcs_ocam cam = a.models[c];
    double x, y;
    if (!cam_project_in_mask(a.mtmc_inv + 16 * c, cam, a.masks + (size_t)c * cam.width * cam.height, a.pos[3 * i], a.pos[3 * i + 1],
                             a.pos[3 * i + 2], x, y))
        return;
    const int oct = a.keys[s].octave;
    if (oct < 0 || oct >= a.n_levels) { *status = MCS_ERR_INVALID; return; }
    ok[s] = 1; u[s] = x; v[s] = y;
}

// ---- previous frame: WindowSearch(F1 = last, F2 = cur) starts from an all-free F2 (ref :333) ----
__global__ void pw_clear_kernel(const PsCamSlots* __restrict__ cams, const int n_cams, const int capacity, int* __restrict__ frame_mp) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_cams * capacity) return;
    if (ps_live(cams, capacity, s)) frame_mp[s] = -1;
}

// ---- previous frame: the skip rules of SearchByProjection(F1 = last, F2 = cur, window) (ref :481-500) ----
// found[p]: p is held by a slot of cur on entry (spMapPointsAlreadyFound).  first[p]: the smallest last-frame slot carrying p
// (mapPt_2_obs_idx); slot order is the reference's visiting order, so the atomicMin picks the keypoint the reference keeps.  Ids of
// cur >= n_points match no valid p and are left out; ids of last >= n_points raise status (their slot is dropped by pf_project).
__global__ void pf_flag_kernel(const PsCamSlots* __restrict__ cur, const PsCamSlots* __restrict__ last, const int n_cams, const int capacity,
                               const int n_points, const int* __restrict__ cur_mp, const int* __restrict__ last_mp, uint8_t* __restrict__ found,
                               int* __restrict__ first, int* __restrict__ status) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_cams * capacity) return;
    if (ps_live(cur, capacity, s)) {
        const int p = cur_mp[s];
        if (p >= 0 && p < n_points) found[p] = 1;
    }
    if (ps_live(last, capacity, s)) {
        const int p = last_mp[s];
        if (p >= n_points) *status = MCS_ERR_INVALID;
        else if (p >= 0) atomicMin(&first[p], s);
    }
}

// Entry k = s * n_cams + c: last-frame slot s qualifies when its point p is valid, not bad, not already found and s is its first
// slot; p is then projected with the current pose into EVERY camera c (ref :509-513), and makes a query where it falls in c's mask.
struct FramesProjArgs {
    const PsCamSlots* last; int n_cams, capacity, n_points;
    const int* last_mp; const uint8_t* bad; const uint8_t* found; const int* first; const double* pos;
    const mcs_ocam* models; const double* mtmc_inv; const uint8_t* masks;
};
__global__ void __launch_bounds__(256) pf_project_kernel(const FramesProjArgs a, uint8_t* __restrict__ ok, double* __restrict__ u,
                                                         double* __restrict__ v) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (long long)a.n_cams * a.n_cams * a.capacity) return;
    const int s = (int)(k / a.n_cams), c = (int)(k - (long long)s * a.n_cams);
    ok[k] = 0;
    if (!ps_live(a.last, a.capacity, s)) return;
    const int i = a.last_mp[s];
    if (i < 0 || i >= a.n_points) return;
    if ((a.bad && a.bad[i]) || a.found[i] || a.first[i] != s) return;
    const mcs_ocam cam = a.models[c];
    double x, y;
    if (!cam_project_in_mask(a.mtmc_inv + 16 * c, cam, a.masks + (size_t)c * cam.width * cam.height, a.pos[3 * i], a.pos[3 * i + 1],
                             a.pos[3 * i + 2], x, y))
        return;
    ok[k] = 1; u[k] = x; v[k] = y;
}

// ---- query build: a count / scan / fill over the entries of a query maker, in the maker's order ----
// A maker has size() entries; valid(k) says whether entry k is a query (and may raise status), make(k) builds it.  sf is the
// launcher's staged scale-factor table.
struct MapPointQueries {         // SearchByProjection(F, vpMapPoints): entry k = point * n_cams + cam, when not bad and in view
    int n_cams, n_points, n_levels;
    const uint8_t* bad; const uint8_t* in_view; const int* level;
    const double* px; const double* py; const double* vcos; const double* sf; double th;
    __host__ __device__ long long size() const { return (long long)n_points * n_cams; }
    __device__ bool valid(long long k, int* status) const {
        if (k >= size()) return false;
        const int i = (int)(k / n_cams);
        if (bad && bad[i]) return false;
        if (!in_view[k]) return false;
        const int lvl = level[k];
        if (lvl < 0 || lvl >= n_levels) {     // the host call refuses such input; here the query is dropped and flagged
            if (status) *status = MCS_ERR_INVALID;
            return false;
        }
        return true;
    }
    __device__ mcs_window_query make(long long k) const {
        const int lvl = level[k];
        double r = vcos[k] > 0.998 ? 2.5 : 4.0;      // RadiusByViewingCos (ref :169-175)
        if (th != 1.0) r *= th;
        mcs_window_query q;
        q.cam = (int)(k % n_cams); q.min_level = lvl - 1; q.max_level = lvl; q.desc_index = (int)(k / n_cams);
        q.x = px[k]; q.y = py[k]; q.r = r * sf[lvl];
        return q;
    }
};

struct LastFrameQueries {        // SearchByProjection(CurrentFrame, LastFrame, th): entry k = last-frame slot, as pl_project_kernel set it
    int n_slots, capacity;
    const uint8_t* ok; const double* u; const double* v; const mcs_keypoint* keys; const double* sf; double th;
    __host__ __device__ long long size() const { return n_slots; }
    __device__ bool valid(long long k, int*) const { return k < n_slots && ok[k]; }
    __device__ mcs_window_query make(long long k) const {
        const int oct = keys[k].octave;
        mcs_window_query q;                          // GetFeaturesInArea(cam, u, v, th * sf[oct], oct - 1, oct + 1)  (ref :2027-2033)
        q.cam = (int)(k / capacity); q.min_level = oct - 1; q.max_level = oct + 1; q.desc_index = (int)k;
        q.x = u[k]; q.y = v[k]; q.r = th * sf[oct];
        return q;
    }
};

struct WindowQueries {           // WindowSearch(F1 = last, F2 = cur, window, ., min_level, max_level): entry k = last-frame slot (ref :344-368)
    int n_slots, capacity, n_points, min_level, max_level;
    const PsCamSlots* last; const mcs_keypoint* keys; const int* last_mp; const uint8_t* bad;
    const double* sf; double window;                         // sf: unused, no level is looked up
    __host__ __device__ long long size() const { return n_slots; }
    __device__ bool valid(long long k, int* status) const {
        if (k >= n_slots) return false;
        const int c = (int)(k / capacity);
        if ((int)k - c * capacity >= min(*last[c].count, capacity)) return false;
        const int p = last_mp[k];
        if (p < 0) return false;
        if (p >= n_points) {
            if (status) *status = MCS_ERR_INVALID;
            return false;
        }
        if (bad && bad[p]) return false;
        const int oct = keys[k].octave;
        if (min_level > 0 && oct < min_level) return false;
        return !(max_level < INT_MAX && oct > max_level);
    }
    __device__ mcs_window_query make(long long k) const {
        mcs_window_query q;                          // GetFeaturesInArea(cam, kp1.pt.x, kp1.pt.y, windowSize)  (ref :366-368)
        q.cam = (int)(k / capacity); q.min_level = -1; q.max_level = -1; q.desc_index = (int)k;
        q.x = (double)keys[k].x; q.y = (double)keys[k].y; q.r = window;
        return q;
    }
};

struct FramesQueries {           // SearchByProjection(F1 = last, F2 = cur, window): entry k = slot * n_cams + cam, as pf_project_kernel set it
    int n_slots, n_cams;
    const uint8_t* ok; const double* u; const double* v; const mcs_keypoint* keys;
    const double* sf; double window;                         // sf: unused, the octave is a level filter only
    __host__ __device__ long long size() const { return (long long)n_slots * n_cams; }
    __device__ bool valid(long long k, int*) const { return k < size() && ok[k]; }
    __device__ mcs_window_query make(long long k) const {
        const int s = (int)(k / n_cams), oct = keys[s].octave;
        mcs_window_query q;                          // GetFeaturesInArea(c, u, v, windowSize, level1, level1)  (ref :515-516)
        q.cam = (int)(k - (long long)s * n_cams); q.min_level = oct; q.max_level = oct; q.desc_index = s;
        q.x = u[k]; q.y = v[k]; q.r = window;
        return q;
    }
};

struct InitQueries {             // SearchForInitialization(F1, F2, vbPrevMatched, ., windowSize): entry k = F1 slot (ref :599-612)
    int n_slots, capacity;
    const PsCamSlots* f1; const mcs_keypoint* keys; const double* prev;   // keys: F1 in slot order; prev [n_slots * 2]
    const double* sf; double window;                         // sf: unused, the octave is a level filter only
    __host__ __device__ long long size() const { return n_slots; }
    __device__ bool valid(long long k, int*) const {
        if (k >= n_slots) return false;
        const int c = (int)(k / capacity);
        return (int)k - c * capacity < min(*f1[c].count, capacity);
    }
    __device__ mcs_window_query make(long long k) const {
        mcs_window_query q;                          // GetFeaturesInArea(cam, prev.x, prev.y, windowSize, level1, level1)  (ref :609-612)
        q.cam = (int)(k / capacity); q.min_level = keys[k].octave; q.max_level = q.min_level; q.desc_index = (int)k;
        q.x = prev[2 * k]; q.y = prev[2 * k + 1]; q.r = window;
        return q;
    }
};

template <class QM>
__global__ void __launch_bounds__(kQbThreads) ps_count_kernel(const QM a, int* __restrict__ block_count, int* __restrict__ status) {
    int total = 0;
    for (int i = 0; i < kQbPer; ++i) {
        const long long k = (long long)blockIdx.x * kQbTile + i * kQbThreads + threadIdx.x;
        total += __syncthreads_count(a.valid(k, status));
    }
    if (threadIdx.x == 0) block_count[blockIdx.x] = total;
}

// exclusive scan of the block counts (one CTA), total -> *nq
__global__ void __launch_bounds__(1024) ps_scan_kernel(const int* __restrict__ block_count, const int nb, int* __restrict__ block_off,
                                                       int* __restrict__ nq) {
    __shared__ int s[1024];
    int carry = 0;
    for (int base = 0; base < nb; base += 1024) {
        const int i = base + threadIdx.x;
        const int v = i < nb ? block_count[i] : 0;
        s[threadIdx.x] = v;
        __syncthreads();
        for (int o = 1; o < 1024; o <<= 1) {
            const int t = threadIdx.x >= o ? s[threadIdx.x - o] : 0;
            __syncthreads();
            s[threadIdx.x] += t;
            __syncthreads();
        }
        if (i < nb) block_off[i] = carry + s[threadIdx.x] - v;
        carry += s[1023];
        __syncthreads();
    }
    if (threadIdx.x == 0) *nq = carry;
}

// The fill of one block's kQbTile entries in the maker's order: emit(k, position) for every valid entry k, positions counted from
// block_off[blockIdx.x] (ps_scan_kernel's exclusive scan of ps_count_kernel's counts).
template <class QM, class Emit>
__device__ __forceinline__ void ps_fill_tile(const QM& a, const int* __restrict__ block_off, const Emit& emit) {
    __shared__ int s_w[kQbThreads / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int run = block_off[blockIdx.x];
    for (int i = 0; i < kQbPer; ++i) {
        const long long k = (long long)blockIdx.x * kQbTile + i * kQbThreads + threadIdx.x;
        const bool v = a.valid(k, nullptr);
        const unsigned m = __ballot_sync(0xffffffffu, v);
        if (lane == 0) s_w[w] = __popc(m);
        __syncthreads();
        int off = run, tot = 0;
        for (int u = 0; u < kQbThreads / 32; ++u) { if (u < w) off += s_w[u]; tot += s_w[u]; }
        if (v) emit(k, off + __popc(m & ((1u << lane) - 1u)));
        run += tot;
        __syncthreads();
    }
}

// ps_fill_kernel keeps its own copy of the tile body: written through ps_fill_tile its SASS changes (the query pointer's load is
// scheduled differently), and the existing searches keep their SASS.
template <class QM>
__global__ void __launch_bounds__(kQbThreads) ps_fill_kernel(const QM a, const int* __restrict__ block_off, mcs_window_query* __restrict__ qry) {
    __shared__ int s_w[kQbThreads / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int run = block_off[blockIdx.x];
    for (int i = 0; i < kQbPer; ++i) {
        const long long k = (long long)blockIdx.x * kQbTile + i * kQbThreads + threadIdx.x;
        const bool v = a.valid(k, nullptr);
        const unsigned m = __ballot_sync(0xffffffffu, v);
        if (lane == 0) s_w[w] = __popc(m);
        __syncthreads();
        int off = run, tot = 0;
        for (int u = 0; u < kQbThreads / 32; ++u) { if (u < w) off += s_w[u]; tot += s_w[u]; }
        if (v) qry[off + __popc(m & ((1u << lane) - 1u))] = a.make(k);
        run += tot;
        __syncthreads();
    }
}

// ---- window search keeping the KB smallest (distance << 16 | visiting position) keys of the candidates not taken ----
// Mirrors window_search_kernel (GetFeaturesInArea, ref src/cMultiFrame.cpp:272-340): same cell range, visiting order, level filter
// and distance.  Every lane ends with the same sorted list.  Returns the number of candidates in the window (taken ones included).
// Taken is called as taken(id), or as taken(id, distance) when it takes a second argument: SearchForInitialization skips a
// candidate by its distance (vMatchedDistance[i2] <= dist, ref :647-648), the other searches by the keypoint alone.
struct NoneTaken { __device__ bool operator()(int) const { return false; } };
template <class Taken> constexpr bool kTakenByDistance = std::is_invocable<const Taken&, int, unsigned>::value;

template <class Taken> __device__ __forceinline__ bool is_taken(const Taken& taken, const int id, const unsigned dist) {
    if constexpr (kTakenByDistance<Taken>) return taken(id, dist);
    else return taken(id);
}

template <int WORDS, bool MASKED, int KB, class Taken>
__device__ __forceinline__ int window_kbest(const WindowFrameDev& f, const mcs_window_query& qq, const uint32_t* __restrict__ qdesc,
                                            const uint32_t* __restrict__ qmask, const Taken& taken, unsigned (&key)[KB], int (&slot)[KB]) {
    constexpr bool BY_DIST = kTakenByDistance<Taken>;
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k < KB; ++k) { key[k] = kNoKey; slot[k] = -1; }
    const int cam = qq.cam;
    const double x = qq.x, y = qq.y, r = qq.r;
    const double wi = f.winv[cam], hi = f.hinv[cam];
    int cx0 = (int)floor((x - 0 - r) * wi); cx0 = max(0, cx0); if (cx0 >= MCS_FRAME_GRID_COLS) return 0;
    int cx1 = (int)ceil((x - 0 + r) * wi);  cx1 = min(MCS_FRAME_GRID_COLS - 1, cx1); if (cx1 < 0) return 0;
    int cy0 = (int)floor((y - 0 - r) * hi); cy0 = max(0, cy0); if (cy0 >= MCS_FRAME_GRID_ROWS) return 0;
    int cy1 = (int)ceil((y - 0 + r) * hi);  cy1 = min(MCS_FRAME_GRID_ROWS - 1, cy1); if (cy1 < 0) return 0;
    uint32_t qw[WORDS], qm[MASKED ? WORDS : 1];
#pragma unroll
    for (int k = 0; k < WORDS; ++k) {
        qw[k] = qdesc[(size_t)qq.desc_index * WORDS + k];
        if (MASKED) qm[k] = qmask[(size_t)qq.desc_index * WORDS + k];
    }
    const bool check = !(qq.min_level == -1 && qq.max_level == -1);
    const bool same = check && qq.min_level == qq.max_level;
    int count = 0;
    for (int ix = cx0; ix <= cx1; ++ix)
        for (int iy = cy0; iy <= cy1; ++iy) {
            const int cell = (cam * MCS_FRAME_GRID_COLS + ix) * MCS_FRAME_GRID_ROWS + iy;
            const int s = f.cell_start[cell], e = f.cell_start[cell + 1];
            for (int base = s; base < e; base += 32) {
                const int it = base + lane;
                bool ok = it < e;
                int id = 0;
                if (ok) {
                    id = f.cell_items[it];
                    const int oct = f.koct[id];
                    if (check && !same) ok = !(oct < qq.min_level || oct > qq.max_level);
                    else if (same) ok = (oct == qq.min_level);
                    if (ok) ok = !(fabs((double)f.kx[id] - x) > r || fabs((double)f.ky[id] - y) > r);
                }
                const unsigned m = __ballot_sync(0xffffffffu, ok);
                const bool cand = ok && (BY_DIST || !is_taken(taken, id, 0u));
                unsigned kk = kNoKey;
                if (cand) {
                    const uint32_t* dd = (const uint32_t*)f.desc + (size_t)id * WORDS;
                    unsigned dist = 0;
                    if (MASKED) {
                        const uint32_t* mm = (const uint32_t*)f.dmask + (size_t)id * WORDS;
#pragma unroll
                        for (int k = 0; k < WORDS; ++k) {
                            const uint32_t xw = qw[k] ^ dd[k];
                            dist += __popc(xw & qm[k]) + __popc(xw & mm[k]);
                        }
                        dist >>= 1;
                    } else {
#pragma unroll
                        for (int k = 0; k < WORDS; ++k) dist += __popc(qw[k] ^ dd[k]);
                    }
                    if (!BY_DIST || !is_taken(taken, id, dist)) kk = (dist << 16) | (unsigned)(count + __popc(m & ((1u << lane) - 1u)));
                }
                unsigned ins = __ballot_sync(0xffffffffu, cand && kk < key[KB - 1]);
                while (ins) {
                    const int b = __ffs(ins) - 1;
                    ins &= ins - 1;
                    unsigned nk = __shfl_sync(0xffffffffu, kk, b);
                    int ns = __shfl_sync(0xffffffffu, id, b);
#pragma unroll
                    for (int k = 0; k < KB; ++k)
                        if (nk < key[k]) { const unsigned tk = key[k]; key[k] = nk; nk = tk; const int ts = slot[k]; slot[k] = ns; ns = ts; }
                }
                count += __popc(m);
            }
        }
    return count;
}

template <int WORDS, bool MASKED>
__global__ void __launch_bounds__(256) ps_list_kernel(const WindowFrameDev f, const mcs_window_query* __restrict__ qry, const int* __restrict__ nq_p,
                                                      const uint32_t* __restrict__ qdesc, const uint32_t* __restrict__ qmask,
                                                      unsigned* __restrict__ lkey, int* __restrict__ lslot, int* __restrict__ lcnt) {
    const int lane = threadIdx.x & 31, nq = *nq_p;
    const int stride = gridDim.x * (blockDim.x >> 5);
    for (int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < nq; q += stride) {
        unsigned key[kPsK]; int slot[kPsK];
        const int n = window_kbest<WORDS, MASKED, kPsK>(f, qry[q], qdesc, qmask, NoneTaken{}, key, slot);
#pragma unroll
        for (int k = 0; k < kPsK; ++k)
            if (lane == k) { lkey[(size_t)q * kPsK + k] = key[k]; lslot[(size_t)q * kPsK + k] = slot[k]; }
        if (lane == 0) lcnt[q] = n;
    }
}

// The decision of one query (warp-uniform) under a "keypoint already taken" predicate.  MCS_RULE_LEVEL_RATIO: best / second best
// free candidate by (distance, visiting position) -- what the sequential strict-< update of ref :138-150 picks -- and the
// acceptance of :154-160.  MCS_RULE_BEST: the best free candidate alone (strict < over the visiting order, ref :2050-2068),
// accepted when its distance is <= th_high (:2070).  MCS_RULE_RATIO: best / second best free candidate, accepted when
// best <= second * nnratio and best <= th_high (WindowSearch :405-416, SearchByProjection(F1, F2) :553-566), in the double form of
// the host replay.  kRuleInit: best / second best candidate not skipped, accepted when best <= th_high and best < second * nnratio
// (SearchForInitialization :662-677); its distance goes to *best_dist.  MCS_RULE_SCW: the best free candidate alone, accepted when
// best <= th_high and it is not contiguous keypoint 0 (SearchByProjection(KF, Scw) :2385, `bestIdx > 0`): slot j = 0 of a camera
// whose first contiguous id (f.cam_first) is 0.  The list decides when it holds as many free entries as the rule reads, or every
// candidate; otherwise the window is scanned again with the predicate.
constexpr int kRuleInit = 100;               // not a public rule: SearchForInitialization's acceptance exists on the device only
template <int RULE, int WORDS, bool MASKED, class Taken>
__device__ __forceinline__ int ps_decide(const WindowFrameDev& f, const mcs_window_query& qq, const unsigned* lk, const int* ls, const int cnt,
                                         const uint32_t* qdesc, const uint32_t* qmask, const Taken& taken, const int th_high,
                                         const double nnratio, int* rescans, int* best_dist = nullptr) {
    static_assert(RULE == MCS_RULE_LEVEL_RATIO || RULE == MCS_RULE_BEST || RULE == MCS_RULE_RATIO || RULE == kRuleInit ||
                  RULE == MCS_RULE_SCW, "device acceptance rules");
    constexpr int NB = RULE == MCS_RULE_BEST || RULE == MCS_RULE_SCW ? 1 : 2;       // free keys the rule reads
    const int lane = threadIdx.x & 31;
    unsigned k = kNoKey; int s = -1; bool fr = false;
    if (lane < kPsK) { k = lk[lane]; s = ls[lane]; fr = k != kNoKey && !is_taken(taken, s, k >> 16); }
    const unsigned fm = __ballot_sync(0xffffffffu, fr);
    unsigned k0 = kNoKey, k1 = kNoKey; int s0 = -1, s1 = -1;
    if (__popc(fm) >= NB || cnt <= kPsK) {
        const int b0 = fm ? __ffs(fm) - 1 : 0;
        const unsigned rest = fm & (fm - 1);
        const int b1 = rest ? __ffs(rest) - 1 : 0;
        const unsigned x0 = __shfl_sync(0xffffffffu, k, b0), x1 = __shfl_sync(0xffffffffu, k, b1);
        const int y0 = __shfl_sync(0xffffffffu, s, b0), y1 = __shfl_sync(0xffffffffu, s, b1);
        if (fm) { k0 = x0; s0 = y0; }
        if (rest) { k1 = x1; s1 = y1; }
    } else {
        unsigned kk[NB]; int ss[NB];
        window_kbest<WORDS, MASKED, NB>(f, qq, qdesc, qmask, taken, kk, ss);
        k0 = kk[0]; s0 = ss[0];
        if constexpr (NB == 2) { k1 = kk[1]; s1 = ss[1]; }
        if (lane == 0 && rescans) atomicAdd(rescans, 1);
    }
    if (s0 < 0) return -1;
    if constexpr (RULE == MCS_RULE_BEST) return (int)(k0 >> 16) <= th_high ? s0 : -1;
    if constexpr (RULE == MCS_RULE_SCW) {
        const int cap = f.n_keys / f.n_cams, c = s0 / cap;
        const bool first = s0 == c * cap && f.cam_first[c] == 0;
        return (int)(k0 >> 16) <= th_high && !first ? s0 : -1;
    }
    if constexpr (RULE == MCS_RULE_RATIO) {
        const int d0 = (int)(k0 >> 16), d1 = s1 >= 0 ? (int)(k1 >> 16) : INT_MAX;
        return (double)d0 <= (double)d1 * nnratio && d0 <= th_high ? s0 : -1;
    }
    if constexpr (RULE == kRuleInit) {
        const int d0 = (int)(k0 >> 16), d1 = s1 >= 0 ? (int)(k1 >> 16) : INT_MAX;
        *best_dist = d0;
        return d0 <= th_high && (double)d0 < (double)d1 * nnratio ? s0 : -1;
    }
    const int d0 = (int)(k0 >> 16), l0 = f.koct[s0];
    const int d1 = s1 >= 0 ? (int)(k1 >> 16) : INT_MAX, l1 = s1 >= 0 ? f.koct[s1] : -1;
    const bool ok = d0 <= th_high && !(l0 == l1 && (double)d0 > nnratio * (double)d1);
    return ok ? s0 : -1;
}

struct PsState {                 // device scratch shared by the acceptance kernels
    const mcs_window_query* qry;
    const unsigned* lkey; const int* lslot; const int* lcnt;
    int* dec;                    // [2][Q] decisions of the last two rounds (accepted slot or -1)
    unsigned* owner;             // [2][n_slots] ((kPsRounds - round) << 24 | smallest accepting query)
    int* ctl;                    // [0] nq  [1] rounds run  [2] rescans  [3] walk start  [4 ..] first changed query of each round
    int Q, n_slots, capacity, th_high;
    double nnratio;
    const int* tag;              // may be NULL: an accepted query writes tag[desc_index] into frame_mp, else desc_index itself
};
__device__ __forceinline__ int ps_tag(const PsState& p, const int desc_index) { return p.tag ? p.tag[desc_index] : desc_index; }
__device__ __forceinline__ int* ps_chg(const PsState& p) { return p.ctl + 4; }

// Round r: every query not yet settled decides, treating a keypoint as taken when frame_mp had it on entry or a query with a
// smaller index accepted it in round r - 1.  Queries below the first one whose decision changed in round r - 1 are final
// (query p reads only decisions of queries < p) and only republish their keypoint.
template <int RULE, int WORDS, bool MASKED>
__global__ void __launch_bounds__(256, 2) ps_round_kernel(const WindowFrameDev f, const PsState p, const int r, const uint32_t* __restrict__ qdesc,
                                                          const uint32_t* __restrict__ qmask, const int* __restrict__ fmp_in) {
    const int* chg = ps_chg(p);
    const int settled = r >= 2 ? chg[r - 1] : 0;
    if (settled == kNoChange) return;                         // converged in an earlier round
    const int lane = threadIdx.x & 31, nq = p.ctl[0];
    if (blockIdx.x == 0 && threadIdx.x == 0) p.ctl[1] = r + 1;
    int* dec_cur = p.dec + (size_t)(r & 1) * p.Q;
    const int* dec_prev = p.dec + (size_t)((r + 1) & 1) * p.Q;
    unsigned* own_cur = p.owner + (size_t)(r & 1) * p.n_slots;
    const unsigned* own_prev = p.owner + (size_t)((r + 1) & 1) * p.n_slots;
    const unsigned ver_cur = (unsigned)(kPsRounds - r) << 24, ver_prev = (unsigned)(kPsRounds - r + 1) << 24;
    const int stride = gridDim.x * (blockDim.x >> 5);
    for (int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < nq; q += stride) {
        if (q < settled) {                                    // dec_cur[q] holds round r - 2, equal to round r - 1 below `settled`
            if (lane == 0) { const int d = dec_cur[q]; if (d >= 0) atomicMin(&own_cur[d], ver_cur | (unsigned)q); }
            continue;
        }
        auto taken = [=](int s) {
            if (fmp_in[s] >= 0) return true;
            if (r == 0) return false;
            const unsigned v = own_prev[s];
            return (v & 0xFF000000u) == ver_prev && (int)(v & 0xFFFFFFu) < q;
        };
        const int d = ps_decide<RULE, WORDS, MASKED>(f, p.qry[q], p.lkey + (size_t)q * kPsK, p.lslot + (size_t)q * kPsK, p.lcnt[q], qdesc,
                                                     qmask, taken, p.th_high, p.nnratio, p.ctl + 2);
        if (lane == 0) {
            dec_cur[q] = d;
            if (d >= 0) atomicMin(&own_cur[d], ver_cur | (unsigned)q);
            if (r >= 1 && d != dec_prev[q]) atomicMin(&p.ctl[4 + r], q);
        }
    }
}

// Writes the final decisions of the settled prefix into frame_mp and counts them; records where the walk has to start.
__global__ void __launch_bounds__(256) ps_finalize_kernel(const PsState p, int* __restrict__ frame_mp, int* __restrict__ nmatches) {
    __shared__ int s_n;
    const int nq = p.ctl[0], rl = p.ctl[1] - 1;
    int S = rl >= 1 ? ps_chg(p)[rl] : 0;
    if (S == kNoChange || S > nq) S = nq;
    const int* dec = p.dec + (size_t)(rl & 1) * p.Q;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    int n = 0;
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < S; q += gridDim.x * blockDim.x) {
        const int d = dec[q];
        if (d >= 0) { frame_mp[d] = ps_tag(p, p.qry[q].desc_index); ++n; }
    }
    if (n) atomicAdd(&s_n, n);
    __syncthreads();
    if (threadIdx.x == 0) {
        if (s_n) atomicAdd(nmatches, s_n);
        if (blockIdx.x == 0) p.ctl[3] = S < nq ? S : -1;
    }
}

// Fallback past the round cap: one warp per camera walks its queries from the first unsettled one in order, with the camera's
// taken keypoints as a bitmap in shared memory.
template <int RULE, int WORDS, bool MASKED>
__global__ void __launch_bounds__(32) ps_walk_kernel(const WindowFrameDev f, const PsState p, const uint32_t* __restrict__ qdesc,
                                                     const uint32_t* __restrict__ qmask, int* __restrict__ frame_mp, int* __restrict__ nmatches) {
    extern __shared__ unsigned s_bits[];
    const int S = p.ctl[3];
    if (S < 0) return;
    const int c = blockIdx.x, lane = threadIdx.x, nq = p.ctl[0], cap = p.capacity;
    const int* fmp = frame_mp + (size_t)c * cap;
    for (int w = lane; w < (cap + 31) / 32; w += 32) {
        unsigned b = 0;
        for (int k = 0; k < 32 && w * 32 + k < cap; ++k) b |= (fmp[w * 32 + k] >= 0 ? 1u : 0u) << k;
        s_bits[w] = b;
    }
    __syncwarp();
    auto taken = [=](int s) { const int j = s - c * cap; return ((s_bits[j >> 5] >> (j & 31)) & 1u) != 0; };
    int nm = 0;
    for (int base = S; base < nq; base += 32) {
        const int q = base + lane;
        unsigned m = __ballot_sync(0xffffffffu, q < nq && p.qry[q].cam == c);
        while (m) {
            const int qi = base + __ffs(m) - 1;
            m &= m - 1;
            const mcs_window_query qq = p.qry[qi];
            const int d = ps_decide<RULE, WORDS, MASKED>(f, qq, p.lkey + (size_t)qi * kPsK, p.lslot + (size_t)qi * kPsK, p.lcnt[qi], qdesc,
                                                         qmask, taken, p.th_high, p.nnratio, p.ctl + 2);
            if (d >= 0) {
                if (lane == 0) {
                    const int j = d - c * cap;
                    s_bits[j >> 5] |= 1u << (j & 31);
                    frame_mp[d] = ps_tag(p, qq.desc_index);
                }
                ++nm;
            }
            __syncwarp();
        }
    }
    if (lane == 0 && nm) atomicAdd(nmatches, nm);
}

__global__ void ps_diag_kernel(const int* __restrict__ ctl, int* __restrict__ diag) {
    diag[0] = ctl[1];        // fixpoint rounds run
    diag[1] = ctl[1] ? ctl[3] : -1;   // first query of the walk, -1 = the rounds settled every query
    diag[2] = ctl[0];        // queries
    diag[3] = ctl[2];        // decisions that rescanned their window
}

// ---- SearchForInitialization: the ordered walk (DESIGN.md section 4) ----
// A later query may take a keypoint away from an earlier one with a strictly smaller distance, so query p needs
// MD(s) = min{ d_q : q < p accepted s } for every candidate s, which no per-keypoint owner word of a round answers.  Cameras are
// independent (a query searches only its own camera of F2), so one warp per camera walks that camera's queries in order with MD
// of the camera's F2 slots in shared memory (16 bits each, 0xFFFF = no acceptance yet: every distance is <= 512).
struct InitWalk {
    const mcs_window_query* qry;
    const unsigned* lkey; const int* lslot; const int* lcnt;
    int* ctl;                    // [0] nq  [2] rescans
    const PsCamSlots* f1; const PsCamSlots* f2;              // device [n_cams]: the counts of both frames
    const mcs_keypoint* keys2;   // F2 in slot order
    int* dec;                    // [Q] the slot each query accepted, or -1
    int* owner;                  // [n_slots] the last query that accepted an F2 slot, -1 on entry
    int n_cams, capacity, th_low;
    double nnratio;
    int* matches12; double* prev; int* nmatches;             // device, F1 slot-indexed / [1]
};

template <int WORDS, bool MASKED>
__global__ void __launch_bounds__(32) pi_walk_kernel(const WindowFrameDev f, const InitWalk w, const uint32_t* __restrict__ qdesc,
                                                     const uint32_t* __restrict__ qmask) {
    extern __shared__ unsigned short s_md[];
    __shared__ unsigned s_key[32 * kPsK];
    __shared__ int s_slot[32 * kPsK], s_cnt[32];
    const int c = blockIdx.x, lane = threadIdx.x, cap = w.capacity, base_slot = c * cap;
    int q0 = 0;                                              // the camera's queries are [q0, q0 + n1): one per F1 slot below the count
    for (int k = 0; k < c; ++k) q0 += min(*w.f1[k].count, cap);
    const int n1 = min(*w.f1[c].count, cap), n2 = min(*w.f2[c].count, cap);
    for (int j = lane; j < n2; j += 32) s_md[j] = 0xFFFF;
    __syncwarp();
    auto skipped = [&](int s, unsigned d) { return s_md[s - base_slot] <= d; };   // vMatchedDistance[i2] <= dist (ref :647-648)
    for (int b = 0; b < n1; b += 32) {
        const int nb = min(32, n1 - b), qb = q0 + b;
        for (int i = lane; i < nb * kPsK; i += 32) {         // the next 32 queries' lists in one coalesced pass
            s_key[i] = w.lkey[(size_t)qb * kPsK + i];
            s_slot[i] = w.lslot[(size_t)qb * kPsK + i];
        }
        if (lane < nb) s_cnt[lane] = w.lcnt[qb + lane];
        __syncwarp();
        for (int i = 0; i < nb; ++i) {
            const int q = qb + i;
            int d0 = 0;
            const int s = ps_decide<kRuleInit, WORDS, MASKED>(f, w.qry[q], s_key + i * kPsK, s_slot + i * kPsK, s_cnt[i], qdesc, qmask,
                                                              skipped, w.th_low, w.nnratio, w.ctl + 2, &d0);
            if (lane == 0) {
                w.dec[q] = s;
                if (s >= 0) { s_md[s - base_slot] = (unsigned short)d0; w.owner[s] = q; }
            }
            __syncwarp();
        }
    }
    // a query's match survives when no later query took its keypoint (ref :666-670); prev moves to the survivors' F2 keypoints
    int nm = 0;
    for (int j = lane; j < n1; j += 32) {
        const int q = q0 + j, s = w.dec[q];
        const bool keep = s >= 0 && w.owner[s] == q;
        w.matches12[base_slot + j] = keep ? s : -1;
        if (keep) {
            const mcs_keypoint kp = w.keys2[s];
            w.prev[2 * (size_t)(base_slot + j)] = (double)kp.x;
            w.prev[2 * (size_t)(base_slot + j) + 1] = (double)kp.y;
            ++nm;
        }
    }
    for (int o = 16; o > 0; o >>= 1) nm += __shfl_xor_sync(0xffffffffu, nm, o);
    if (lane == 0 && nm) atomicAdd(w.nmatches, nm);
}

__global__ void pi_diag_kernel(const int* __restrict__ ctl, int* __restrict__ diag) {
    diag[0] = ctl[0];        // queries
    diag[1] = ctl[2];        // decisions that rescanned their window
}

// FirstInitialization's fill (ref src/cTracking.cpp:383-386): prev = the keypoint position as doubles, for every slot below the count
__global__ void pi_seed_kernel(const PsCamSlots* __restrict__ cams, const int n_cams, const int capacity, double* __restrict__ prev) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_cams * capacity) return;
    const int c = s / capacity, j = s - c * capacity;
    if (j >= min(*cams[c].count, capacity)) return;
    const mcs_keypoint kp = cams[c].kps[j];
    prev[2 * (size_t)s] = (double)kp.x;
    prev[2 * (size_t)s + 1] = (double)kp.y;
}

// ---- Fuse (ref :1265-1418, :1420-1567, :1570-1719): n_kf target key frames searched as one frame of n_kf * n_cams images ----
// A Fuse query takes nothing from another query (the "already occupied" test lives in the host bookkeeping), so there are no
// rounds: every (key frame k, query q, camera c) entry projects, searches its window in image k * n_cams + c and decides alone.
// qmap[p]: the first query position holding map point p (>= n_q: none); an id >= n_points drops its query and raises status.
__global__ void fu_qmap_kernel(const int* __restrict__ query_mp, const int n_q, const int n_points, int* __restrict__ qmap,
                               int* __restrict__ status) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n_q) return;
    const int p = query_mp[q];
    if (p >= n_points) *status = MCS_ERR_INVALID;
    else if (p >= 0) atomicMin(&qmap[p], q);
}

// The membership pre-filter: held[k * n_q + qmap[p]] = 1 for every point p a slot of key frame k's row holds (below the camera's
// count).  Queries holding the same point share the flag of its first position.
__global__ void fu_held_kernel(const PsCamSlots* __restrict__ slots, const int* const* __restrict__ kf_mp, const int n_kf, const int n_cams,
                               const int capacity, const int n_q, const int n_points, const int* __restrict__ qmap, uint8_t* __restrict__ held) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (long long)n_kf * n_cams * capacity) return;
    const int img = (int)(g / capacity), j = (int)(g - (long long)img * capacity), k = img / n_cams;
    const int* mp = kf_mp[k];
    if (!mp || j >= min(*slots[img].count, capacity)) return;
    const int p = mp[(size_t)(img - k * n_cams) * capacity + j];
    if (p < 0 || p >= n_points) return;
    const int q = qmap[p];
    if (q < n_q) held[(size_t)k * n_q + q] = 1;
}

// The range test and the predicted level of a projected point at distance d: false outside [dmin, dmax], else lv =
// std::lower_bound(vfScaleFactors, d / dmin), clamped to the last level.
__device__ __forceinline__ bool predict_level(const double d, const double dmin, const double dmax, const double* sf, const int n_levels,
                                              int& lv) {
    if (d < dmin || d > dmax) return false;
    const double ratio = d / dmin;
    lv = 0;
    while (lv < n_levels && sf[lv] < ratio) ++lv;
    if (lv >= n_levels) lv = n_levels - 1;
    return true;
}

// Entry e = (k * n_q + q) * n_cams + c: query q's point, when not NULL, not bad and not held by key frame k, projected with
// k's MtMc_inv into camera c (WorldToCamHom_fast, mirror mask), its distance to k's centre in the range [min, max] and its
// level predicted, in the operation order of the host projection (api._project): dist3D a float for :1265 / :1420, a double for
// :1570 (ref :1301, :1472, :1624).  -fmad=false keeps the norm free of FMA contraction.
struct FuseProjArgs {
    int n_kf, n_cams, n_q, n_points, n_levels; bool float_dist;
    const int* query_mp; const uint8_t* bad; const uint8_t* held; const int* qmap;
    const double* pos; const double* dmin; const double* dmax;
    const mcs_ocam* models; const double* mtmc_inv; const double* ow; const uint8_t* masks; const double* sf;
};
__global__ void __launch_bounds__(256) fu_project_kernel(const FuseProjArgs a, uint8_t* __restrict__ ok, double* __restrict__ u,
                                                         double* __restrict__ v, int* __restrict__ level) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)a.n_kf * a.n_q * a.n_cams) return;
    const long long kq = e / a.n_cams;
    const int c = (int)(e - kq * a.n_cams), k = (int)(kq / a.n_q), q = (int)(kq - (long long)k * a.n_q);
    ok[e] = 0;
    const int p = a.query_mp[q];
    if (p < 0 || p >= a.n_points) return;
    if ((a.bad && a.bad[p]) || a.held[(size_t)k * a.n_q + a.qmap[p]]) return;
    const mcs_ocam cam = a.models[c];
    const double P0 = a.pos[3 * p], P1 = a.pos[3 * p + 1], P2 = a.pos[3 * p + 2];
    double x, y;
    if (!cam_project_in_mask(a.mtmc_inv + 16 * ((size_t)k * a.n_cams + c), cam, a.masks + (size_t)c * cam.width * cam.height, P0, P1, P2, x, y))
        return;
    const double* O = a.ow + 3 * k;
    const double o0 = P0 - O[0], o1 = P1 - O[1], o2 = P2 - O[2];
    double d = sqrt((o0 * o0 + o1 * o1) + o2 * o2);
    if (a.float_dist) d = (double)__double2float_rn(d);
    int lv;
    if (!predict_level(d, a.dmin[p], a.dmax[p], a.sf, a.n_levels, lv)) return;
    ok[e] = 1; u[e] = x; v[e] = y; level[e] = lv;
}

// The query of entry k of a projection (fu_project / s3_project / scw_project_kernel set ok, u, v and level):
// GetFeaturesInArea(cam, u, v, th * sf[l]) on levels {l - 1, l}.  `at` gives the entry's camera and descriptor row.
template <class At> struct ProjectedQueries {
    long long n; const uint8_t* ok; const double* u; const double* v; const int* level; const double* sf; double th;
    At at;
    __host__ __device__ long long size() const { return n; }
    __device__ bool valid(long long k, int*) const { return k < n && ok[k]; }
    __device__ mcs_window_query make(long long k) const {
        const int lvl = level[k];
        mcs_window_query q;
        at(k, q.cam, q.desc_index);
        q.min_level = lvl - 1; q.max_level = lvl; q.x = u[k]; q.y = v[k]; q.r = th * sf[lvl];
        return q;
    }
};
struct FuseAt {                  // entry e = (k * n_q + q) * n_cams + c: image k * n_cams + c, the row of query q's map point
    int n_q, n_cams; const int* query_mp;
    __device__ void operator()(long long e, int& cam, int& row) const {
        const long long kq = e / n_cams;
        const int c = (int)(e - kq * n_cams), k = (int)(kq / n_q);
        cam = k * n_cams + c; row = query_mp[kq - (long long)k * n_q];
    }
};
struct Sim3At {                  // entry = slot s of key frame a: camera s / capacity, the row of the slot's map point
    int capacity; const int* mp;
    __device__ void operator()(long long s, int& cam, int& row) const { row = mp[s]; cam = (int)(s / capacity); }
};
struct ScwAt {                   // entry i of vpPoints: the camera scw_project_kernel found, the row of the entry's map point
    const int* qcam; const int* points;
    __device__ void operator()(long long i, int& cam, int& row) const { cam = qcam[i]; row = points[i]; }
};

// entry[i] = the maker entry of query i: ps_fill_kernel's fill, writing the entry index instead of the query
template <class QM>
__global__ void __launch_bounds__(kQbThreads) fu_entry_kernel(const QM a, const int* __restrict__ block_off, int* __restrict__ entry) {
    ps_fill_tile(a, block_off, [&](long long k, int o) { entry[o] = (int)k; });
}

// MCS_FUSE_NEIGHBOUR / MCS_FUSE_SIM3: the best candidate (strict < over the visiting order, ref :1345-1356) is the first key of
// the query's list, which holds every candidate's key when nothing is taken; kept when its distance is <= th_low (:1359).
__global__ void __launch_bounds__(256) fu_best_kernel(const int* __restrict__ nq_p, const unsigned* __restrict__ lkey,
                                                      const int* __restrict__ lslot, const int th_low, int* __restrict__ dec) {
    const int nq = *nq_p;
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x) {
        const unsigned k0 = lkey[(size_t)q * kPsK];
        dec[q] = k0 != kNoKey && (int)(k0 >> 16) <= th_low ? lslot[(size_t)q * kPsK] : -1;
    }
}

// MCS_FUSE_FIRST: the distance is discarded (ref :1506-1514, `dist` stays 0), so the first candidate of the window in visiting
// order that passes the level filter wins, whatever the distances the list sorted by.  One warp per query walks the window in
// window_kbest's order and stops at the first candidate; a query whose list counted none is not walked.  The cell range, the
// item order and the level / radius filter below must stay those of window_kbest (which keeps its own copy: its SASS is shared
// by every device search); the MCS_FUSE_FIRST parity tests pin them against the host window search.
__global__ void __launch_bounds__(256) fu_first_kernel(const WindowFrameDev f, const mcs_window_query* __restrict__ qry, const int* __restrict__ nq_p,
                                                       const int* __restrict__ lcnt, const int th_low, int* __restrict__ dec) {
    const int lane = threadIdx.x & 31, nq = *nq_p;
    const int stride = gridDim.x * (blockDim.x >> 5);
    for (int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < nq; q += stride) {
        int first = -1;
        if (lcnt[q] > 0 && 0 <= th_low) {
            const mcs_window_query qq = qry[q];
            const int cam = qq.cam;
            const double x = qq.x, y = qq.y, r = qq.r;
            const double wi = f.winv[cam], hi = f.hinv[cam];
            const int cx0 = max(0, (int)floor((x - 0 - r) * wi)), cx1 = min(MCS_FRAME_GRID_COLS - 1, (int)ceil((x - 0 + r) * wi));
            const int cy0 = max(0, (int)floor((y - 0 - r) * hi)), cy1 = min(MCS_FRAME_GRID_ROWS - 1, (int)ceil((y - 0 + r) * hi));
            const bool check = !(qq.min_level == -1 && qq.max_level == -1);
            const bool same = check && qq.min_level == qq.max_level;
            for (int ix = cx0; ix <= cx1 && first < 0; ++ix)
                for (int iy = cy0; iy <= cy1 && first < 0; ++iy) {
                    const int cell = (cam * MCS_FRAME_GRID_COLS + ix) * MCS_FRAME_GRID_ROWS + iy;
                    const int s = f.cell_start[cell], e = f.cell_start[cell + 1];
                    for (int base = s; base < e && first < 0; base += 32) {
                        const int it = base + lane;
                        bool ok = it < e;
                        int id = 0;
                        if (ok) {
                            id = f.cell_items[it];
                            const int oct = f.koct[id];
                            if (check && !same) ok = !(oct < qq.min_level || oct > qq.max_level);
                            else if (same) ok = (oct == qq.min_level);
                            if (ok) ok = !(fabs((double)f.kx[id] - x) > r || fabs((double)f.ky[id] - y) > r);
                        }
                        const unsigned m = __ballot_sync(0xffffffffu, ok);
                        if (m) first = __shfl_sync(0xffffffffu, id, __ffs(m) - 1);
                    }
                }
        }
        if (lane == 0) dec[q] = first;
    }
}

struct FuseHitQueries {          // the queries with a hit, in query order (= the reference's (key frame, query, camera) order)
    long long Q; const int* nq; const int* dec;
    __host__ __device__ long long size() const { return Q; }
    __device__ bool valid(long long i, int*) const { return i < Q && i < *nq && dec[i] >= 0; }
};

// The hit rows: row o = (k, q, slot in k) of the o-th query with a hit; rows past max_hits are counted (ps_scan_kernel writes the
// true total) but not written, and raise MCS_ERR_CAPACITY unless status already holds an error.
__global__ void __launch_bounds__(kQbThreads) fu_hits_kernel(const FuseHitQueries a, const int* __restrict__ block_off, const int* __restrict__ entry,
                                                             const int n_q, const int n_cams, const int capacity, const int max_hits,
                                                             int* __restrict__ hits, int* __restrict__ status) {
    ps_fill_tile(a, block_off, [&](long long k, int o) {
        if (o < max_hits) {
            const int e = entry[k], kq = e / n_cams, kf = kq / n_q;
            hits[3 * (size_t)o] = kf;
            hits[3 * (size_t)o + 1] = kq - kf * n_q;
            hits[3 * (size_t)o + 2] = a.dec[k] - kf * n_cams * capacity;
        } else {
            atomicCAS(status, MCS_OK, MCS_ERR_CAPACITY);
        }
    });
}

// ---- SearchBySim3(KF1, KF2, vpMatches12, s12, R12, t12, th) (ref :1721-1988) ----
// Nothing is skipped as taken in either direction, so each direction is Fuse's stateless decision (fu_best_kernel under th_high)
// over one query per slot of the key frame whose points are carried over, and a mutual check joins the two.
// The transforms of one direction: a's pose (R, t: GetPoseInverse's rotation and translation, row-major) and the similarity into
// b's rig frame (sR, st), 24 doubles.
struct Sim3Xf { double R[9], t[3], sR[9], st[3]; };

// Slot s = c * capacity + j (j below camera c's count) of key frame a: its point p = mp[s] when p exists, s is not skipped (skip_mp:
// matches12 on entry, >= 0 = already matched; skip: already2, non-zero = already matched), and p is not bad.  Then, in the order and
// arithmetic of the reference (cv::Matx products, no FMA): pa = R * X + t, pb = sR * pa + st, p4 = mc_inv[c] * (pb, 1); the query is
// dropped when pb.z < 0 (the RIG frame's z), when WorldToImg(p4) falls outside camera c's mirror mask, or when |p4| (a double) lies
// outside [min, max]; else its level is lower_bound over the scale factors, clamped.  An id >= n_points in mp or skip_mp drops the
// slot and raises status.
struct Sim3ProjArgs {
    const PsCamSlots* a; int n_cams, capacity, n_points, n_levels;
    const int* mp; const int* skip_mp; const uint8_t* skip; const uint8_t* bad;
    const double* pos; const double* dmin; const double* dmax;
    const mcs_ocam* models; const Sim3Xf* xf; const double* mc_inv; const uint8_t* masks; const double* sf;
};
__global__ void __launch_bounds__(256) s3_project_kernel(const Sim3ProjArgs a, uint8_t* __restrict__ ok, double* __restrict__ u,
                                                         double* __restrict__ v, int* __restrict__ level, int* __restrict__ status) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n_cams * a.capacity) return;
    const int c = s / a.capacity;
    ok[s] = 0;
    if (!ps_live(a.a, a.capacity, s)) return;
    if (a.skip_mp) {                              // checked first: an invalid matches12 entry raises status whatever mp holds
        const int m = a.skip_mp[s];
        if (m >= a.n_points) { *status = MCS_ERR_INVALID; return; }
        if (m >= 0) return;
    }
    const int p = a.mp[s];
    if (p < 0) return;
    if (p >= a.n_points) { *status = MCS_ERR_INVALID; return; }
    if ((a.skip && a.skip[s]) || (a.bad && a.bad[p])) return;
    const Sim3Xf x = *a.xf;
    const double X0 = a.pos[3 * p], X1 = a.pos[3 * p + 1], X2 = a.pos[3 * p + 2];
    double pa[3], pb[3], p4[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) pa[k] = ((x.R[3 * k] * X0 + x.R[3 * k + 1] * X1) + x.R[3 * k + 2] * X2) + x.t[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) pb[k] = ((x.sR[3 * k] * pa[0] + x.sR[3 * k + 1] * pa[1]) + x.sR[3 * k + 2] * pa[2]) + x.st[k];
    const double* M = a.mc_inv + 16 * c;
#pragma unroll
    for (int k = 0; k < 3; ++k) p4[k] = ((M[4 * k] * pb[0] + M[4 * k + 1] * pb[1]) + M[4 * k + 2] * pb[2]) + M[4 * k + 3] * 1.0;
    if (pb[2] < 0.0) return;
    const mcs_ocam cam = a.models[c];
    double x_, y_;
    cam_world_to_img(cam, p4[0], p4[1], p4[2], x_, y_);
    const int ur = __double2int_rn(x_), vr = __double2int_rn(y_);
    if (ur >= cam.width || ur <= 0 || vr >= cam.height || vr <= 0) return;
    if (!a.masks[(size_t)c * cam.width * cam.height + (size_t)vr * cam.width + ur]) return;
    const double d = sqrt((p4[0] * p4[0] + p4[1] * p4[1]) + p4[2] * p4[2]);
    int lv;
    if (!predict_level(d, a.dmin[p], a.dmax[p], a.sf, a.n_levels, lv)) return;
    ok[s] = 1; u[s] = x_; v[s] = y_; level[s] = lv;
}

// best[entry[q]] = dec[q]: a direction's decisions by slot of the key frame carried over (best starts at -1)
__global__ void s3_scatter_kernel(const int* __restrict__ nq_p, const int* __restrict__ entry, const int* __restrict__ dec, int* __restrict__ best) {
    const int nq = *nq_p;
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x) best[entry[q]] = dec[q];
}

// The agreement (ref :1964-1985): matches12[s1] = mp2[s2] where b1[s1] = s2 and b2[s2] = s1; nfound counts them.
__global__ void __launch_bounds__(256) s3_mutual_kernel(const PsCamSlots* __restrict__ kf1, const int n_cams, const int capacity,
                                                        const int* __restrict__ b1, const int* __restrict__ b2, const int* __restrict__ mp2,
                                                        int* __restrict__ matches12, int* __restrict__ nfound) {
    __shared__ int s_n;
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    if (s < n_cams * capacity) {
        const int s2 = ps_live(kf1, capacity, s) ? b1[s] : -1;
        if (s2 >= 0 && b2[s2] == s) {
            matches12[s] = mp2[s2];
            atomicAdd(&s_n, 1);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0 && s_n) atomicAdd(nfound, s_n);
}

// ---- SearchByProjection(pKF, Scw, vpPoints, vpMatched, th) (ref :2265-2392) ----
// first[c]: the first contiguous keypoint id of camera c (the counts before it, each clamped to the capacity); first[n_cams]: the
// key frame's keypoints.
__global__ void scw_first_kernel(const PsCamSlots* __restrict__ cams, const int n_cams, const int capacity, int* __restrict__ first) {
    int acc = 0;
    for (int c = 0; c < n_cams; ++c) { first[c] = acc; acc += min(*cams[c].count, capacity); }
    first[n_cams] = acc;
}

// found[p] = 1 for every point a slot of vpMatched holds on entry (spAlreadyFound).  Ids >= n_points mark their keypoint taken and
// find no point.
__global__ void scw_found_kernel(const PsCamSlots* __restrict__ cams, const int n_cams, const int capacity, const int n_points,
                                 const int* __restrict__ matched, uint8_t* __restrict__ found) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_cams * capacity) return;
    if (!ps_live(cams, capacity, s)) return;
    const int p = matched[s];
    if (p >= 0 && p < n_points) found[p] = 1;
}

// Entry i of vpPoints: its point p, when not NULL, not bad and not already found, is projected into the camera of CONTIGUOUS
// KEYPOINT i of the key frame (keypoint_to_cam.find(iMP), :2307) with the Sim3's rigid pose (WorldToCamHom_fast, mirror mask), its
// double distance to ow tested against [min, max] and its level predicted, as fu_project_kernel does for MCS_FUSE_SIM3.  An entry
// at or beyond the key frame's keypoints (where the reference dereferences end(): undefined) and an id >= n_points are dropped and
// raise status.
struct ScwProjArgs {
    int n_q, n_cams, n_points, n_levels;
    const int* points; const uint8_t* bad; const uint8_t* found; const int* first;
    const double* pos; const double* dmin; const double* dmax;
    const mcs_ocam* models; const double* mtmc_inv; const double* ow; const uint8_t* masks; const double* sf;
};
__global__ void __launch_bounds__(256) scw_project_kernel(const ScwProjArgs a, uint8_t* __restrict__ ok, double* __restrict__ u,
                                                          double* __restrict__ v, int* __restrict__ level, int* __restrict__ qcam,
                                                          int* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n_q) return;
    ok[i] = 0;
    const int p = a.points[i];
    if (p < 0) return;
    if (p >= a.n_points) { *status = MCS_ERR_INVALID; return; }
    if ((a.bad && a.bad[p]) || a.found[p]) return;
    if (i >= a.first[a.n_cams]) { *status = MCS_ERR_INVALID; return; }
    int c = 0;
    while (i >= a.first[c + 1]) ++c;
    const mcs_ocam cam = a.models[c];
    const double P0 = a.pos[3 * p], P1 = a.pos[3 * p + 1], P2 = a.pos[3 * p + 2];
    double x, y;
    if (!cam_project_in_mask(a.mtmc_inv + 16 * c, cam, a.masks + (size_t)c * cam.width * cam.height, P0, P1, P2, x, y)) return;
    const double o0 = P0 - a.ow[0], o1 = P1 - a.ow[1], o2 = P2 - a.ow[2];
    const double d = sqrt((o0 * o0 + o1 * o1) + o2 * o2);
    int lv;
    if (!predict_level(d, a.dmin[p], a.dmax[p], a.sf, a.n_levels, lv)) return;
    ok[i] = 1; u[i] = x; v[i] = y; level[i] = lv; qcam[i] = c;
}

}  // namespace

int proj_search_max_rounds() { return kPsRounds; }

namespace {

// frame_prepare_kernel's camera table for a search without camera models: it reads only width and height (no rays)
std::vector<mcs_ocam> cam_sizes(const PsFrameArgs& a) {
    std::vector<mcs_ocam> hc(a.n_cams);
    std::memset(hc.data(), 0, sizeof(mcs_ocam) * a.n_cams);
    for (int c = 0; c < a.n_cams; ++c) { hc[c].width = a.cam_w[c]; hc[c].height = a.cam_h[c]; }
    return hc;
}

// What the front end of the searches leaves for an acceptance stage, in one stream-ordered scratch block the caller releases: the
// frame searched in slot order with its grid, the queries in the maker's order and their lists, and the acceptance scratch.
struct PsFront {
    StreamScratch sc;
    WindowFrameDev f;
    const mcs_keypoint* keys;    // the searched frame in slot order
    const mcs_window_query* qry; const unsigned* lkey; const int* lslot; const int* lcnt;
    const int* qoff;                                         // the query fill's block offsets (kQbTile entries of the maker per block)
    int* ctl; int* dec; unsigned* owner;                     // PsState's; owner starts at 0xFFFFFFFF
    const uint32_t* qd; const uint32_t* qk;                  // the query descriptors and masks (qk NULL unless masked)
    long long Q;                                             // queries at most (the maker's size)
    int sms, wblocks;
};

// The front end from the query maker on: the frame view of `a` in slot order and its grid, the queries in the maker's order and
// their lists.  slots, cams: the searched frame's slot table and camera table [a.n_cams] on the device.  qdesc / qmask: the query
// descriptors, row desc_index.  cam_first (may be NULL): the device [n_cams + 1] first contiguous ids of SearchByProjection(KF,
// Scw); the frame view then carries the rows ps_gather_kernel<true> picks, and the view's cam_first is set for MCS_RULE_SCW.
template <class QM>
cudaError_t ps_front(const PsFrameArgs& a, const QM& qm, const PsCamSlots* slots, const mcs_ocam* cams, const int* cam_first,
                     const uint8_t* qdesc, const uint8_t* qmask, PsFront& fr, cudaStream_t st) {
    const int NS = a.n_cams * a.capacity;
    const int ncell = a.n_cams * MCS_FRAME_GRID_COLS * MCS_FRAME_GRID_ROWS;
    const long long Q = qm.size();
    const int nb = (int)((Q + kQbTile - 1) / kQbTile);
    const size_t db = (size_t)NS * a.dim;
    int sms = 0;
    cudaError_t e = sm_count(sms);
    if (e != cudaSuccess) return e;
    StreamScratch& sc = fr.sc;
    e = sc.alloc({sizeof(mcs_keypoint) * NS, 4ull * NS, 4ull * NS, 4ull * NS, 4ull * NS, db, a.masked ? db : 0,    // keys key_cam kx ky koct desc dmask
                  4ull * NS, 4ull * ncell, 4ull * (ncell + 1), 4ull * NS, 8ull * a.n_cams, 8ull * a.n_cams,         // cell_of cursor start items winv hinv
                  4ull * (nb + 1), 4ull * (nb + 1), 4ull * (4 + kPsRounds),                                         // block counts / offsets, ctl
                  sizeof(mcs_window_query) * Q, 4ull * Q * kPsK, 4ull * Q * kPsK, 4ull * Q, 8ull * Q, 8ull * NS},   // qry lkey lslot lcnt dec owner
                 st);
    if (e != cudaSuccess) return e;
    mcs_keypoint* keys = sc.at<mcs_keypoint>(0); int* key_cam = sc.at<int>(1); float* kx = sc.at<float>(2); float* ky = sc.at<float>(3);
    int* koct = sc.at<int>(4); uint8_t* desc = sc.at<uint8_t>(5); uint8_t* dmask = a.masked ? sc.at<uint8_t>(6) : nullptr;
    int* cell_of = sc.at<int>(7); int* cursor = sc.at<int>(8); int* cell_start = sc.at<int>(9); int* cell_items = sc.at<int>(10);
    double* winv = sc.at<double>(11); double* hinv = sc.at<double>(12);
    int* bcount = sc.at<int>(13); int* boff = sc.at<int>(14); int* ctl = sc.at<int>(15);
    mcs_window_query* qry = sc.at<mcs_window_query>(16); unsigned* lkey = sc.at<unsigned>(17); int* lslot = sc.at<int>(18);
    int* lcnt = sc.at<int>(19); int* dec = sc.at<int>(20); unsigned* owner = sc.at<unsigned>(21);

    e = cudaMemsetAsync(ctl, 0, 16, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(ctl + 4, 0x7F, 4 * kPsRounds, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(owner, 0xFF, 8ull * NS, st);
    if (e != cudaSuccess) return e;

    // frame view in slot order and its grid (the kernel the host entry points build their grid with)
    if (cam_first)
        ps_gather_kernel<true><<<(NS + 255) / 256, 256, 0, st>>>(slots, cam_first, a.n_cams, a.capacity, a.dim, a.masked, keys, key_cam, desc, dmask);
    else
        ps_gather_kernel<false><<<(NS + 255) / 256, 256, 0, st>>>(slots, nullptr, a.n_cams, a.capacity, a.dim, a.masked, keys, key_cam, desc, dmask);
    e = launch_frame_prepare(keys, key_cam, NS, cams, a.n_cams, kx, ky, koct, nullptr, cell_of, cursor, cell_start, cell_items, winv, hinv, st);
    // queries in the reference's order
    if (e == cudaSuccess && nb > 0) {
        ps_count_kernel<<<nb, kQbThreads, 0, st>>>(qm, bcount, a.status);
        ps_scan_kernel<<<1, 1024, 0, st>>>(bcount, nb, boff, ctl);
        ps_fill_kernel<<<nb, kQbThreads, 0, st>>>(qm, boff, qry);
        e = cudaGetLastError();
    }
    fr.f = WindowFrameDev{a.n_cams, NS, a.dim, kx, ky, koct, desc, dmask, cell_start, cell_items, winv, hinv, cam_first};
    fr.keys = keys;
    fr.qry = qry; fr.lkey = lkey; fr.lslot = lslot; fr.lcnt = lcnt; fr.qoff = boff; fr.ctl = ctl; fr.dec = dec; fr.owner = owner;
    fr.qd = (const uint32_t*)qdesc; fr.qk = a.masked ? (const uint32_t*)qmask : nullptr;
    fr.Q = Q; fr.sms = sms;
    fr.wblocks = (int)std::min<long long>((Q + 7) / 8, (long long)sms * 16);
    if (e == cudaSuccess && Q > 0) {
        with_desc_width(a.dim, a.masked, [&](auto W, auto M) {
            ps_list_kernel<W, M><<<fr.wblocks, 256, 0, st>>>(fr.f, qry, ctl, fr.qd, fr.qk, lkey, lslot, lcnt);
        });
        e = cudaGetLastError();
    }
    return e;
}

// Both searches from the query maker on: the front end, then the rounds and the walk under RULE.  tag: see PsState.  slots, cams,
// cam_first: see ps_front.  The caller has zeroed a.nmatches and a.status.
template <int RULE, class QM>
cudaError_t ps_search(const PsFrameArgs& a, const QM& qm, const double nnratio, const uint8_t* qdesc, const uint8_t* qmask, const int* tag,
                      const PsCamSlots* slots, const mcs_ocam* cams, const int* cam_first, cudaStream_t st) {
    const int NS = a.n_cams * a.capacity;
    PsFront fr;
    cudaError_t e = ps_front(a, qm, slots, cams, cam_first, qdesc, qmask, fr, st);
    const long long Q = fr.Q;
    if (e == cudaSuccess && Q > 0) {
        const PsState p{fr.qry, fr.lkey, fr.lslot, fr.lcnt, fr.dec, fr.owner, fr.ctl, (int)Q, NS, a.capacity, a.th_high, nnratio, tag};
        const int fblocks = (int)std::min<long long>((Q + 255) / 256, (long long)fr.sms * 4);
        const size_t walk_smem = 4ull * ((a.capacity + 31) / 32);
        with_desc_width(a.dim, a.masked, [&](auto W, auto M) {
            for (int r = 0; r < kPsRounds; ++r) ps_round_kernel<RULE, W, M><<<fr.wblocks, 256, 0, st>>>(fr.f, p, r, fr.qd, fr.qk, a.frame_mp);
            ps_finalize_kernel<<<fblocks, 256, 0, st>>>(p, a.frame_mp, a.nmatches);
            ps_walk_kernel<RULE, W, M><<<a.n_cams, 32, walk_smem, st>>>(fr.f, p, fr.qd, fr.qk, a.frame_mp, a.nmatches);
        });
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && a.diag) ps_diag_kernel<<<1, 1, 0, st>>>(fr.ctl, a.diag);
    if (e == cudaSuccess) e = cudaGetLastError();
    return fr.sc.release(e);
}

cudaError_t ps_zero_outputs(const PsFrameArgs& a, cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(a.nmatches, 0, 4, st);
    if (e == cudaSuccess && a.status) e = cudaMemsetAsync(a.status, 0, 4, st);     // NULL: a search whose input cannot be invalid
    return e;
}

// What the searches between two frames share, in the launcher's one stream-ordered scratch block: its own pieces (`own`, from
// piece 0 on), the last frame in slot order, and the staged slot tables of cur and last, camera table (the models when the search
// projects, else the image sizes), mtmc_inv (searches that project) and scale factors.  The caller releases `sc`, whatever the
// result.
struct TwoFrameScratch {
    StreamScratch sc;
    const PsCamSlots* cur; const PsCamSlots* last; const mcs_ocam* cams; const double* mtmc_inv; const double* sf;
    mcs_keypoint* keys; uint8_t* desc; uint8_t* dmask;      // the last frame in slot order (dmask NULL unless masked)
};

// Allocates and stages those pieces, zeroes the outputs and gathers the last frame into slot order (without a grid).
cudaError_t ps_open_two_frames(const PsTwoFrameArgs& a, std::vector<size_t> own, TwoFrameScratch& t, cudaStream_t st) {
    const int NS = a.n_cams * a.capacity;
    const size_t db = (size_t)NS * a.dim, k = own.size();
    own.insert(own.end(), {sizeof(mcs_keypoint) * NS, db, a.masked ? db : 0});
    const bool pose = a.models != nullptr;
    const std::vector<mcs_ocam> sizes = pose ? std::vector<mcs_ocam>() : cam_sizes(a);
    cudaError_t e = open_scratch(t.sc, own, st, host_in(t.cur, a.cams, a.n_cams), host_in(t.last, a.last, a.n_cams),
                                 host_in(t.cams, pose ? a.models : sizes.data(), a.n_cams), host_in(t.mtmc_inv, a.mtmc_inv, pose ? 16 * a.n_cams : 0),
                                 host_in(t.sf, a.sf, a.n_levels));
    if (e != cudaSuccess) return e;
    t.keys = t.sc.at<mcs_keypoint>(k); t.desc = t.sc.at<uint8_t>(k + 1); t.dmask = a.masked ? t.sc.at<uint8_t>(k + 2) : nullptr;
    e = ps_zero_outputs(a, st);
    if (e == cudaSuccess) {
        ps_gather_kernel<false><<<(NS + 255) / 256, 256, 0, st>>>(t.last, nullptr, a.n_cams, a.capacity, a.dim, a.masked, t.keys, nullptr, t.desc,
                                                                  t.dmask);
        e = cudaGetLastError();
    }
    return e;
}

}  // namespace

cudaError_t launch_search_by_projection(const ProjSearchArgs& a, cudaStream_t st) {
    cudaError_t e = ps_zero_outputs(a, st);
    if (e != cudaSuccess) return e;
    const std::vector<mcs_ocam> sizes = cam_sizes(a);
    const PsCamSlots* slots; const mcs_ocam* cams; const double* sf;
    StreamScratch sc;
    e = open_scratch(sc, {}, st, host_in(slots, a.cams, a.n_cams), host_in(cams, sizes.data(), a.n_cams), host_in(sf, a.sf, a.n_levels));
    if (e == cudaSuccess) {
        const MapPointQueries qm{a.n_cams, a.n_points, a.n_levels, a.bad, a.in_view, a.level, a.px, a.py, a.vcos, sf, a.th};
        e = ps_search<MCS_RULE_LEVEL_RATIO>(a, qm, a.nnratio, a.mp_desc, a.mp_dmask, nullptr, slots, cams, nullptr, st);
    }
    return sc.release(e);
}

// The last frame's queries (pl_project_kernel), then the current frame searched under MCS_RULE_BEST with the last frame's
// descriptors as the query rows and last_mp as the tags.
cudaError_t launch_search_by_projection_last(const ProjSearchLastArgs& a, cudaStream_t st) {
    const int NS = a.n_cams * a.capacity;
    TwoFrameScratch t;
    cudaError_t e = ps_open_two_frames(a, {(size_t)NS, 8ull * NS, 8ull * NS}, t, st);      // ok u v
    if (e != cudaSuccess) return t.sc.release(e);
    uint8_t* ok = t.sc.at<uint8_t>(0); double* u = t.sc.at<double>(1); double* v = t.sc.at<double>(2);
    const LastProjArgs pa{t.last, a.n_cams, a.capacity, a.n_levels, a.n_points, t.keys, a.last_mp, a.last_outlier, a.bad, a.world_pos,
                          t.cams, t.mtmc_inv, a.masks};
    pl_project_kernel<<<(NS + 255) / 256, 256, 0, st>>>(pa, ok, u, v, a.status);
    e = cudaGetLastError();
    if (e == cudaSuccess) {
        const LastFrameQueries qm{NS, a.capacity, ok, u, v, t.keys, t.sf, a.th};
        e = ps_search<MCS_RULE_BEST>(a, qm, 0.0, t.desc, t.dmask, a.last_mp, t.cur, t.cams, nullptr, st);
    }
    return t.sc.release(e);
}

// WindowSearch: cur_mp cleared below each camera's count, then the current frame searched under MCS_RULE_RATIO with one query per
// qualifying last-frame slot and last_mp as the tags.
cudaError_t launch_window_search_device(const WindowSearchDevArgs& a, cudaStream_t st) {
    const int NS = a.n_cams * a.capacity;
    TwoFrameScratch t;
    cudaError_t e = ps_open_two_frames(a, {}, t, st);
    if (e != cudaSuccess) return t.sc.release(e);
    pw_clear_kernel<<<(NS + 255) / 256, 256, 0, st>>>(t.cur, a.n_cams, a.capacity, a.frame_mp);
    e = cudaGetLastError();
    if (e == cudaSuccess) {
        const WindowQueries qm{NS, a.capacity, a.n_points, a.min_level, a.max_level, t.last, t.keys, a.last_mp, a.bad, nullptr, a.window};
        e = ps_search<MCS_RULE_RATIO>(a, qm, a.nnratio, t.desc, t.dmask, a.last_mp, t.cur, t.cams, nullptr, st);
    }
    return t.sc.release(e);
}

// SearchByProjection(F1 = last, F2 = cur): the skip flags (pf_flag_kernel), the (slot, camera) projections (pf_project_kernel),
// then the current frame searched under MCS_RULE_RATIO with last_mp as the tags.
cudaError_t launch_search_by_projection_frames(const SearchFramesDevArgs& a, cudaStream_t st) {
    const int NS = a.n_cams * a.capacity;
    const size_t NK = (size_t)NS * a.n_cams;
    TwoFrameScratch t;
    cudaError_t e = ps_open_two_frames(a, {(size_t)a.n_points, 4ull * a.n_points, NK, 8 * NK, 8 * NK}, t, st);   // found first ok u v
    if (e != cudaSuccess) return t.sc.release(e);
    uint8_t* found = t.sc.at<uint8_t>(0); int* first = t.sc.at<int>(1);
    uint8_t* ok = t.sc.at<uint8_t>(2); double* u = t.sc.at<double>(3); double* v = t.sc.at<double>(4);
    if (a.n_points > 0) e = cudaMemsetAsync(found, 0, a.n_points, st);
    if (e == cudaSuccess && a.n_points > 0) e = cudaMemsetAsync(first, 0x7F, 4ull * a.n_points, st);     // above every slot
    if (e == cudaSuccess) {
        pf_flag_kernel<<<(NS + 255) / 256, 256, 0, st>>>(t.cur, t.last, a.n_cams, a.capacity, a.n_points, a.frame_mp, a.last_mp, found, first,
                                                         a.status);
        const FramesProjArgs pa{t.last, a.n_cams, a.capacity, a.n_points, a.last_mp, a.bad, found, first, a.world_pos, t.cams, t.mtmc_inv,
                                a.masks};
        pf_project_kernel<<<(unsigned)((NK + 255) / 256), 256, 0, st>>>(pa, ok, u, v);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        const FramesQueries qm{NS, a.n_cams, ok, u, v, t.keys, nullptr, a.window};
        e = ps_search<MCS_RULE_RATIO>(a, qm, a.nnratio, t.desc, t.dmask, a.last_mp, t.cur, t.cams, nullptr, st);
    }
    return t.sc.release(e);
}

// SearchForInitialization(F1 = last, F2 = cur): one query per F1 slot below its count, centred on prev, then the ordered walk
// (pi_walk_kernel) instead of the rounds.
cudaError_t launch_search_for_initialization(const InitSearchDevArgs& a, cudaStream_t st) {
    TwoFrameScratch t;
    cudaError_t e = ps_open_two_frames(a, {}, t, st);
    if (e != cudaSuccess) return t.sc.release(e);
    const InitQueries qm{a.n_cams * a.capacity, a.capacity, t.last, t.keys, a.prev, nullptr, (double)a.window};
    PsFront fr;
    e = ps_front(a, qm, t.cur, t.cams, nullptr, t.desc, t.dmask, fr, st);
    if (e == cudaSuccess && fr.Q > 0) {
        const InitWalk w{fr.qry, fr.lkey, fr.lslot, fr.lcnt, fr.ctl, t.last, t.cur, fr.keys, fr.dec, (int*)fr.owner, a.n_cams, a.capacity,
                         a.th_high, a.nnratio, a.matches12, a.prev, a.nmatches};
        const size_t smem = 2ull * a.capacity;              // MD of one camera's F2 slots
        with_desc_width(a.dim, a.masked, [&](auto W, auto M) {
            // The opt-in is set on every call: without it the static lists and MD together must fit in 48 KB, which capacities
            // from 23 489 up do not (per device, so a set attribute cannot be remembered across devices either).
            e = cudaFuncSetAttribute(pi_walk_kernel<W, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e == cudaSuccess) pi_walk_kernel<W, M><<<a.n_cams, 32, smem, st>>>(fr.f, w, fr.qd, fr.qk);
        });
        if (e == cudaSuccess) e = cudaGetLastError();
    }
    if (e == cudaSuccess && a.diag) pi_diag_kernel<<<1, 1, 0, st>>>(fr.ctl, a.diag);
    if (e == cudaSuccess) e = cudaGetLastError();
    return t.sc.release(fr.sc.release(e));
}

// Fuse for n_kf key frames: membership pre-filter (fu_qmap / fu_held), the (k, q, c) projections (fu_project), the front end over
// the n_kf * n_cams images with the projected queries, the stateless decision (fu_best or fu_first), then a count / scan / fill of
// the hits in query order.  Scratch beyond the front end's: 4 * n_points + n_kf * n_q bytes for the pre-filter and 33 bytes per
// entry.
cudaError_t launch_fuse_device(const FuseDevArgs& a, cudaStream_t st) {
    const int nk = a.n_kf, nc = a.n_kf_cams, NI = nk * nc;
    const long long QE = (long long)nk * a.n_q * nc;
    const int nb = (int)((QE + kQbTile - 1) / kQbTile);
    cudaError_t e = cudaMemsetAsync(a.n_hits, 0, 4, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(a.status, 0, 4, st);
    if (e != cudaSuccess) return e;
    std::vector<mcs_ocam> models;            // the camera table of the searched frame's NI images; fu_project reads the first nc
    for (int k = 0; k < nk; ++k) models.insert(models.end(), a.pts.models, a.pts.models + nc);
    const PsCamSlots* slots; const int* const* kf_mp; const double* mtmc_inv; const double* ow; const mcs_ocam* cams; const double* sf;
    StreamScratch sc;
    e = open_scratch(sc, {4ull * a.pts.n_points, (size_t)nk * a.n_q,                                                                    // qmap held
                          (size_t)QE, 8ull * QE, 8ull * QE, 4ull * QE, 4ull * QE, 4ull * QE, 4ull * (nb + 1), 4ull * (nb + 1)},          // ok u v level entry dec
                     st, host_in(slots, a.cams, NI), host_in(kf_mp, a.kf_mp, nk), host_in(mtmc_inv, a.mtmc_inv, 16 * NI), host_in(ow, a.ow, 3 * nk),
                     host_in(cams, models.data(), NI), host_in(sf, a.sf, a.n_levels));
    if (e != cudaSuccess) return sc.release(e);
    int* qmap = sc.at<int>(0); uint8_t* held = sc.at<uint8_t>(1);
    uint8_t* ok = sc.at<uint8_t>(2); double* u = sc.at<double>(3); double* v = sc.at<double>(4); int* level = sc.at<int>(5);
    int* entry = sc.at<int>(6); int* dec = sc.at<int>(7); int* bcount = sc.at<int>(8); int* boff = sc.at<int>(9);
    if (a.pts.n_points > 0) e = cudaMemsetAsync(qmap, 0x7F, 4ull * a.pts.n_points, st);     // above every query position
    if (e == cudaSuccess && nk * a.n_q > 0) e = cudaMemsetAsync(held, 0, (size_t)nk * a.n_q, st);
    if (e != cudaSuccess) return sc.release(e);
    if (a.n_q > 0) {
        fu_qmap_kernel<<<(a.n_q + 255) / 256, 256, 0, st>>>(a.query_mp, a.n_q, a.pts.n_points, qmap, a.status);
        const long long ns = (long long)NI * a.capacity;
        fu_held_kernel<<<(unsigned)((ns + 255) / 256), 256, 0, st>>>(slots, kf_mp, nk, nc, a.capacity, a.n_q, a.pts.n_points, qmap, held);
        const FuseProjArgs pa{nk, nc, a.n_q, a.pts.n_points, a.n_levels, a.variant != MCS_FUSE_SIM3, a.query_mp, a.pts.bad, held, qmap,
                              a.pts.world_pos, a.pts.min_dist, a.pts.max_dist, cams, mtmc_inv, ow, a.pts.masks, sf};
        fu_project_kernel<<<(unsigned)((QE + 255) / 256), 256, 0, st>>>(pa, ok, u, v, level);
        e = cudaGetLastError();
    }
    PsFront fr;
    if (e == cudaSuccess) {
        const ProjectedQueries<FuseAt> qm{QE, ok, u, v, level, sf, a.th, {a.n_q, nc, a.query_mp}};
        e = ps_front(a, qm, slots, cams, nullptr, a.pts.desc, a.pts.dmask, fr, st);
        if (e == cudaSuccess && nb > 0) {
            fu_entry_kernel<<<nb, kQbThreads, 0, st>>>(qm, fr.qoff, entry);
            if (a.variant == MCS_FUSE_FIRST) {
                fu_first_kernel<<<fr.wblocks, 256, 0, st>>>(fr.f, fr.qry, fr.ctl, fr.lcnt, a.th_high, dec);
            } else {
                const int blocks = (int)std::min<long long>((QE + 255) / 256, (long long)fr.sms * 8);
                fu_best_kernel<<<blocks, 256, 0, st>>>(fr.ctl, fr.lkey, fr.lslot, a.th_high, dec);
            }
            const FuseHitQueries hq{QE, fr.ctl, dec};
            ps_count_kernel<<<nb, kQbThreads, 0, st>>>(hq, bcount, nullptr);
            ps_scan_kernel<<<1, 1024, 0, st>>>(bcount, nb, boff, a.n_hits);
            fu_hits_kernel<<<nb, kQbThreads, 0, st>>>(hq, boff, entry, a.n_q, nc, a.capacity, a.max_hits, a.hits, a.status);
            e = cudaGetLastError();
        }
    }
    return sc.release(fr.sc.release(e));
}

// SearchBySim3: per direction the slot projections (s3_project_kernel), the front end over the other key frame with the projected
// queries, Fuse's stateless decision under th_high and the scatter of the decisions to slots; then the mutual check.  The
// projection and list scratch of direction 1 is reused by direction 2 in stream order.
cudaError_t launch_search_by_sim3(const Sim3SearchDevArgs& a, cudaStream_t st) {
    const int NS = a.n_cams * a.capacity, nb = (NS + kQbTile - 1) / kQbTile;
    static_assert(sizeof(Sim3Xf) == 24 * sizeof(double), "two directions of 24 doubles");
    cudaError_t e = ps_zero_outputs(a, st);
    if (e != cudaSuccess) return e;
    const PsCamSlots* s1; const PsCamSlots* s2; const mcs_ocam* models; const double* mc_inv; const Sim3Xf* xf; const double* sf;
    StreamScratch sc;
    e = open_scratch(sc, {(size_t)NS, 8ull * NS, 8ull * NS, 4ull * NS, 4ull * NS, 4ull * NS, 4ull * NS, 4ull * NS}, st,        // ok u v level entry dec b1 b2
                     host_in(s1, a.kf1, a.n_cams), host_in(s2, a.cams, a.n_cams), host_in(models, a.pts.models, a.n_cams),
                     host_in(mc_inv, a.mc_inv, 16 * a.n_cams), host_in(xf, (const Sim3Xf*)a.xf, 2), host_in(sf, a.sf, a.n_levels));
    if (e != cudaSuccess) return sc.release(e);
    uint8_t* ok = sc.at<uint8_t>(0); double* u = sc.at<double>(1); double* v = sc.at<double>(2); int* level = sc.at<int>(3);
    int* entry = sc.at<int>(4); int* dec = sc.at<int>(5); int* b1 = sc.at<int>(6); int* b2 = sc.at<int>(7);
    e = cudaMemsetAsync(b1, 0xFF, 4ull * NS, st);        // no decision yet: -1
    if (e == cudaSuccess) e = cudaMemsetAsync(b2, 0xFF, 4ull * NS, st);
    int sms = 0;
    if (e == cudaSuccess) e = sm_count(sms);
    const int blocks = (int)std::min<long long>((NS + 255) / 256, (long long)sms * 8);
    for (int dir = 0; dir < 2 && e == cudaSuccess; ++dir) {
        const bool one = dir == 0;                           // direction 1: KF1's points into KF2; direction 2: KF2's into KF1
        const int* mp = one ? a.mp1 : a.mp2;
        const Sim3ProjArgs pa{one ? s1 : s2, a.n_cams, a.capacity, a.pts.n_points, a.n_levels, mp, one ? a.matches12 : nullptr,
                              one ? nullptr : a.already2, a.pts.bad, a.pts.world_pos, a.pts.min_dist, a.pts.max_dist, models, xf + dir, mc_inv,
                              a.pts.masks, sf};
        s3_project_kernel<<<(NS + 255) / 256, 256, 0, st>>>(pa, ok, u, v, level, a.status);
        e = cudaGetLastError();
        const ProjectedQueries<Sim3At> qm{NS, ok, u, v, level, sf, a.th, {a.capacity, mp}};
        PsFront fr;
        if (e == cudaSuccess) e = ps_front(a, qm, one ? s2 : s1, models, nullptr, a.pts.desc, a.pts.dmask, fr, st);
        if (e == cudaSuccess) {
            fu_entry_kernel<<<nb, kQbThreads, 0, st>>>(qm, fr.qoff, entry);
            fu_best_kernel<<<blocks, 256, 0, st>>>(fr.ctl, fr.lkey, fr.lslot, a.th_high, dec);
            s3_scatter_kernel<<<blocks, 256, 0, st>>>(fr.ctl, entry, dec, one ? b1 : b2);
            e = cudaGetLastError();
        }
        e = fr.sc.release(e);
    }
    if (e == cudaSuccess) {
        s3_mutual_kernel<<<(NS + 255) / 256, 256, 0, st>>>(s1, a.n_cams, a.capacity, b1, b2, a.mp2, a.matches12, a.nmatches);
        e = cudaGetLastError();
    }
    return sc.release(e);
}

// SearchByProjection(KF, Scw): the first contiguous ids (scw_first_kernel), spAlreadyFound (scw_found_kernel), the entry projections
// (scw_project_kernel), then the rounds and the walk under MCS_RULE_SCW over ps_gather_kernel<true>'s view, with the map-point ids
// as the tags (desc_index).
cudaError_t launch_search_by_projection_scw(const ScwSearchDevArgs& a, cudaStream_t st) {
    const int NS = a.n_cams * a.capacity;
    cudaError_t e = ps_zero_outputs(a, st);
    if (e != cudaSuccess) return e;
    const PsCamSlots* slots; const mcs_ocam* models; const double* mtmc_inv; const double* ow; const double* sf;
    StreamScratch sc;
    e = open_scratch(sc, {4ull * (a.n_cams + 1), (size_t)a.pts.n_points,                                                   // first found
                          (size_t)a.n_q, 8ull * a.n_q, 8ull * a.n_q, 4ull * a.n_q, 4ull * a.n_q},                          // ok u v level qcam
                     st, host_in(slots, a.cams, a.n_cams), host_in(models, a.pts.models, a.n_cams), host_in(mtmc_inv, a.mtmc_inv, 16 * a.n_cams),
                     host_in(ow, a.ow, 3), host_in(sf, a.sf, a.n_levels));
    if (e != cudaSuccess) return sc.release(e);
    int* first = sc.at<int>(0); uint8_t* found = sc.at<uint8_t>(1);
    uint8_t* ok = sc.at<uint8_t>(2); double* u = sc.at<double>(3); double* v = sc.at<double>(4); int* level = sc.at<int>(5);
    int* qcam = sc.at<int>(6);
    if (a.pts.n_points > 0) e = cudaMemsetAsync(found, 0, a.pts.n_points, st);
    if (e != cudaSuccess) return sc.release(e);
    scw_first_kernel<<<1, 1, 0, st>>>(slots, a.n_cams, a.capacity, first);
    scw_found_kernel<<<(NS + 255) / 256, 256, 0, st>>>(slots, a.n_cams, a.capacity, a.pts.n_points, a.frame_mp, found);
    if (a.n_q > 0) {
        const ScwProjArgs pa{a.n_q, a.n_cams, a.pts.n_points, a.n_levels, a.points, a.pts.bad, found, first, a.pts.world_pos, a.pts.min_dist,
                             a.pts.max_dist, models, mtmc_inv, ow, a.pts.masks, sf};
        scw_project_kernel<<<(a.n_q + 255) / 256, 256, 0, st>>>(pa, ok, u, v, level, qcam, a.status);
    }
    e = cudaGetLastError();
    if (e == cudaSuccess) {
        const ProjectedQueries<ScwAt> qm{a.n_q, ok, u, v, level, sf, (double)a.th, {qcam, a.points}};
        e = ps_search<MCS_RULE_SCW>(a, qm, 0.0, a.pts.desc, a.pts.dmask, nullptr, slots, models, first, st);
    }
    return sc.release(e);
}

cudaError_t launch_search_for_initialization_seed(const PsCamSlots* f1, int n_cams, int capacity, double* prev, cudaStream_t st) {
    const int NS = n_cams * capacity;
    const PsCamSlots* slots;
    StreamScratch sc;
    cudaError_t e = open_scratch(sc, {}, st, host_in(slots, f1, n_cams));
    if (e == cudaSuccess) {
        pi_seed_kernel<<<(NS + 255) / 256, 256, 0, st>>>(slots, n_cams, capacity, prev);
        e = cudaGetLastError();
    }
    return sc.release(e);
}

}  // namespace mcs
