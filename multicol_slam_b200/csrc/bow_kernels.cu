// bow_kernels.cu -- bag-of-words kernels (SURVEY 8f rank 4)
//   bow_descend_kernel : TemplatedVocabulary::transform(feature, word, weight, nid, levelsup)
//                        (ref ThirdParty/DBoW2/DBoW2/TemplatedVocabulary.h:1218-1261, FORB::distance FORB.cpp:84-104):
//                        16 lanes per descriptor, lane j scores child j of the current node, the group takes the first minimum.
//   group_distance_kernel : the distance half of cORBmatcher::SearchByBoW(KF, F) (ref src/cORBmatcher.cpp:205-262): one warp
//                        per key-frame keypoint, distances to every frame keypoint of the same vocabulary node, in list order.
//   bv_* kernels        : ComputeBoW on a frame in packed feature buffers, both containers built on the device (further down).
//   bs_search_kernel    : SearchByBoW(KF_i, F) whole, for a batch of key frames: one warp per (key frame, node) follows the
//                        reference's order inside the node; no distance list, the acceptance on the device (further down).
#include <climits>

#include "mcs_common.cuh"
#include "kernels.h"

namespace mcs {

constexpr int kBowGroup = 16;

// The descent of one descriptor (qa, qb) by its 16-lane group: `node` ends at the leaf, `at_level` at the ancestor `nid_level`
// steps below the root (0 when nid_level <= 0, -1 when the leaf is shallower).
__device__ __forceinline__ void bow_descend(const VocabularyDev& v, const uint4 qa, const uint4 qb, const int nid_level, const int gl,
                                            const unsigned gmask, int& node, int& at_level) {
    int level = 0;
    node = 0; at_level = nid_level <= 0 ? 0 : -1;
    for (;;) {
        const int c0 = __ldg(v.child_off + node), nc = __ldg(v.child_off + node + 1) - c0;
        if (nc == 0) break;                                                     // leaf (the root always has children)
        ++level;
        unsigned best = 0xFFFFFFFFu;                                            // distance << 16 | child position: first minimum wins
        for (int j = gl; j < nc; j += kBowGroup) {
            const int id = __ldg(v.child_ids + c0 + j);
            const uint4 da = __ldg(v.desc + 2 * (size_t)id), db = __ldg(v.desc + 2 * (size_t)id + 1);
            const unsigned d = __popc(qa.x ^ da.x) + __popc(qa.y ^ da.y) + __popc(qa.z ^ da.z) + __popc(qa.w ^ da.w) +
                               __popc(qb.x ^ db.x) + __popc(qb.y ^ db.y) + __popc(qb.z ^ db.z) + __popc(qb.w ^ db.w);
            best = min(best, (d << 16) | (unsigned)j);
        }
#pragma unroll
        for (int o = kBowGroup / 2; o; o >>= 1) best = min(best, __shfl_xor_sync(gmask, best, o, kBowGroup));
        node = __ldg(v.child_ids + c0 + (int)(best & 0xFFFFu));
        if (level == nid_level) at_level = node;
    }
}

__global__ void __launch_bounds__(256)
bow_descend_kernel(const VocabularyDev v, const uint4* __restrict__ desc, const int n, const int nid_level,
                   int* __restrict__ word, double* __restrict__ weight, int* __restrict__ node_out) {
    const int gi = (blockIdx.x * blockDim.x + threadIdx.x) / kBowGroup;          // descriptor of this group
    if (gi >= n) return;                                                        // whole groups leave together
    const int lane = threadIdx.x & 31, gl = lane & (kBowGroup - 1);
    const unsigned gmask = 0xFFFFu << (lane & ~(kBowGroup - 1));
    const uint4 qa = __ldg(desc + 2 * (size_t)gi), qb = __ldg(desc + 2 * (size_t)gi + 1);
    int node, at_level;
    bow_descend(v, qa, qb, nid_level, gl, gmask, node, at_level);
    if (gl == 0) {
        if (word) word[gi] = __ldg(v.word_of_node + node);
        if (weight) weight[gi] = __ldg(v.weight + node);
        if (node_out) node_out[gi] = at_level >= 0 ? at_level : node;            // shallower leaf: see include/mcs_b200.h
    }
}

cudaError_t launch_bow_descend(const VocabularyDev& v, const uint8_t* desc, int n, int levelsup, int* word, double* weight,
                               int* node, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    const long long threads = (long long)n * kBowGroup;
    bow_descend_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(v, (const uint4*)desc, n, v.L - levelsup, word, weight, node);
    return cudaGetLastError();
}

template <int WORDS, bool MASKED>
__global__ void __launch_bounds__(256)
group_distance_kernel(const GroupQuery* __restrict__ queries, const int nq, const uint32_t* __restrict__ desc1,
                      const uint32_t* __restrict__ mask1, const uint32_t* __restrict__ desc2, const uint32_t* __restrict__ mask2,
                      const int* __restrict__ cand, int* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int qi = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (qi >= nq) return;
    const GroupQuery q = queries[qi];
    uint32_t qw[WORDS], qm[MASKED ? WORDS : 1];
#pragma unroll
    for (int k = 0; k < WORDS; ++k) {
        qw[k] = __ldg(desc1 + (size_t)q.feature * WORDS + k);
        if (MASKED) qm[k] = __ldg(mask1 + (size_t)q.feature * WORDS + k);
    }
    for (int j = lane; j < q.cand_count; j += 32) {
        const int id = __ldg(cand + q.cand_start + j);
        const uint32_t* dd = desc2 + (size_t)id * WORDS;
        unsigned dist = 0;
        if (MASKED) {
            const uint32_t* mm = mask2 + (size_t)id * WORDS;
#pragma unroll
            for (int k = 0; k < WORDS; ++k) {
                const uint32_t xw = qw[k] ^ __ldg(dd + k);
                dist += __popc(xw & qm[k]) + __popc(xw & __ldg(mm + k));
            }
            dist >>= 1;                                                         // DescriptorDistance64Masked (ref :2452-2474)
        } else {
#pragma unroll
            for (int k = 0; k < WORDS; ++k) dist += __popc(qw[k] ^ __ldg(dd + k));
        }
        out[q.out_off + j] = (int)dist;
    }
}

cudaError_t launch_group_distance(const GroupQuery* queries, int nq, const uint8_t* desc1, const uint8_t* mask1, const uint8_t* desc2,
                                  const uint8_t* mask2, const int* cand, int dim, int* out, cudaStream_t st) {
    if (nq <= 0) return cudaSuccess;
    if (!desc_width_ok(dim)) return cudaErrorInvalidValue;
    const int blocks = (int)(((long long)nq * 32 + 255) / 256);
    const bool masked = mask1 && mask2;
    with_desc_width(dim, masked, [&](auto W, auto M) {
        group_distance_kernel<W, M><<<blocks, 256, 0, st>>>(queries, nq, (const uint32_t*)desc1, (const uint32_t*)mask1, (const uint32_t*)desc2,
                                                            (const uint32_t*)mask2, cand, out);
    });
    return cudaGetLastError();
}


// ------------------------------------------------------------------------------------------------
// ComputeBoW on a frame in packed feature buffers (mcs_bow_vectors_device)
// ------------------------------------------------------------------------------------------------
// Both containers of transform(features, BowVector&, FeatureVector&, levelsup) are a stable sort of the live features (word weight
// > 0) by a key, node id or word id, whose result is unique; it is built without a sort:
//   bv_descend_kernel     the descent per slot, reading the camera's descriptor section in place; counts the live slots per node id
//                         and per word id in two dense counter arrays
//   bv_tile_count / emit  a two-pass scan over each counter array in tiles of kBvTile ids that compacts the non-empty ids --
//                         ascending, as std::map iterates -- into fv_nodes + fv_offsets and bow_words + bow_values, and leaves
//                         every node's rank in its counter
//   bv_scatter_kernel     the live slots into their node's segment, in arrival order
//   bv_place_kernel       every slot to the position inside its segment that equals the number of smaller slots there
//   bv_normalize_kernel   the BowVector's "/ nb" or norm: the sum runs over the words in ascending order on one thread, because the
//                         double additions must happen in the order the host code makes them
namespace {

constexpr int kBvThreads = 256, kBvPer = 8, kBvTile = kBvThreads * kBvPer;

struct BvKeys {                 // one key space: node ids (FeatureVector) or word ids (BowVector)
    int* cnt;                   // [n] live slots per id; bv_tile_emit leaves the id's rank there (-1 beyond cap)
    int n;
    int* ids; int* offsets;     // compacted output: [cap] ids, [cap + 1] CSR offsets (NULL for words)
    int* n_out; int cap;
};

__global__ void __launch_bounds__(256)
bv_descend_kernel(const VocabularyDev v, const PsCamSlots* __restrict__ cams, const int n_slots, const int capacity, const int nid_level,
                  int* __restrict__ word_out, double* __restrict__ weight_out, int* __restrict__ node_out, int* __restrict__ key_node,
                  double* __restrict__ wt, int* __restrict__ cnt_node, int* __restrict__ cnt_word, int* __restrict__ word_rep) {
    const int s = (blockIdx.x * blockDim.x + threadIdx.x) / kBowGroup;          // slot of this group
    if (s >= n_slots) return;
    const int lane = threadIdx.x & 31, gl = lane & (kBowGroup - 1);
    const unsigned gmask = 0xFFFFu << (lane & ~(kBowGroup - 1));
    const int c = s / capacity, j = s - c * capacity;
    const PsCamSlots cs = cams[c];
    if (j >= min(*cs.count, capacity)) {                                        // not a keypoint: whole groups leave together
        if (gl == 0) key_node[s] = -1;
        return;
    }
    const uint4* q = (const uint4*)cs.desc + 2 * (size_t)j;
    const uint4 qa = __ldg(q), qb = __ldg(q + 1);
    int node, at_level;
    bow_descend(v, qa, qb, nid_level, gl, gmask, node, at_level);
    if (gl == 0) {
        const int w = __ldg(v.word_of_node + node), nd = at_level >= 0 ? at_level : node;
        const double wgt = __ldg(v.weight + node);
        if (word_out) word_out[s] = w;
        if (weight_out) weight_out[s] = wgt;
        if (node_out) node_out[s] = nd;
        const bool live = wgt > 0;                                              // stopped words are in neither vector (ref :1157-1161)
        key_node[s] = live ? nd : -1;
        if (live) {
            wt[s] = wgt;
            atomicAdd(cnt_node + nd, 1);
            atomicAdd(cnt_word + w, 1);
            word_rep[w] = s;                                                    // any slot of the word: they all carry its weight
        }
    }
}

// exclusive scan of x over the block; `total` = the block's sum.  x packs (non-empty ids << 32 | slots).
__device__ __forceinline__ unsigned long long bv_block_exclusive(const unsigned long long x, unsigned long long& total) {
    __shared__ unsigned long long wsum[kBvThreads / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    unsigned long long inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, inc, o);
        if (lane >= o) inc += y;
    }
    __syncthreads();                                                            // wsum may still be read from an earlier call
    if (lane == 31) wsum[w] = inc;
    __syncthreads();
    unsigned long long before = 0;
    total = 0;
#pragma unroll
    for (int i = 0; i < kBvThreads / 32; ++i) {
        if (i < w) before += wsum[i];
        total += wsum[i];
    }
    return before + inc - x;
}

// blockIdx.y = 0: node ids, 1: word ids.  tile_sums[y * max_tiles + tile] = (non-empty ids << 32 | slots) of the tile.
__global__ void __launch_bounds__(kBvThreads)
bv_tile_count_kernel(const BvKeys nodes, const BvKeys words, const int max_tiles, unsigned long long* __restrict__ tile_sums) {
    const BvKeys d = blockIdx.y ? words : nodes;
    const int first = blockIdx.x * kBvTile + threadIdx.x * kBvPer;
    if (blockIdx.x * kBvTile >= d.n) return;
    unsigned long long x = 0;
#pragma unroll
    for (int k = 0; k < kBvPer; ++k) {
        const int c = first + k < d.n ? d.cnt[first + k] : 0;
        if (c > 0) x += (1ull << 32) + (unsigned)c;
    }
    unsigned long long total;
    bv_block_exclusive(x, total);
    if (threadIdx.x == 0) tile_sums[blockIdx.y * max_tiles + blockIdx.x] = total;
}

__global__ void __launch_bounds__(kBvThreads)
bv_tile_emit_kernel(const BvKeys nodes, const BvKeys words, const int max_tiles, const unsigned long long* __restrict__ tile_sums,
                    const double* __restrict__ wt, const int* __restrict__ word_rep, const bool accumulate,
                    double* __restrict__ bow_values, int* __restrict__ status) {
    const BvKeys d = blockIdx.y ? words : nodes;
    const int tile = blockIdx.x, first = tile * kBvTile + threadIdx.x * kBvPer;
    if (tile * kBvTile >= d.n) return;
    unsigned long long x = 0, base;
    for (int t = threadIdx.x; t < tile; t += kBvThreads) x += tile_sums[blockIdx.y * max_tiles + t];
    bv_block_exclusive(x, base);                                                // everything in the tiles before this one
    int c[kBvPer];
    x = 0;
#pragma unroll
    for (int k = 0; k < kBvPer; ++k) {
        c[k] = first + k < d.n ? d.cnt[first + k] : 0;
        if (c[k] > 0) x += (1ull << 32) + (unsigned)c[k];
    }
    unsigned long long total;
    unsigned long long at = base + bv_block_exclusive(x, total);
#pragma unroll
    for (int k = 0; k < kBvPer; ++k) {
        if (c[k] <= 0) continue;
        const int r = (int)(at >> 32), off = (int)(at & 0xFFFFFFFFu), id = first + k;
        if (r < d.cap) d.ids[r] = id;
        if (d.offsets) {
            if (r <= d.cap) d.offsets[r] = off;                                 // rank cap closes the last segment that fits
            d.cnt[id] = r < d.cap ? r : -1;
        } else {
            // BowVector::addWeight adds the word's weight once per feature, in feature order; addIfNotExist keeps the first
            // (ref BowVector.cpp:34-59).  Every feature of a word carries the same weight, so the order is immaterial and the
            // number of additions is not.
            const double w = wt[word_rep[id]];
            double sum = w;
            if (accumulate)
                for (int i = 1; i < c[k]; ++i) sum += w;
            bow_values[r] = sum;                                                // cap = the number of slots: every word fits
        }
        at += (1ull << 32) + (unsigned)c[k];
    }
    if ((tile + 1) * kBvTile >= d.n && threadIdx.x == 0) {                      // the last tile knows the totals
        const unsigned long long all = base + total;
        const int n_ids = (int)(all >> 32);
        *d.n_out = min(n_ids, d.cap);
        if (d.offsets && n_ids <= d.cap) d.offsets[n_ids] = (int)(all & 0xFFFFFFFFu);
        if (n_ids > d.cap) *status = MCS_ERR_CAPACITY;
    }
}

__global__ void __launch_bounds__(256)
bv_scatter_kernel(const int n_slots, const int* __restrict__ key_node, const int* __restrict__ rank_of, const int* __restrict__ offsets,
                  int* __restrict__ fill, int* __restrict__ slot_rank, int* __restrict__ unordered) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    const int nd = key_node[s];
    const int r = nd < 0 ? -1 : rank_of[nd];
    slot_rank[s] = r;
    if (r >= 0) unordered[offsets[r] + atomicAdd(fill + r, 1)] = s;
}

// features inside a node ascend (std::map<NodeId, vector<unsigned>> filled in feature order): slot s goes to the position that
// equals the number of smaller slots of its segment.  One thread per slot, a segment's length of reads each.
__global__ void __launch_bounds__(256)
bv_place_kernel(const int n_slots, const int* __restrict__ slot_rank, const int* __restrict__ offsets, const int* __restrict__ unordered,
                int* __restrict__ fv_features) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    const int r = slot_rank[s];
    if (r < 0) return;
    const int lo = offsets[r], hi = offsets[r + 1];
    int pos = 0;
    for (int i = lo; i < hi; ++i) pos += unordered[i] < s;
    fv_features[lo + pos] = s;
}

constexpr int kBvNormChunk = 2048;
// ref TemplatedVocabulary.h:1165-1171 and BowVector::normalize (BowVector.cpp:63-87), in the operation order of mcs_bow_vectors
__global__ void __launch_bounds__(256)
bv_normalize_kernel(double* __restrict__ vals, const int* __restrict__ n_bow, const int scoring, const bool accumulate) {
    __shared__ double buf[kBvNormChunk];
    __shared__ double norm_s;
    const int nb = *n_bow;
    if (nb <= 0) return;
    const bool must = scoring != 5, l2 = scoring == 1;                          // mustNormalize (ref ScoringObject.h:74-89)
    if (!must) {
        if (accumulate) {
            const double nd = (double)nb;
            for (int i = threadIdx.x; i < nb; i += blockDim.x) vals[i] /= nd;
        }
        return;
    }
    double norm = 0.0;
    for (int base = 0; base < nb; base += kBvNormChunk) {
        const int m = min(kBvNormChunk, nb - base);
        for (int i = threadIdx.x; i < m; i += blockDim.x) {
            const double x = vals[base + i];
            buf[i] = l2 ? x * x : fabs(x);
        }
        __syncthreads();
        if (threadIdx.x == 0)
            for (int i = 0; i < m; ++i) norm += buf[i];                         // ascending word order, one addition after another
        __syncthreads();
    }
    if (threadIdx.x == 0) norm_s = l2 ? sqrt(norm) : norm;
    __syncthreads();
    const double nrm = norm_s;
    if (nrm > 0.0)
        for (int i = threadIdx.x; i < nb; i += blockDim.x) vals[i] /= nrm;
}

}  // namespace

cudaError_t launch_bow_vectors_device(const VocabularyDev& v, const BowVectorsDevArgs& a, cudaStream_t st) {
    const int NS = a.n_cams * a.capacity;
    const int n_fill = a.max_nodes < NS ? a.max_nodes : NS;                     // a frame holds at most NS nodes
    const int tiles_n = (v.n_nodes + kBvTile - 1) / kBvTile, tiles_w = (a.n_words + kBvTile - 1) / kBvTile;
    const int max_tiles = tiles_n > tiles_w ? tiles_n : tiles_w;
    // the three cleared arrays first, in one block
    StreamScratch sc;
    const PsCamSlots* cams;
    cudaError_t e = open_scratch(sc, {4ull * v.n_nodes, 4ull * a.n_words, 4ull * n_fill,            // cnt_node cnt_word fill
                                      4ull * NS, 8ull * NS, 4ull * a.n_words,                     // key_node wt word_rep
                                      4ull * NS, 4ull * NS, 16ull * max_tiles},                   // slot_rank unordered tile_sums
                                 st, host_in(cams, a.cams, a.n_cams));
    if (e != cudaSuccess) return sc.release(e);
    int* cnt_node = sc.at<int>(0); int* cnt_word = sc.at<int>(1); int* fill = sc.at<int>(2);
    int* key_node = sc.at<int>(3); double* wt = sc.at<double>(4); int* word_rep = sc.at<int>(5);
    int* slot_rank = sc.at<int>(6); int* unordered = sc.at<int>(7); unsigned long long* tile_sums = sc.at<unsigned long long>(8);
    e = cudaMemsetAsync(cnt_node, 0, sc.at<uint8_t>(3) - sc.at<uint8_t>(0), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(a.status, 0, 4, st);
    if (e == cudaSuccess) {
        const BvKeys nodes{cnt_node, v.n_nodes, a.fv_nodes, a.fv_offsets, a.n_fv, a.max_nodes};
        const BvKeys words{cnt_word, a.n_words, a.bow_words, nullptr, a.n_bow, NS};
        const bool accumulate = a.weighting == 0 || a.weighting == 1;           // TF_IDF, TF
        const int sb = (NS + 255) / 256;
        bv_descend_kernel<<<(unsigned)(((long long)NS * kBowGroup + 255) / 256), 256, 0, st>>>(
            v, cams, NS, a.capacity, v.L - a.levelsup, a.word, a.weight, a.node, key_node, wt, cnt_node, cnt_word, word_rep);
        bv_tile_count_kernel<<<dim3(max_tiles, 2), kBvThreads, 0, st>>>(nodes, words, max_tiles, tile_sums);
        bv_tile_emit_kernel<<<dim3(max_tiles, 2), kBvThreads, 0, st>>>(nodes, words, max_tiles, tile_sums, wt, word_rep, accumulate,
                                                                       a.bow_values, a.status);
        bv_scatter_kernel<<<sb, 256, 0, st>>>(NS, key_node, cnt_node, a.fv_offsets, fill, slot_rank, unordered);
        bv_place_kernel<<<sb, 256, 0, st>>>(NS, slot_rank, a.fv_offsets, unordered, a.fv_features);
        bv_normalize_kernel<<<1, 256, 0, st>>>(a.bow_values, a.n_bow, a.scoring, accumulate);
        e = cudaGetLastError();
    }
    return sc.release(e);
}

// ------------------------------------------------------------------------------------------------
// SearchByBoW(KF_i, F) for a batch of key frames (mcs_search_by_bow_device), ref src/cORBmatcher.cpp:179-324
// ------------------------------------------------------------------------------------------------
// A frame keypoint lies in exactly one node of F.mFeatVec and "already matched" is read and written only inside that node's
// list, so the (key frame, common node) groups are independent; only the key-frame keypoints inside one group depend on each
// other's acceptances.  One warp takes a group and follows the reference's order literally: the key-frame slots of the node one
// after another, the lanes striding the frame's list, the accepted candidate's match_mp entry being the taken flag the next
// keypoint reads.
namespace {

struct BowSearchDev {
    int n_kf, n_cams, capacity, max_nodes, n_points, th_low;
    double nnratio;
    const PsCamSlots* kf_cams; const PsCamSlots* cur_cams; const BowFrameDev* kfs; BowFrameDev cur;
    const uint8_t* bad;
    int* match_mp; int* match_slot; int* nmatches; int* status;
};

// both outputs start at -1 below each camera's count of the current frame (the reference starts from an all-NULL vector, :185)
__global__ void __launch_bounds__(256) bs_clear_kernel(const BowSearchDev a) {
    const int NS = a.n_cams * a.capacity;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.n_kf) a.nmatches[t] = 0;
    if (t == 0) *a.status = MCS_OK;
    if (t >= (long long)a.n_kf * NS) return;
    const int s = (int)(t % NS), c = s / a.capacity, j = s - c * a.capacity;
    if (j >= min(*a.cur_cams[c].count, a.capacity)) return;
    a.match_mp[t] = -1;
    if (a.match_slot) a.match_slot[t] = -1;
}

// the packed descriptor (and mask) row of slot s, or NULL when s is no keypoint of the frame
__device__ __forceinline__ bool bs_row(const PsCamSlots* __restrict__ cams, const int n_slots, const int capacity, const int words,
                                       const int s, const uint32_t*& desc, const uint32_t*& mask) {
    if ((unsigned)s >= (unsigned)n_slots) return false;
    const int c = s / capacity, j = s - c * capacity;
    const PsCamSlots cs = cams[c];
    if (j >= min(*cs.count, capacity)) return false;
    desc = (const uint32_t*)cs.desc + (size_t)j * words;
    mask = (const uint32_t*)cs.dmask + (size_t)j * words;
    return true;
}

template <int WORDS, bool MASKED>
__global__ void __launch_bounds__(256) bs_search_kernel(const BowSearchDev a) {
    const int lane = threadIdx.x & 31;
    const int NS = a.n_cams * a.capacity;
    const long long n_items = (long long)a.n_kf * a.max_nodes, n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
    const int n_cur = min(*a.cur.n_fv, a.max_nodes);
    for (long long item = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; item < n_items; item += n_warps) {
        const int k = (int)(item / a.max_nodes), ia = (int)(item - (long long)k * a.max_nodes);
        const BowFrameDev kf = a.kfs[k];
        if (ia >= min(*kf.n_fv, a.max_nodes)) continue;
        const int node = kf.fv_nodes[ia];
        int lo = 0, hi = n_cur;                                                 // the node in the frame's ascending list
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (a.cur.fv_nodes[mid] < node) lo = mid + 1; else hi = mid;
        }
        if (lo >= n_cur || a.cur.fv_nodes[lo] != node) continue;
        const int cs = a.cur.fv_offsets[lo], cc = a.cur.fv_offsets[lo + 1] - cs;
        const int q0 = kf.fv_offsets[ia], q1 = kf.fv_offsets[ia + 1];
        if (cc <= 0) continue;
        const PsCamSlots* kcams = a.kf_cams + (size_t)k * a.n_cams;
        volatile int* taken = a.match_mp + (size_t)k * NS;                      // written by this warp between its reads
        int found = 0;
        for (int q = q0; q < q1; ++q) {
            const int s1 = kf.fv_features[q];
            const uint32_t* qd; const uint32_t* qmk;
            if (!bs_row(kcams, NS, a.capacity, WORDS, s1, qd, qmk)) { if (lane == 0) *a.status = MCS_ERR_INVALID; continue; }
            const int mp = kf.mp[s1];
            if (mp < 0) continue;                                               // no map point (ref :212-216)
            if (mp >= a.n_points) { if (lane == 0) *a.status = MCS_ERR_INVALID; continue; }
            if (a.bad && a.bad[mp]) continue;
            uint32_t qw[WORDS], qm[MASKED ? WORDS : 1];
#pragma unroll
            for (int w = 0; w < WORDS; ++w) {
                qw[w] = __ldg(qd + w);
                if (MASKED) qm[w] = __ldg(qmk + w);
            }
            // per lane: (distance << 32 | list position) of its best, and its second-best distance; positions ascend per lane, so
            // a smaller key is a strictly smaller distance, as the reference's `<` asks
            unsigned long long k1 = ~0ull;
            unsigned d2 = 0xFFFFFFFFu;
            for (int j = lane; j < cc; j += 32) {
                const int s2 = a.cur.fv_features[cs + j];
                const uint32_t* dd; const uint32_t* mm;
                if (!bs_row(a.cur_cams, NS, a.capacity, WORDS, s2, dd, mm)) { *a.status = MCS_ERR_INVALID; continue; }
                if (taken[s2] >= 0) continue;                                   // vpMapPointMatches[realIdxF] (ref :237)
                unsigned dist = 0;
                if (MASKED) {
#pragma unroll
                    for (int w = 0; w < WORDS; ++w) {
                        const uint32_t xw = qw[w] ^ __ldg(dd + w);
                        dist += __popc(xw & qm[w]) + __popc(xw & __ldg(mm + w));
                    }
                    dist >>= 1;                                                 // DescriptorDistance64Masked (ref :2452-2474)
                } else {
#pragma unroll
                    for (int w = 0; w < WORDS; ++w) dist += __popc(qw[w] ^ __ldg(dd + w));
                }
                const unsigned long long key = ((unsigned long long)dist << 32) | (unsigned)j;
                if (key < k1) {
                    if (k1 != ~0ull) d2 = (unsigned)(k1 >> 32);
                    k1 = key;
                } else if (dist < d2) d2 = dist;
            }
            unsigned long long kmin = k1;
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                const unsigned long long y = __shfl_xor_sync(0xFFFFFFFFu, kmin, o);
                kmin = y < kmin ? y : kmin;
            }
            if (kmin == ~0ull) continue;                                        // every candidate is taken
            // the second best over all: the winner lane's second, every other lane's best
            unsigned second = k1 == kmin ? d2 : (unsigned)(k1 >> 32);           // k1 = ~0: 0xFFFFFFFF, no candidate
#pragma unroll
            for (int o = 16; o; o >>= 1) second = min(second, __shfl_xor_sync(0xFFFFFFFFu, second, o));
            const int best = (int)(kmin >> 32), best2 = second == 0xFFFFFFFFu ? INT_MAX : (int)second;
            if (best <= a.th_low && (double)best < a.nnratio * (double)best2) { // ref :264-268
                if (lane == 0) {
                    const int s2 = a.cur.fv_features[cs + (int)(kmin & 0xFFFFFFFFu)];
                    taken[s2] = mp;
                    if (a.match_slot) a.match_slot[(size_t)k * NS + s2] = s1;
                }
                ++found;
            }
            __syncwarp();                                                       // the next keypoint's lanes read the flag
        }
        if (lane == 0 && found) atomicAdd(a.nmatches + k, found);
    }
}

}  // namespace

cudaError_t launch_search_by_bow_device(const BowSearchDevArgs& a, cudaStream_t st) {
    const int NS = a.n_cams * a.capacity;
    BowSearchDev d{a.n_kf, a.n_cams, a.capacity, a.max_nodes, a.n_points, a.th_low, a.nnratio, nullptr, nullptr, nullptr, a.cur,
                   a.bad, a.match_mp, a.match_slot, a.nmatches, a.status};
    StreamScratch sc;
    cudaError_t e = open_scratch(sc, {}, st, host_in(d.kf_cams, a.kf_cams, (size_t)a.n_cams * a.n_kf), host_in(d.cur_cams, a.cur_cams, a.n_cams),
                                 host_in(d.kfs, a.kfs, a.n_kf));
    if (e == cudaSuccess) {
        const long long cells = (long long)a.n_kf * NS, items = (long long)a.n_kf * a.max_nodes;
        bs_clear_kernel<<<(unsigned)((cells + 255) / 256), 256, 0, st>>>(d);
        // a warp per (key frame, node) up to a grid that fills the device several times over; beyond it the warps stride
        const long long blocks = (items + 7) / 8;
        const unsigned grid = (unsigned)(blocks < 16384 ? blocks : 16384);
        with_desc_width(a.dim, a.masked, [&](auto W, auto M) { bs_search_kernel<W, M><<<grid, 256, 0, st>>>(d); });
        e = cudaGetLastError();
    }
    return sc.release(e);
}

}  // namespace mcs
