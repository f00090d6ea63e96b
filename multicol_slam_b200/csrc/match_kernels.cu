// match_kernels.cu -- sm_90a kernels of the matcher half of the hot path.
//
//   M2 hamming_topk_kernel : all-pairs bit-level Hamming distance (ref src/cORBmatcher.cpp:2438-2474)
//                            of nq queries against nd database descriptors, K best (distance, index)
//                            per query.  One thread owns one query (descriptor words in registers),
//                            database tiles are staged in shared memory with 128-bit loads and broadcast.
//                            Bound by the POPC issue rate, not HBM (SURVEY.md 7, hard part 7).
//   M1/M3 window_search_kernel : GetFeaturesInArea (ref src/cMultiFrame.cpp:272-340) + distance to every
//                            candidate, one warp per query, candidates emitted in the reference's visiting
//                            order (cell-x outer, cell-y inner, insertion order inside a cell).
#include "cam_model.cuh"
#include "mcs_common.cuh"
#include "kernels.h"

namespace mcs {

constexpr int kTopKMax = 8;
constexpr int kDbTile = 256;
constexpr int kTopkThreads = 128;


// ---- bit-sliced population count (Harley-Seal carry-save adders) -------------------------------------------------
// POPC issues at 16 lanes/clk/SM on sm_90 (4x slower than LOP3), which makes a plain popcount loop
// the bottleneck of brute-force Hamming.  A carry-save adder (2 LOP3) turns three words into a "ones" and a "twos"
// word; reducing 16 (8) words this way needs 9 (4) POPC instead of 16 (8).
// (a ^ b) & c in one LOP3 (immLut = (0xF0 ^ 0xCC) & 0xAA); the compiler otherwise keeps the shared xor separate
__device__ __forceinline__ uint32_t xor_and(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d;
    asm("lop3.b32 %0, %1, %2, %3, 0x28;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ void csa(uint32_t a, uint32_t b, uint32_t c, uint32_t& sum, uint32_t& carry) {
    sum = a ^ b ^ c;                       // LOP3 0x96
    carry = (a & b) | (c & (a | b));       // LOP3 0xE8 (majority)
}
__device__ __forceinline__ unsigned popc_sum8(const uint32_t (&w)[8]) {
    uint32_t s0, c0, s1, c1, s2, c2, t0, d0;
    csa(w[0], w[1], w[2], s0, c0);
    csa(w[3], w[4], w[5], s1, c1);
    csa(s0, s1, w[6], s2, c2);
    csa(c0, c1, c2, t0, d0);
    return __popc(s2) + __popc(w[7]) + 2 * __popc(t0) + 4 * __popc(d0);
}
// 16 words (masked distance): two carry-save levels on the ones, none on the twos -- 14 LOP3 + 9 POPC.  LOP3 (64 lanes/clk/SM)
// and POPC (16 lanes/clk/SM) issue concurrently, so the cheapest split loads both about equally.  Greedy stream matcher,
// H100 80GB HBM3, 400 W limit, bench.py config 2, 2 alternating runs: this split 6.71 / 6.69 ms, MCS_M2_TREE=1 7.27 / 7.03 ms, =2 7.07 / 7.00 ms.
#ifndef MCS_M2_TREE
#define MCS_M2_TREE 0                // 0: 7 carry-save adders + 9 POPC, 1: 5 + 11, 2: 6 + 10 (A/B builds)
#endif
__device__ __forceinline__ void popc_sum16(const uint32_t (&w)[16], unsigned& ones_out, unsigned& twos_out) {
    uint32_t s0, c0, s1, c1, s2, c2, s3, c3, s4, c4;
    csa(w[0], w[1], w[2], s0, c0);
    csa(w[3], w[4], w[5], s1, c1);
    csa(w[6], w[7], w[8], s2, c2);
    csa(w[9], w[10], w[11], s3, c3);
    csa(w[12], w[13], w[14], s4, c4);
#if MCS_M2_TREE == 1
    const unsigned ones = __popc(s0) + __popc(s1) + __popc(s2) + __popc(s3) + __popc(s4) + __popc(w[15]);
    const unsigned twos = __popc(c0) + __popc(c1) + __popc(c2) + __popc(c3) + __popc(c4);
#elif MCS_M2_TREE == 2
    uint32_t a0, b0;
    csa(s0, s1, s2, a0, b0);
    const unsigned ones = __popc(a0) + __popc(s3) + __popc(s4) + __popc(w[15]);
    const unsigned twos = __popc(c0) + __popc(c1) + __popc(c2) + __popc(c3) + __popc(c4) + __popc(b0);
#else
    uint32_t a0, b0, a1, b1;
    csa(s0, s1, s2, a0, b0);
    csa(s3, s4, w[15], a1, b1);
    const unsigned ones = __popc(a0) + __popc(a1);
    const unsigned twos = __popc(c0) + __popc(c1) + __popc(c2) + __popc(c3) + __popc(c4) + __popc(b0) + __popc(b1);
#endif
    ones_out += ones; twos_out += twos;
}
// sum over k of popc(x_k) [unmasked] or (popc(x_k & qm_k) + popc(x_k & dm_k)) / 2 [masked: the integer division of ref :2472
// applied to the carry-save form, (ones + 2 twos) >> 1 == twos + (ones >> 1)], x_k = q_k ^ d_k
template <int WORDS, bool MASKED>
__device__ __forceinline__ unsigned hamming_words(const uint32_t (&qw)[WORDS], const uint32_t* qm, const uint32_t* dd, const uint32_t* dm) {
    unsigned dist = 0;
    if (MASKED) {
        unsigned ones = 0, twos = 0;
#pragma unroll
        for (int h = 0; h < WORDS; h += 8) {
            uint32_t w[16];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                if (h + k < WORDS) {
                    w[2 * k] = xor_and(qw[h + k], dd[h + k], qm[h + k]);
                    w[2 * k + 1] = xor_and(qw[h + k], dd[h + k], dm[h + k]);
                } else { w[2 * k] = 0; w[2 * k + 1] = 0; }
            }
            popc_sum16(w, ones, twos);
        }
        unsigned half;                       // (inline shift: the compiler otherwise wraps the plain `ones >> 1` in two 16-bit masks)
        asm("shr.u32 %0, %1, 1;" : "=r"(half) : "r"(ones));
        dist = twos + half;
    } else {
#pragma unroll
        for (int h = 0; h < WORDS; h += 8) {
            uint32_t w[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) w[k] = (h + k < WORDS) ? (qw[h + k] ^ dd[h + k]) : 0u;
            dist += popc_sum8(w);
        }
    }
    return dist;
}

// (Parking candidates in a per-thread shared-memory queue and inserting them with all lanes together -- the insertion below runs
// with few active lanes -- was tried and was slower: the vote + queue traffic per pair costs more than the divergent insertions.)
// Keys are 32 bits: distance << kTopkShift | database index (index < 2^21, distance <= 512), the list length KT is a compile-time
// constant (4 or 8): see hamming_stream_kernel.
constexpr int kTopkShift = 21;
template <int WORDS, bool MASKED, int KT>
__global__ void __launch_bounds__(kTopkThreads)
hamming_topk_kernel(const uint32_t* __restrict__ q, const uint32_t* __restrict__ qmask, const int nq,
                    const uint32_t* __restrict__ d, const uint32_t* __restrict__ dmask, const int nd,
                    const uint8_t* __restrict__ skip, const int K, const int chunk, const unsigned bound,
                    unsigned* __restrict__ part /* [splits][nq][kTopKMax] */) {
    __shared__ __align__(16) uint32_t s_d[kDbTile * WORDS];
    __shared__ __align__(16) uint32_t s_m[MASKED ? kDbTile * WORDS : 4];
    __shared__ uint8_t s_skip[kDbTile];

    const int qi = blockIdx.x * kTopkThreads + threadIdx.x;
    const bool active = qi < nq;
    uint32_t qw[WORDS], qm[MASKED ? WORDS : 1];
#pragma unroll
    for (int k = 0; k < WORDS; ++k) {
        qw[k] = active ? q[(size_t)qi * WORDS + k] : 0u;
        if (MASKED) qm[k] = active ? qmask[(size_t)qi * WORDS + k] : 0u;
    }
    constexpr unsigned kNone = 0xFFFFFFFFu;
    unsigned best[KT];
#pragma unroll
    for (int k = 0; k < KT; ++k) best[k] = kNone;
    unsigned worst = min(bound, 0x7FFu);   // a pair is listed only below the K-th best so far and the caller's bound

    const int j0 = blockIdx.y * chunk, j1 = min(j0 + chunk, nd);
    for (int t0 = j0; t0 < j1; t0 += kDbTile) {
        const int tn = min(kDbTile, j1 - t0);
        __syncthreads();
        {   // 128-bit coalesced staging of the database tile
            const uint4* src = (const uint4*)(d + (size_t)t0 * WORDS);
            uint4* dst = (uint4*)s_d;
            for (int i = threadIdx.x; i < tn * WORDS / 4; i += kTopkThreads) dst[i] = src[i];
            if (MASKED) {
                const uint4* msrc = (const uint4*)(dmask + (size_t)t0 * WORDS);
                uint4* mdst = (uint4*)s_m;
                for (int i = threadIdx.x; i < tn * WORDS / 4; i += kTopkThreads) mdst[i] = msrc[i];
            }
            for (int i = threadIdx.x; i < tn; i += kTopkThreads) s_skip[i] = skip ? skip[t0 + i] : 0;
        }
        __syncthreads();
        for (int j = 0; j < tn; ++j) {
            if (s_skip[j]) continue;       // uniform across the CTA
            // bit-level Hamming distance; masked form = (popc(x&ma) + popc(x&mb)) / 2, integer division (ref :2472)
            const unsigned dist = hamming_words<WORDS, MASKED>(qw, qm, s_d + j * WORDS, s_m + j * WORDS);
            if (dist < worst) {            // strict: equal distances keep the earlier index; entries at or beyond `bound` are not listed
                unsigned key = (dist << kTopkShift) | (unsigned)(t0 + j);
#pragma unroll
                for (int k = 0; k < KT; ++k) {
                    if (k < K) { const unsigned lo = min(key, best[k]); key = max(key, best[k]); best[k] = lo; }
                }
                unsigned w = best[0];
#pragma unroll
                for (int k = 1; k < KT; ++k) if (k < K) w = best[k];
                if (w != kNone) worst = min(worst, w >> kTopkShift);
            }
        }
    }
    if (active) {
        unsigned* o = part + ((size_t)blockIdx.y * nq + qi) * kTopKMax;
#pragma unroll
        for (int k = 0; k < kTopKMax; ++k) o[k] = k < KT ? best[k < KT ? k : 0] : kNone;
    }
}

__global__ void topk_merge_kernel(const unsigned* __restrict__ part, const int splits, const int nq, const int K,
                                  int* __restrict__ topk_idx, int* __restrict__ topk_dist) {
    const int qi = blockIdx.x * blockDim.x + threadIdx.x;
    if (qi >= nq) return;
    constexpr unsigned kNone = 0xFFFFFFFFu;
    unsigned best[kTopKMax];
#pragma unroll
    for (int k = 0; k < kTopKMax; ++k) best[k] = kNone;
    for (int s = 0; s < splits; ++s) {
        const unsigned* p = part + ((size_t)s * nq + qi) * kTopKMax;
        for (int i = 0; i < K; ++i) {
            unsigned key = p[i];
            if (key == kNone) break;
#pragma unroll
            for (int k = 0; k < kTopKMax; ++k) {
                if (k < K) { const unsigned lo = min(key, best[k]); key = max(key, best[k]); best[k] = lo; }
            }
        }
    }
    for (int k = 0; k < K; ++k) {
        const bool none = best[k] == kNone;
        topk_idx[(size_t)qi * K + k] = none ? -1 : (int)(best[k] & ((1u << kTopkShift) - 1u));
        topk_dist[(size_t)qi * K + k] = none ? 0x7FFFFFFF : (int)(best[k] >> kTopkShift);
    }
}

cudaError_t launch_hamming_topk(const uint8_t* q, const uint8_t* qmask, int nq, const uint8_t* d, const uint8_t* dmask,
                                int nd, const uint8_t* db_skip, int dim, int K, unsigned bound, int* topk_idx, int* topk_dist,
                                cudaStream_t st) {
    if (K < 1 || K > kTopKMax || (dim != 16 && dim != 32 && dim != 64) || nd >= (1 << kTopkShift)) return cudaErrorInvalidValue;
    if (nq <= 0) return cudaSuccess;
    const int qblocks = (nq + kTopkThreads - 1) / kTopkThreads;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    // enough CTAs for ~4 waves; database chunks are multiples of the tile
    int splits = (4 * sms * 8 + qblocks - 1) / qblocks;
    const int tiles = (nd + kDbTile - 1) / kDbTile;
    splits = max(1, min(splits, tiles));
    const int chunk = ((tiles + splits - 1) / splits) * kDbTile;
    splits = max(1, (nd + chunk - 1) / chunk);
    // partial top-K lists of the database splits: stream-ordered scratch owned by THIS call (cudaMallocAsync pool), so that
    // concurrent callers -- the reference runs its matchers from three threads -- and different streams never share it
    const size_t need = (size_t)splits * nq * kTopKMax * sizeof(unsigned);
    unsigned* g_part = nullptr;
    cudaError_t e = keep_pool_memory();
    if (e != cudaSuccess) return e;
    e = cudaMallocAsync((void**)&g_part, need, st);
    if (e != cudaSuccess) return e;
    dim3 grid(qblocks, splits);
    const bool masked = qmask && dmask;
#define MCS_TOPK2(W, M, KT) hamming_topk_kernel<W, M, KT><<<grid, kTopkThreads, 0, st>>>((const uint32_t*)q, (const uint32_t*)qmask, nq, \
        (const uint32_t*)d, (const uint32_t*)dmask, nd, db_skip, K, chunk, bound, g_part)
#define MCS_TOPK(W, M) { if (K <= 4) MCS_TOPK2(W, M, 4); else MCS_TOPK2(W, M, 8); }
    if (dim == 16) { if (masked) MCS_TOPK(4, true) else MCS_TOPK(4, false) }
    else if (dim == 32) { if (masked) MCS_TOPK(8, true) else MCS_TOPK(8, false) }
    else { if (masked) MCS_TOPK(16, true) else MCS_TOPK(16, false) }
#undef MCS_TOPK2
#undef MCS_TOPK
    topk_merge_kernel<<<(nq + 127) / 128, 128, 0, st>>>(g_part, splits, nq, K, topk_idx, topk_dist);
    e = cudaGetLastError();
    const cudaError_t ef = cudaFreeAsync(g_part, st);        // after the merge in stream order
    return e != cudaSuccess ? e : ef;
}

// Stream matching: image i = (frame f, camera c) is matched against image i - n_cams = (f-1, c); both live in
// fixed-size slots of `capacity` descriptors, the valid counts are read on the device (no host sync).
// One thread owns one query; the (<= capacity) database descriptors of the previous frame are staged tile by
// tile in shared memory.  Output: K best (index, distance) per query slot, (-1, INT_MAX) where none.
// The per-thread list holds 32-bit keys (distance << 16 | slot; slots < 65536, distances <= 512) and its length KT is a compile-time
// constant (4 or 8): the sorted insertion -- executed by the one or two lanes of a warp that have a candidate -- is 3 instructions
// per list position instead of ~6 on 64-bit keys over all 8 positions.
template <int WORDS, bool MASKED, int KT>
__global__ void __launch_bounds__(kTopkThreads)
hamming_stream_kernel(const uint32_t* __restrict__ desc, const uint32_t* __restrict__ dmask, const int* __restrict__ counts,
                      const int n_cams, const int capacity, const int K, const int img_lo, const unsigned bound,
                      int* __restrict__ out_idx, int* __restrict__ out_dist) {
    __shared__ __align__(16) uint32_t s_d[kDbTile * WORDS];
    __shared__ __align__(16) uint32_t s_m[MASKED ? kDbTile * WORDS : 4];
    const int img = blockIdx.y + img_lo;
    const int qi = blockIdx.x * kTopkThreads + threadIdx.x;
    const bool has_prev = img >= n_cams;                 // frame 0 has no predecessor
    const int nq = has_prev ? min(counts[img], capacity) : 0;
    const int nd = has_prev ? min(counts[img - n_cams], capacity) : 0;
    if ((int)(blockIdx.x * kTopkThreads) >= nq) {        // nothing to match in this block: mark the slots empty
        if (qi < capacity)
            for (int k = 0; k < K; ++k) {
                out_idx[((size_t)img * capacity + qi) * K + k] = -1;
                out_dist[((size_t)img * capacity + qi) * K + k] = 0x7FFFFFFF;
            }
        return;
    }
    const bool active = qi < nq;
    const uint32_t* q = desc + ((size_t)img * capacity + qi) * WORDS;
    const uint32_t* qmk = MASKED ? dmask + ((size_t)img * capacity + qi) * WORDS : nullptr;
    uint32_t qw[WORDS], qm[MASKED ? WORDS : 1];
#pragma unroll
    for (int k = 0; k < WORDS; ++k) {
        qw[k] = active ? q[k] : 0u;
        if (MASKED) qm[k] = active ? qmk[k] : 0u;
    }
    constexpr unsigned kNone = 0xFFFFFFFFu;
    unsigned best[KT];
#pragma unroll
    for (int k = 0; k < KT; ++k) best[k] = kNone;
    unsigned worst = min(bound, 0xFFFFu);                // a pair is listed only below the K-th best so far and the caller's bound
    const uint32_t* dbase = desc + (size_t)(img - n_cams) * capacity * WORDS;
    const uint32_t* mbase = MASKED ? dmask + (size_t)(img - n_cams) * capacity * WORDS : nullptr;
    for (int t0 = 0; t0 < nd; t0 += kDbTile) {
        const int tn = min(kDbTile, nd - t0);
        __syncthreads();
        {
            const uint4* src = (const uint4*)(dbase + (size_t)t0 * WORDS);
            uint4* dst = (uint4*)s_d;
            for (int i = threadIdx.x; i < tn * WORDS / 4; i += kTopkThreads) dst[i] = src[i];
            if (MASKED) {
                const uint4* msrc = (const uint4*)(mbase + (size_t)t0 * WORDS);
                uint4* mdst = (uint4*)s_m;
                for (int i = threadIdx.x; i < tn * WORDS / 4; i += kTopkThreads) mdst[i] = msrc[i];
            }
        }
        __syncthreads();
#pragma unroll 2
        for (int j = 0; j < tn; ++j) {
            // bit-level Hamming distance; masked form = (popc(x&ma) + popc(x&mb)) / 2, integer division (ref :2472)
            const unsigned dist = hamming_words<WORDS, MASKED>(qw, qm, s_d + j * WORDS, s_m + j * WORDS);
            if (dist < worst) {                          // strict: equal distances keep the earlier slot
                unsigned key = (dist << 16) | (unsigned)(t0 + j);
#pragma unroll
                for (int k = 0; k < KT; ++k) {
                    if (k < K) { const unsigned lo = min(key, best[k]); key = max(key, best[k]); best[k] = lo; }
                }
                unsigned w = best[0];
#pragma unroll
                for (int k = 1; k < KT; ++k) if (k < K) w = best[k];
                if (w != kNone) worst = min(worst, w >> 16);
            }
        }
    }
    if (qi < capacity) {
        int* oi = out_idx + ((size_t)img * capacity + qi) * K;
        int* od = out_dist + ((size_t)img * capacity + qi) * K;
#pragma unroll
        for (int k = 0; k < KT; ++k) {
            if (k < K) {
                const bool none = !active || best[k] == kNone;
                oi[k] = none ? -1 : (int)(best[k] & 0xFFFFu);
                od[k] = none ? 0x7FFFFFFF : (int)(best[k] >> 16);
            }
        }
    }
}

cudaError_t launch_hamming_stream(const uint8_t* desc, const uint8_t* dmask, const int* counts, int img_lo, int img_count,
                                  int n_cams, int capacity, int dim, int K, unsigned bound, int* out_idx, int* out_dist, cudaStream_t st) {
    if (K < 1 || K > kTopKMax || (dim != 16 && dim != 32 && dim != 64) || capacity > 65535) return cudaErrorInvalidValue;
    if (img_count < 1) return cudaSuccess;
    dim3 grid((capacity + kTopkThreads - 1) / kTopkThreads, img_count);
    const bool masked = dmask != nullptr;
#define MCS_HS2(W, M, KT) hamming_stream_kernel<W, M, KT><<<grid, kTopkThreads, 0, st>>>((const uint32_t*)desc, (const uint32_t*)dmask, counts, \
        n_cams, capacity, K, img_lo, bound, out_idx, out_dist)
#define MCS_HS(W, M) { if (K <= 4) MCS_HS2(W, M, 4); else MCS_HS2(W, M, 8); }
    if (dim == 16) { if (masked) MCS_HS(4, true) else MCS_HS(4, false) }
    else if (dim == 32) { if (masked) MCS_HS(8, true) else MCS_HS(8, false) }
    else { if (masked) MCS_HS(16, true) else MCS_HS(16, false) }
#undef MCS_HS
#undef MCS_HS2
    return cudaGetLastError();
}

// Greedy acceptance of SearchByBoW(KF1, KF2) (ref src/cORBmatcher.cpp:899-961) over the K-best lists of the stream matcher, on
// the device: one warp per image; the lanes fetch the lists of 32 queries at a time (coalesced), lane 0 walks them in order.
// The lists are sorted by (distance, index) -- the reference's strict `<` scan order -- and were computed without knowledge of
// which database entries earlier queries have taken.  With u0, u1 the first two list entries still unmatched and dK the
// distance of the last list entry (every entry NOT in the list is at least that far), a query is decided from its list when
//   two unmatched entries are in it (best = u0, second = u1), or the list holds every database entry, or
//   one is (best = u0): rejected if u0 >= th_low, accepted if u0 < nnratio * dK (the true second is >= dK), or
//   none is: rejected if dK >= th_low.
// Otherwise the warp rescans the whole previous image for this one query (exact best / second among the unmatched entries), so
// the result never depends on K; redo[] stays 0 and is kept for interface stability.
#ifndef MCS_REPLAY_THREADS
#define MCS_REPLAY_THREADS 256
#endif
constexpr int kReplayThreads = MCS_REPLAY_THREADS;   // stream matcher: <= 65535 database entries per image, many images in flight
constexpr int kBfReplayThreads = 1024;       // key-frame database: one CTA per query set scans up to ~1.5 M entries per rescan
constexpr int kKeyShift = 21;                // rescan keys = distance << 21 | index (index < 2^21, distance <= 512)

template <int THREADS>
__device__ __forceinline__ void named_bar(int id) { asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(THREADS) : "memory"); }

// One pass over this thread's share of the unmatched database entries for up to R queries at once (rows[0..n)): per query the two
// smallest (distance << kKeyShift | index) keys.  The database words are loaded once per entry whatever n is; a rescan is bound
// by the latency of those loads, so the extra queries ride along almost for free.
template <int WORDS, bool MASKED, int THREADS, int R>
__device__ __forceinline__ void replay_scan(const uint32_t* __restrict__ qd, const uint32_t* __restrict__ qmk, const int* rows, const int n,
                                            const uint32_t* __restrict__ dd, const uint32_t* __restrict__ dm, const int id_lo,
                                            const int id_hi, const unsigned* s_taken /* bit (id - id_lo) */, const int tid,
                                            unsigned (&k1)[R], unsigned (&k2)[R]) {
    uint32_t qw[R][WORDS], qm[R][MASKED ? WORDS : 1];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int row = rows[r < n ? r : 0];
        const uint4* qp = reinterpret_cast<const uint4*>(qd + (size_t)row * WORDS);
#pragma unroll
        for (int k = 0; k < WORDS / 4; ++k) { const uint4 t = qp[k]; qw[r][4 * k] = t.x; qw[r][4 * k + 1] = t.y; qw[r][4 * k + 2] = t.z; qw[r][4 * k + 3] = t.w; }
        if (MASKED) {
            const uint4* qmp = reinterpret_cast<const uint4*>(qmk + (size_t)row * WORDS);
#pragma unroll
            for (int k = 0; k < WORDS / 4; ++k) { const uint4 t = qmp[k]; qm[r][4 * k] = t.x; qm[r][4 * k + 1] = t.y; qm[r][4 * k + 2] = t.z; qm[r][4 * k + 3] = t.w; }
        }
        k1[r] = 0xFFFFFFFFu; k2[r] = 0xFFFFFFFFu;
    }
#pragma unroll 2
    for (int id = id_lo + tid; id < id_hi; id += THREADS) {
        if (s_taken[(id - id_lo) >> 5] >> ((id - id_lo) & 31) & 1u) continue;
        const uint4* dp = reinterpret_cast<const uint4*>(dd + (size_t)id * WORDS);
        const uint4* mp = MASKED ? reinterpret_cast<const uint4*>(dm + (size_t)id * WORDS) : nullptr;
        uint32_t dw[WORDS], mw[MASKED ? WORDS : 1];
#pragma unroll
        for (int k = 0; k < WORDS / 4; ++k) {
            const uint4 t = dp[k]; dw[4 * k] = t.x; dw[4 * k + 1] = t.y; dw[4 * k + 2] = t.z; dw[4 * k + 3] = t.w;
            if (MASKED) { const uint4 u = mp[k]; mw[4 * k] = u.x; mw[4 * k + 1] = u.y; mw[4 * k + 2] = u.z; mw[4 * k + 3] = u.w; }
        }
#pragma unroll
        for (int r = 0; r < R; ++r) {
            if (r >= n) break;
            // the list kernels' distance (carry-save popcount: 9 POPC instead of 16 per masked 256-bit pair -- a rescan is bound by the
            // POPC rate of the SM as soon as the descriptors come from shared memory)
            const unsigned dist = hamming_words<WORDS, MASKED>(qw[r], qm[r], dw, mw);
            const unsigned key = (dist << kKeyShift) | (unsigned)id;
            if (key < k1[r]) { k2[r] = k1[r]; k1[r] = key; } else if (key < k2[r]) k2[r] = key;
        }
    }
    // warp: smallest and second smallest of the 64 keys per query (keys are unique: the index is part of the key)
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const unsigned B = __reduce_min_sync(0xffffffffu, k1[r]);
        const unsigned S = __reduce_min_sync(0xffffffffu, k1[r] == B ? k2[r] : k1[r]);
        k1[r] = B; k2[r] = S;
    }
}

// Queries served by one pass over the previous image.  3 (the pass also serving the next undecided queries of the chunk) was slower
// than 1 on the Lafida stream -- a pass is not purely latency-bound (8 entries x 50 instructions per thread and query), and the
// look-ahead results are often invalidated by the matches in between.  The code path stays (R is a template parameter).
constexpr int kRescanBatch = 1;
// decision of one query from its K-best list under the current matched bits, evaluated by a single lane (look-ahead only)
__device__ __forceinline__ int list_code(const int* li, const int* ld, const int K, const unsigned* s_taken, const int th_low, const double nnratio) {
    int best1 = 0x7FFFFFFF, best2 = 0x7FFFFFFF, found = 0, dK = 0x7FFFFFFF;
    bool complete = false;
    for (int k = 0; k < K; ++k) {
        const int id = li[k];
        if (id < 0) { complete = true; break; }
        dK = ld[k];
        if (s_taken[id >> 5] >> (id & 31) & 1u) continue;
        if (found == 0) best1 = ld[k]; else best2 = ld[k];
        if (++found == 2) break;
    }
    if (found == 2 || complete) return (best1 < th_low && (double)best1 < nnratio * (double)best2) ? 1 : 0;
    if (found == 1) return !(best1 < th_low) ? 0 : ((double)best1 < nnratio * (double)dK ? 1 : 2);
    return !(dK < th_low) ? 0 : 2;
}

struct ReplayShared {
    int cmd;                                  // queries in the published batch (>= 1), -1 = the walk is over
    int bq[kRescanBatch];                     // their rows
    unsigned k1[32][kRescanBatch], k2[32][kRescanBatch];      // per warp: two smallest keys per batch query
    int pq[kRescanBatch];                     // look-ahead results of the last batch: query row (-1 = none), best, second
    unsigned pB[kRescanBatch], pS[kRescanBatch];
};

// Several CTAs per query set (key-frame database): the leader CTA walks the queries; for a rescan it publishes the query in global
// memory, every helper CTA scans its own shard of the database and delivers the two smallest keys, the leader scans shard 0
// meanwhile and folds the partials.  Helpers learn which entries were matched since the last rescan from a log the leader appends
// to.  All CTAs must be co-resident (cooperative launch): helpers spin on cmd_seq.
constexpr int kCoopMax = 16;                 // helpers per query set
struct CoopSeg {                             // one per query set, zeroed by the host before the launch
    int cmd_seq;                             // rescans published so far; -1 = the walk is over
    int cmd_query;                           // query (row relative to the set) of the latest rescan
    int log_len;                             // entries of the set's log valid for the latest rescan
    int done;                                // helper deliveries, cumulative
    unsigned partial[2 * kCoopMax];
};
struct CoopLeader { CoopSeg* seg; int* log; int helpers; int shard_hi; };   // helpers == 0: plain single-CTA walk

// The ordered walk over one query set (queries 0..nq-1 of the given rows, lists [nq][K]) against one database of nd entries whose
// "already matched" bits live in s_taken.  Warp 0 walks the queries in order (lane 0 decides from the list); the other warps
// sleep on a named barrier and wake only for a rescan, where all THREADS threads split the database.  Every thread of the CTA
// must call this; returns the number of matches in warp 0 (other warps: 0).
// R > 1: a rescan pass also serves the next queries of the current 32-query chunk that cannot be decided from their lists right
// now (look-ahead).  Such a result stays exact as long as neither its best nor its second entry has been matched in between (the
// minimum and second minimum of a set do not change when OTHER elements leave it); that is checked when the walk gets there.
template <int WORDS, bool MASKED, int THREADS, int R>
__device__ __forceinline__ int replay_core(const int* __restrict__ list_idx, const int* __restrict__ list_dist, const int K, const int nq,
                                           const uint8_t* __restrict__ valid1, const uint32_t* __restrict__ qd,
                                           const uint32_t* __restrict__ qmk, const uint32_t* __restrict__ dd,
                                           const uint32_t* __restrict__ dmk, const int nd, const int th_low, const double nnratio,
                                           int* __restrict__ matches12, int* s_li, int* s_ld, unsigned* s_taken, ReplayShared* sh,
                                           uint32_t* s_qc /* [2][32][WORDS]: descriptors (and masks) of the current 32-query chunk */,
                                           const CoopLeader coop = CoopLeader{nullptr, nullptr, 0, 0}) {
    // rescans read their query from this chunk copy (sh->bq holds the chunk-relative row): no global-memory round trip between the
    // decision to rescan and the scan itself
    const uint32_t* s_qd = s_qc;
    const uint32_t* s_qm = MASKED ? s_qc + 32 * WORDS : nullptr;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int scan_hi = coop.helpers ? coop.shard_hi : nd;          // this CTA's share of a rescan
    int nlog = 0, seq = 0;
    if (warp != 0) {
        for (;;) {
            named_bar<THREADS>(1);
            const int cmd = *(volatile int*)&sh->cmd;
            if (cmd < 0) return 0;
            unsigned k1[R], k2[R];
            replay_scan<WORDS, MASKED, THREADS, R>(s_qd, s_qm, sh->bq, cmd, dd, dmk, 0, scan_hi, s_taken, tid, k1, k2);
            if (lane == 0) {
#pragma unroll
                for (int r = 0; r < R; ++r) { sh->k1[warp][r] = k1[r]; sh->k2[warp][r] = k2[r]; }
            }
            named_bar<THREADS>(2);
        }
    }
    int nm = 0;
    if (lane < kRescanBatch) sh->pq[lane] = -1;
    __syncwarp();
    for (int q0 = 0; q0 < nq; q0 += 32) {
        const int nchunk = min(32, nq - q0);
        for (int i = lane; i < nchunk * K; i += 32) {
            s_li[i] = list_idx[(size_t)q0 * K + i];
            s_ld[i] = list_dist[(size_t)q0 * K + i];
        }
        for (int i = lane; i < nchunk * (WORDS / 4); i += 32) {
            reinterpret_cast<uint4*>(s_qc)[i] = reinterpret_cast<const uint4*>(qd + (size_t)q0 * WORDS)[i];
            if (MASKED) reinterpret_cast<uint4*>(s_qc + 32 * WORDS)[i] = reinterpret_cast<const uint4*>(qmk + (size_t)q0 * WORDS)[i];
        }
        __syncwarp();
        for (int t = 0; t < nchunk; ++t) {
            // Decision from the list, evaluated by the whole warp: lane k looks at list entry k (K <= 8), two ballots give the
            // unmatched entries in list order -- no serial chain of dependent shared-memory loads per entry.
            //   code 0 no match, 1 match bestIdx, 2 undecided from the list
            int code = 0, bestIdx = -1;
            {
                const unsigned kmask = (1u << K) - 1u;
                const int id = lane < K ? s_li[t * K + lane] : -1;
                const int dl = lane < K ? s_ld[t * K + lane] : 0x7FFFFFFF;
                const bool valid = id >= 0;
                const bool open = valid && !(s_taken[id >> 5] >> (id & 31) & 1u);
                const unsigned m_valid = __ballot_sync(0xffffffffu, valid) & kmask;
                const unsigned m_open = __ballot_sync(0xffffffffu, open) & kmask;
                const bool complete = m_valid != kmask;                 // a -1 entry: the list holds every database entry that matters
                const int found = min(__popc(m_open), 2);
                const int first = m_open ? __ffs(m_open) - 1 : 0;
                const unsigned rest = m_open & ~(1u << first);
                const int second = rest ? __ffs(rest) - 1 : 0, lastv = m_valid ? 31 - __clz(m_valid) : 0;
                const int best1 = found >= 1 ? __shfl_sync(0xffffffffu, dl, first) : 0x7FFFFFFF;
                const int best2 = found >= 2 ? __shfl_sync(0xffffffffu, dl, second) : 0x7FFFFFFF;
                const int dK = m_valid ? __shfl_sync(0xffffffffu, dl, lastv) : 0x7FFFFFFF;      // every entry NOT in the list is at least this far
                bestIdx = found >= 1 ? __shfl_sync(0xffffffffu, id, first) : -1;
                if (valid1 && !valid1[q0 + t]) code = 0;
                else if (found == 2 || complete) code = (best1 < th_low && (double)best1 < nnratio * (double)best2) ? 1 : 0;
                else if (found == 1) code = !(best1 < th_low) ? 0 : ((double)best1 < nnratio * (double)dK ? 1 : 2);
                else code = !(dK < th_low) ? 0 : 2;
            }
            if (code == 2) {
                unsigned B = 0xFFFFFFFFu, S = 0xFFFFFFFFu;
                bool have = false;
                if (R > 1) {                                // a look-ahead result of an earlier pass, still exact?
#pragma unroll
                    for (int r = 1; r < R; ++r)
                        if (sh->pq[r] == q0 + t) {
                            const unsigned pb = sh->pB[r], ps = sh->pS[r];
                            const unsigned bi = pb & ((1u << kKeyShift) - 1u), si = ps & ((1u << kKeyShift) - 1u);
                            const bool gone = (pb != 0xFFFFFFFFu && (s_taken[bi >> 5] >> (bi & 31) & 1u)) ||
                                              (ps != 0xFFFFFFFFu && (s_taken[si >> 5] >> (si & 31) & 1u));
                            if (!gone) { B = pb; S = ps; have = true; }
                        }
                }
                if (!have) {
                    // exact rescan of the database: two smallest (distance, index) keys among the unmatched entries, for this query
                    // and (R > 1) for the next queries of the chunk that are undecided under the current matched bits
                    int n = 1;
                    unsigned cand = 0u;
                    if (R > 1) {
                        int c = 0;
                        if (lane > t && lane < nchunk && !(valid1 && !valid1[q0 + lane]))
                            c = list_code(s_li + lane * K, s_ld + lane * K, K, s_taken, th_low, nnratio);
                        cand = __ballot_sync(0xffffffffu, c == 2);
                        n += min(__popc(cand), R - 1);
                    }
                    if (lane == 0) {
                        sh->cmd = n;
                        sh->bq[0] = t;                     // chunk-relative rows (see s_qd)
                        unsigned cm = cand;
                        for (int r = 1; r < n; ++r) { sh->bq[r] = __ffs(cm) - 1; cm &= cm - 1u; }
                        if (coop.helpers) {                 // publish the rescan to the helper CTAs before scanning shard 0 here (R == 1)
                            coop.seg->cmd_query = q0 + t;
                            coop.seg->log_len = nlog;
                            __threadfence();
                            atomicExch(&coop.seg->cmd_seq, ++seq);
                        }
                    }
                    named_bar<THREADS>(1);
                    unsigned k1[R], k2[R];
                    replay_scan<WORDS, MASKED, THREADS, R>(s_qd, s_qm, sh->bq, n, dd, dmk, 0, scan_hi, s_taken, tid, k1, k2);
                    if (lane == 0) {
#pragma unroll
                        for (int r = 0; r < R; ++r) { sh->k1[0][r] = k1[r]; sh->k2[0][r] = k2[r]; }
                    }
                    named_bar<THREADS>(2);
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        const unsigned a1 = lane < THREADS / 32 ? sh->k1[lane][r] : 0xFFFFFFFFu;
                        const unsigned a2 = lane < THREADS / 32 ? sh->k2[lane][r] : 0xFFFFFFFFu;
                        const unsigned Br = __reduce_min_sync(0xffffffffu, a1);
                        const unsigned Sr = __reduce_min_sync(0xffffffffu, a1 == Br ? a2 : a1);
                        if (r == 0) { B = Br; S = Sr; }
                        else if (lane == 0) { sh->pq[r] = r < n ? q0 + sh->bq[r] : -1; sh->pB[r] = Br; sh->pS[r] = Sr; }
                    }
                    if (coop.helpers) {                     // fold the helpers' partial minima (lanes 0..helpers-1), own shard in lane 31
                        if (lane == 0) {
                            while (*(volatile int*)&coop.seg->done < seq * coop.helpers) {}
                            __threadfence();
                        }
                        __syncwarp();
                        const unsigned a1 = lane < coop.helpers ? *(volatile unsigned*)&coop.seg->partial[2 * lane] : (lane == 31 ? B : 0xFFFFFFFFu);
                        const unsigned a2 = lane < coop.helpers ? *(volatile unsigned*)&coop.seg->partial[2 * lane + 1] : (lane == 31 ? S : 0xFFFFFFFFu);
                        B = __reduce_min_sync(0xffffffffu, a1);
                        S = __reduce_min_sync(0xffffffffu, a1 == B ? a2 : a1);
                    }
                }
                const int best1 = B == 0xFFFFFFFFu ? 0x7FFFFFFF : (int)(B >> kKeyShift), best2 = S == 0xFFFFFFFFu ? 0x7FFFFFFF : (int)(S >> kKeyShift);
                bestIdx = (int)(B & ((1u << kKeyShift) - 1u));
                code = (best1 < th_low && (double)best1 < nnratio * (double)best2) ? 1 : 0;
            }
            if (code == 1) {
                if (lane == 0) {
                    matches12[q0 + t] = bestIdx;
                    s_taken[bestIdx >> 5] |= 1u << (bestIdx & 31);
                    if (coop.helpers) coop.log[nlog] = bestIdx;      // visible to the helpers with the fence of the next publication
                }
                ++nm; ++nlog;
            }
            __syncwarp();
        }
    }
    if (lane == 0) {
        sh->cmd = -1;
        if (coop.helpers) atomicExch(&coop.seg->cmd_seq, -1);
    }
    named_bar<THREADS>(1);
    return nm;
}

// helper CTA of a cooperative walk: scans database entries [lo, hi) for every rescan the leader publishes
template <int WORDS, bool MASKED, int THREADS>
__device__ __forceinline__ void replay_helper(CoopSeg* cs, const int* log, const int helper /* 0-based */, const uint32_t* __restrict__ qd,
                                              const uint32_t* __restrict__ qmk, const uint32_t* __restrict__ dd,
                                              const uint32_t* __restrict__ dmk, const int lo, const int hi, unsigned* s_taken /* bit (id - lo) */,
                                              ReplayShared* sh) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int seen = 0, applied = 0;
    for (;;) {
        if (tid == 0) {
            int sq;
            while ((sq = *(volatile int*)&cs->cmd_seq) == seen) {}
            sh->cmd = sq;
        }
        __syncthreads();
        const int sq = sh->cmd;
        if (sq < 0) return;
        seen = sq;
        __threadfence();
        const int q = *(volatile int*)&cs->cmd_query, len = *(volatile int*)&cs->log_len;
        for (int i = applied + tid; i < len; i += THREADS) {
            const int id = *(volatile const int*)&log[i];
            if (id >= lo && id < hi) atomicOr(&s_taken[(id - lo) >> 5], 1u << ((id - lo) & 31));
        }
        applied = len;
        __syncthreads();
        unsigned k1[1], k2[1];
        if (tid == 0) sh->bq[0] = q;
        __syncthreads();
        replay_scan<WORDS, MASKED, THREADS, 1>(qd, qmk, sh->bq, 1, dd, dmk, lo, hi, s_taken, tid, k1, k2);
        if (lane == 0) { sh->k1[warp][0] = k1[0]; sh->k2[warp][0] = k2[0]; }
        __syncthreads();
        if (warp == 0) {
            const unsigned a1 = lane < THREADS / 32 ? sh->k1[lane][0] : 0xFFFFFFFFu;
            const unsigned a2 = lane < THREADS / 32 ? sh->k2[lane][0] : 0xFFFFFFFFu;
            const unsigned B = __reduce_min_sync(0xffffffffu, a1);
            const unsigned S = __reduce_min_sync(0xffffffffu, a1 == B ? a2 : a1);
            if (lane == 0) {
                *(volatile unsigned*)&cs->partial[2 * helper] = B;
                *(volatile unsigned*)&cs->partial[2 * helper + 1] = S;
                __threadfence();
                atomicAdd(&cs->done, 1);
            }
        }
        // sh->cmd is rewritten only after thread 0 has seen the next publication, which the leader issues after this delivery
    }
}

// Stream matcher: one CTA per image; queries = the image's slots, database = the same camera's image one frame earlier.
template <int WORDS, bool MASKED>
__global__ void __launch_bounds__(kReplayThreads)
stream_replay_kernel(const int* __restrict__ list_idx, const int* __restrict__ list_dist, const int* __restrict__ counts,
                     const uint32_t* __restrict__ desc, const uint32_t* __restrict__ dmask,
                     const int n_cams, const int capacity, const int K, const int img_lo, const int th_low, const double nnratio,
                     int* __restrict__ matches12, int* __restrict__ nmatches, int* __restrict__ redo) {
    extern __shared__ int s_mem[];
    int* s_li = s_mem;                              // [32][K]
    int* s_ld = s_mem + 32 * K;                     // [32][K]
    unsigned* s_taken = (unsigned*)(s_mem + 64 * K);   // [(capacity + 31) / 32]
    __shared__ ReplayShared sh;
    __shared__ __align__(16) uint32_t s_qc[(MASKED ? 2 : 1) * 32 * WORDS];
    const int img = blockIdx.x + img_lo, tid = threadIdx.x;
    const bool has_prev = img >= n_cams;
    const int nq = has_prev ? min(counts[img], capacity) : 0;
    const int nd = has_prev ? min(counts[img - n_cams], capacity) : 0;
    const size_t q_row0 = (size_t)img * capacity, d_row0 = has_prev ? (size_t)(img - n_cams) * capacity : 0;
    for (int i = tid; i < (capacity + 31) / 32; i += kReplayThreads) s_taken[i] = 0u;
    for (int i = tid; i < capacity; i += kReplayThreads) matches12[q_row0 + i] = -1;
    __syncthreads();
    const int nm = replay_core<WORDS, MASKED, kReplayThreads, kRescanBatch>(list_idx + q_row0 * K, list_dist + q_row0 * K, K, nq, nullptr, desc + q_row0 * WORDS,
                                                              MASKED ? dmask + q_row0 * WORDS : nullptr, desc + d_row0 * WORDS,
                                                              MASKED ? dmask + d_row0 * WORDS : nullptr, nd, th_low, nnratio,
                                                              matches12 + q_row0, s_li, s_ld, s_taken, &sh, s_qc);
    if (tid == 0) { nmatches[img] = nm; redo[img] = 0; }
}

// The same walk with the previous image's descriptors (and masks) RESIDENT IN SHARED MEMORY: a rescan then reads its 8 x 64 bytes
// per thread from shared memory instead of L2, a fraction of the latency, at the price of one CTA per SM (capacity x 2 x dim
// bytes, 129 KB for 2016 slots of mdBRIEF-256).  Used when the launch holds no more images than the device has SMs -- a chunk of the
// host-facing stream pipeline, whose last acceptance launch is the un-overlapped tail of the call; a full 384-image step keeps the
// kernel above (2.6 CTAs per SM in flight hide each other's latency, and the extraction kernels of the next step share the SMs).
// (256 threads as in the kernel above; 1024 -- more warps of its own for the CTA that is alone on its SM -- was no better)
constexpr int kSmemReplayThreads = kReplayThreads;
template <int WORDS, bool MASKED>
__global__ void __launch_bounds__(kSmemReplayThreads, 1)
stream_replay_smem_kernel(const int* __restrict__ list_idx, const int* __restrict__ list_dist, const int* __restrict__ counts,
                          const uint32_t* __restrict__ desc, const uint32_t* __restrict__ dmask,
                          const int n_cams, const int capacity, const int K, const int img_lo, const int th_low, const double nnratio,
                          int* __restrict__ matches12, int* __restrict__ nmatches, int* __restrict__ redo) {
    extern __shared__ __align__(16) int s_mem[];
    uint32_t* s_db = (uint32_t*)s_mem;                                     // [capacity][WORDS]
    uint32_t* s_dbm = s_db + (MASKED ? (size_t)capacity * WORDS : 0);      // [capacity][WORDS]
    int* s_li = (int*)(s_dbm + (size_t)capacity * WORDS);                  // [32][K]
    int* s_ld = s_li + 32 * K;                                             // [32][K]
    unsigned* s_taken = (unsigned*)(s_ld + 32 * K);                        // [(capacity + 31) / 32]
    __shared__ ReplayShared sh;
    __shared__ __align__(16) uint32_t s_qc[(MASKED ? 2 : 1) * 32 * WORDS];
    const int img = blockIdx.x + img_lo, tid = threadIdx.x;
    const bool has_prev = img >= n_cams;
    const int nq = has_prev ? min(counts[img], capacity) : 0;
    const int nd = has_prev ? min(counts[img - n_cams], capacity) : 0;
    const size_t q_row0 = (size_t)img * capacity, d_row0 = has_prev ? (size_t)(img - n_cams) * capacity : 0;
    for (int i = tid; i < (capacity + 31) / 32; i += kSmemReplayThreads) s_taken[i] = 0u;
    for (int i = tid; i < capacity; i += kSmemReplayThreads) matches12[q_row0 + i] = -1;
    if (nq > 0) {
        const uint4* src = (const uint4*)(desc + d_row0 * WORDS);
        for (int i = tid; i < nd * WORDS / 4; i += kSmemReplayThreads) ((uint4*)s_db)[i] = src[i];
        if (MASKED) {
            const uint4* msrc = (const uint4*)(dmask + d_row0 * WORDS);
            for (int i = tid; i < nd * WORDS / 4; i += kSmemReplayThreads) ((uint4*)s_dbm)[i] = msrc[i];
        }
    }
    __syncthreads();
    const int nm = replay_core<WORDS, MASKED, kSmemReplayThreads, kRescanBatch>(list_idx + q_row0 * K, list_dist + q_row0 * K, K, nq, nullptr, desc + q_row0 * WORDS,
                                                              MASKED ? dmask + q_row0 * WORDS : nullptr, s_db, MASKED ? s_dbm : nullptr, nd, th_low,
                                                              nnratio, matches12 + q_row0, s_li, s_ld, s_taken, &sh, s_qc);
    if (tid == 0) { nmatches[img] = nm; redo[img] = 0; }
}

cudaError_t launch_stream_replay(const int* list_idx, const int* list_dist, const int* counts, const uint8_t* desc, const uint8_t* dmask,
                                 int dim, int img_lo, int n_images, int n_cams, int capacity, int K, int th_low, double nnratio,
                                 int* matches12, int* nmatches, int* redo, cudaStream_t st) {
    if (n_images < 1) return cudaSuccess;
    if (capacity > 65535 || (dim != 16 && dim != 32 && dim != 64)) return cudaErrorInvalidValue;
    const size_t smem = (size_t)64 * K * 4 + (size_t)((capacity + 31) / 32) * 4;
    const bool masked = dmask != nullptr;
    // one wave of images: the database of every image fits beside its walk (see stream_replay_smem_kernel)
    int dev = 0, sms = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return e;
    const size_t smem_db = smem + (size_t)capacity * dim * (masked ? 2 : 1) + 16;
    if (n_images <= sms && smem_db <= 200u * 1024u) {
        const void* fn = nullptr;
#define MCS_SRS(W, M) fn = (const void*)stream_replay_smem_kernel<W, M>
        if (dim == 16) { if (masked) MCS_SRS(4, true); else MCS_SRS(4, false); }
        else if (dim == 32) { if (masked) MCS_SRS(8, true); else MCS_SRS(8, false); }
        else { if (masked) MCS_SRS(16, true); else MCS_SRS(16, false); }
#undef MCS_SRS
        e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_db);     // per device, set every time
        if (e != cudaSuccess) return e;
        const uint32_t *d32 = (const uint32_t*)desc, *m32 = (const uint32_t*)dmask;
        void* args[] = {(void*)&list_idx, (void*)&list_dist, (void*)&counts, (void*)&d32, (void*)&m32, (void*)&n_cams, (void*)&capacity, (void*)&K,
                        (void*)&img_lo, (void*)&th_low, (void*)&nnratio, (void*)&matches12, (void*)&nmatches, (void*)&redo};
        return cudaLaunchKernel(fn, dim3(n_images), dim3(kSmemReplayThreads), args, smem_db, st);
    }
#define MCS_SR(W, M) stream_replay_kernel<W, M><<<n_images, kReplayThreads, smem, st>>>(list_idx, list_dist, counts, (const uint32_t*)desc, \
        (const uint32_t*)dmask, n_cams, capacity, K, img_lo, th_low, nnratio, matches12, nmatches, redo)
    if (dim == 16) { if (masked) MCS_SR(4, true); else MCS_SR(4, false); }
    else if (dim == 32) { if (masked) MCS_SR(8, true); else MCS_SR(8, false); }
    else { if (masked) MCS_SR(16, true); else MCS_SR(16, false); }
#undef MCS_SR
    return cudaGetLastError();
}

// Key-frame database: one CTA per query set (seg[s] .. seg[s+1]) against the same nd database entries, each set with its own
// "already matched" bits (initialised from valid2), as separate SearchByBoW(KF1, KF2) calls of the reference would have.
template <int WORDS, bool MASKED>
__global__ void __launch_bounds__(kBfReplayThreads)
bruteforce_replay_kernel(const int* __restrict__ list_idx, const int* __restrict__ list_dist, const int K,
                         const uint32_t* __restrict__ q, const uint32_t* __restrict__ qm, const uint8_t* __restrict__ valid1,
                         const int* __restrict__ seg, const uint32_t* __restrict__ d, const uint32_t* __restrict__ dm,
                         const uint8_t* __restrict__ valid2, const int nd, const int th_low, const double nnratio,
                         int* __restrict__ matches12, int* __restrict__ nmatches, CoopSeg* __restrict__ coop_seg, int* __restrict__ coop_log,
                         const int helpers) {
    extern __shared__ int s_mem[];
    int* s_li = s_mem;
    int* s_ld = s_mem + 32 * K;
    unsigned* s_taken = (unsigned*)(s_mem + 64 * K);   // leader: [(nd + 31) / 32]; helper: its shard only
    __shared__ ReplayShared sh;
    __shared__ __align__(16) uint32_t s_qc[(MASKED ? 2 : 1) * 32 * WORDS];
    const int s = blockIdx.x / (helpers + 1), role = blockIdx.x - s * (helpers + 1), tid = threadIdx.x;   // role 0 = leader
    const int q0 = seg[s], nq = seg[s + 1] - q0;
    // shards: leader [0, cut), helper h (1-based role) [cut + (h-1) * per, ...): equal shares, the leader takes one too
    const int per = (nd + helpers) / (helpers + 1);
    const int lo = role * per, hi = min(nd, lo + per);
    const int bit_lo = role == 0 ? 0 : lo, bit_hi = role == 0 ? nd : hi;                 // the leader needs every bit for the list walk
    for (int w = tid; w < (bit_hi - bit_lo + 31) / 32; w += kBfReplayThreads) {
        unsigned bits = 0u;
        if (valid2)
            for (int k = 0; k < 32 && bit_lo + w * 32 + k < bit_hi; ++k) bits |= (valid2[bit_lo + w * 32 + k] ? 0u : 1u) << k;
        s_taken[w] = bits;
    }
    if (role == 0)
        for (int i = tid; i < nq; i += kBfReplayThreads) matches12[q0 + i] = -1;
    __syncthreads();
    if (role != 0) {
        replay_helper<WORDS, MASKED, kBfReplayThreads>(coop_seg + s, coop_log + q0, role - 1, q + (size_t)q0 * WORDS, MASKED ? qm + (size_t)q0 * WORDS : nullptr,
                                                       d, dm, lo, hi, s_taken, &sh);
        return;
    }
    const CoopLeader cl{helpers ? coop_seg + s : nullptr, helpers ? coop_log + q0 : nullptr, helpers, helpers ? hi : nd};
    const int nm = replay_core<WORDS, MASKED, kBfReplayThreads, 1>(list_idx + (size_t)q0 * K, list_dist + (size_t)q0 * K, K, nq, valid1 ? valid1 + q0 : nullptr,
                                                                q + (size_t)q0 * WORDS, MASKED ? qm + (size_t)q0 * WORDS : nullptr, d, dm, nd, th_low,
                                                                nnratio, matches12 + q0, s_li, s_ld, s_taken, &sh, s_qc, cl);
    if (tid == 0) nmatches[s] = nm;
}

cudaError_t launch_bruteforce_replay(const int* list_idx, const int* list_dist, int K, const uint8_t* q, const uint8_t* qm, const uint8_t* valid1,
                                     const int* seg, int n_seg, int nq_total, const uint8_t* d, const uint8_t* dm, const uint8_t* valid2, int nd, int dim,
                                     int th_low, double nnratio, int* matches12, int* nmatches, cudaStream_t st) {
    if (n_seg < 1) return cudaSuccess;
    if (nd >= (1 << kKeyShift) || (dim != 16 && dim != 32 && dim != 64)) return cudaErrorInvalidValue;
    const size_t smem = (size_t)64 * K * 4 + (size_t)((nd + 31) / 32) * 4;
    if (smem > 200 * 1024) return cudaErrorInvalidValue;
    const bool masked = qm && dm;
    int dev = 0, sms = 0, coop_ok = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&coop_ok, cudaDevAttrCooperativeLaunch, dev);
    if (e != cudaSuccess) return e;
    const void* fn = nullptr;
#define MCS_BR(W, M) fn = (const void*)bruteforce_replay_kernel<W, M>
    if (dim == 16) { if (masked) MCS_BR(4, true); else MCS_BR(4, false); }
    else if (dim == 32) { if (masked) MCS_BR(8, true); else MCS_BR(8, false); }
    else { if (masked) MCS_BR(16, true); else MCS_BR(16, false); }
#undef MCS_BR
    if (smem > 48 * 1024) {
        e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    // helper CTAs per query set: only worth it for a large database (a rescan of a few thousand entries is faster than a
    // round trip through global memory), and only as many as can be co-resident with every leader
    int per_sm = 0, helpers = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kBfReplayThreads, smem);
    if (e != cudaSuccess) return e;
    if (coop_ok && nd >= 32768) helpers = std::max(0, std::min(kCoopMax, per_sm * sms / n_seg - 1));
    CoopSeg* cseg = nullptr; int* clog = nullptr;
    if (helpers) {
        e = keep_pool_memory();
        if (e == cudaSuccess) e = cudaMallocAsync((void**)&cseg, sizeof(CoopSeg) * n_seg, st);
        if (e == cudaSuccess) e = cudaMallocAsync((void**)&clog, sizeof(int) * (size_t)std::max(nq_total, 1), st);
        if (e == cudaSuccess) e = cudaMemsetAsync(cseg, 0, sizeof(CoopSeg) * n_seg, st);
        if (e != cudaSuccess) return e;
    }
    const uint32_t *q32 = (const uint32_t*)q, *qm32 = (const uint32_t*)qm, *d32 = (const uint32_t*)d, *dm32 = (const uint32_t*)dm;
    void* args[] = {(void*)&list_idx, (void*)&list_dist, (void*)&K, (void*)&q32, (void*)&qm32, (void*)&valid1, (void*)&seg, (void*)&d32, (void*)&dm32,
                    (void*)&valid2, (void*)&nd, (void*)&th_low, (void*)&nnratio, (void*)&matches12, (void*)&nmatches, (void*)&cseg, (void*)&clog,
                    (void*)&helpers};
    const dim3 grid(n_seg * (helpers + 1)), block(kBfReplayThreads);
    if (helpers) e = cudaLaunchCooperativeKernel(fn, grid, block, args, smem, st);       // co-residency guaranteed or the launch fails
    else e = cudaLaunchKernel(fn, grid, block, args, smem, st);
    if (helpers) { cudaFreeAsync(cseg, st); cudaFreeAsync(clog, st); }
    return e != cudaSuccess ? e : cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// window search
// ------------------------------------------------------------------------------------------------
template <int WORDS, bool MASKED>
__global__ void __launch_bounds__(256)
window_search_kernel(const WindowFrameDev f, const mcs_window_query* __restrict__ queries, const int nq,
                     const uint32_t* __restrict__ qdesc, const uint32_t* __restrict__ qmask, const int max_cand,
                     int* __restrict__ cand_idx, int* __restrict__ cand_dist, int* __restrict__ cand_count) {
    const int lane = threadIdx.x & 31;
    const int qi = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (qi >= nq) return;
    const mcs_window_query qq = queries[qi];
    const int cam = qq.cam;
    const double x = qq.x, y = qq.y, r = qq.r;
    // cell range (ref src/cMultiFrame.cpp:280-298): floor/ceil of double products, early outs
    const double wi = f.winv[cam], hi = f.hinv[cam];
    int count = 0;
    bool empty = false;
    int cx0 = (int)floor((x - 0 - r) * wi); cx0 = max(0, cx0); if (cx0 >= MCS_FRAME_GRID_COLS) empty = true;
    int cx1 = (int)ceil((x - 0 + r) * wi);  cx1 = min(MCS_FRAME_GRID_COLS - 1, cx1); if (cx1 < 0) empty = true;
    int cy0 = (int)floor((y - 0 - r) * hi); cy0 = max(0, cy0); if (cy0 >= MCS_FRAME_GRID_ROWS) empty = true;
    int cy1 = (int)ceil((y - 0 + r) * hi);  cy1 = min(MCS_FRAME_GRID_ROWS - 1, cy1); if (cy1 < 0) empty = true;
    if (!empty) {
        uint32_t qw[WORDS], qm[MASKED ? WORDS : 1];
#pragma unroll
        for (int k = 0; k < WORDS; ++k) {
            qw[k] = qdesc[(size_t)qq.desc_index * WORDS + k];
            if (MASKED) qm[k] = qmask[(size_t)qq.desc_index * WORDS + k];
        }
        const bool check = !(qq.min_level == -1 && qq.max_level == -1);
        const bool same = check && qq.min_level == qq.max_level;
        int* oi = cand_idx + (size_t)qi * max_cand;
        int* od = cand_dist + (size_t)qi * max_cand;
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
                        // abs(kp.pt.x - x) > r with float - double -> double (ref :328)
                        if (ok) ok = !(fabs((double)f.kx[id] - x) > r || fabs((double)f.ky[id] - y) > r);
                    }
                    int row = id;
                    if (f.cam_first) {           // SearchByProjection(KF, Scw): contiguous id used as the row of camera `cam`
                        row = f.cam_first[cam] + id;
                        ok = ok && row < f.cam_first[cam + 1];
                    }
                    const unsigned m = __ballot_sync(0xffffffffu, ok);
                    if (ok) {
                        const int pos = count + __popc(m & ((1u << lane) - 1u));
                        if (pos < max_cand) {
                            const uint32_t* dd = (const uint32_t*)f.desc + (size_t)row * WORDS;
                            unsigned dist = 0;
                            if (MASKED) {
                                const uint32_t* mm = (const uint32_t*)f.dmask + (size_t)row * WORDS;
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
                            oi[pos] = id;
                            od[pos] = (int)dist;
                        }
                    }
                    count += __popc(m);
                }
            }
    }
    if (lane == 0) cand_count[qi] = count;
}

cudaError_t launch_window_search(const WindowFrameDev& f, const mcs_window_query* q, int nq, const uint8_t* qdesc,
                                 const uint8_t* qmask, int max_cand, int* cand_idx, int* cand_dist, int* cand_count,
                                 cudaStream_t st) {
    if (nq <= 0) return cudaSuccess;
    const int blocks = (nq * 32 + 255) / 256;
    const bool masked = qmask && f.dmask;
#define MCS_WS(W, M) window_search_kernel<W, M><<<blocks, 256, 0, st>>>(f, q, nq, (const uint32_t*)qdesc, (const uint32_t*)qmask, \
        max_cand, cand_idx, cand_dist, cand_count)
    if (f.dim == 16) { if (masked) MCS_WS(4, true); else MCS_WS(4, false); }
    else if (f.dim == 32) { if (masked) MCS_WS(8, true); else MCS_WS(8, false); }
    else if (f.dim == 64) { if (masked) MCS_WS(16, true); else MCS_WS(16, false); }
    else return cudaErrorInvalidValue;
#undef MCS_WS
    return cudaGetLastError();
}

// Candidate lists [nq][max_cand] -> one dense array in query order (off = exclusive prefix sum of min(count, max_cand)): the host
// copies back the candidates that exist instead of nq * max_cand slots (SearchByProjection over 50 k map points x 8 views: 3 MB
// instead of 200 MB).
__global__ void compact_lists_kernel(const int* __restrict__ idx, const int* __restrict__ dist, const int* __restrict__ count,
                                     const int* __restrict__ off, const int nq, const int max_cand, int* __restrict__ oidx,
                                     int* __restrict__ odist) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    const int n = min(count[q], max_cand), o = off[q];
    for (int k = 0; k < n; ++k) {
        oidx[o + k] = idx[(size_t)q * max_cand + k];
        odist[o + k] = dist[(size_t)q * max_cand + k];
    }
}
cudaError_t launch_compact_lists(const int* idx, const int* dist, const int* count, const int* off, int nq, int max_cand, int* oidx, int* odist,
                                 cudaStream_t st) {
    if (nq <= 0) return cudaSuccess;
    compact_lists_kernel<<<(nq + 255) / 256, 256, 0, st>>>(idx, dist, count, off, nq, max_cand, oidx, odist);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// frame epilogue of the cMultiFrame constructor (ref src/cMultiFrame.cpp:143-184, :342-353): bearing rays + 64x48 grid (CSR)
// ------------------------------------------------------------------------------------------------
// One CTA of 1024 threads per frame.  cell_of / cursor are global scratch ([n_keys], [n_cell]).
__global__ void __launch_bounds__(1024)
frame_prepare_kernel(const mcs_keypoint* __restrict__ keys, const int* __restrict__ key_cam, const int n_keys,
                     const mcs_ocam* __restrict__ cams, const int n_cams, float* __restrict__ kx, float* __restrict__ ky,
                     int* __restrict__ koct, double* __restrict__ rays, int* __restrict__ cell_of, int* __restrict__ cursor,
                     int* __restrict__ cell_start, int* __restrict__ cell_items, double* __restrict__ winv, double* __restrict__ hinv) {
    __shared__ int s_part[1024];
    const int tid = threadIdx.x;
    const int n_cell = n_cams * MCS_FRAME_GRID_COLS * MCS_FRAME_GRID_ROWS;
    for (int c = tid; c < n_cams; c += 1024) {
        winv[c] = (double)MCS_FRAME_GRID_COLS / (double)cams[c].width;       // mfGridElementWidthInv (ref :154-157)
        hinv[c] = (double)MCS_FRAME_GRID_ROWS / (double)cams[c].height;
    }
    for (int c = tid; c <= n_cell; c += 1024) cell_start[c] = 0;
    __syncthreads();
    // rays, SoA copies, cell of every keypoint, histogram
    for (int i = tid; i < n_keys; i += 1024) {
        const mcs_keypoint k = keys[i];
        const int c = key_cam[i];
        kx[i] = k.x; ky[i] = k.y; koct[i] = k.octave;
        if (rays) {
            double x, y, z;
            cam_img_to_world(cams[c], (double)k.x, (double)k.y, x, y, z);
            rays[3 * i] = x; rays[3 * i + 1] = y; rays[3 * i + 2] = z;
        }
        // PosInGrid: cvRound((pt - mnMin) * inv): float - int -> float, times double (ref :345-346)
        const int px = __double2int_rn((double)(k.x - 0.f) * ((double)MCS_FRAME_GRID_COLS / (double)cams[c].width));
        const int py = __double2int_rn((double)(k.y - 0.f) * ((double)MCS_FRAME_GRID_ROWS / (double)cams[c].height));
        int cell = -1;
        if (px >= 0 && px < MCS_FRAME_GRID_COLS && py >= 0 && py < MCS_FRAME_GRID_ROWS) {
            cell = (c * MCS_FRAME_GRID_COLS + px) * MCS_FRAME_GRID_ROWS + py;
            atomicAdd(&cell_start[cell + 1], 1);
        }
        cell_of[i] = cell;
    }
    __syncthreads();
    // inclusive scan of cell_start[1..n_cell] (contiguous chunk per thread + block scan of the chunk sums)
    const int chunk = (n_cell + 1023) / 1024;
    const int lo = 1 + tid * chunk, hi = min(lo + chunk, n_cell + 1);
    int sum = 0;
    for (int c = lo; c < hi; ++c) sum += cell_start[c];
    s_part[tid] = sum;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const int v = tid >= o ? s_part[tid - o] : 0;
        __syncthreads();
        s_part[tid] += v;
        __syncthreads();
    }
    int run = tid ? s_part[tid - 1] : 0;
    for (int c = lo; c < hi; ++c) { run += cell_start[c]; cell_start[c] = run; }
    __syncthreads();
    for (int c = tid; c < n_cell; c += 1024) cursor[c] = cell_start[c];
    __syncthreads();
    for (int i = tid; i < n_keys; i += 1024) {
        const int cell = cell_of[i];
        if (cell >= 0) cell_items[atomicAdd(&cursor[cell], 1)] = i;
    }
    __syncthreads();
    // insertion order inside a cell = ascending keypoint index (the constructor pushes in index order, ref :176-181)
    for (int c = tid; c < n_cell; c += 1024) {
        const int a = cell_start[c], b = cell_start[c + 1];
        for (int i = a + 1; i < b; ++i) {
            const int v = cell_items[i];
            int j = i - 1;
            while (j >= a && cell_items[j] > v) { cell_items[j + 1] = cell_items[j]; --j; }
            cell_items[j + 1] = v;
        }
    }
}

cudaError_t launch_frame_prepare(const mcs_keypoint* keys, const int* key_cam, int n_keys, const mcs_ocam* cams, int n_cams, float* kx,
                                 float* ky, int* koct, double* rays, int* cell_of, int* cursor, int* cell_start, int* cell_items,
                                 double* winv, double* hinv, cudaStream_t st) {
    frame_prepare_kernel<<<1, 1024, 0, st>>>(keys, key_cam, n_keys, cams, n_cams, kx, ky, koct, rays, cell_of, cursor, cell_start,
                                             cell_items, winv, hinv);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// projection front-end: isInFrustum for every (map point, camera)   (ref src/cMultiFrame.cpp:218-270)
// ------------------------------------------------------------------------------------------------
__global__ void frustum_kernel(const int n_cams, const double* __restrict__ mtmc_inv, const double* __restrict__ mtmc,
                               const mcs_ocam* __restrict__ cams, const uint8_t* __restrict__ masks, const int n_points,
                               const double* __restrict__ pos, const double* __restrict__ nrm, const double* __restrict__ dmin,
                               const double* __restrict__ dmax, const double* __restrict__ sf, const int n_levels,
                               uint8_t* __restrict__ in_view, int* __restrict__ level, double* __restrict__ px, double* __restrict__ py,
                               double* __restrict__ vcos) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_points * n_cams) return;
    const int i = t / n_cams, c = t - i * n_cams;
    in_view[t] = 0; level[t] = 0; px[t] = 0.0; py[t] = 0.0; vcos[t] = 0.0;
    const double P0 = pos[3 * i], P1 = pos[3 * i + 1], P2 = pos[3 * i + 2];
    // ptRot = MtMc_inv[c] * (P,1): cv::Matx product, s = 0 + a0 b0 + a1 b1 + a2 b2 + a3 b3 in this order, no FMA
    const double* M = mtmc_inv + 16 * c;
    double r[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) r[k] = ((M[4 * k] * P0 + M[4 * k + 1] * P1) + M[4 * k + 2] * P2) + M[4 * k + 3] * 1.0;
    const mcs_ocam cam = cams[c];
    double u, v;
    cam_world_to_img(cam, r[0], r[1], r[2], u, v);
    // isPointInMirrorMask(u, v, 0)  (ref src/cam_model_omni.cpp:163-178)
    const int ur = __double2int_rn(u), vr = __double2int_rn(v);
    if (ur >= cam.width || ur <= 0 || vr >= cam.height || vr <= 0) return;
    if (masks[(size_t)c * cam.width * cam.height + (size_t)vr * cam.width + ur] == 0) return;
    // distance to the camera centre, scale-invariance region
    const double* T = mtmc + 16 * c;
    const double o0 = P0 - T[3], o1 = P1 - T[7], o2 = P2 - T[11];
    const double dist = sqrt((o0 * o0 + o1 * o1) + o2 * o2);
    if (dist < dmin[i] || dist > dmax[i]) return;
    const double viewCos = ((o0 * nrm[3 * i] + o1 * nrm[3 * i + 1]) + o2 * nrm[3 * i + 2]) / dist;
    const double ratio = dist / dmin[i];
    int lv = 0;                                   // std::lower_bound(mvScaleFactors, ratio)
    while (lv < n_levels && sf[lv] < ratio) ++lv;
    if (lv >= n_levels) lv = n_levels - 1;
    in_view[t] = 1; px[t] = u; py[t] = v; level[t] = lv; vcos[t] = viewCos;
}

cudaError_t launch_frustum(int n_cams, const double* mtmc_inv, const double* mtmc, const mcs_ocam* cams, const uint8_t* masks,
                           int n_points, const double* pos, const double* nrm, const double* dmin, const double* dmax, const double* sf,
                           int n_levels, uint8_t* in_view, int* level, double* px, double* py, double* vcos, cudaStream_t st) {
    const long long n = (long long)n_points * n_cams;
    if (n <= 0) return cudaSuccess;
    frustum_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(n_cams, mtmc_inv, mtmc, cams, masks, n_points, pos, nrm, dmin, dmax, sf,
                                                                n_levels, in_view, level, px, py, vcos);
    return cudaGetLastError();
}

}  // namespace mcs
