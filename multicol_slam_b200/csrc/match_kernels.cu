// match_kernels.cu -- sm_90a kernels of the matcher half of the hot path.
//
//   M2 hamming_topk_kernel : all-pairs bit-level Hamming distance (ref src/cORBmatcher.cpp:2438-2474)
//                            of nq queries against nd database descriptors, K best (distance, index)
//                            per query, as binary matrix products on the tensor cores (BMMA AND.POPC, see
//                            "K-best lists on the binary tensor cores" below).  A warp owns 32 queries (fragments in
//                            registers), database tiles are staged in shared memory.  Not bound by HBM.
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
// H100 80GB HBM3, 400 W limit, bench.py config 2, 2 alternating runs: this split (7 carry-save adders + 9 POPC) 6.71 / 6.69 ms,
// 5 + 11: 7.27 / 7.03 ms, 6 + 10: 7.07 / 7.00 ms.
__device__ __forceinline__ void popc_sum16(const uint32_t (&w)[16], unsigned& ones_out, unsigned& twos_out) {
    uint32_t s0, c0, s1, c1, s2, c2, s3, c3, s4, c4;
    csa(w[0], w[1], w[2], s0, c0);
    csa(w[3], w[4], w[5], s1, c1);
    csa(w[6], w[7], w[8], s2, c2);
    csa(w[9], w[10], w[11], s3, c3);
    csa(w[12], w[13], w[14], s4, c4);
    uint32_t a0, b0, a1, b1;
    csa(s0, s1, s2, a0, b0);
    csa(s3, s4, w[15], a1, b1);
    const unsigned ones = __popc(a0) + __popc(a1);
    const unsigned twos = __popc(c0) + __popc(c1) + __popc(c2) + __popc(c3) + __popc(c4) + __popc(b0) + __popc(b1);
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

// ---- K-best lists on the binary tensor cores -------------------------------------------------------------------------------------
// Query a (mask m1) against database entry b (mask m2), x = a ^ b, [u|v].[s|t] = popc(u & s) + popc(v & t) (AND-popcount over
// the concatenation):
//   masked:   T = popc(a&m1) + popc(b&m2) + [m1|a].[b|m2] - 2 [a&m1|a].[b|b&m2] = popc(x&m1) + popc(x&m2),  dist = T >> 1
//             (the integer division of ref :2472)
//   unmasked: dist = popc(a) + popc(b) - 2 a.b
// The dot products of 16 queries x 8 entries are one mma.sync.m16n8k256 .b1 AND.POPC (BMMA) per 256 bits of operand: masked
// 2 / 4 / 8 BMMAs per 16x8 tile at 16 / 32 / 64 bytes, unmasked 1 / 1 / 2 (the second half of a 16-byte k256 step is zero).
// .xor.popc would give popc(x) directly, but sm_90 lowers it to two AND BMMAs plus inversions.  Measured rate (tools/bmma_rate.cu,
// H100 80GB HBM3, 400 W limit): 0.66 BMMA/clk/SM with 8 or more warps of 4 independent chains, i.e. 21 masked 32-byte pairs/clk/SM,
// where the carry-save popcount on the CUDA cores (popc_sum16) is capped near 1.8 by the POPC issue rate.
// Operand layout: the k dimension is a sequence of 128-bit half chunks (word w of a descriptor is word t = w % 4 of half chunk
// w / 4); a k256 step takes two of them, and lane (g, t) holds word t of both for rows g and g + 8 (A) and column g (B).  A warp
// owns 32 queries (two m16 tiles) and keeps their fragments in registers; database tiles are staged in shared memory with each
// row's words permuted so that a lane's words of all half chunks are adjacent (one 32/64/128-bit load, the warp reads one
// contiguous block: no bank conflicts).  b & m2 is formed in registers.
// Epilogue: 3 integer instructions per pair (value, compare); one warp vote skips the rest when no lane has a pair below its
// threshold.  The 4 lanes of a quad see the same 4 query rows over disjoint columns (2 of every 8), and together hold one sorted
// K-best list per row, KT / 4 keys per lane (lane t positions t KT/4 ..).  A pair is a candidate iff its key is below the row's
// K-th key kK (every lane of the quad knows it; for the columns still to come this is distance < dK, see bmma_klists); keys are
// unique (the index is part of the key), so this is exact, and ties keep the earlier index.  Candidates are appended to the
// lane's buffer in shared memory and folded in batches: per row, each lane sorts its buffer, a quad butterfly keeps the KT
// smallest of the four, and they are merged with the list -- a fixed network per row, whatever the busiest lane buffered.  H100 80GB HBM3, 700 W limit, bench.py
// config 2, the greedy matcher's list kernel (tools/m2_split.py): 3.92 ms with one insertion per slot into per-lane lists, 1.76 ms
// with per-lane lists, the candidate buffer and a bound shared by the quad, 1.23-1.24 ms with one list per row; 0.65 ms when
// nothing is listed (th_low = 0).
// Keys are 32 bits: distance << SHIFT | index (SHIFT 16 for the stream matcher's slots, kTopkShift for the key-frame database).
constexpr int kTopkShift = 21;
constexpr unsigned kColOff = 0x40000u;       // cd of a column that is not listed (beyond the database, skipped): its value exceeds
                                             // every threshold (<= 2 * 0xFFFF) whatever the stale operand bits contribute
// CTAs per SM the list kernels are compiled for (a register budget: 128 per thread, 168 for the 64-byte masked fragments).  Without
// it ptxas kept some instantiations at 72 registers and reloaded A fragments from local memory in the inner loop.
template <int WORDS, bool MASKED>
constexpr int kListMinBlocks = (MASKED && WORDS == 16) ? 3 : 4;
// Candidate keys a lane buffers per query row before the warp folds them into the lists (bmma_klists).  7 keeps the 64-byte masked
// kernels' static shared memory under 48 KB.
constexpr int kCandDepth = 7;
template <int WORDS, bool MASKED>
struct BmmaTile {                            // one staged database tile, rows permuted (see above)
    uint32_t b[kDbTile * WORDS];
    uint32_t m[MASKED ? kDbTile * WORDS : 4];
    unsigned cd[kDbTile];                    // popc(b & m2) (masked) / popc(b), kColOff for a column that is not listed
    unsigned cand[kTopkThreads / 32][4][kCandDepth][32];    // [warp][row r][entry][lane]: the lanes' candidate buffers
};

__device__ __forceinline__ void cmp_swap(unsigned& a, unsigned& b) { const unsigned lo = min(a, b); b = max(a, b); a = lo; }
// ascending sort of 8 keys, 19 compare-exchanges (Knuth, TAOCP 5.3.4)
__device__ __forceinline__ void sort8(unsigned (&x)[8]) {
    constexpr int kNet[19][2] = {{0, 2}, {1, 3}, {4, 6}, {5, 7}, {0, 4}, {1, 5}, {2, 6}, {3, 7}, {0, 1}, {2, 3},
                                 {4, 5}, {6, 7}, {2, 4}, {3, 5}, {1, 4}, {3, 6}, {1, 2}, {3, 4}, {5, 6}};
#pragma unroll
    for (int i = 0; i < 19; ++i) cmp_swap(x[kNet[i][0]], x[kNet[i][1]]);
}
// x[0, N) <- the N smallest of x[0, N) and y[0, N), both ascending, in ascending order: min(x[i], y[N-1-i]) is a bitonic sequence
// holding them, then a bitonic merge sorts it
template <int N>
__device__ __forceinline__ void merge_lowest(unsigned (&x)[8], const unsigned (&y)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) x[i] = min(x[i], y[N - 1 - i]);
#pragma unroll
    for (int j = N / 2; j > 0; j /= 2)
#pragma unroll
        for (int i = 0; i < N; ++i)
            if (!(i & j)) cmp_swap(x[i], x[i + j]);
}

__device__ __forceinline__ void bmma_and_popc(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
template <int H>
__device__ __forceinline__ void lds_words(const uint32_t* p, uint32_t (&w)[H]) {
    if constexpr (H == 4) { const uint4 v = *reinterpret_cast<const uint4*>(p); w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w; }
    else if constexpr (H == 2) { const uint2 v = *reinterpret_cast<const uint2*>(p); w[0] = v.x; w[1] = v.y; }
    else w[0] = p[0];
}

// Database entries [t0, t0 + tn) of d (dm) into the tile; skip[i] != 0 leaves entry i out of the lists.
template <int WORDS, bool MASKED>
__device__ __forceinline__ void bmma_stage(BmmaTile<WORDS, MASKED>& s, const uint32_t* __restrict__ d, const uint32_t* __restrict__ dm,
                                           const uint8_t* __restrict__ skip, const int t0, const int tn) {
    constexpr int H = WORDS / 4;
    for (int j = threadIdx.x; j < kDbTile; j += kTopkThreads) {
        unsigned cd = kColOff;
        if (j < tn && !(skip && skip[t0 + j])) {
            uint32_t w[WORDS], mw[WORDS];
            const uint4* src = reinterpret_cast<const uint4*>(d + (size_t)(t0 + j) * WORDS);
            const uint4* msrc = MASKED ? reinterpret_cast<const uint4*>(dm + (size_t)(t0 + j) * WORDS) : nullptr;
#pragma unroll
            for (int k = 0; k < H; ++k) {
                const uint4 v = src[k]; w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
                if (MASKED) { const uint4 u = msrc[k]; mw[4 * k] = u.x; mw[4 * k + 1] = u.y; mw[4 * k + 2] = u.z; mw[4 * k + 3] = u.w; }
            }
            cd = 0;
#pragma unroll
            for (int k = 0; k < WORDS; ++k) cd += __popc(MASKED ? (w[k] & mw[k]) : w[k]);
            uint32_t pw[WORDS], pm[WORDS];                       // word 4h + t at t * H + h
#pragma unroll
            for (int k = 0; k < WORDS; ++k) { pw[(k & 3) * H + (k >> 2)] = w[k]; pm[(k & 3) * H + (k >> 2)] = mw[k]; }
#pragma unroll
            for (int k = 0; k < H; ++k) {
                reinterpret_cast<uint4*>(s.b + j * WORDS)[k] = make_uint4(pw[4 * k], pw[4 * k + 1], pw[4 * k + 2], pw[4 * k + 3]);
                if (MASKED) reinterpret_cast<uint4*>(s.m + j * WORDS)[k] = make_uint4(pm[4 * k], pm[4 * k + 1], pm[4 * k + 2], pm[4 * k + 3]);
            }
        }
        s.cd[j] = cd;
    }
}

// The K-best lists of the CTA's 128 queries (rows 0 .. nq_cta - 1 of q / qm; rows beyond are not listed) against database entries
// [j0, j1) of d / dm that skip does not exclude, listing only distances below worst0.  Every thread of the CTA must call this.
// emit(row, k, key) receives, from the lane of the quad that holds it, key k < KT of the CTA row (kNone past the list's end).
template <int WORDS, bool MASKED, int KT, int SHIFT, class Emit>
__device__ __forceinline__ void bmma_klists(const uint32_t* __restrict__ q, const uint32_t* __restrict__ qm, const int nq_cta,
                                            const uint32_t* __restrict__ d, const uint32_t* __restrict__ dm, const uint8_t* __restrict__ skip,
                                            const int j0, const int j1, const int K, const unsigned worst0, BmmaTile<WORDS, MASKED>& s,
                                            Emit&& emit) {
    constexpr int H = WORDS / 4;                                   // 128-bit half chunks of a descriptor
    constexpr int STEPS = MASKED ? H : (H + 1) / 2;                // k256 steps per product
    constexpr unsigned kNone = 0xFFFFFFFFu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    // rows r = 0..3 of this lane: m-tile r >> 1, row g + 8 * (r & 1) of it
    uint32_t qa[4][H], qx[4][H], qam[4][H];         // a, m1, a & m1: word t of every half chunk
    unsigned cq[4], thr[4];                                        // popc(a & m1) / popc(a); value threshold (2 * worst masked)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int row = warp * 32 + (r >> 1) * 16 + (r & 1) * 8 + g;
        const bool act = row < nq_cta;
        unsigned c = 0;
#pragma unroll
        for (int h = 0; h < H; ++h) {
            qa[r][h] = act ? q[(size_t)row * WORDS + 4 * h + t] : 0u;
            if constexpr (MASKED) {
                qx[r][h] = act ? qm[(size_t)row * WORDS + 4 * h + t] : 0u;
                qam[r][h] = qa[r][h] & qx[r][h];
                c += __popc(qam[r][h]);
            } else {
                c += __popc(qa[r][h]);
            }
        }
        c += __shfl_xor_sync(0xffffffffu, c, 1);
        c += __shfl_xor_sync(0xffffffffu, c, 2);
        cq[r] = c;
        thr[r] = act ? (MASKED ? 2 * worst0 : worst0) : 0u;
    }
    constexpr int P = KT / 4;                                      // list positions per lane
    static_assert(KT % 4 == 0 && KT <= 8 && kCandDepth <= 7, "a fold sorts one lane's buffer in 8 registers");
    unsigned list[4][P];                                           // row r: positions t P .. t P + P - 1 of its list
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int p = 0; p < P; ++p) list[r][p] = kNone;
    unsigned* cand = &s.cand[warp][0][0][lane];                    // row r, entry i at cand[(r * kCandDepth + i) * 32]
    int cnt[4] = {0, 0, 0, 0};
    // Fold the quad's buffered keys of each row into its list: every lane sorts its own, two butterfly rounds leave the KT smallest
    // of the quad's in every lane, and merging them with the list gives the new list in every lane; lane t keeps its positions.
    // A pair is a candidate iff its key is below the row's K-th key kK.  Every column visited after a fold has a larger index than
    // every column before it, kK's included, so for those columns key < kK is distance < dK, dK the distance of kK: the threshold
    // on the value is exact and strict.  The list only improves, so a pair that was not buffered has K smaller keys in the list.
    auto fold = [&]() {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            if (!__any_sync(0xffffffffu, cnt[r] > 0)) continue;
            unsigned x[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) x[i] = i < cnt[r] ? cand[(r * kCandDepth + i) * 32] : kNone;
            cnt[r] = 0;
            sort8(x);
#pragma unroll
            for (int m = 1; m <= 2; m <<= 1) {
                unsigned y[KT];
#pragma unroll
                for (int i = 0; i < KT; ++i) y[i] = __shfl_xor_sync(0xffffffffu, x[i], m);
                merge_lowest<KT>(x, y);
            }
            unsigned y[KT];
#pragma unroll
            for (int k = 0; k < KT; ++k) y[k] = __shfl_sync(0xffffffffu, list[r][k % P], (lane & ~3) | (k / P));
            merge_lowest<KT>(x, y);
#pragma unroll
            for (int p = 0; p < P; ++p) {
                unsigned v = x[p];
#pragma unroll
                for (int u = 1; u < 4; ++u) if (t == u) v = x[u * P + p];
                list[r][p] = v;
            }
            unsigned w = x[0];
#pragma unroll
            for (int k = 1; k < KT; ++k) if (k < K) w = x[k];
            if (w != kNone) thr[r] = min(thr[r], (w >> SHIFT) * (MASKED ? 2 : 1));
        }
    };

    for (int t0 = j0; t0 < j1; t0 += kDbTile) {
        const int tn = min(kDbTile, j1 - t0);
        __syncthreads();
        bmma_stage<WORDS, MASKED>(s, d, dm, skip, t0, tn);
        __syncthreads();
        for (int n0 = 0; n0 < tn; n0 += 8) {
            uint32_t bw[H], mw[H], bmw[H];
            lds_words<H>(s.b + (n0 + g) * WORDS + t * H, bw);
            if constexpr (MASKED) {
                lds_words<H>(s.m + (n0 + g) * WORDS + t * H, mw);
#pragma unroll
                for (int h = 0; h < H; ++h) bmw[h] = bw[h] & mw[h];
            }
            const uint2 cd = *reinterpret_cast<const uint2*>(s.cd + n0 + 2 * t);
            unsigned v[4][2];                                      // row r, column 2t + c
            bool any = false;
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                const int r0 = 2 * mt, r1 = 2 * mt + 1;
                int c1[4] = {0, 0, 0, 0};
#pragma unroll
                for (int st = 0; st < STEPS; ++st) {
                    // half chunks 2st, 2st + 1 of A = [m1|a] (masked) / [a], B = [b|m2] / [b]
                    const int h0 = 2 * st, h1 = 2 * st + 1;
                    if constexpr (MASKED) {
                        bmma_and_popc(c1, h0 < H ? qx[r0][h0] : qa[r0][h0 - H], h0 < H ? qx[r1][h0] : qa[r1][h0 - H],
                                      h1 < H ? qx[r0][h1] : qa[r0][h1 - H], h1 < H ? qx[r1][h1] : qa[r1][h1 - H],
                                      h0 < H ? bw[h0] : mw[h0 - H], h1 < H ? bw[h1] : mw[h1 - H]);
                    } else {
                        bmma_and_popc(c1, qa[r0][h0], qa[r1][h0], h1 < H ? qa[r0][h1] : 0u, h1 < H ? qa[r1][h1] : 0u,
                                      bw[h0], h1 < H ? bw[h1] : 0u);
                    }
                }
                if constexpr (MASKED) {
                    int c2[4] = {0, 0, 0, 0};                      // [a&m1|a].[b|b&m2]
#pragma unroll
                    for (int st = 0; st < STEPS; ++st) {
                        const int h0 = 2 * st, h1 = 2 * st + 1;
                        bmma_and_popc(c2, h0 < H ? qam[r0][h0] : qa[r0][h0 - H], h0 < H ? qam[r1][h0] : qa[r1][h0 - H],
                                      h1 < H ? qam[r0][h1] : qa[r0][h1 - H], h1 < H ? qam[r1][h1] : qa[r1][h1 - H],
                                      h0 < H ? bw[h0] : bmw[h0 - H], h1 < H ? bw[h1] : bmw[h1 - H]);
                    }
#pragma unroll
                    for (int i = 0; i < 4; ++i) c1[i] -= 2 * c2[i];
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int r = 2 * mt + (i >> 1);
                    const unsigned val = cq[r] + (i & 1 ? cd.y : cd.x) + (MASKED ? c1[i] : -2 * c1[i]);
                    v[r][i & 1] = val;
                    any |= val < thr[r];
                }
            }
            // candidates below the threshold go to this lane's buffer, in column order; the warp folds them in when some lane's
            // buffer for a row could not take another step's two columns.  A step where no lane has a candidate costs one vote.
            if (__any_sync(0xffffffffu, any)) {
                if (any) {
#pragma unroll
                    for (int r = 0; r < 4; ++r)
#pragma unroll
                        for (int c = 0; c < 2; ++c)
                            if (v[r][c] < thr[r]) {
                                cand[(r * kCandDepth + cnt[r]) * 32] = ((MASKED ? v[r][c] >> 1 : v[r][c]) << SHIFT) | (unsigned)(t0 + n0 + 2 * t + c);
                                ++cnt[r];
                            }
                }
                if (__any_sync(0xffffffffu, max(max(cnt[0], cnt[1]), max(cnt[2], cnt[3])) > kCandDepth - 2)) fold();
            }
        }
    }
    fold();
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int row = warp * 32 + (r >> 1) * 16 + (r & 1) * 8 + g;
#pragma unroll
        for (int p = 0; p < P; ++p) {
            const int k = t * P + p;
            emit(row, k, k < K ? list[r][p] : kNone);
        }
    }
}

template <int WORDS, bool MASKED, int KT>
__global__ void __launch_bounds__(kTopkThreads, kListMinBlocks<WORDS, MASKED>)
hamming_topk_kernel(const uint32_t* __restrict__ q, const uint32_t* __restrict__ qmask, const int nq,
                    const uint32_t* __restrict__ d, const uint32_t* __restrict__ dmask, const int nd,
                    const uint8_t* __restrict__ skip, const int K, const int chunk, const unsigned bound,
                    unsigned* __restrict__ part /* [splits][nq][kTopKMax] */) {
    __shared__ __align__(16) BmmaTile<WORDS, MASKED> s;
    const int qb = blockIdx.x * kTopkThreads;
    const int j0 = blockIdx.y * chunk, j1 = min(j0 + chunk, nd);
    bmma_klists<WORDS, MASKED, KT, kTopkShift>(q + (size_t)qb * WORDS, MASKED ? qmask + (size_t)qb * WORDS : nullptr, nq - qb, d, dmask,
                                               skip, j0, j1, K, min(bound, 0x7FFu), s, [=](int row, int k, unsigned key) {
        if (qb + row >= nq) return;
        unsigned* o = part + ((size_t)blockIdx.y * nq + qb + row) * kTopKMax;
        o[k] = key;
        if (k == KT - 1)
            for (int j = KT; j < kTopKMax; ++j) o[j] = 0xFFFFFFFFu;
    });
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

// The database chunks of the K-best list kernels for cta_q CTAs of queries and a database of at most n_db entries: enough CTAs for
// ~4 waves, chunks a multiple of the tile, and `splits` chunks cover n_db.  An empty database is one empty chunk.
struct ListPlan { int chunk, splits; };
ListPlan list_plan(const int sms, const long long cta_q, const int n_db) {
    const int tiles = (n_db + kDbTile - 1) / kDbTile;
    const int splits = (int)std::max(1LL, std::min((long long)tiles, (4LL * sms * 8 + cta_q - 1) / cta_q));
    const int chunk = std::max(1, (tiles + splits - 1) / splits) * kDbTile;
    return {chunk, std::max(1, (n_db + chunk - 1) / chunk)};
}

cudaError_t launch_hamming_topk(const uint8_t* q, const uint8_t* qmask, int nq, const uint8_t* d, const uint8_t* dmask,
                                int nd, const uint8_t* db_skip, int dim, int K, unsigned bound, int* topk_idx, int* topk_dist,
                                cudaStream_t st) {
    if (K < 1 || K > kTopKMax || !desc_width_ok(dim) || nd >= (1 << kTopkShift)) return cudaErrorInvalidValue;
    if (nq <= 0) return cudaSuccess;
    const int qblocks = (nq + kTopkThreads - 1) / kTopkThreads;
    int sms = 0;
    cudaError_t e = sm_count(sms);
    if (e != cudaSuccess) return e;
    const ListPlan pl = list_plan(sms, qblocks, nd);
    // partial top-K lists of the database splits: stream-ordered scratch owned by THIS call, so that concurrent callers -- the
    // reference runs its matchers from three threads -- and different streams never share it
    StreamScratch sc;
    e = sc.alloc({(size_t)pl.splits * nq * kTopKMax * sizeof(unsigned)}, st);
    if (e != cudaSuccess) return e;
    unsigned* part = sc.at<unsigned>(0);
    dim3 grid(qblocks, pl.splits);
    const bool masked = qmask && dmask;
    with_desc_width(dim, masked, [&](auto W, auto M) {
        with_list_len(K, [&](auto KT) {
            hamming_topk_kernel<W, M, KT><<<grid, kTopkThreads, 0, st>>>((const uint32_t*)q, (const uint32_t*)qmask, nq, (const uint32_t*)d,
                                                                         (const uint32_t*)dmask, nd, db_skip, K, pl.chunk, bound, part);
        });
    });
    topk_merge_kernel<<<(nq + 127) / 128, 128, 0, st>>>(part, pl.splits, nq, K, topk_idx, topk_dist);
    return sc.release(cudaGetLastError());                   // frees after the merge in stream order
}

// Stream matching: image i = (frame f, camera c) is matched against image i - n_cams = (f-1, c); both live in
// fixed-size slots of `capacity` descriptors, the valid counts are read on the device (no host sync).
// A CTA lists 128 query slots against the (<= capacity) database descriptors of the previous frame, staged tile by tile in
// shared memory (bmma_klists).  Output: K best (index, distance) per query slot, (-1, INT_MAX) where none.
// Keys are 32 bits (distance << 16 | slot; slots < 65536, distances <= 512) and the list length KT is a compile-time constant
// (4 or 8): the sorted insertion is 3 instructions per list position instead of ~6 on 64-bit keys over all 8 positions.
template <int WORDS, bool MASKED, int KT>
__global__ void __launch_bounds__(kTopkThreads, kListMinBlocks<WORDS, MASKED>)
hamming_stream_kernel(const uint32_t* __restrict__ desc, const uint32_t* __restrict__ dmask, const int* __restrict__ counts,
                      const int n_cams, const int capacity, const int K, const int img_lo, const unsigned bound,
                      int* __restrict__ out_idx, int* __restrict__ out_dist) {
    __shared__ __align__(16) BmmaTile<WORDS, MASKED> s;
    const int img = blockIdx.y + img_lo;
    const int qb = blockIdx.x * kTopkThreads;
    const bool has_prev = img >= n_cams;                 // frame 0 has no predecessor
    const int nq = has_prev ? min(counts[img], capacity) : 0;
    const int nd = has_prev ? min(counts[img - n_cams], capacity) : 0;
    if (qb >= nq) {                                      // nothing to match in this block: mark the slots empty
        const int qi = qb + threadIdx.x;
        if (qi < capacity)
            for (int k = 0; k < K; ++k) {
                out_idx[((size_t)img * capacity + qi) * K + k] = -1;
                out_dist[((size_t)img * capacity + qi) * K + k] = 0x7FFFFFFF;
            }
        return;
    }
    const size_t q_row0 = (size_t)img * capacity + qb, d_row0 = (size_t)(img - n_cams) * capacity;
    bmma_klists<WORDS, MASKED, KT, 16>(desc + q_row0 * WORDS, MASKED ? dmask + q_row0 * WORDS : nullptr, nq - qb, desc + d_row0 * WORDS,
                                       MASKED ? dmask + d_row0 * WORDS : nullptr, nullptr, 0, nd, K, min(bound, 0xFFFFu), s,
                                       [=](int row, int k, unsigned key) {
        if (qb + row >= capacity || k >= K) return;
        const bool none = qb + row >= nq || key == 0xFFFFFFFFu;
        out_idx[(q_row0 + row) * K + k] = none ? -1 : (int)(key & 0xFFFFu);
        out_dist[(q_row0 + row) * K + k] = none ? 0x7FFFFFFF : (int)(key >> 16);
    });
}

cudaError_t launch_hamming_stream(const uint8_t* desc, const uint8_t* dmask, const int* counts, int img_lo, int img_count,
                                  int n_cams, int capacity, int dim, int K, unsigned bound, int* out_idx, int* out_dist, cudaStream_t st) {
    if (K < 1 || K > kTopKMax || !desc_width_ok(dim) || capacity > 65535) return cudaErrorInvalidValue;
    if (img_count < 1) return cudaSuccess;
    dim3 grid((capacity + kTopkThreads - 1) / kTopkThreads, img_count);
    const bool masked = dmask != nullptr;
    with_desc_width(dim, masked, [&](auto W, auto M) {
        with_list_len(K, [&](auto KT) {
            hamming_stream_kernel<W, M, KT><<<grid, kTopkThreads, 0, st>>>((const uint32_t*)desc, (const uint32_t*)dmask, counts, n_cams,
                                                                           capacity, K, img_lo, bound, out_idx, out_dist);
        });
    });
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
constexpr int kReplayThreads = 256;         // stream matcher: <= 65535 database entries per image, many images in flight
constexpr int kBfReplayThreads = 1024;       // key-frame database: one CTA per query set scans up to ~1.5 M entries per rescan
constexpr int kKeyShift = 21;                // rescan keys = distance << 21 | index (index < 2^21, distance <= 512)

template <int THREADS>
__device__ __forceinline__ void named_bar(int id) { asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(THREADS) : "memory"); }

// One pass over this thread's share of the unmatched database entries for query row `row`: the two smallest
// (distance << kKeyShift | index) keys of the warp.
template <int WORDS, bool MASKED, int THREADS>
__device__ __forceinline__ void replay_scan(const uint32_t* __restrict__ qd, const uint32_t* __restrict__ qmk, const int row,
                                            const uint32_t* __restrict__ dd, const uint32_t* __restrict__ dm, const int id_lo,
                                            const int id_hi, const unsigned* s_taken /* bit (id - id_lo) */, const int tid,
                                            unsigned& k1, unsigned& k2) {
    uint32_t qw[WORDS], qm[MASKED ? WORDS : 1];
    const uint4* qp = reinterpret_cast<const uint4*>(qd + (size_t)row * WORDS);
#pragma unroll
    for (int k = 0; k < WORDS / 4; ++k) { const uint4 t = qp[k]; qw[4 * k] = t.x; qw[4 * k + 1] = t.y; qw[4 * k + 2] = t.z; qw[4 * k + 3] = t.w; }
    if (MASKED) {
        const uint4* qmp = reinterpret_cast<const uint4*>(qmk + (size_t)row * WORDS);
#pragma unroll
        for (int k = 0; k < WORDS / 4; ++k) { const uint4 t = qmp[k]; qm[4 * k] = t.x; qm[4 * k + 1] = t.y; qm[4 * k + 2] = t.z; qm[4 * k + 3] = t.w; }
    }
    k1 = 0xFFFFFFFFu; k2 = 0xFFFFFFFFu;
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
        // the list kernels' distance (carry-save popcount: 9 POPC instead of 16 per masked 256-bit pair -- a rescan is bound by the
        // POPC rate of the SM as soon as the descriptors come from shared memory)
        const unsigned dist = hamming_words<WORDS, MASKED>(qw, qm, dw, mw);
        const unsigned key = (dist << kKeyShift) | (unsigned)id;
        if (key < k1) { k2 = k1; k1 = key; } else if (key < k2) k2 = key;
    }
    // warp: smallest and second smallest of the 64 keys (keys are unique: the index is part of the key)
    const unsigned B = __reduce_min_sync(0xffffffffu, k1);
    const unsigned S = __reduce_min_sync(0xffffffffu, k1 == B ? k2 : k1);
    k1 = B; k2 = S;
}

// A pass serves one query.  Letting it also serve the next undecided queries of the chunk (look-ahead) was slower on the Lafida
// stream, and the look-ahead results are often invalidated by the matches in between.
struct ReplayShared {
    int cmd;                                  // 0 while the walk runs, -1 once it is over (helper CTAs: the rescan sequence)
    int bq;                                   // the rescan's query row
    unsigned k1[32], k2[32];                  // per warp: the two smallest keys
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
template <int WORDS, bool MASKED, int THREADS>
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
            unsigned k1, k2;
            replay_scan<WORDS, MASKED, THREADS>(s_qd, s_qm, sh->bq, dd, dmk, 0, scan_hi, s_taken, tid, k1, k2);
            if (lane == 0) { sh->k1[warp] = k1; sh->k2[warp] = k2; }
            named_bar<THREADS>(2);
        }
    }
    int nm = 0;
    if (lane == 0) sh->cmd = 0;
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
                // exact rescan of the database: two smallest (distance, index) keys among the unmatched entries
                if (lane == 0) {
                    sh->bq = t;                            // chunk-relative row (see s_qd)
                    if (coop.helpers) {                     // publish the rescan to the helper CTAs before scanning shard 0 here
                        coop.seg->cmd_query = q0 + t;
                        coop.seg->log_len = nlog;
                        __threadfence();
                        atomicExch(&coop.seg->cmd_seq, ++seq);
                    }
                }
                named_bar<THREADS>(1);
                unsigned k1, k2;
                replay_scan<WORDS, MASKED, THREADS>(s_qd, s_qm, t, dd, dmk, 0, scan_hi, s_taken, tid, k1, k2);
                if (lane == 0) { sh->k1[0] = k1; sh->k2[0] = k2; }
                named_bar<THREADS>(2);
                const unsigned w1 = lane < THREADS / 32 ? sh->k1[lane] : 0xFFFFFFFFu;
                const unsigned w2 = lane < THREADS / 32 ? sh->k2[lane] : 0xFFFFFFFFu;
                unsigned B = __reduce_min_sync(0xffffffffu, w1);
                unsigned S = __reduce_min_sync(0xffffffffu, w1 == B ? w2 : w1);
                if (coop.helpers) {                         // fold the helpers' partial minima (lanes 0..helpers-1), own shard in lane 31
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
        unsigned k1, k2;
        replay_scan<WORDS, MASKED, THREADS>(qd, qmk, q, dd, dmk, lo, hi, s_taken, tid, k1, k2);
        if (lane == 0) { sh->k1[warp] = k1; sh->k2[warp] = k2; }
        __syncthreads();
        if (warp == 0) {
            const unsigned a1 = lane < THREADS / 32 ? sh->k1[lane] : 0xFFFFFFFFu;
            const unsigned a2 = lane < THREADS / 32 ? sh->k2[lane] : 0xFFFFFFFFu;
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

// Stream matcher: one CTA per image; queries = the image's slots, database = the same camera's image one frame earlier.  The
// shared memory `s_mem` holds, in order, the database (DB_SMEM: descriptors, then masks, [capacity][WORDS] each), the list chunk
// ([32][K] indices, [32][K] distances) and the "already matched" bits ([(capacity + 31) / 32]).  Every thread of the CTA calls this.
template <int WORDS, bool MASKED, bool DB_SMEM>
__device__ __forceinline__ void stream_replay(const int* __restrict__ list_idx, const int* __restrict__ list_dist, const int* __restrict__ counts,
                                              const uint32_t* __restrict__ desc, const uint32_t* __restrict__ dmask, const int n_cams,
                                              const int capacity, const int K, const int img_lo, const int th_low, const double nnratio,
                                              int* __restrict__ matches12, int* __restrict__ nmatches, int* __restrict__ redo, int* s_mem) {
    uint32_t* s_db = (uint32_t*)s_mem;
    uint32_t* s_dbm = s_db + (DB_SMEM && MASKED ? (size_t)capacity * WORDS : 0);
    int* s_li = DB_SMEM ? (int*)(s_dbm + (size_t)capacity * WORDS) : s_mem;
    int* s_ld = s_li + 32 * K;
    unsigned* s_taken = (unsigned*)(s_ld + 32 * K);
    __shared__ ReplayShared sh;
    __shared__ __align__(16) uint32_t s_qc[(MASKED ? 2 : 1) * 32 * WORDS];
    const int img = blockIdx.x + img_lo, tid = threadIdx.x;
    const bool has_prev = img >= n_cams;
    const int nq = has_prev ? min(counts[img], capacity) : 0;
    const int nd = has_prev ? min(counts[img - n_cams], capacity) : 0;
    const size_t q_row0 = (size_t)img * capacity, d_row0 = has_prev ? (size_t)(img - n_cams) * capacity : 0;
    for (int i = tid; i < (capacity + 31) / 32; i += kReplayThreads) s_taken[i] = 0u;
    for (int i = tid; i < capacity; i += kReplayThreads) matches12[q_row0 + i] = -1;
    if (DB_SMEM && nq > 0) {
        const uint4* src = (const uint4*)(desc + d_row0 * WORDS);
        for (int i = tid; i < nd * WORDS / 4; i += kReplayThreads) ((uint4*)s_db)[i] = src[i];
        if (MASKED) {
            const uint4* msrc = (const uint4*)(dmask + d_row0 * WORDS);
            for (int i = tid; i < nd * WORDS / 4; i += kReplayThreads) ((uint4*)s_dbm)[i] = msrc[i];
        }
    }
    __syncthreads();
    const uint32_t* dd = DB_SMEM ? s_db : desc + d_row0 * WORDS;
    const uint32_t* dm = MASKED ? (DB_SMEM ? s_dbm : dmask + d_row0 * WORDS) : nullptr;
    const int nm = replay_core<WORDS, MASKED, kReplayThreads>(list_idx + q_row0 * K, list_dist + q_row0 * K, K, nq, nullptr, desc + q_row0 * WORDS,
                                                              MASKED ? dmask + q_row0 * WORDS : nullptr, dd, dm, nd, th_low, nnratio,
                                                              matches12 + q_row0, s_li, s_ld, s_taken, &sh, s_qc);
    if (tid == 0) { nmatches[img] = nm; redo[img] = 0; }
}

template <int WORDS, bool MASKED>
__global__ void __launch_bounds__(kReplayThreads)
stream_replay_kernel(const int* __restrict__ list_idx, const int* __restrict__ list_dist, const int* __restrict__ counts,
                     const uint32_t* __restrict__ desc, const uint32_t* __restrict__ dmask,
                     const int n_cams, const int capacity, const int K, const int img_lo, const int th_low, const double nnratio,
                     int* __restrict__ matches12, int* __restrict__ nmatches, int* __restrict__ redo) {
    extern __shared__ int s_mem[];
    stream_replay<WORDS, MASKED, false>(list_idx, list_dist, counts, desc, dmask, n_cams, capacity, K, img_lo, th_low, nnratio, matches12,
                                        nmatches, redo, s_mem);
}

// The same walk with the previous image's descriptors (and masks) RESIDENT IN SHARED MEMORY: a rescan then reads its 8 x 64 bytes
// per thread from shared memory instead of L2, a fraction of the latency, at the price of one CTA per SM (capacity x 2 x dim
// bytes, 129 KB for 2016 slots of mdBRIEF-256).  Used when the launch holds no more images than the device has SMs -- a chunk of the
// host-facing stream pipeline, whose last acceptance launch is the un-overlapped tail of the call; a full 384-image step keeps the
// kernel above (2.6 CTAs per SM in flight hide each other's latency, and the extraction kernels of the next step share the SMs).
// (256 threads as in the kernel above; 1024 -- more warps of its own for the CTA that is alone on its SM -- was no better)
template <int WORDS, bool MASKED>
__global__ void __launch_bounds__(kReplayThreads, 1)
stream_replay_smem_kernel(const int* __restrict__ list_idx, const int* __restrict__ list_dist, const int* __restrict__ counts,
                          const uint32_t* __restrict__ desc, const uint32_t* __restrict__ dmask,
                          const int n_cams, const int capacity, const int K, const int img_lo, const int th_low, const double nnratio,
                          int* __restrict__ matches12, int* __restrict__ nmatches, int* __restrict__ redo) {
    extern __shared__ __align__(16) int s_mem[];
    stream_replay<WORDS, MASKED, true>(list_idx, list_dist, counts, desc, dmask, n_cams, capacity, K, img_lo, th_low, nnratio, matches12,
                                       nmatches, redo, s_mem);
}

cudaError_t launch_stream_replay(const int* list_idx, const int* list_dist, const int* counts, const uint8_t* desc, const uint8_t* dmask,
                                 int dim, int img_lo, int n_images, int n_cams, int capacity, int K, int th_low, double nnratio,
                                 int* matches12, int* nmatches, int* redo, cudaStream_t st) {
    if (n_images < 1) return cudaSuccess;
    if (capacity > 65535 || !desc_width_ok(dim)) return cudaErrorInvalidValue;
    const size_t smem = (size_t)64 * K * 4 + (size_t)((capacity + 31) / 32) * 4;
    const bool masked = dmask != nullptr;
    int sms = 0;
    cudaError_t e = sm_count(sms);
    if (e != cudaSuccess) return e;
    // one wave of images: the database of every image fits beside its walk (see stream_replay_smem_kernel)
    const size_t smem_db = smem + (size_t)capacity * dim * (masked ? 2 : 1) + 16;
    const bool db_smem = n_images <= sms && smem_db <= kReplaySmemMax;
    with_desc_width(dim, masked, [&](auto W, auto M) {
        auto* kern = db_smem ? stream_replay_smem_kernel<W, M> : stream_replay_kernel<W, M>;
        if (db_smem) e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_db);   // per device, set every time
        if (e == cudaSuccess)
            kern<<<n_images, kReplayThreads, db_smem ? smem_db : smem, st>>>(list_idx, list_dist, counts, (const uint32_t*)desc,
                                                                             (const uint32_t*)dmask, n_cams, capacity, K, img_lo, th_low,
                                                                             nnratio, matches12, nmatches, redo);
    });
    return e != cudaSuccess ? e : cudaGetLastError();
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
    const int nm = replay_core<WORDS, MASKED, kBfReplayThreads>(list_idx + (size_t)q0 * K, list_dist + (size_t)q0 * K, K, nq, valid1 ? valid1 + q0 : nullptr,
                                                                q + (size_t)q0 * WORDS, MASKED ? qm + (size_t)q0 * WORDS : nullptr, d, dm, nd, th_low,
                                                                nnratio, matches12 + q0, s_li, s_ld, s_taken, &sh, s_qc, cl);
    if (tid == 0) nmatches[s] = nm;
}

cudaError_t launch_bruteforce_replay(const int* list_idx, const int* list_dist, int K, const uint8_t* q, const uint8_t* qm, const uint8_t* valid1,
                                     const int* seg, int n_seg, int nq_total, const uint8_t* d, const uint8_t* dm, const uint8_t* valid2, int nd, int dim,
                                     int th_low, double nnratio, int* matches12, int* nmatches, cudaStream_t st) {
    if (n_seg < 1) return cudaSuccess;
    if (nd >= (1 << kKeyShift) || !desc_width_ok(dim)) return cudaErrorInvalidValue;
    const size_t smem = bruteforce_replay_smem(K, nd);
    if (smem > kReplaySmemMax) return cudaErrorInvalidValue;
    const bool masked = qm && dm;
    int dev = 0, sms = 0, coop_ok = 0;
    cudaError_t e = sm_count(sms);
    if (e == cudaSuccess) e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&coop_ok, cudaDevAttrCooperativeLaunch, dev);
    if (e != cudaSuccess) return e;
    const void* fn = nullptr;
    with_desc_width(dim, masked, [&](auto W, auto M) { fn = (const void*)bruteforce_replay_kernel<W, M>; });
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
    StreamScratch sc;
    CoopSeg* cseg = nullptr; int* clog = nullptr;
    if (helpers) {
        e = sc.alloc({sizeof(CoopSeg) * n_seg, sizeof(int) * (size_t)std::max(nq_total, 1)}, st);
        if (e != cudaSuccess) return e;
        cseg = sc.at<CoopSeg>(0); clog = sc.at<int>(1);
        e = cudaMemsetAsync(cseg, 0, sizeof(CoopSeg) * n_seg, st);
        if (e != cudaSuccess) return sc.release(e);
    }
    const uint32_t *q32 = (const uint32_t*)q, *qm32 = (const uint32_t*)qm, *d32 = (const uint32_t*)d, *dm32 = (const uint32_t*)dm;
    void* args[] = {(void*)&list_idx, (void*)&list_dist, (void*)&K, (void*)&q32, (void*)&qm32, (void*)&valid1, (void*)&seg, (void*)&d32, (void*)&dm32,
                    (void*)&valid2, (void*)&nd, (void*)&th_low, (void*)&nnratio, (void*)&matches12, (void*)&nmatches, (void*)&cseg, (void*)&clog,
                    (void*)&helpers};
    const dim3 grid(n_seg * (helpers + 1)), block(kBfReplayThreads);
    if (helpers) e = cudaLaunchCooperativeKernel(fn, grid, block, args, smem, st);       // co-residency guaranteed or the launch fails
    else e = cudaLaunchKernel(fn, grid, block, args, smem, st);
    return sc.release(e != cudaSuccess ? e : cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------
// SearchByBoW(KF1, KF_k) for n_kf candidates (ref src/cORBmatcher.cpp:885-966, mcs_search_by_bow_keyframes_device)
// ------------------------------------------------------------------------------------------------
// Frame 0 is KF1, frame 1 + k candidate k, NS = n_cams * capacity slots each.  The number of valid slots is known only on the
// device, so every grid is sized from NS and the kernels read the real counts (nvalid) there.
//   kk_gather_kernel  one CTA per frame: the valid slots (below the camera's count, map-point id >= 0 and not bad) in slot order,
//                     compacted into descriptor / mask rows [f][NS] with their slots (c2s) and the number of them (nvalid[f]).
//   seg_lists_kernel<KfSegs>  the K-best lists of every (candidate, KF1 query) pair on the binary tensor cores (bmma_klists), one
//                     CTA per (candidate, 128 queries, database chunk); topk_merge_kernel merges the chunks' partial lists.
//   kk_replay_kernel  one CTA per candidate: the reference's ordered walk (replay_core) with the candidate's own "taken" bits, then
//                     compact indices back to slots and map-point ids.
// Compaction keeps slot order, so a compact index is the reference's contiguous order among the valid keypoints: ties broken by
// index in the lists and the rescans are the reference's strict `<` scan order.
// FREE_ROWS selects the rows of SearchForTriangulationRaw instead (tr_* below): the slots whose map-point id is -1, each row with
// its bearing ray ([f][NS][3], cam_img_to_world of the keypoint, models [n_cams]), and each camera's first row (seg [f][n_cams + 1],
// the last entry = nvalid[f]); n_points, bad and status are then unused.
template <bool FREE_ROWS>
__global__ void __launch_bounds__(1024)
kk_gather_kernel(const PsCamSlots* __restrict__ cams, const int* const* __restrict__ mp, const int n_cams, const int capacity, const int dim,
                 const bool masked, const int n_points, const uint8_t* __restrict__ bad, uint8_t* __restrict__ desc, uint8_t* __restrict__ dmask,
                 int* __restrict__ c2s, int* __restrict__ nvalid, int* __restrict__ status, const mcs_ocam* __restrict__ models,
                 double* __restrict__ rays, int* __restrict__ seg) {
    __shared__ int s_warp[32];
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int NS = n_cams * capacity, n16 = dim / 16;
    const PsCamSlots* fc = cams + (size_t)f * n_cams;
    const int* m = mp[f];
    const size_t row0 = (size_t)f * NS;
    int base = 0;
    for (int s0 = 0; s0 < NS; s0 += 1024) {
        const int s = s0 + tid, c = s / capacity, j = s - c * capacity;
        bool ok = false;
        if (s < NS && j < min(*fc[c].count, capacity)) {
            const int id = m[s];
            if constexpr (FREE_ROWS) ok = id == -1;
            else if (id >= n_points) *status = MCS_ERR_INVALID;            // dropped; the other slots are unaffected
            else ok = id >= 0 && !(bad && bad[id]);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, ok);
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < 32; ++w) { const int v = s_warp[w]; before += w < warp ? v : 0; total += v; }
        if constexpr (FREE_ROWS) {
            if (s < NS && j == 0) seg[(size_t)f * (n_cams + 1) + c] = base + before + __popc(bal & ((1u << lane) - 1u));
        }
        if (ok) {
            const size_t r = row0 + base + before + __popc(bal & ((1u << lane) - 1u));
            c2s[r] = s;
            const uint4* src = reinterpret_cast<const uint4*>(fc[c].desc + (size_t)j * dim);
            for (int h = 0; h < n16; ++h) reinterpret_cast<uint4*>(desc + r * dim)[h] = src[h];
            if (masked) {
                const uint4* msrc = reinterpret_cast<const uint4*>(fc[c].dmask + (size_t)j * dim);
                for (int h = 0; h < n16; ++h) reinterpret_cast<uint4*>(dmask + r * dim)[h] = msrc[h];
            }
            if constexpr (FREE_ROWS) {                                 // mvKeysRays (ref src/cMultiFrame.cpp:145-151)
                const mcs_keypoint k = fc[c].kps[j];
                double x, y, z;
                cam_img_to_world(models[c], (double)k.x, (double)k.y, x, y, z);
                rays[3 * r] = x; rays[3 * r + 1] = y; rays[3 * r + 2] = z;
            }
        }
        base += total;
        __syncthreads();                                               // s_warp is rewritten by the next chunk
    }
    if (tid == 0) {
        nvalid[f] = base;
        if constexpr (FREE_ROWS) seg[(size_t)f * (n_cams + 1) + n_cams] = base;
    }
}

// The rows segment g of a segmented list kernel reads and writes: queries q_row .. q_row + nq - 1 and database entries
// d_row .. d_row + nd - 1 of the gathered descriptors, partial-list rows o_row .. o_row + n_out - 1 (n_out >= nq): rows past nq
// get empty lists.  Row numbers fit an int: the entry points keep every search's gathered rows below 2^31.
struct SegRows { int q_row, nq, d_row, nd, o_row, n_out; };

// CTA x = (segment g, query block), y = database chunk; part [chunks][part_rows][kTopKMax].  Seg maps g to its SegRows on the device.
// Every chunk's CTA of a block writes the block's rows below n_out, as empty lists where it has no query or no database entry, so that
// the merge reads defined keys for every such row.  Distances are listed below `bound`, clamped to the keys' 11-bit distance field.
template <class Seg, int WORDS, bool MASKED>
__global__ void __launch_bounds__(kTopkThreads, kListMinBlocks<WORDS, MASKED>)
seg_lists_kernel(const uint32_t* __restrict__ desc, const uint32_t* __restrict__ dmask, const Seg seg, const int qblocks,
                 const size_t part_rows, const int chunk, const unsigned bound, unsigned* __restrict__ part) {
    __shared__ __align__(16) BmmaTile<WORDS, MASKED> s;
    const int g = blockIdx.x / qblocks, qb = (blockIdx.x - g * qblocks) * kTopkThreads;
    const SegRows r = seg(g);
    if (qb >= r.n_out) return;
    const int j0 = blockIdx.y * chunk, j1 = min(j0 + chunk, r.nd);
    unsigned* o = part + (blockIdx.y * part_rows + (size_t)r.o_row + qb) * kTopKMax;
    if (qb >= r.nq || j0 >= j1) {
        for (int i = threadIdx.x; i < min(kTopkThreads, r.n_out - qb) * kTopKMax; i += kTopkThreads) o[i] = 0xFFFFFFFFu;
        return;
    }
    const size_t q_row = (size_t)r.q_row + qb, d_row = r.d_row;
    bmma_klists<WORDS, MASKED, kTopKMax, kTopkShift>(desc + q_row * WORDS, MASKED ? dmask + q_row * WORDS : nullptr, r.nq - qb,
                                                     desc + d_row * WORDS, MASKED ? dmask + d_row * WORDS : nullptr, nullptr, j0, j1,
                                                     kTopKMax, min(bound, 0x7FFu), s, [=](int row, int kk, unsigned key) {
        if (qb + row < r.n_out) o[(size_t)row * kTopKMax + kk] = key;
    });
}

// SearchByBoW(KF1, KF_k): segment k lists frame 0's valid rows against frame 1 + k's (counts nvalid), into rows k * NS .. of part;
// every one of the NS rows is written.
struct KfSegs {
    const int* nvalid; int NS;
    __device__ SegRows operator()(const int k) const {
        return {0, nvalid[0], (1 + k) * NS, nvalid[1 + k], k * NS, NS};
    }
};

// Threads of the acceptance CTA: 512 leaves 128 registers per thread, where replay_core at 1024 spills with 64 (the masked
// 32- and 64-byte instances); a rescan of a key frame's few thousand valid slots is still a handful of entries per thread.
constexpr int kKfReplayThreads = 512;

// One CTA per candidate k: its ordered walk over the merged lists [n_kf][NS][kTopKMax] into m12c (compact database indices), then the
// outputs: -1 for every KF1 slot below its camera's count, the candidate's map-point id and slot for the accepted ones.
template <int WORDS, bool MASKED>
__global__ void __launch_bounds__(kKfReplayThreads, 1)
kk_replay_kernel(const int* __restrict__ list_idx, const int* __restrict__ list_dist, const uint32_t* __restrict__ desc,
                 const uint32_t* __restrict__ dmask, const int* __restrict__ nvalid, const int* __restrict__ c2s,
                 const PsCamSlots* __restrict__ kf1, const int* const* __restrict__ mp, const int n_cams, const int capacity,
                 const int th_low, const double nnratio, int* __restrict__ m12c, int* __restrict__ matches12, int* __restrict__ match_slot,
                 int* __restrict__ nmatches) {
    constexpr int K = kTopKMax;
    extern __shared__ int s_mem[];
    int* s_li = s_mem;
    int* s_ld = s_mem + 32 * K;
    unsigned* s_taken = (unsigned*)(s_mem + 64 * K);
    __shared__ ReplayShared sh;
    __shared__ __align__(16) uint32_t s_qc[(MASKED ? 2 : 1) * 32 * WORDS];
    const int k = blockIdx.x, tid = threadIdx.x, NS = n_cams * capacity;
    const int nq = nvalid[0], nd = nvalid[1 + k];
    const size_t o0 = (size_t)k * NS, d_row0 = (size_t)(1 + k) * NS;
    for (int w = tid; w < (nd + 31) / 32; w += kKfReplayThreads) s_taken[w] = 0u;
    for (int i = tid; i < nq; i += kKfReplayThreads) m12c[o0 + i] = -1;
    __syncthreads();
    const int nm = replay_core<WORDS, MASKED, kKfReplayThreads>(list_idx + o0 * K, list_dist + o0 * K, K, nq, nullptr, desc,
                                                                MASKED ? dmask : nullptr, desc + d_row0 * WORDS,
                                                                MASKED ? dmask + d_row0 * WORDS : nullptr, nd, th_low, nnratio, m12c + o0,
                                                                s_li, s_ld, s_taken, &sh, s_qc);
    if (tid == 0) nmatches[k] = nm;
    for (int s = tid; s < NS; s += kKfReplayThreads) {
        const int c = s / capacity;
        if (s - c * capacity < min(*kf1[c].count, capacity)) {
            matches12[o0 + s] = -1;
            if (match_slot) match_slot[o0 + s] = -1;
        }
    }
    __syncthreads();
    const int* mpk = mp[1 + k];
    for (int q = tid; q < nq; q += kKfReplayThreads) {
        const int b = m12c[o0 + q];
        if (b < 0) continue;
        const int s1 = c2s[q], s2 = c2s[d_row0 + b];
        matches12[o0 + s1] = mpk[s2];
        if (match_slot) match_slot[o0 + s1] = s2;
    }
}

cudaError_t launch_search_by_bow_keyframes(const BowKfSearchDevArgs& a, cudaStream_t st) {
    constexpr int K = kTopKMax;
    const int n_fr = a.n_kf + 1, NS = a.n_cams * a.capacity, n_rows = a.n_kf * NS;
    int sms = 0;
    cudaError_t e = sm_count(sms);
    if (e != cudaSuccess) return e;
    // chunks of the database from the upper bound NS on every frame's valid slots
    const int qblocks = (NS + kTopkThreads - 1) / kTopkThreads;
    const long long cta_q = (long long)qblocks * a.n_kf;
    const ListPlan pl = list_plan(sms, cta_q, NS);
    const size_t rows = (size_t)n_fr * NS, lists = (size_t)n_rows * K;
    StreamScratch sc;
    const PsCamSlots* cams;
    const int* const* mp;
    e = open_scratch(sc, {rows * a.dim, a.masked ? rows * a.dim : 0, rows * 4, (size_t)n_fr * 4, (size_t)pl.splits * lists * 4, lists * 4,
                          lists * 4, (size_t)n_rows * 4}, st, host_in(cams, a.cams, (size_t)a.n_cams * n_fr), host_in(mp, a.mp, n_fr));
    if (e != cudaSuccess) return sc.release(e);
    uint8_t* desc = sc.at<uint8_t>(0); uint8_t* dmask = a.masked ? sc.at<uint8_t>(1) : nullptr;
    int* c2s = sc.at<int>(2); int* nvalid = sc.at<int>(3);
    unsigned* part = sc.at<unsigned>(4); int* lidx = sc.at<int>(5); int* ldist = sc.at<int>(6); int* m12c = sc.at<int>(7);
    e = cudaMemsetAsync(a.status, 0, sizeof(int), st);                                      // MCS_OK
    if (e != cudaSuccess) return sc.release(e);
    kk_gather_kernel<false><<<n_fr, 1024, 0, st>>>(cams, mp, a.n_cams, a.capacity, a.dim, a.masked, a.n_points, a.bad, desc, dmask, c2s,
                                                   nvalid, a.status, nullptr, nullptr, nullptr);
    const size_t smem = bruteforce_replay_smem(K, NS);
    with_desc_width(a.dim, a.masked, [&](auto W, auto M) {
        const uint32_t *d32 = (const uint32_t*)desc, *m32 = (const uint32_t*)dmask;
        seg_lists_kernel<KfSegs, W, M><<<dim3((unsigned)cta_q, pl.splits), kTopkThreads, 0, st>>>(
            d32, m32, KfSegs{nvalid, NS}, qblocks, (size_t)n_rows, pl.chunk, greedy_dist_bound(a.th_low, a.nnratio), part);
        topk_merge_kernel<<<(n_rows + 127) / 128, 128, 0, st>>>(part, pl.splits, n_rows, K, lidx, ldist);
        auto* kern = kk_replay_kernel<W, M>;
        if (smem > 48 * 1024) e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess)
            kern<<<a.n_kf, kKfReplayThreads, smem, st>>>(lidx, ldist, d32, m32, nvalid, c2s, cams, mp, a.n_cams, a.capacity, a.th_low, a.nnratio,
                                                         m12c, a.matches12, a.match_slot, a.nmatches);
    });
    return sc.release(e != cudaSuccess ? e : cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------
// SearchForTriangulationRaw(KF1, KF2) (ref src/cORBmatcher.cpp:968-1107, mcs_search_for_triangulation_device)
// ------------------------------------------------------------------------------------------------
// Frame 0 is KF1, frame 1 KF2, NS = n_cams * capacity slots each.  A query only sees the keypoints of its own camera, so past the
// gather everything runs on camera segments: seg[f][c] .. seg[f][c + 1] are camera c's rows of frame f, and a database index is
// relative to its segment (< capacity <= 65535, inside the lists' and the rescans' 21-bit index).
//   kk_gather_kernel<true>  one CTA per frame: the free slots (map-point id -1) in slot order, their rays and the segments.
//   seg_lists_kernel<CamSegs>  the K-best (distance, index) lists, distance <= th_low, of every KF1 row against the KF2 rows of
//                           its camera (bmma_klists), one CTA per (camera, 128 queries, database chunk); topk_merge_kernel merges.
//   tr_epi_kernel           CheckDistEpipolarLine of every list entry, one thread per (row, entry).
//   tr_walk_kernel          one CTA per camera: the reference's ordered walk over the camera's queries with the camera's "taken"
//                           bits, then the KF2 slot of each match into matches12.
// The reference walks a query's candidates (distance <= th_low, not taken) in (distance, index) order while distance <= 2 * best
// and takes the first that passes the epipolar test: the winner is the smallest (distance, index) candidate that passes, accepted
// iff its distance <= 2 * best.  From a list made before any query took anything: best = its first open (untaken) entry, since every
// entry before it is taken and every key after it or not listed is larger; the winner = its first open entry that passes.  Without
// one, a list with a -1 entry holds every candidate, so there is none; a full list bounds every key not listed by its last
// distance dK, so there is none within 2 * best when dK > 2 * best.  Otherwise (a full list with no open entry, or with no open
// entry that passes and dK <= 2 * best) the query is undecided from its list, and the whole CTA rescans the camera's segment.
// Compaction keeps slot order, so (distance, index) order inside a camera is the reference's (distance, contiguous index) order.
constexpr int kTrWalkThreads = 256;          // a camera segment is <= 65535 rows: a rescan is <= 293 rows per scanning thread

struct TriWalkShared {
    int cmd;                                  // 0 while the walk runs, -1 once it is over
    int bq;                                   // the rescan's chunk-relative query
    unsigned k1[kTrWalkThreads / 32], k2[kTrWalkThreads / 32];     // per scanning warp (1 ..): smallest open key, smallest that passes
};

// Camera segment c lists KF1's rows of camera c against KF2's, into the same rows of part [chunks][NS][kTopKMax]; the rows past
// its queries are the next camera's, so n_out = nq.
struct CamSegs {
    const int* seg; int n_cams, NS;
    __device__ SegRows operator()(const int c) const {
        const int q_lo = seg[c], nq = seg[c + 1] - q_lo, d_lo = seg[n_cams + 1 + c];
        return {q_lo, nq, NS + d_lo, seg[n_cams + 2 + c] - d_lo, q_lo, nq};
    }
};

// flag [NS][kTopKMax]: CheckDistEpipolarLine(ray1, ray2, E[c][c], epi) of KF1 row `row` and its list entry (0 for an empty entry)
__global__ void tr_epi_kernel(const int* __restrict__ list_idx, const double* __restrict__ rays, const int* __restrict__ seg,
                              const int* __restrict__ c2s, const int* __restrict__ nvalid, const double* __restrict__ E, const int n_cams,
                              const int capacity, const double epi, uint8_t* __restrict__ flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, row = i / kTopKMax, NS = n_cams * capacity;
    if (row >= nvalid[0]) return;
    const int id = list_idx[i];
    if (id < 0) { flag[i] = 0; return; }
    const int c = c2s[row] / capacity;
    flag[i] = cam_epipolar_ok(rays + (size_t)row * 3, rays + ((size_t)NS + seg[n_cams + 1 + c] + id) * 3, E + 9 * c, epi) ? 1 : 0;
}

// One pass over this thread's share of the camera's database rows [0, nd) (dd / dm / r2 start at the segment; the scanning warps
// are warps 1 .. of the CTA) for the query descriptor qd (qm) and ray r1: the smallest key (distance << kKeyShift | index) over the
// rows not taken with distance <= th_low (k1), and over those that also pass the epipolar test (k2), each reduced over the warp.
// The test runs only for a key below k2.
template <int WORDS, bool MASKED>
__device__ __forceinline__ void tr_scan(const uint32_t* qd, const uint32_t* qmk, const double* r1, const uint32_t* __restrict__ dd,
                                        const uint32_t* __restrict__ dm, const double* __restrict__ r2, const int nd, const unsigned* s_taken,
                                        const double* E, const double epi, const int th_low, unsigned& k1, unsigned& k2) {
    uint32_t qw[WORDS], qm[MASKED ? WORDS : 1];
#pragma unroll
    for (int k = 0; k < WORDS; ++k) { qw[k] = qd[k]; if (MASKED) qm[k] = qmk[k]; }
    const double ray1[3] = {r1[0], r1[1], r1[2]};
    k1 = 0xFFFFFFFFu; k2 = 0xFFFFFFFFu;
    for (int id = threadIdx.x - 32; id < nd; id += kTrWalkThreads - 32) {
        if (s_taken[id >> 5] >> (id & 31) & 1u) continue;
        const uint4* dp = reinterpret_cast<const uint4*>(dd + (size_t)id * WORDS);
        const uint4* mp = MASKED ? reinterpret_cast<const uint4*>(dm + (size_t)id * WORDS) : nullptr;
        uint32_t dw[WORDS], mw[MASKED ? WORDS : 1];
#pragma unroll
        for (int k = 0; k < WORDS / 4; ++k) {
            const uint4 t = dp[k]; dw[4 * k] = t.x; dw[4 * k + 1] = t.y; dw[4 * k + 2] = t.z; dw[4 * k + 3] = t.w;
            if (MASKED) { const uint4 u = mp[k]; mw[4 * k] = u.x; mw[4 * k + 1] = u.y; mw[4 * k + 2] = u.z; mw[4 * k + 3] = u.w; }
        }
        const unsigned dist = hamming_words<WORDS, MASKED>(qw, qm, dw, mw);
        if ((int)dist > th_low) continue;
        const unsigned key = (dist << kKeyShift) | (unsigned)id;
        k1 = min(k1, key);
        if (key < k2 && cam_epipolar_ok(ray1, r2 + 3 * (size_t)id, E, epi)) k2 = key;
    }
    k1 = __reduce_min_sync(0xffffffffu, k1);
    k2 = __reduce_min_sync(0xffffffffu, k2);
}

// One CTA per camera c.  Warp 0 walks the camera's queries in order and decides from the lists with the whole warp (lane k holds
// entry k; ballots give the open and the open passing entries); the other warps sleep on a named barrier and wake only for a
// rescan, which they alone run: the walk then holds no call of the double division's slow path, whose calling convention would
// make ptxas spill the walk's state.  Every KF1 slot of the camera below its count gets -1 or the KF2 slot it matched.
template <int WORDS, bool MASKED>
__global__ void __launch_bounds__(kTrWalkThreads)
tr_walk_kernel(const int* __restrict__ list_idx, const int* __restrict__ list_dist, const uint8_t* __restrict__ list_epi,
               const uint32_t* __restrict__ desc, const uint32_t* __restrict__ dmask, const double* __restrict__ rays,
               const int* __restrict__ seg, const int* __restrict__ c2s, const PsCamSlots* __restrict__ kf1, const double* __restrict__ E,
               const int n_cams, const int capacity, const int th_low, const double epi, int* __restrict__ matches12,
               int* __restrict__ nmatches, int* __restrict__ diag) {
    constexpr int K = kTopKMax, THREADS = kTrWalkThreads;
    extern __shared__ unsigned s_taken[];                              // [(capacity + 31) / 32]: bit = segment index of KF2
    __shared__ int s_li[32 * K], s_ld[32 * K];
    __shared__ uint8_t s_fl[32 * K];
    __shared__ __align__(16) uint32_t s_qc[(MASKED ? 2 : 1) * 32 * WORDS];   // the chunk's query descriptors (and masks)
    __shared__ double s_qr[32 * 3], s_E[9];
    __shared__ TriWalkShared sh;
    const int c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, NS = n_cams * capacity;
    const int q_lo = seg[c], nq = seg[c + 1] - q_lo, d_lo = seg[n_cams + 1 + c], nd = seg[n_cams + 2 + c] - d_lo;
    const int n1 = min(*kf1[c].count, capacity);
    for (int j = tid; j < n1; j += THREADS) matches12[(size_t)c * capacity + j] = -1;
    for (int w = tid; w < (nd + 31) / 32; w += THREADS) s_taken[w] = 0u;
    if (tid < 9) s_E[tid] = E[9 * c + tid];
    __syncthreads();
    const uint32_t* dd = desc + ((size_t)NS + d_lo) * WORDS;
    const uint32_t* dm = MASKED ? dmask + ((size_t)NS + d_lo) * WORDS : nullptr;
    const double* r2 = rays + ((size_t)NS + d_lo) * 3;
    const uint32_t* s_qm = s_qc + (MASKED ? 32 * WORDS : 0);
    if (warp != 0) {
        for (;;) {
            named_bar<THREADS>(1);
            if (*(volatile int*)&sh.cmd < 0) return;
            const int b = sh.bq;
            unsigned k1, k2;
            tr_scan<WORDS, MASKED>(s_qc + b * WORDS, s_qm + b * WORDS, s_qr + 3 * b, dd, dm, r2, nd, s_taken, s_E, epi, th_low, k1, k2);
            if (lane == 0) { sh.k1[warp] = k1; sh.k2[warp] = k2; }
            named_bar<THREADS>(2);
        }
    }
    int nm = 0, rescans = 0;
    if (lane == 0) sh.cmd = 0;
    const unsigned kmask = (1u << K) - 1u;
    for (int q0 = 0; q0 < nq; q0 += 32) {
        const int nchunk = min(32, nq - q0);
        const size_t r0 = (size_t)q_lo + q0;
        for (int i = lane; i < nchunk * K; i += 32) {
            s_li[i] = list_idx[r0 * K + i];
            s_ld[i] = list_dist[r0 * K + i];
            s_fl[i] = list_epi[r0 * K + i];
        }
        for (int i = lane; i < nchunk * (WORDS / 4); i += 32) {
            reinterpret_cast<uint4*>(s_qc)[i] = reinterpret_cast<const uint4*>(desc + r0 * WORDS)[i];
            if (MASKED) reinterpret_cast<uint4*>(s_qc + 32 * WORDS)[i] = reinterpret_cast<const uint4*>(dmask + r0 * WORDS)[i];
        }
        for (int i = lane; i < nchunk * 3; i += 32) s_qr[i] = rays[r0 * 3 + i];
        __syncwarp();
        for (int t = 0; t < nchunk; ++t) {
            //   code 0 no match, 1 match `win`, 2 undecided from the list
            int code, win;
            {
                const int id = lane < K ? s_li[t * K + lane] : -1;
                const int dl = lane < K ? s_ld[t * K + lane] : 0x7FFFFFFF;
                const bool open = id >= 0 && !(s_taken[id >> 5] >> (id & 31) & 1u);
                const unsigned m_valid = __ballot_sync(0xffffffffu, id >= 0);
                const unsigned m_open = __ballot_sync(0xffffffffu, open);
                const unsigned m_pass = __ballot_sync(0xffffffffu, open && s_fl[t * K + lane] != 0);
                const int best = __shfl_sync(0xffffffffu, dl, m_open ? __ffs(m_open) - 1 : 0);
                const int wl = m_pass ? __ffs(m_pass) - 1 : 0;
                const int wd = __shfl_sync(0xffffffffu, dl, wl), dK = __shfl_sync(0xffffffffu, dl, K - 1);
                win = __shfl_sync(0xffffffffu, id, wl);
                if (m_pass) code = wd <= 2 * best ? 1 : 0;
                else if (m_valid != kmask) code = 0;                   // the list holds every candidate
                else if (!m_open) code = 2;
                else code = dK <= 2 * best ? 2 : 0;
            }
            if (code == 2) {
                // exact rescan of the camera's database: the smallest open key, and the smallest open key that passes
                if (lane == 0) sh.bq = t;
                named_bar<THREADS>(1);
                named_bar<THREADS>(2);
                const bool w = lane >= 1 && lane < THREADS / 32;
                const unsigned B = __reduce_min_sync(0xffffffffu, w ? sh.k1[lane] : 0xFFFFFFFFu);
                const unsigned W = __reduce_min_sync(0xffffffffu, w ? sh.k2[lane] : 0xFFFFFFFFu);
                code = W != 0xFFFFFFFFu && (W >> kKeyShift) <= 2 * (B >> kKeyShift) ? 1 : 0;
                win = (int)(W & ((1u << kKeyShift) - 1u));
                ++rescans;
            }
            if (code == 1) {
                if (lane == 0) {
                    matches12[c2s[r0 + t]] = c2s[(size_t)NS + d_lo + win];
                    s_taken[win >> 5] |= 1u << (win & 31);
                }
                ++nm;
            }
            __syncwarp();
        }
    }
    if (lane == 0) sh.cmd = -1;
    named_bar<THREADS>(1);
    if (lane == 0) {
        atomicAdd(nmatches, nm);
        if (diag) { atomicAdd(diag, nq); atomicAdd(diag + 1, rescans); }
    }
}

cudaError_t launch_search_for_triangulation(const TriSearchDevArgs& a, cudaStream_t st) {
    constexpr int K = kTopKMax;
    const int nc = a.n_cams, NS = nc * a.capacity;
    int sms = 0;
    cudaError_t e = sm_count(sms);
    if (e != cudaSuccess) return e;
    // chunks of a camera's database from the upper bound `capacity` on its free rows
    const int qblocks = (a.capacity + kTopkThreads - 1) / kTopkThreads;
    const long long cta_q = (long long)qblocks * nc;
    const ListPlan pl = list_plan(sms, cta_q, a.capacity);
    const size_t rows = (size_t)2 * NS, lists = (size_t)NS * K;
    StreamScratch sc;
    const PsCamSlots* cams;
    const int* const* mp;
    const mcs_ocam* models;
    const double* E;
    e = open_scratch(sc, {rows * a.dim, a.masked ? rows * a.dim : 0, rows * 4, 2 * 4, (size_t)2 * (nc + 1) * 4, rows * 24,
                          (size_t)pl.splits * lists * 4, lists * 4, lists * 4, lists},
                     st, host_in(cams, a.cams, 2 * (size_t)nc), host_in(mp, a.mp, 2), host_in(models, a.models, nc), host_in(E, a.E, 9 * (size_t)nc));
    if (e != cudaSuccess) return sc.release(e);
    uint8_t* desc = sc.at<uint8_t>(0); uint8_t* dmask = a.masked ? sc.at<uint8_t>(1) : nullptr;
    int* c2s = sc.at<int>(2); int* nvalid = sc.at<int>(3); int* seg = sc.at<int>(4); double* rays = sc.at<double>(5);
    unsigned* part = sc.at<unsigned>(6); int* lidx = sc.at<int>(7); int* ldist = sc.at<int>(8); uint8_t* flag = sc.at<uint8_t>(9);
    e = cudaMemsetAsync(a.nmatches, 0, sizeof(int), st);
    if (e == cudaSuccess && a.diag) e = cudaMemsetAsync(a.diag, 0, 2 * sizeof(int), st);
    if (e != cudaSuccess) return sc.release(e);
    kk_gather_kernel<true><<<2, 1024, 0, st>>>(cams, mp, nc, a.capacity, a.dim, a.masked, 0, nullptr, desc, dmask, c2s, nvalid, nullptr,
                                               models, rays, seg);
    // distances <= th_low are listed (bmma_klists lists those below its bound)
    const unsigned bound = a.th_low < 0 ? 0u : (unsigned)(a.th_low + 1LL);
    const size_t smem = (size_t)((a.capacity + 31) / 32) * 4;
    with_desc_width(a.dim, a.masked, [&](auto W, auto M) {
        const uint32_t *d32 = (const uint32_t*)desc, *m32 = (const uint32_t*)dmask;
        seg_lists_kernel<CamSegs, W, M><<<dim3((unsigned)cta_q, pl.splits), kTopkThreads, 0, st>>>(d32, m32, CamSegs{seg, nc, NS}, qblocks,
                                                                                                   (size_t)NS, pl.chunk, bound, part);
        topk_merge_kernel<<<(NS + 127) / 128, 128, 0, st>>>(part, pl.splits, NS, K, lidx, ldist);
        tr_epi_kernel<<<(unsigned)((lists + 255) / 256), 256, 0, st>>>(lidx, rays, seg, c2s, nvalid, E, nc, a.capacity, a.epi_thresh, flag);
        tr_walk_kernel<W, M><<<nc, kTrWalkThreads, smem, st>>>(lidx, ldist, flag, d32, m32, rays, seg, c2s, cams, E, nc, a.capacity, a.th_low,
                                                               a.epi_thresh, a.matches12, a.nmatches, a.diag);
    });
    return sc.release(cudaGetLastError());
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
    if (!desc_width_ok(f.dim)) return cudaErrorInvalidValue;
    const int blocks = (nq * 32 + 255) / 256;
    const bool masked = qmask && f.dmask;
    with_desc_width(f.dim, masked, [&](auto W, auto M) {
        window_search_kernel<W, M><<<blocks, 256, 0, st>>>(f, q, nq, (const uint32_t*)qdesc, (const uint32_t*)qmask, max_cand, cand_idx,
                                                           cand_dist, cand_count);
    });
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
                               double* __restrict__ vcos, const uint8_t* __restrict__ skip) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_points * n_cams) return;
    const int i = t / n_cams, c = t - i * n_cams;
    if (skip && skip[i]) return;                  // already matched / bad (ref src/cTracking.cpp:985-988): keeps its last entries
    in_view[t] = 0; level[t] = 0; px[t] = 0.0; py[t] = 0.0; vcos[t] = 0.0;
    const double P0 = pos[3 * i], P1 = pos[3 * i + 1], P2 = pos[3 * i + 2];
    const mcs_ocam cam = cams[c];
    double u, v;
    if (!cam_project_in_mask(mtmc_inv + 16 * c, cam, masks + (size_t)c * cam.width * cam.height, P0, P1, P2, u, v)) return;
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
                           int n_levels, uint8_t* in_view, int* level, double* px, double* py, double* vcos, const uint8_t* skip,
                           cudaStream_t st) {
    const long long n = (long long)n_points * n_cams;
    if (n <= 0) return cudaSuccess;
    frustum_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(n_cams, mtmc_inv, mtmc, cams, masks, n_points, pos, nrm, dmin, dmax, sf,
                                                                n_levels, in_view, level, px, py, vcos, skip);
    return cudaGetLastError();
}

}  // namespace mcs
