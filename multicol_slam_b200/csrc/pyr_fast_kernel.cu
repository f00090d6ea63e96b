// pyr_fast_kernel.cu -- K1: per pyramid level, ONE fused kernel
//     resize(level l-1 -> l)  +  5x5 box blur  +  FAST-9/16 score  +  per-cell 3x3 NMS  +  mirror-mask filter
// (ref src/mdBRIEFextractorOct.cpp:1158-1201 ComputePyramid, :863-949 cell loop, :1301 boxFilter; OpenCV
// resize / boxFilter / FAST arithmetic restated in SURVEY.md Appendix A.1 / A.3 / A.5).
//
// One CTA owns a 64x32 tile of level l.  The source region of level l-1 is staged in shared memory with 128-bit
// loads, the tile (+4 px ring, REFLECT_101 at the image border) is resized once and kept in three shared forms:
// bytes (for the stores) and two 16-bit-per-pixel copies offset by one pixel, so that ANY horizontally adjacent
// pixel pair is one aligned 32-bit word.  Blur and FAST then run on pixel PAIRS with the packed 16x2 integer
// SIMD of sm_90a (16x2 adds, DPX three-way min / max):
//   * box blur: 5 packed loads + 4 packed adds give the horizontal 5-sums of two pixels;
//   * FAST: E_k = ring_k - centre (packed), 9-arc minima / maxima by two 3-input min (max) levels
//     (M3_k = min3(E_k,E_k+1,E_k+2), M9_k = min3(M3_k,M3_k+3,M3_k+6)), branch-free exact cornerScore for every
//     pixel pair: score = max over arcs of max(min9(E), -max9(E)) - 1, corner iff that maximum exceeds the threshold.
// The kernel is bound by integer issue rate, not by HBM (DESIGN.md, K1): on the order of a hundred thread-instructions per
// pixel against a few bytes of DRAM traffic.
#include <cstring>
#include <cuda.h>
#include <cudaTypedefs.h>

#include "kernels.h"
#include "mcs_common.cuh"

namespace mcs {

// ---- TMA staging (cp.async.bulk.tensor + mbarrier) ---------------------------------------------------------------------------
// The source region of a tile is one box of a 3-D tensor map (x bytes, y rows, image) over the level l-1 buffer: a single thread
// issues the bulk copy, the hardware writes the box into shared memory (rows past the image are zero-filled) and signals an
// mbarrier, while the other threads fill the per-tile tables.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "MBAR_WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra MBAR_DONE_%=;\n"
        "bra MBAR_WAIT_%=;\n"
        "MBAR_DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(smem_u32(dst)), "l"((unsigned long long)map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)) : "memory");
}

#ifndef MCS_K1_MINB
#define MCS_K1_MINB 6                        // resident CTAs per SM the register budget is cut for (6 needs <= 40 registers)
#endif
#ifndef MCS_K1_TMA
#define MCS_K1_TMA 1                         // 0: stage the source region with __ldg + st.shared (A/B builds)
#endif
constexpr int kThreads = 256;
constexpr int kSrcWB = 176;                 // staged source row stride (bytes, multiple of 16)
constexpr int kT8S = 80;                    // byte tile row stride
constexpr int kT16S = 72;                   // 16-bit tile row stride (elements)
constexpr int kScoreS = 68;                 // score tile row stride in 16-bit elements (66 used)
constexpr int kWarpCorners = (kTH / (kThreads / 32)) * (kTW / 2);   // a warp owns kTH/8 rows; strict 3x3 maxima are never adjacent in a row

__device__ __forceinline__ unsigned vneg2(unsigned a) { return __vadd2(~a, 0x00010001u); }

// packed cornerScore<16> margin of a pixel pair: C = centre pair, R[k] = ring pairs -> max over the 16 arcs of
// max(min9(R-C), min9(C-R)) per 16-bit lane (signed).  min over an arc of (R_k - C) = (min over the arc of R_k) - C, so the
// arc minima / maxima are taken on the ring values themselves and the centre enters once at the end.
__device__ __forceinline__ unsigned fast_margin2(unsigned C, const unsigned (&E)[16]) {
    unsigned mn3[16], mx3[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        mn3[k] = __vimin3_s16x2(E[k], E[(k + 1) & 15], E[(k + 2) & 15]);
        mx3[k] = __vimax3_s16x2(E[k], E[(k + 1) & 15], E[(k + 2) & 15]);
    }
    unsigned mn9[16], mx9[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        mn9[k] = __vimin3_s16x2(mn3[k], mn3[(k + 3) & 15], mn3[(k + 6) & 15]);
        mx9[k] = __vimax3_s16x2(mx3[k], mx3[(k + 3) & 15], mx3[(k + 6) & 15]);
    }
    unsigned bright = __vimax3_s16x2(mn9[0], mn9[1], mn9[2]);
    unsigned darkn = __vimin3_s16x2(mx9[0], mx9[1], mx9[2]);
#pragma unroll
    for (int k = 3; k < 15; k += 2) {
        bright = __vimax3_s16x2(bright, mn9[k], mn9[k + 1]);
        darkn = __vimin3_s16x2(darkn, mx9[k], mx9[k + 1]);
    }
    bright = __vmaxs2(bright, mn9[15]);                     // max over arcs of the arc minimum of the ring
    darkn = __vmins2(darkn, mx9[15]);                       // min over arcs of the arc maximum
    return __vmaxs2(__vsub2(bright, C), __vsub2(C, darkn)); // values in 0..255: no 16-bit overflow
}

__global__ void __launch_bounds__(kThreads, MCS_K1_MINB)
pyr_fast_kernel(const __grid_constant__ CUtensorMap src_map, const int use_tma,
                const LevelGeom g, const int level, const int nlevels, const int fast_th, const int src_aligned,
                const uint8_t* __restrict__ src, const size_t src_img_bytes,
                uint8_t* __restrict__ dst, uint8_t* __restrict__ dst_blur,
                const uint8_t* __restrict__ mask0, const int mask_w, const size_t mask_bytes,
                const int* __restrict__ cam_of_image, const uint8_t* __restrict__ tile_flags, const int tiles_total,
                uint32_t* __restrict__ raw, const size_t raw_img_stride, int* __restrict__ raw_count) {
    __shared__ __align__(128) uint8_t s_src[kSrcH * kSrcWB];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ __align__(16) uint8_t s_t8[kTileH * kT8S];
    __shared__ __align__(16) uint16_t s_a0[kTileH * kT16S];          // s_a0[y][x]   = px(x)
    __shared__ __align__(16) uint16_t s_a1[kTileH * kT16S];          // s_a1[y][i]   = px(i+1)
    __shared__ __align__(16) uint32_t s_h[(kTH + 4) * (kTW / 2)];    // packed horizontal 5-sums of pixel pairs
    __shared__ uint32_t s_ml[kTW / 2], s_mr[kTW / 2], s_mu[kTH], s_md[kTH];   // NMS lane masks (same-cell neighbours)
    __shared__ int16_t s_xs0[kTileW], s_xs1[kTileW], s_xa0[kTileW], s_xa1[kTileW];
    __shared__ int16_t s_ys0[kTileH], s_ys1[kTileH], s_yb0[kTileH], s_yb1[kTileH];
    __shared__ int16_t s_cellx[kTW + 2], s_celly[kTH + 2];
    __shared__ int16_t s_mx[kTW], s_my[kTH];                          // level-0 mask coordinates of the tile's pixels
    __shared__ int s_wn[kThreads / 32], s_base;

    // 16-bit score tiles (two copies offset by one pixel, like the pixel tiles); they reuse the source staging
    // area, which is dead once the tile has been resized
    uint16_t* s_s0 = (uint16_t*)s_src;                                  // s_s0[y][x] = score(x),   x = score-tile column
    uint16_t* s_s1 = (uint16_t*)s_src + (kTH + 2) * kScoreS;            // s_s1[y][i] = score(i+1)
    // corner list, one segment per warp (no atomics while collecting): lives in the 16-bit pixel tile, which is dead once the FAST
    // margins are computed (phases b, c; the barrier before phase d separates them from phase e)
    uint32_t* s_list = (uint32_t*)s_a0;
    static_assert((kThreads / 32) * kWarpCorners * 4 <= kTileH * kT16S * 2, "corner list must fit into the dead pixel tile");
    static_assert(2 * (kTH + 2) * kScoreS * 2 <= kSrcH * kSrcWB, "score tiles must fit into the staging area");
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int b = blockIdx.z;
    const int X0 = blockIdx.x * kTW, Y0 = blockIdx.y * kTH;
    const uint8_t* simg = src + (size_t)b * src_img_bytes;
    // FAST + NMS only where the tile holds at least one pixel inside the camera's mask: a corner is reported only if its own
    // mask pixel is set (mask applied after NMS, SURVEY A.5), and the scores of its 8 neighbours come from this CTA's own halo
    const int cam_b = cam_of_image[b];
    const int tile_flag = tile_flags[(size_t)cam_b * tiles_total + g.tile_off + blockIdx.y * g.tiles_x + blockIdx.x];
    const bool fast_on = tile_flag != 0, mask_full = tile_flag == 2;      // 2: every pixel of the tile is inside the mask

    // output-space range needed by this tile; after REFLECT_101 everything lies inside it
    const int xa = max(X0 - kHalo, 0), xb = min(X0 + kTW + kHalo, g.w) - 1;
    const int ya = max(Y0 - kHalo, 0), yb = min(Y0 + kTH + kHalo, g.h) - 1;
    const int sx_lo = g.xofs[xa], sx_hi = min(g.xofs[xb] + 1, g.sw - 1);
    const int sy_lo = min(max((int)g.yofs[ya], 0), g.sh - 1), sy_hi = min(max(g.yofs[yb] + 1, 0), g.sh - 1);
    const int sx_base = sx_lo & ~15;
    const int wb = use_tma ? g.box_w : kSrcWB;                          // row stride of the staged region in bytes
    if (tid == 0) {
        if (use_tma) {
            // the barrier is initialised and armed by the same thread that issues the copy; every other thread first sees it
            // after the __syncthreads below, then waits for phase 0
            mbar_init(&s_bar, 1);
            mbar_expect_tx(&s_bar, (uint32_t)(g.box_w * g.box_h));
            tma_load_3d(s_src, &src_map, sx_base, sy_lo, b, &s_bar);
        }
    }

    // ---- per-tile slices of the resize / cell tables ----
    if (tid < kTileW) {
        // rows/columns further than the ring beyond the image are never consumed: clamp them into the staged range
        const int rx = min(max(reflect101(X0 - kHalo + tid, g.w), xa), xb);
        const int sx = g.xofs[rx];
        s_xs0[tid] = (int16_t)(sx - sx_base);
        s_xs1[tid] = (int16_t)(min(sx + 1, g.sw - 1) - sx_base);
        s_xa0[tid] = g.xa0[rx]; s_xa1[tid] = g.xa1[rx];
    } else if (tid >= 96 && tid < 96 + kTileH) {
        const int t = tid - 96;
        const int ry = min(max(reflect101(Y0 - kHalo + t, g.h), ya), yb);
        const int sy = g.yofs[ry];
        s_ys0[t] = (int16_t)(min(max(sy, 0), g.sh - 1) - sy_lo);
        s_ys1[t] = (int16_t)(min(max(sy + 1, 0), g.sh - 1) - sy_lo);
        s_yb0[t] = g.yb0[ry]; s_yb1[t] = g.yb1[ry];
    } else if (tid >= 144 && tid < 144 + kTW + 2) {
        const int x = X0 - 1 + tid - 144;
        s_cellx[tid - 144] = (x >= 0 && x < g.w) ? g.cellx[x] : (int16_t)-1;
    }
    if (tid < kTH + 2) {
        const int y = Y0 - 1 + tid;
        s_celly[tid] = (y >= 0 && y < g.h) ? g.celly[y] : (int16_t)-1;
    } else if (tid >= 64 && tid < 64 + kTW) {
        const int x = X0 + tid - 64;
        s_mx[tid - 64] = x < g.w ? g.mx0[x] : (int16_t)0;
    } else if (tid >= 128 && tid < 128 + kTH) {
        const int y = Y0 + tid - 128;
        s_my[tid - 128] = y < g.h ? g.my0[y] : (int16_t)0;
    }
    // ---- stage the source rows: by TMA (above), or -- caller images with an unaligned base / stride -- 16-byte chunks per warp ----
    if (!use_tma) {
        const int nrows = sy_hi - sy_lo + 1;
        if (src_aligned) {
            const int nchunks = ((sx_hi - sx_base) >> 4) + 1;
            if (nchunks <= 8) {          // scale factors <= 1.5: four rows per warp instruction
                const int c = lane & 7;
                for (int r = wid * 4 + (lane >> 3); r < nrows; r += kThreads / 8)
                    if (c < nchunks)
                        *(uint4*)(s_src + r * kSrcWB + c * 16) =
                            __ldg((const uint4*)(simg + (size_t)(sy_lo + r) * g.spitch + sx_base + c * 16));
            } else {
                for (int r = wid; r < nrows; r += kThreads / 32)
                    for (int c = lane; c < nchunks; c += 32)
                        *(uint4*)(s_src + r * kSrcWB + c * 16) =
                            __ldg((const uint4*)(simg + (size_t)(sy_lo + r) * g.spitch + sx_base + c * 16));
            }
        } else {   // caller-supplied image with an unaligned base or stride (level 0 only)
            const int nb = sx_hi - sx_base + 1;
            for (int r = wid; r < nrows; r += kThreads / 32)
                for (int c = lane; c < nb; c += 32) {
                    const int x = sx_base + c;
                    s_src[r * kSrcWB + c] = x < g.sw ? simg[(size_t)(sy_lo + r) * g.spitch + x] : (uint8_t)0;
                }
        }
    }
    __syncthreads();
    if (use_tma) mbar_wait(&s_bar, 0);

    // ---- bilinear resize (OpenCV 11-bit fixed point) into the three tile forms; a thread owns a pixel-pair column ----
    if (tid < (kTileW / 2) * 7) {
        const int pc = tid % (kTileW / 2), rg = tid / (kTileW / 2);      // 36 pair columns x 7 row groups
        const int tx = 2 * pc;
        const int xs00 = s_xs0[tx], xs01 = s_xs1[tx], xs10 = s_xs0[tx + 1], xs11 = s_xs1[tx + 1];
        const int a00 = s_xa0[tx], a01 = s_xa1[tx], a10 = s_xa0[tx + 1], a11 = s_xa1[tx + 1];
#pragma unroll
        for (int ty = rg; ty < kTileH; ty += 7) {
            const uint8_t* r0 = s_src + s_ys0[ty] * wb;
            const uint8_t* r1 = s_src + s_ys1[ty] * wb;
            const int b0 = s_yb0[ty], b1 = s_yb1[ty];
            int v0, v1;
            if (level == 0) {            // identity resize: the general formula reduces to a copy
                v0 = r0[xs00]; v1 = r0[xs10];
            } else {
                const int h00 = r0[xs00] * a00 + r0[xs01] * a01, h01 = r1[xs00] * a00 + r1[xs01] * a01;
                const int h10 = r0[xs10] * a10 + r0[xs11] * a11, h11 = r1[xs10] * a10 + r1[xs11] * a11;
                v0 = (((b0 * (h00 >> 4)) >> 16) + ((b1 * (h01 >> 4)) >> 16) + 2) >> 2;
                v1 = (((b0 * (h10 >> 4)) >> 16) + ((b1 * (h11 >> 4)) >> 16) + 2) >> 2;
                v0 = min(max(v0, 0), 255); v1 = min(max(v1, 0), 255);
            }
            *(uint16_t*)(s_t8 + ty * kT8S + tx) = (uint16_t)(v0 | (v1 << 8));
            *(uint32_t*)(s_a0 + ty * kT16S + tx) = (uint32_t)v0 | ((uint32_t)v1 << 16);
            if (tx > 0) s_a1[ty * kT16S + tx - 1] = (uint16_t)v0;
            s_a1[ty * kT16S + tx] = (uint16_t)v1;
        }
    }
    __syncthreads();

    // same-cell masks for the packed NMS: pair column j holds pixels x = 2j, 2j+1 (score-tile columns x+1, x+2)
    if (tid < kTW / 2) {
        const int c0 = s_cellx[2 * tid], c1 = s_cellx[2 * tid + 1], c2 = s_cellx[2 * tid + 2], c3 = s_cellx[2 * tid + 3];
        s_ml[tid] = (c0 == c1 ? 0xFFFFu : 0u) | (c1 == c2 ? 0xFFFF0000u : 0u);     // left  neighbours of (x, x+1)
        s_mr[tid] = (c2 == c1 ? 0xFFFFu : 0u) | (c3 == c2 ? 0xFFFF0000u : 0u);     // right neighbours of (x, x+1)
    } else if (tid >= 64 && tid < 64 + kTH) {
        const int y = tid - 64;
        s_mu[y] = s_celly[y] == s_celly[y + 1] ? 0xFFFFFFFFu : 0u;
        s_md[y] = s_celly[y + 2] == s_celly[y + 1] ? 0xFFFFFFFFu : 0u;
    }
    uint8_t* dimg = dst + (size_t)b * g.img_bytes;
    uint8_t* bimg = dst_blur + (size_t)b * g.img_bytes;
    // ---- (a) store the unblurred tile, 4 px per thread ----
#pragma unroll
    for (int i = tid; i < kTH * (kTW / 4); i += kThreads) {
        const int y = i >> 4, x4 = (i & 15) * 4;
        if (Y0 + y < g.h && X0 + x4 < g.pitch)
            *(uint32_t*)(dimg + (size_t)(Y0 + y) * g.pitch + X0 + x4) = *(const uint32_t*)(s_t8 + (y + kHalo) * kT8S + x4 + kHalo);
    }
    // ---- (b) packed horizontal 5-sums of pixel pairs (rows Y0-2 .. Y0+33) ----
#pragma unroll
    for (int i = tid; i < (kTH + 4) * (kTW / 2); i += kThreads) {
        const int y = i >> 5, j = i & 31;
        const uint32_t* w0 = (const uint32_t*)(s_a0 + (y + kHalo - 2) * kT16S) + (kHalo / 2 + j);   // pair (x, x+1), x = tile col 4+2j
        const uint32_t* w1 = (const uint32_t*)(s_a1 + (y + kHalo - 2) * kT16S) + (kHalo / 2 + j);   // pair (x+1, x+2)
        s_h[i] = __vadd2(__vadd2(__vadd2(w0[-1], w1[-1]), __vadd2(w0[0], w1[0])), w0[1]);
    }
    // ---- (c) FAST margins of pixel pairs on the tile + 1 ring; pairs start at tile column 3 (odd) ----
    if (fast_on)
#pragma unroll
    for (int i = tid; i < (kTH + 2) * ((kTW + 2) / 2); i += kThreads) {
        const int y = i / ((kTW + 2) / 2), j = i - y * ((kTW + 2) / 2);
        const int sx = 2 * j;                                   // score-tile column of the first pixel of the pair
        const bool in0 = s_cellx[sx] >= 0, in1 = s_cellx[sx + 1] >= 0, iny = s_celly[y] >= 0;
        unsigned s0 = 0, s1 = 0;
        if (iny && (in0 || in1)) {
            // centre pair (px, px+1) with px = tile col 3+2j (odd) -> word j+1 of the odd copy; even dx -> odd copy, odd dx -> even copy
            const uint32_t* o = (const uint32_t*)(s_a1 + (y + kHalo - 1) * kT16S) + (j + 1);
            const uint32_t* e = (const uint32_t*)(s_a0 + (y + kHalo - 1) * kT16S) + (j + 2);   // pair starting at px+1
            constexpr int S = kT16S / 2;                         // row stride in words
            const unsigned C = o[0];
            unsigned R[16];
            R[0] = o[3 * S];       R[1] = e[3 * S];        R[2] = o[2 * S + 1];   R[3] = e[S + 1];
            R[4] = e[1];           R[5] = e[-S + 1];       R[6] = o[-2 * S + 1];  R[7] = e[-3 * S];
            R[8] = o[-3 * S];      R[9] = e[-3 * S - 1];   R[10] = o[-2 * S - 1]; R[11] = e[-S - 2];
            R[12] = e[-2];         R[13] = e[S - 2];       R[14] = o[2 * S - 1];  R[15] = e[3 * S - 1];
            const unsigned m = fast_margin2(C, R);
            const int m0 = (int)(short)(m & 0xFFFFu), m1 = (int)(short)(m >> 16);
            s0 = (in0 && m0 > fast_th) ? (unsigned)(m0 - 1) : 0u;
            s1 = (in1 && m1 > fast_th) ? (unsigned)(m1 - 1) : 0u;
        }
        *(uint32_t*)(s_s0 + y * kScoreS + sx) = s0 | (s1 << 16);
        if (sx > 0) s_s1[y * kScoreS + sx - 1] = (uint16_t)s0;
        s_s1[y * kScoreS + sx] = (uint16_t)s1;
    }
    __syncthreads();

    // ---- (d) blurred tile: vertical 5-sum of the packed row sums, (S+12)/25, 4 px per thread ----
#pragma unroll
    for (int i = tid; i < kTH * (kTW / 4); i += kThreads) {
        const int y = i >> 4, q = i & 15;
        if (Y0 + y < g.h && X0 + 4 * q < g.pitch) {
            const uint32_t* h = s_h + y * (kTW / 2) + 2 * q;
            const unsigned p0 = __vadd2(__vadd2(__vadd2(h[0], h[32]), __vadd2(h[64], h[96])), h[128]);
            const unsigned p1 = __vadd2(__vadd2(__vadd2(h[1], h[33]), __vadd2(h[65], h[97])), h[129]);
            // (S + 12) / 25 == ((S + 12) * 5243) >> 17 for S <= 6375 (checked exhaustively in tests)
            const unsigned o0 = (((p0 & 0xFFFFu) + 12u) * 5243u) >> 17, o1 = (((p0 >> 16) + 12u) * 5243u) >> 17;
            const unsigned o2 = (((p1 & 0xFFFFu) + 12u) * 5243u) >> 17, o3 = (((p1 >> 16) + 12u) * 5243u) >> 17;
            *(uint32_t*)(bimg + (size_t)(Y0 + y) * g.pitch + X0 + 4 * q) = o0 | (o1 << 8) | (o2 << 16) | (o3 << 24);
        }
    }
    // ---- (e) per-cell 3x3 non-max suppression on pixel pairs (packed 16x2), mask filter, tile-local compaction ----
    // Pair j of row y = pixels x = 2j, 2j+1 = score-tile columns 2j+1, 2j+2: centre word from the odd copy, left /
    // right neighbour pairs from the even copy.  A neighbour outside the pixel's FAST cell counts as 0 (cv::FAST runs per cell).
    if (!fast_on) return;                                   // uniform for the CTA: no corner can come out of this tile
    const uint8_t* m0p = mask0 + (size_t)cam_b * mask_bytes;
    // A warp owns one tile row per pass (32 pixel pairs), every lane evaluates its pair branch-free and the warp VOTES: two
    // ballots give the number of surviving corners and each lane's slot in the warp's own list segment (a per-corner divergent
    // append runs with few active lanes, and a per-pass shared atomic still costs a visible share of the instructions).  The
    // level-0 mask is only consulted when the row segment holds a strict maximum at all.
    int wn = 0;                                             // corners this warp has collected (warp-uniform)
#pragma unroll
    for (int i = tid; i < kTH * (kTW / 2); i += kThreads) {
        const int y = i >> 5, j = i & 31;
        const uint32_t* e0 = (const uint32_t*)(s_s0 + y * kScoreS) + j;          // row y-1 of the interior row y (score row y)
        const uint32_t* o0 = (const uint32_t*)(s_s1 + y * kScoreS) + j;
        constexpr int S = kScoreS / 2;
        const unsigned C = o0[S];
        const unsigned ml = s_ml[j], mr = s_mr[j], mu = s_mu[y], md = s_md[y];
        const unsigned up = __vimax3_u16x2(e0[0] & ml & mu, o0[0] & mu, e0[1] & mr & mu);
        const unsigned dn = __vimax3_u16x2(e0[2 * S] & ml & md, o0[2 * S] & md, e0[2 * S + 1] & mr & md);
        const unsigned nm = __vimax3_u16x2(up, dn, __vmaxu2(e0[S] & ml, e0[S + 1] & mr));
        const int sv0 = (int)(C & 0xFFFFu), sv1 = (int)(C >> 16);
        // strict maximum of its 3x3 (implies a non-zero score), then the mask of its own pixel (mask applied after NMS)
        bool k0 = sv0 > (int)(nm & 0xFFFFu), k1 = sv1 > (int)(nm >> 16);
        unsigned b0 = __ballot_sync(0xffffffffu, k0), b1 = __ballot_sync(0xffffffffu, k1);
        if (b0 | b1) {                                                           // warp-uniform: some pixel of this row segment is a maximum
            if (!mask_full) {                                                    // CTA-uniform: tiles on the mask border only
                if (k0) k0 = m0p[(size_t)s_my[y] * mask_w + s_mx[2 * j]] != 0;
                if (k1) k1 = m0p[(size_t)s_my[y] * mask_w + s_mx[2 * j + 1]] != 0;
                b0 = __ballot_sync(0xffffffffu, k0); b1 = __ballot_sync(0xffffffffu, k1);
            }
            const int n0 = __popc(b0);
            const unsigned lt = (1u << lane) - 1u;
            uint32_t* wl = s_list + wid * kWarpCorners + wn;
            if (k0) wl[__popc(b0 & lt)] = pack_corner(X0 + 2 * j, Y0 + y, sv0);
            if (k1) wl[n0 + __popc(b1 & lt)] = pack_corner(X0 + 2 * j + 1, Y0 + y, sv1);
            wn += n0 + __popc(b1);
        }
    }
    if (lane == 0) s_wn[wid] = wn;
    __syncthreads();
    int n = 0, my_off = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
        if (w == wid) my_off = n;
        n += s_wn[w];
    }
    if (n == 0) return;
    if (tid == 0) s_base = atomicAdd(&raw_count[b * nlevels + level], n);
    __syncthreads();
    uint32_t* rlist = raw + (size_t)b * raw_img_stride + g.raw_off;
    for (int i = lane; i < wn; i += 32) {
        const int pos = s_base + my_off + i;
        if (pos < g.raw_cap) rlist[pos] = s_list[wid * kWarpCorners + i];
    }
}

// tight caller rows -> 64-byte aligned pitch (the host entry points copy H2D linearly, then re-pitch on the device:
// a 2-D DMA of 754-byte rows is several times slower than a linear copy)
__global__ void repitch_kernel(const uint8_t* __restrict__ src, int src_stride, uint8_t* __restrict__ dst, int dst_pitch, int width,
                               size_t rows) {
    const size_t row = blockIdx.x;
    if (row >= rows) return;
    const uint8_t* s = src + row * src_stride;
    uint8_t* d = dst + row * dst_pitch;
    for (int x = threadIdx.x; x < dst_pitch; x += blockDim.x) d[x] = x < width ? s[x] : (uint8_t)0;
}
void launch_repitch(const uint8_t* src, int src_stride, uint8_t* dst, int dst_pitch, int width, size_t rows, cudaStream_t st) {
    repitch_kernel<<<(unsigned)rows, 256, 0, st>>>(src, src_stride, dst, dst_pitch, width, rows);
}

void launch_pyr_fast(const PyramidGeom& G, int level, int n_images, const uint8_t* src, size_t src_img_bytes,
                     uint8_t* dst, uint8_t* dst_blur, const uint8_t* mask0, int mask_w, size_t mask_bytes,
                     const int* cam_of_image, const uint8_t* tile_flags, uint32_t* raw, int* raw_count, cudaStream_t st) {
    const LevelGeom& g = G.lv[level];
    dim3 grid(g.tiles_x, g.tiles_y, n_images);
    const int aligned = (((uintptr_t)src & 15) == 0 && (g.spitch & 15) == 0 && (src_img_bytes & 15) == 0) ? 1 : 0;
    // tensor map of the source: (row bytes, rows, images), box = the level's staged region.  Encoding is a host-side table fill
    // (no driver round trip), done per launch because the base address and the batch size are per call.
    CUtensorMap map;
    std::memset(&map, 0, sizeof(map));
    int use_tma = 0;
#if MCS_K1_TMA
    static PFN_cuTensorMapEncodeTiled_v12000 encode = [] {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || qr != cudaDriverEntryPointSuccess) fn = nullptr;
        return (PFN_cuTensorMapEncodeTiled_v12000)fn;
    }();
    if (encode && aligned && g.box_w * g.box_h <= kSrcH * kSrcWB) {
        const cuuint64_t dims[3] = {(cuuint64_t)g.spitch, (cuuint64_t)g.sh, (cuuint64_t)n_images};
        const cuuint64_t strides[2] = {(cuuint64_t)g.spitch, (cuuint64_t)src_img_bytes};
        const cuuint32_t box[3] = {(cuuint32_t)g.box_w, (cuuint32_t)g.box_h, 1u};
        const cuuint32_t estr[3] = {1u, 1u, 1u};
        use_tma = encode(&map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, (void*)src, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
    }
#endif
    pyr_fast_kernel<<<grid, kThreads, 0, st>>>(map, use_tma, g, level, G.nlevels, G.fast_threshold, aligned, src, src_img_bytes, dst, dst_blur,
                                               mask0, mask_w, mask_bytes, cam_of_image, tile_flags, G.tiles_total, raw, G.raw_total,
                                               raw_count);
}

}  // namespace mcs
