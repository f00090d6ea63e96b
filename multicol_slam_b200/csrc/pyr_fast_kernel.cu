// pyr_fast_kernel.cu -- K1: per pyramid level, ONE fused kernel
//     resize(level l-1 -> l)  +  5x5 box blur  +  FAST-9/16 score  +  per-cell 3x3 NMS  +  mirror-mask filter
// (ref src/mdBRIEFextractorOct.cpp:1158-1201 ComputePyramid, :863-949 cell loop, :1301 boxFilter; OpenCV
// resize / boxFilter / FAST arithmetic restated in SURVEY.md Appendix A.1 / A.3 / A.5).
//
// One CTA owns a 64x64 tile of level l.  The source region of level l-1 is staged in shared memory by TMA (or 128-bit
// loads), the tile (+4 px ring, REFLECT_101 at the image border) is resized once and kept in two shared 16-bit-per-pixel
// copies offset by one pixel, so that ANY horizontally adjacent pixel pair is one aligned 32-bit word (the level's bytes are
// stored from the even copy).  Blur and FAST then run on pixel PAIRS with the packed 16x2 integer
// SIMD of sm_90a (16x2 adds, DPX three-way min / max):
//   * box blur: 5 packed loads + 4 packed adds give the horizontal 5-sums of two pixels;
//   * FAST: E_k = ring_k - centre (packed), 9-arc minima / maxima by two 3-input min (max) levels
//     (M3_k = min3(E_k,E_k+1,E_k+2), M9_k = min3(M3_k,M3_k+3,M3_k+6)), branch-free exact cornerScore for every
//     pixel pair: score = max over arcs of max(min9(E), -max9(E)) - 1, corner iff that maximum exceeds the threshold.
// The kernel is bound by integer issue rate, not by HBM (DESIGN.md, K1): on the order of a hundred thread-instructions per
// pixel against a few bytes of DRAM traffic.
#include <algorithm>
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

// block index read from the special register where it is used: asm volatile keeps the compiler from holding the first read live
// across the FAST phase, where it would be spilled at the 40-register budget
__device__ __forceinline__ int ctaid_x() { int v; asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(v)); return v; }
__device__ __forceinline__ int ctaid_y() { int v; asm volatile("mov.u32 %0, %%ctaid.y;" : "=r"(v)); return v; }
__device__ __forceinline__ int ctaid_z() { int v; asm volatile("mov.u32 %0, %%ctaid.z;" : "=r"(v)); return v; }

// Phase split of the kernel's time: tools/k1_split.py --split builds this file with -DMCS_K1_SPLIT_EXIT=n into a library of its own,
// whose CTAs return after the staging and the tables (1), after the resize (2) or after FAST (3).  The shipped build has no exit.
#ifdef MCS_K1_SPLIT_EXIT
#define K1_SPLIT_EXIT(n) if (MCS_K1_SPLIT_EXIT == (n)) return
#else
#define K1_SPLIT_EXIT(n)
#endif

// resident CTAs per SM the register budget is cut for: 5 allows 48 registers, enough for FAST without spills.  Shared memory
// (23 KB of pixel tiles and tables plus 17.3 KB of staging at scale 1.2) also allows 5 (DESIGN.md, K1)
constexpr int kMinBlocks = 5;
constexpr int kThreads = 256;
constexpr int kT16S = 72;                   // 16-bit tile row stride (elements)
constexpr int kScoreS = 68;                 // score tile row stride in 16-bit elements (66 used)
// the score tile and the packed row sums reuse the staging area, which is dead once the tile has been resized
constexpr int kScoreBytes = (kTH + 2) * kScoreS * 2;
constexpr int kRowSumBytes = (kTH + 4) * (kTW / 2) * 4;
constexpr int kStagingMin = kScoreBytes + kRowSumBytes;
static_assert(kScoreBytes % 16 == 0, "row sums start 16-byte aligned");
// corner slots per warp: a warp owns kTH/8 = 8 tile rows.  Inside a FAST cell two strict 3x3 maxima are never adjacent in a row, but the
// NMS counts a neighbour in another cell as 0, so the last pixel of a cell and the first of the next can both be maxima.  Cells are
// at least 30 px wide (nCols = int(width / 30), checked by build_geometry), so a 64-px row meets at most 4 cells and holds at most
// sum ceil(piece / 2) <= (64 + 4) / 2 = 34 maxima (tests/test_k1_bounds_cpu.py runs every level width)
constexpr int kWarpCorners = (kTH / (kThreads / 32)) * (kTW / 2 + 2);

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

// packed FAST margins of the pixel pair (px, px+1), px odd: o = word of the odd copy holding the pair, e = word of the even copy
// holding (px+1, px+2).  Even ring offsets dx read the odd copy, odd dx the even one.
__device__ __forceinline__ unsigned fast_pair_margin(const uint32_t* o, const uint32_t* e) {
    constexpr int S = kT16S / 2;                             // row stride in words
    unsigned R[16];
    R[0] = o[3 * S];       R[1] = e[3 * S];        R[2] = o[2 * S + 1];   R[3] = e[S + 1];
    R[4] = e[1];           R[5] = e[-S + 1];       R[6] = o[-2 * S + 1];  R[7] = e[-3 * S];
    R[8] = o[-3 * S];      R[9] = e[-3 * S - 1];   R[10] = o[-2 * S - 1]; R[11] = e[-S - 2];
    R[12] = e[-2];         R[13] = e[S - 2];       R[14] = o[2 * S - 1];  R[15] = e[3 * S - 1];
    return fast_margin2(o[0], R);
}

// score pair of packed margins m: margin - 1 where the margin exceeds th2 (the threshold in both 16-bit lanes), else 0
__device__ __forceinline__ unsigned fast_pair_score(unsigned m, unsigned th2) {
    return __vsub2(m, 0x00010001u) & __vcmpgts2(m, th2);
}

__global__ void __launch_bounds__(kThreads, kMinBlocks)
pyr_fast_kernel(const __grid_constant__ CUtensorMap src_map, const int use_tma,
                const LevelGeom g, const int level, const int nlevels, const int fast_th, const int src_aligned,
                const uint8_t* __restrict__ src, const size_t src_img_bytes,
                uint8_t* __restrict__ dst, uint8_t* __restrict__ dst_blur,
                const uint8_t* __restrict__ mask0, const int mask_w, const size_t mask_bytes,
                const int* __restrict__ cam_of_image, const uint8_t* __restrict__ tile_flags, const int tiles_total,
                uint32_t* __restrict__ raw, const size_t raw_img_stride, int* __restrict__ raw_count) {
    extern __shared__ __align__(128) uint8_t s_src[];                  // staged source rows: box_h x kSrcWB bytes (launcher)
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ __align__(16) uint16_t s_a0[kTileH * kT16S];          // s_a0[y][x]   = px(x)
    __shared__ __align__(16) uint16_t s_a1[kTileH * kT16S];          // s_a1[y][i]   = px(i+1)
    __shared__ uint32_t s_ml[kTW / 2], s_mr[kTW / 2], s_mu[kTH], s_md[kTH];   // NMS lane masks (same-cell neighbours)
    __shared__ int16_t s_xs0[kTileW], s_xs1[kTileW], s_xa0[kTileW], s_xa1[kTileW];
    __shared__ int16_t s_ys0[kTileH], s_ys1[kTileH], s_yb0[kTileH], s_yb1[kTileH];
    __shared__ int16_t s_cellx[kTW + 2], s_celly[kTH + 2];
    __shared__ int16_t s_mx[kTW], s_my[kTH];                          // level-0 mask coordinates of the tile's pixels
    __shared__ int s_wn[kThreads / 32], s_base, s_cam, s_flag;

    // 16-bit score tile; it reuses the source staging area, which is dead once the tile has been resized.  The NMS forms the
    // odd-aligned score pairs from two aligned words with a byte permute.
    uint16_t* s_s0 = (uint16_t*)s_src;                                  // s_s0[y][x] = score(x),   x = score-tile column
    uint32_t* s_h = (uint32_t*)(s_src + kScoreBytes);                   // packed horizontal 5-sums of pixel pairs
    // corner list, one segment per warp (no atomics while collecting): lives in the 16-bit pixel tile, which is dead once the FAST
    // margins are computed (phases b, c; the barrier before phase d separates them from phase e)
    uint32_t* s_list = (uint32_t*)s_a0;
    static_assert((kThreads / 32) * kWarpCorners * 4 <= kTileH * kT16S * 2, "corner list must fit into the dead pixel tile");
    // the launcher sizes the staging area to at least kStagingMin
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int b = blockIdx.z;
    const int X0 = blockIdx.x * kTW, Y0 = blockIdx.y * kTH;
    const uint8_t* simg = src + (size_t)b * src_img_bytes;
    // output-space range needed by this tile; after REFLECT_101 everything lies inside it
    const int xa = max(X0 - kHalo, 0), xb = min(X0 + kTW + kHalo, g.w) - 1;
    const int ya = max(Y0 - kHalo, 0), yb = min(Y0 + kTH + kHalo, g.h) - 1;
    const int sx_lo = g.xofs[xa], sx_hi = min(g.xofs[xb] + 1, g.sw - 1);
    const int sy_lo = min(max((int)g.yofs[ya], 0), g.sh - 1), sy_hi = min(max(g.yofs[yb] + 1, 0), g.sh - 1);
    const int sx_base = sx_lo & ~15;
    if (tid == 0) {
        if (use_tma) {
            // the barrier is initialised and armed by the same thread that issues the copy; every other thread first sees it
            // after the __syncthreads below, then waits for phase 0
            mbar_init(&s_bar, 1);
            mbar_expect_tx(&s_bar, (uint32_t)(g.box_w * g.box_h));
            tma_load_3d(s_src, &src_map, sx_base, sy_lo, b, &s_bar);
        }
    }

    // FAST + NMS only where the tile holds at least one pixel inside the camera's mask: a corner is reported only if its own
    // mask pixel is set (mask applied after NMS, SURVEY A.5), and the scores of its 8 neighbours come from this CTA's own halo.
    // One thread reads the camera and the tile's flag; the other threads read them from shared memory where they are used,
    // so that they hold no registers through FAST.
    if (tid == 32) {
        const int cam_b = cam_of_image[b];
        s_cam = cam_b;
        s_flag = tile_flags[(size_t)cam_b * tiles_total + g.tile_off + blockIdx.y * g.tiles_x + blockIdx.x];
    }

    // ---- per-tile slices of the resize / cell tables ----
    bool in_cells = true;                 // this thread's score-tile row / column lies inside a FAST cell
    if (tid < kTileW) {
        // rows/columns further than the ring beyond the image are never consumed: clamp them into the staged range
        const int rx = min(max(reflect101(X0 - kHalo + tid, g.w), xa), xb);
        const int sx = g.xofs[rx];
        s_xs0[tid] = (int16_t)(sx - sx_base);
        s_xs1[tid] = (int16_t)(min(sx + 1, g.sw - 1) - sx_base);
        s_xa0[tid] = g.xa0[rx]; s_xa1[tid] = g.xa1[rx];
    } else if (tid >= kTileW && tid < kTileW + kTileH) {
        const int t = tid - kTileW;
        const int ry = min(max(reflect101(Y0 - kHalo + t, g.h), ya), yb);
        const int sy = g.yofs[ry];
        s_ys0[t] = (int16_t)(min(max(sy, 0), g.sh - 1) - sy_lo);
        s_ys1[t] = (int16_t)(min(max(sy + 1, 0), g.sh - 1) - sy_lo);
        s_yb0[t] = g.yb0[ry]; s_yb1[t] = g.yb1[ry];
    } else if (tid >= kTileW + kTileH && tid < kTileW + kTileH + kTW + 2) {
        const int x = X0 - 1 + tid - (kTileW + kTileH);
        const int16_t c = (x >= 0 && x < g.w) ? g.cellx[x] : (int16_t)-1;
        s_cellx[tid - (kTileW + kTileH)] = c;
        in_cells = c >= 0;
    }
    if (tid < kTH + 2) {
        const int y = Y0 - 1 + tid;
        const int16_t c = (y >= 0 && y < g.h) ? g.celly[y] : (int16_t)-1;
        s_celly[tid] = c;
        in_cells = in_cells && c >= 0;
    } else if (tid >= 96 && tid < 96 + kTW) {
        const int x = X0 + tid - 96;
        s_mx[tid - 96] = x < g.w ? g.mx0[x] : (int16_t)0;
    } else if (tid >= 96 + kTW && tid < 96 + kTW + kTH) {
        const int y = Y0 + tid - (96 + kTW);
        s_my[tid - (96 + kTW)] = y < g.h ? g.my0[y] : (int16_t)0;
    }
    static_assert(kTileW + kTileH + kTW + 2 <= kThreads && kTH + 2 <= 96 && 96 + kTW + kTH <= kThreads, "one table entry per thread");
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
    // every pixel of the score tile (tile + 1 ring) lies inside some FAST cell, and so inside the level: FAST needs no per-pixel test
    const bool fast_inner = __syncthreads_and(in_cells);
    if (use_tma) mbar_wait(&s_bar, 0);
    K1_SPLIT_EXIT(1);
    const int wb = use_tma ? g.box_w : kSrcWB;                          // row stride of the staged region in bytes

    if (level == 0 && ctaid_x() * kTW >= kHalo && ctaid_x() * kTW + kTW + kHalo <= g.w) {
        // ---- identity resize of a tile whose columns (with the ring) need no reflection: a word copy of the staged rows ----
        // staged column X0 - kHalo lies at byte (X0 - kHalo) & 15 (sx_base = (X0 - kHalo) & ~15), a multiple of 4
        static_assert(kTW % 16 == 0 && kHalo % 4 == 0 && kTileW % 4 == 0, "level-0 word copy needs word-aligned tile columns");
        constexpr int kQ = kTileW / 4, kRG = kThreads / kQ;              // 18 words per row, 14 row groups
        if (tid < kQ * kRG) {
            const int q = tid % kQ;
            const uint8_t* s_row = s_src + ((ctaid_x() * kTW - kHalo) & 15) + 4 * q;
#pragma unroll
            for (int ty = tid / kQ; ty < kTileH; ty += kRG) {
                const uint32_t* r = (const uint32_t*)(s_row + s_ys0[ty] * wb);
                const uint32_t w = r[0], wn = r[1];                         // pixels 4q .. 4q+3, 4q+4 .. 4q+7
                const uint32_t a0 = __byte_perm(w, 0u, 0x4140), a1 = __byte_perm(w, 0u, 0x4342);
                *(uint2*)(s_a0 + ty * kT16S + 4 * q) = make_uint2(a0, a1);
                *(uint2*)(s_a1 + ty * kT16S + 4 * q) = make_uint2(__byte_perm(w, 0u, 0x4241), __byte_perm(a1, wn, 0x1412));
            }
        }
    } else if (tid < (kTileW / 2) * (kThreads / (kTileW / 2))) {
        // ---- bilinear resize (OpenCV 11-bit fixed point) into the three tile forms; a thread owns a pixel-pair column ----
        constexpr int kRG = kThreads / (kTileW / 2);
        const int pc = tid % (kTileW / 2), rg = tid / (kTileW / 2);      // 36 pair columns x 7 row groups
        const int tx = 2 * pc;
        const int xs00 = s_xs0[tx], xs01 = s_xs1[tx], xs10 = s_xs0[tx + 1], xs11 = s_xs1[tx + 1];
        const int a00 = s_xa0[tx], a01 = s_xa1[tx], a10 = s_xa0[tx + 1], a11 = s_xa1[tx + 1];
#pragma unroll
        for (int ty = rg; ty < kTileH; ty += kRG) {
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
            *(uint32_t*)(s_a0 + ty * kT16S + tx) = (uint32_t)v0 | ((uint32_t)v1 << 16);
            if (tx > 0) s_a1[ty * kT16S + tx - 1] = (uint16_t)v0;
            s_a1[ty * kT16S + tx] = (uint16_t)v1;
        }
    }
    __syncthreads();
    K1_SPLIT_EXIT(2);

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
    // ---- (a) store the unblurred tile, 4 px per thread, packed from the even 16-bit copy ----
#pragma unroll
    for (int i = tid; i < kTH * (kTW / 4); i += kThreads) {
        const int y = i >> 4, x4 = (i & 15) * 4;
        if (Y0 + y < g.h && X0 + x4 < g.pitch) {
            const uint2 p = *(const uint2*)(s_a0 + (y + kHalo) * kT16S + x4 + kHalo);
            *(uint32_t*)(dimg + (size_t)(Y0 + y) * g.pitch + X0 + x4) = __byte_perm(p.x, p.y, 0x6420);
        }
    }
    // ---- (b) packed horizontal 5-sums of pixel pairs (rows Y0-2 .. Y0+kTH+1) ----
#pragma unroll
    for (int i = tid; i < (kTH + 4) * (kTW / 2); i += kThreads) {
        const int y = i >> 5, j = i & 31;
        const uint32_t* w0 = (const uint32_t*)(s_a0 + (y + kHalo - 2) * kT16S) + (kHalo / 2 + j);   // pair (x, x+1), x = tile col 4+2j
        const uint32_t* w1 = (const uint32_t*)(s_a1 + (y + kHalo - 2) * kT16S) + (kHalo / 2 + j);   // pair (x+1, x+2)
        s_h[i] = __vadd2(__vadd2(__vadd2(w0[-1], w1[-1]), __vadd2(w0[0], w1[0])), w0[1]);
    }
    // ---- (c) FAST scores of pixel pairs on the tile + 1 ring: score-tile row y, pair j = score-tile columns 2j, 2j+1, centre
    // pixel px = tile col 3+2j (odd) -> word j+1 of the odd copy, pair (px+1, px+2) -> word j+2 of the even copy ----
    constexpr int kPJ = (kTW + 2) / 2;                          // 33 pairs per score-tile row
    static_assert(kTH % 8 == 0 && kTW == 64 && kThreads == 256, "FAST: one lane per pair column, a warp per score-tile row");
    if (s_flag != 0) {                                          // CTA-uniform
        const unsigned th2 = (unsigned)fast_th * 0x00010001u;   // 1 <= fast_th <= 254 (checked by the host)
        // score of pair j on row y; pixels outside every FAST cell get a threshold no margin exceeds (margins are at most 255)
        // rather than a mask on the score: one register less across the margin, which keeps FAST free of spills.  A warp skips
        // the margins of a pair set outside the cells.  Tiles inside the cell grid (fast_inner, most of them) test nothing.
        auto score = [&](const uint32_t* o, const uint32_t* e, unsigned in) -> unsigned {
            return in ? fast_pair_score(fast_pair_margin(o, e), (th2 & in) | (0x7FFF7FFFu & ~in)) : 0u;
        };
        auto cells = [&](int y, int j) -> unsigned {
            if (fast_inner) return ~0u;
            return s_celly[y] < 0 ? 0u : (s_cellx[2 * j] >= 0 ? 0xFFFFu : 0u) | (s_cellx[2 * j + 1] >= 0 ? 0xFFFF0000u : 0u);
        };
        // lane = pair column 0..31 on rows wid, wid + 8, ..: addresses formed once, rows 8 apart are compile-time offsets
        {
            const uint32_t* o = (const uint32_t*)(s_a1 + (wid + kHalo - 1) * kT16S) + (lane + 1);
            const uint32_t* e = (const uint32_t*)(s_a0 + (wid + kHalo - 1) * kT16S) + (lane + 2);
            uint32_t* sc = (uint32_t*)(s_s0 + wid * kScoreS) + lane;
#pragma unroll
            for (int k = 0; k < kTH / 8; ++k)                   // 8 rows further: 8 * kT16S / 2 words in the pixel tiles
                sc[k * 4 * kScoreS] = score(o + k * 4 * kT16S, e + k * 4 * kT16S, cells(wid + 8 * k, lane));
        }
        // the rest: rows kTH, kTH + 1 (warps 0, 1) and pair column 32 of every row (threads 64 .. 64 + kTH + 1)
        if (tid < 2 * 32 + kTH + 2) {
            const int y = tid < 64 ? kTH + (tid >> 5) : tid - 64, j = tid < 64 ? lane : kPJ - 1;
            const uint32_t* o = (const uint32_t*)(s_a1 + (y + kHalo - 1) * kT16S) + (j + 1);
            const uint32_t* e = (const uint32_t*)(s_a0 + (y + kHalo - 1) * kT16S) + (j + 2);
            *((uint32_t*)(s_s0 + y * kScoreS) + j) = score(o, e, cells(y, j));
        }
    }
    __syncthreads();
    K1_SPLIT_EXIT(3);
    const int tx0 = ctaid_x() * kTW, ty0 = ctaid_y() * kTH, img = ctaid_z();   // X0, Y0, b again (see ctaid_x)
    uint8_t* bimg = dst_blur + (size_t)img * g.img_bytes;

    // ---- (d) blurred tile: vertical 5-sum of the packed row sums, (S+12)/25, 4 px per thread ----
#pragma unroll
    for (int i = tid; i < kTH * (kTW / 4); i += kThreads) {
        const int y = i >> 4, q = i & 15;
        if (ty0 + y < g.h && tx0 + 4 * q < g.pitch) {
            const uint32_t* h = s_h + y * (kTW / 2) + 2 * q;
            const unsigned p0 = __vadd2(__vadd2(__vadd2(h[0], h[32]), __vadd2(h[64], h[96])), h[128]);
            const unsigned p1 = __vadd2(__vadd2(__vadd2(h[1], h[33]), __vadd2(h[65], h[97])), h[129]);
            // (S + 12) / 25 == ((S + 12) * 5243) >> 17 for S <= 6375 (checked exhaustively in tests)
            const unsigned o0 = (((p0 & 0xFFFFu) + 12u) * 5243u) >> 17, o1 = (((p0 >> 16) + 12u) * 5243u) >> 17;
            const unsigned o2 = (((p1 & 0xFFFFu) + 12u) * 5243u) >> 17, o3 = (((p1 >> 16) + 12u) * 5243u) >> 17;
            *(uint32_t*)(bimg + (size_t)(ty0 + y) * g.pitch + tx0 + 4 * q) = o0 | (o1 << 8) | (o2 << 16) | (o3 << 24);
        }
    }
    // ---- (e) per-cell 3x3 non-max suppression on pixel pairs (packed 16x2), mask filter, tile-local compaction ----
    // Pair j of row y = pixels x = 2j, 2j+1 = score-tile columns 2j+1, 2j+2: the high half of word j and the low half of word j+1
    // (one byte permute), left / right neighbour pairs are words j and j+1 themselves.  A neighbour outside the pixel's FAST cell
    // counts as 0 (cv::FAST runs per cell).
    const int tile_flag = s_flag;
    if (tile_flag == 0) return;                             // uniform for the CTA: no corner can come out of this tile
    const bool mask_full = tile_flag == 2;                  // 2: every pixel of the tile is inside the mask
    const uint8_t* m0p = mask0 + (size_t)s_cam * mask_bytes;
    // A warp owns one tile row per pass (32 pixel pairs), every lane evaluates its pair branch-free and the warp VOTES: two
    // ballots give the number of surviving corners and each lane's slot in the warp's own list segment (a per-corner divergent
    // append runs with few active lanes, and a per-pass shared atomic still costs a visible share of the instructions).  The
    // level-0 mask is only consulted when the row segment holds a strict maximum at all.
    int wn = 0;                                             // corners this warp has collected (warp-uniform)
#pragma unroll
    for (int i = tid; i < kTH * (kTW / 2); i += kThreads) {
        const int y = i >> 5, j = i & 31;
        const uint32_t* e0 = (const uint32_t*)(s_s0 + y * kScoreS) + j;          // row y-1 of the interior row y (score row y)
        constexpr int S = kScoreS / 2;
        const unsigned u0 = e0[0], u1 = e0[1], c0 = e0[S], c1 = e0[S + 1], d0 = e0[2 * S], d1 = e0[2 * S + 1];
        const unsigned C = __byte_perm(c0, c1, 0x5432);
        const unsigned ml = s_ml[j], mr = s_mr[j], mu = s_mu[y], md = s_md[y];
        const unsigned up = __vimax3_u16x2(u0 & ml & mu, __byte_perm(u0, u1, 0x5432) & mu, u1 & mr & mu);
        const unsigned dn = __vimax3_u16x2(d0 & ml & md, __byte_perm(d0, d1, 0x5432) & md, d1 & mr & md);
        const unsigned nm = __vimax3_u16x2(up, dn, __vmaxu2(c0 & ml, c1 & mr));
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
            if (k0) wl[__popc(b0 & lt)] = pack_corner(tx0 + 2 * j, ty0 + y, sv0);
            if (k1) wl[n0 + __popc(b1 & lt)] = pack_corner(tx0 + 2 * j + 1, ty0 + y, sv1);
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
    if (tid == 0) s_base = atomicAdd(&raw_count[img * nlevels + level], n);
    __syncthreads();
    uint32_t* rlist = raw + (size_t)img * raw_img_stride + g.raw_off;
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

cudaError_t launch_pyr_fast(const PyramidGeom& G, int level, int n_images, const uint8_t* src, size_t src_img_bytes,
                            uint8_t* dst, uint8_t* dst_blur, const uint8_t* mask0, int mask_w, size_t mask_bytes,
                            const int* cam_of_image, const uint8_t* tile_flags, uint32_t* raw, int* raw_count, cudaStream_t st) {
    const LevelGeom& g = G.lv[level];
    // staging sized for this level's source region (box_w <= kSrcWB, box_h <= kSrcH: build_geometry refuses larger), so that
    // levels at small scale factors keep 4 CTAs per SM.  The opt-in above 48 KB is per device: set on every launch.
    const int staging = std::max(g.box_h * kSrcWB, kStagingMin);
    cudaError_t e = cudaFuncSetAttribute(pyr_fast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSrcH * kSrcWB);
    if (e != cudaSuccess) return e;
    dim3 grid(g.tiles_x, g.tiles_y, n_images);
    const int aligned = (((uintptr_t)src & 15) == 0 && (g.spitch & 15) == 0 && (src_img_bytes & 15) == 0) ? 1 : 0;
    // tensor map of the source: (row bytes, rows, images), box = the level's staged region.  Encoding is a host-side table fill
    // (no driver round trip), done per launch because the base address and the batch size are per call.  Sources with an
    // unaligned base or stride are staged with __ldg instead (use_tma = 0).
    CUtensorMap map;
    std::memset(&map, 0, sizeof(map));
    int use_tma = 0;
    static PFN_cuTensorMapEncodeTiled_v12000 encode = [] {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || qr != cudaDriverEntryPointSuccess) fn = nullptr;
        return (PFN_cuTensorMapEncodeTiled_v12000)fn;
    }();
    if (encode && aligned) {
        const cuuint64_t dims[3] = {(cuuint64_t)g.spitch, (cuuint64_t)g.sh, (cuuint64_t)n_images};
        const cuuint64_t strides[2] = {(cuuint64_t)g.spitch, (cuuint64_t)src_img_bytes};
        const cuuint32_t box[3] = {(cuuint32_t)g.box_w, (cuuint32_t)g.box_h, 1u};
        const cuuint32_t estr[3] = {1u, 1u, 1u};
        use_tma = encode(&map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, (void*)src, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
    }
    pyr_fast_kernel<<<grid, kThreads, staging, st>>>(map, use_tma, g, level, G.nlevels, G.fast_threshold, aligned, src, src_img_bytes, dst,
                                                     dst_blur, mask0, mask_w, mask_bytes, cam_of_image, tile_flags, G.tiles_total, raw,
                                                     G.raw_total, raw_count);
    return cudaGetLastError();
}

}  // namespace mcs
