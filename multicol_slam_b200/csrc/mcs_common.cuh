// mcs_common.cuh -- shared host/device definitions of the sm_90a feature pipeline.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>
#include "../../include/mcs_b200.h"

namespace mcs {

constexpr int kEdge = 25;        // EDGE_THRESHOLD  (ref src/mdBRIEFextractorOct.cpp:85)
constexpr int kHalfPatch = 16;   // HALF_PATCH_SIZE (ref :84)
constexpr int kMaxLevels = MCS_MAX_LEVELS;

// K1 tiling: one CTA produces a TW x TH tile of level l (+ kHalo ring kept in shared memory)
constexpr int kTW = 64, kTH = 32, kHalo = 4;
constexpr int kTileW = kTW + 2 * kHalo;     // 72
constexpr int kTileH = kTH + 2 * kHalo;     // 40
constexpr int kSrcH = 88;                   // staged source rows, enough for scale factors <= 2
constexpr int kMaxNodes = 2048;             // octree nodes alive at once (>= max(quota + 8, 4 * nodes_ini) of every level)

// Per-level geometry + look-up tables (device pointers into one blob built by the host).
struct LevelGeom {
    int w, h, pitch;              // level size, row pitch in bytes (multiple of 64)
    int sw, sh, spitch;           // source (level l-1, or the input image for l == 0)
    int tiles_x, tiles_y;
    int tile_off;                 // offset of this level's tiles in the per-camera tile-flag table
    int box_w, box_h;             // TMA box of the staged source region: bytes per row (multiple of 16) x rows, covers every tile
    int raw_cap;                  // capacity of the raw corner list of this level (per image)
    int quota;                    // mnFeaturesPerLevel[l]
    int sel_cap;                  // max(quota + 3, 4 * nodes_ini): the most keypoints DistributeOctTree returns
    int sel_off;                  // offset of this level's selected-keypoint slots (per image)
    int n_cols, n_rows, w_cell, h_cell;   // FAST cell grid (ref :876-949)
    int nodes_ini;                // octree roots (ref :640)
    double hX;                    // octree root width (ref :642)
    float scale;                  // (float)mvScaleFactor[l]
    float patch_size;             // (float)(int)(32*mvScaleFactor[l])
    size_t img_bytes;             // pitch*h : per-image stride of this level's buffers
    size_t raw_off;               // element offset of this level's raw list inside a per-image raw block
    // LUTs (device)
    const int16_t* xofs;  const int16_t* xa0; const int16_t* xa1;   // [w] resize: source column, weights
    const int16_t* yofs;  const int16_t* yb0; const int16_t* yb1;   // [h]
    const int16_t* cellx; const int16_t* celly;                     // [w]/[h] FAST cell index or -1
    const int16_t* mx0;   const int16_t* my0;                       // [w]/[h] level-0 mask coordinates
};

struct PyramidGeom {
    int nlevels;
    int width, height;
    int fast_threshold;
    int desc_size;
    int do_dbrief, learn_masks;
    int cap;                       // output slots per image
    int sel_total;                 // sum of sel_cap
    size_t raw_total;              // sum of raw_cap (elements per image)
    int tiles_total;               // sum of tiles_x * tiles_y
    int node_cap;                  // K2's node table per (image, level): max(quota + 8, 4 * nodes_ini) over the levels, multiple of 32
    LevelGeom lv[kMaxLevels];
};

// raw corner packing: x:12 | y:12 | score:8
__host__ __device__ inline uint32_t pack_corner(int x, int y, int s) {
    return ((uint32_t)x << 20) | ((uint32_t)y << 8) | (uint32_t)s;
}
__host__ __device__ inline int corner_x(uint32_t c) { return (int)(c >> 20); }
__host__ __device__ inline int corner_y(uint32_t c) { return (int)((c >> 8) & 0xFFF); }
__host__ __device__ inline int corner_s(uint32_t c) { return (int)(c & 0xFF); }

__host__ __device__ inline int reflect101(int p, int n) {
    if (p < 0) p = -p;
    if (p >= n) p = 2 * (n - 1) - p;
    return p;
}

// descriptor widths (bytes) the Hamming kernels are built for
inline bool desc_width_ok(const int dim) { return dim == 16 || dim == 32 || dim == 64; }

// The descriptor-width dispatch of the Hamming kernels: calls f(W, M) with W = std::integral_constant<int, dim / 4> (the 32-bit
// words of a descriptor) and M = std::integral_constant<bool, masked>, so that `kern<W, M>` names one instantiation per width and
// mask.  Any dim other than 16 and 32 takes the 64-byte path; callers that refuse other widths test desc_width_ok first.
template <class F>
inline void with_desc_width(const int dim, const bool masked, F&& f) {
    using std::integral_constant;
    const auto with_mask = [&](auto W) {
        if (masked) f(W, std::true_type{});
        else f(W, std::false_type{});
    };
    if (dim == 16) with_mask(integral_constant<int, 4>{});
    else if (dim == 32) with_mask(integral_constant<int, 8>{});
    else with_mask(integral_constant<int, 16>{});
}

// The list-length dispatch of the K-best kernels: calls f(KT) with KT = std::integral_constant<int, 4> for K <= 4 and
// std::integral_constant<int, 8> otherwise, the compile-time length of the lists that hold K entries.
template <class F>
inline void with_list_len(const int K, F&& f) {
    if (K <= 4) f(std::integral_constant<int, 4>{});
    else f(std::integral_constant<int, 8>{});
}

}  // namespace mcs
