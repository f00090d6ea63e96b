// mcs_api.cu -- C-ABI host layer of libmcs_b200.so (see include/mcs_b200.h): the error message, the camera-model helpers and
// the extractor with its extract-and-match stream pipeline.
//
// Host responsibilities only: parameter tables of the extractor constructor (ref
// src/mdBRIEFextractorOct.cpp:134-203), per-image-size geometry / look-up tables, device buffers and
// kernel launches.  The matcher entry points live in mcs_match_api.cu.
// There is no CPU implementation of the image or distance arithmetic in this library: without a CUDA
// device every compute entry point fails with MCS_ERR_NO_DEVICE.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "api_check.h"
#include "cam_model.cuh"
#include "kernels.h"
#include "mcs_common.cuh"
#include "packed_frame.h"

using namespace mcs;

static thread_local std::string g_err;
int mcs_fail(int code, const std::string& msg) { g_err = msg; return code; }

namespace {

static const signed char kPairs[2048] = {
#include "brief_pairs_64.inc"
};

inline int cv_round(double v) { return (int)lrint(v); }
inline int cv_floor(double v) { int i = (int)v; return i - (i > v); }
inline int cv_ceil(double v) { int i = (int)v; return i + (i < v); }
inline short sat_short_round(float v) { int i = (int)lrintf(v); return (short)std::min(std::max(i, -32768), 32767); }

// device memory owned by the extractor: freed with it (the caller makes the extractor's device current)
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
    cudaError_t ensure(size_t count) {
        if (count <= n) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; n = 0;
        cudaError_t e = cudaMalloc((void**)&p, count * sizeof(T));
        if (e != cudaSuccess) return e;
        n = count;
        // unused tail slots of the fixed-size outputs read back as zeros.  The memset runs on the legacy default stream, the
        // extractor works on non-blocking streams: wait for it, or it could overtake-zero freshly written data (allocation is rare).
        e = cudaMemset(p, 0, count * sizeof(T));
        if (e != cudaSuccess) return e;
        return cudaDeviceSynchronize();
    }
};

}  // namespace

struct mcs_extractor {
    mcs_extractor_params p;
    int device = 0;
    std::vector<double> sf, isf;
    std::vector<int> quota;
    int capacity = 0;
    cudaStream_t stream = nullptr;

    // geometry for the current image size
    PyramidGeom G;
    int geom_w = 0, geom_h = 0, geom_stride = 0;
    DevBuf<uint8_t> lut_blob;
    DevBuf<PyramidGeom> G_dev;

    // device buffers (grown on demand)
    int B_cap = 0;
    DevBuf<uint8_t> in_images;
    DevBuf<uint8_t> lvl[kMaxLevels], blur[kMaxLevels];
    DevBuf<uint8_t> masks;
    DevBuf<mcs_ocam> cams;
    DevBuf<int> cam_of_image;
    const int* coi_last = nullptr;      // camera-of-image table the last run used (device)
    DevBuf<uint32_t> raw;
    DevBuf<uint16_t> node_of;
    DevBuf<int> raw_count, sel_count, status, counts;
    DevBuf<uint32_t> sel_xys;
    DevBuf<mcs_keypoint> kps;
    DevBuf<uint8_t> desc, dmask;
    int last_n_images = 0;
    DevBuf<int> match_idx, match_dist, m12, nmat, redo;
    DevBuf<uint8_t> in_tight;
    cudaStream_t s_copy = nullptr, s_out = nullptr, s_match = nullptr;
    // distortion tables, rebuilt when the camera set changes
    std::vector<mcs_ocam> lut_cams;
    std::vector<uint8_t> masks_host;    // what ex->masks holds
    std::vector<int16_t> h_mx[kMaxLevels], h_my[kMaxLevels];   // host copies of the level -> level-0 mask coordinate maps
    DevBuf<uint8_t> tile_flags;         // [n_cams][tiles_total]: the K1 tile holds a pixel inside the camera's mask
    bool tile_flags_valid = false;
    DevBuf<double> lut_coef;
    DevBuf<DistortLut> luts;
    // small host-buffer calls (mcs_extract_batch with <= kGraphMaxImages images: what cMultiFrame's constructor issues per frame):
    // pinned staging on both sides and the whole copy-in / K1..K3 / copy-out sequence kept as an instantiated CUDA graph
    uint8_t* pin_in = nullptr;  size_t pin_in_bytes = 0;
    uint8_t* pin_out = nullptr; size_t pin_out_bytes = 0;
    cudaGraphExec_t sf_exec = nullptr;
    struct SfKey { int n = 0, w = 0, h = 0, stride = 0, capacity = 0; bool dm = false; std::vector<int> coi; std::vector<mcs_ocam> cams; } sf_key;
    bool sf_valid = false;
    long long sf_replays = 0;
    bool profiling = false;
    bool tier_on = false;
    DevBuf<unsigned long long> tier;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
};

namespace {

// ---- extractor tables: everything that depends only on the params (ref :151-179) ----------------
int init_tables(mcs_extractor* ex, const mcs_extractor_params* p) {
    if (p->use_agast) return mcs_fail(MCS_ERR_UNSUPPORTED, "AGAST detector is not built (north star: FAST-9)");
    if (p->fast_agast_type != 2) return mcs_fail(MCS_ERR_UNSUPPORTED, "only FastFeatureDetector::TYPE_9_16 (type 2) is built");
    if (p->nlevels < 1 || p->nlevels > kMaxLevels) return mcs_fail(MCS_ERR_INVALID, "nlevels must be in [1,16]");
    if (p->desc_size != 16 && p->desc_size != 32 && p->desc_size != 64) return mcs_fail(MCS_ERR_INVALID, "desc_size must be 16, 32 or 64");
    if (p->nfeatures < 1 || !(p->scale_factor > 1.0f) || p->fast_threshold < 1 || p->fast_threshold > 254)
        return mcs_fail(MCS_ERR_INVALID, "bad nfeatures / scale_factor / fast_threshold");
    ex->p = *p;
    const double sfd = (double)p->scale_factor;
    ex->sf.resize(p->nlevels); ex->isf.resize(p->nlevels); ex->quota.resize(p->nlevels);
    ex->sf[0] = 1; ex->isf[0] = 1;
    for (int i = 1; i < p->nlevels; ++i) ex->sf[i] = ex->sf[i - 1] * sfd;
    const double inv = 1.0 / sfd;
    for (int i = 1; i < p->nlevels; ++i) ex->isf[i] = ex->isf[i - 1] * inv;
    const double factor = 1.0 / sfd;
    double nd = p->nfeatures * (1 - factor) / (1 - std::pow(factor, p->nlevels));
    int sum = 0;
    for (int l = 0; l < p->nlevels - 1; ++l) {
        ex->quota[l] = cv_round(nd);
        sum += ex->quota[l];
        nd *= factor;
    }
    ex->quota[p->nlevels - 1] = std::max(p->nfeatures - sum, 0);
    ex->capacity = 0;
    for (int l = 0; l < p->nlevels; ++l) {
        if (ex->quota[l] + 8 > kMaxNodes) return mcs_fail(MCS_ERR_UNSUPPORTED, "nfeatures too large for the octree node table");
        ex->capacity += std::max(ex->quota[l] + 2, 16);
    }
    return MCS_OK;
}

// ---- geometry: everything that depends only on (width, height, params) ------------------------
struct LutOffsets { size_t xofs, xa0, xa1, yofs, yb0, yb1, cellx, celly, mx0, my0; };

// ex->G without its table pointers, the tables (blob, off) and the refusals of a geometry: host only
int plan_geometry(mcs_extractor* ex, int W, int H, int in_stride, std::vector<int16_t>& blob, LutOffsets* off) {
    PyramidGeom& G = ex->G;
    std::memset(&G, 0, sizeof(G));
    const int L = ex->p.nlevels;
    G.nlevels = L; G.width = W; G.height = H;
    G.fast_threshold = ex->p.fast_threshold; G.desc_size = ex->p.desc_size;
    G.do_dbrief = ex->p.do_dbrief; G.learn_masks = ex->p.learn_masks;
    if (W >= 4096 || H >= 4096) return mcs_fail(MCS_ERR_UNSUPPORTED, "images larger than 4095 px are not supported");

    std::vector<int16_t> pmx, pmy;
    size_t raw_off = 0;
    int sel_off = 0;
    for (int l = 0; l < L; ++l) {
        LevelGeom& g = G.lv[l];
        g.w = cv_round((double)W * ex->isf[l]);
        g.h = cv_round((double)H * ex->isf[l]);
        if (g.w < 2 * kEdge + 8 || g.h < 2 * kEdge + 8)
            return mcs_fail(MCS_ERR_UNSUPPORTED, "pyramid level smaller than 58 px");
        g.pitch = (g.w + 63) & ~63;
        g.img_bytes = (size_t)g.pitch * g.h;
        g.sw = l ? G.lv[l - 1].w : W; g.sh = l ? G.lv[l - 1].h : H;
        g.spitch = l ? G.lv[l - 1].pitch : in_stride;
        g.tiles_x = (g.w + kTW - 1) / kTW; g.tiles_y = (g.h + kTH - 1) / kTH;
        g.scale = (float)ex->sf[l];
        g.patch_size = (float)(int)(32 * ex->sf[l]);
        g.quota = ex->quota[l];
        // resize tables (OpenCV resize INTER_LINEAR, SURVEY Appendix A.1)
        std::vector<int16_t> xofs(g.w), xa0(g.w), xa1(g.w), yofs(g.h), yb0(g.h), yb1(g.h), mx(g.w), my(g.h);
        if (l) {
            const double scale_x = 1.0 / ((double)g.w / g.sw), scale_y = 1.0 / ((double)g.h / g.sh);
            // the staged source region of a 72x72 tile must fit kSrcWB x kSrcH = 176 x 152 bytes: (72*s + 17) <= 176, (72*s + 2) <= 152
            if (scale_x > 2.08 || scale_y > 2.08) return mcs_fail(MCS_ERR_UNSUPPORTED, "scale factors above 2 are not supported");
            for (int dx = 0; dx < g.w; ++dx) {
                float fx = (float)((dx + 0.5) * scale_x - 0.5);
                int sx = cv_floor(fx);
                fx -= sx;
                if (sx < 0) { fx = 0; sx = 0; }
                if (sx >= g.sw - 1) { fx = 0; sx = g.sw - 1; }
                xofs[dx] = (int16_t)sx;
                xa0[dx] = sat_short_round((1.f - fx) * 2048.f);
                xa1[dx] = sat_short_round(fx * 2048.f);
                mx[dx] = pmx[std::min(cv_floor(dx * scale_x), g.sw - 1)];
            }
            for (int dy = 0; dy < g.h; ++dy) {
                float fy = (float)((dy + 0.5) * scale_y - 0.5);
                int sy = cv_floor(fy);
                fy -= sy;
                yofs[dy] = (int16_t)sy;
                yb0[dy] = sat_short_round((1.f - fy) * 2048.f);
                yb1[dy] = sat_short_round(fy * 2048.f);
                my[dy] = pmy[std::min(cv_floor(dy * scale_y), g.sh - 1)];
            }
        } else {
            for (int x = 0; x < g.w; ++x) { xofs[x] = (int16_t)x; xa0[x] = 2048; xa1[x] = 0; mx[x] = (int16_t)x; }
            for (int y = 0; y < g.h; ++y) { yofs[y] = (int16_t)y; yb0[y] = 2048; yb1[y] = 0; my[y] = (int16_t)y; }
        }
        pmx = mx; pmy = my;
        ex->h_mx[l] = mx; ex->h_my[l] = my;
        {   // staged source region of the widest / tallest tile (same index arithmetic as pyr_fast_kernel): the TMA box of the level
            int bw = 16, bh = 1;
            for (int tx = 0; tx < g.tiles_x; ++tx) {
                const int xa = std::max(tx * kTW - kHalo, 0), xb = std::min(tx * kTW + kTW + kHalo, g.w) - 1;
                const int lo = xofs[xa] & ~15, hi = std::min(xofs[xb] + 1, g.sw - 1);
                bw = std::max(bw, hi - lo + 1);
            }
            for (int ty = 0; ty < g.tiles_y; ++ty) {
                const int ya = std::max(ty * kTH - kHalo, 0), yb = std::min(ty * kTH + kTH + kHalo, g.h) - 1;
                const int lo = std::min(std::max((int)yofs[ya], 0), g.sh - 1), hi = std::min(std::max(yofs[yb] + 1, 0), g.sh - 1);
                bh = std::max(bh, hi - lo + 1);
            }
            g.box_w = (bw + 15) & ~15; g.box_h = bh;
            if (g.box_w > kSrcWB || g.box_h > kSrcH) return mcs_fail(MCS_ERR_UNSUPPORTED, "K1 source region larger than its staging");
        }
        // FAST cell grid (ref :876-949, SURVEY Appendix A.6)
        std::vector<int16_t> cellx(g.w, -1), celly(g.h, -1);
        const int minB = kEdge - 3, maxBX = g.w - kEdge + 3, maxBY = g.h - kEdge + 3;
        const double width = maxBX - minB, height = maxBY - minB;
        g.n_cols = (int)(width / 30.0); g.n_rows = (int)(height / 30.0);
        if (g.n_cols < 1 || g.n_rows < 1) return mcs_fail(MCS_ERR_UNSUPPORTED, "level too small for the 30 px cell grid");
        g.w_cell = (int)std::ceil(width / g.n_cols); g.h_cell = (int)std::ceil(height / g.n_rows);
        // K1 sizes its per-warp corner segments for tile rows that cross at most 3 cell edges (kWarpCorners)
        if (g.w_cell < 30) return mcs_fail(MCS_ERR_UNSUPPORTED, "FAST cells narrower than 30 px");
        if ((long long)g.n_cols * g.n_rows * g.w_cell * g.h_cell >= (1 << 24))
            return mcs_fail(MCS_ERR_UNSUPPORTED, "cell-order key overflow");
        for (int i = 0; i < g.n_rows; ++i) {
            const double iniY = minB + i * g.h_cell;
            double maxY = iniY + g.h_cell + 6;
            if (iniY >= maxBY - 3) continue;
            if (maxY > maxBY) maxY = maxBY;
            for (int y = (int)iniY + 3; y < (int)maxY - 3; ++y) celly[y] = (int16_t)i;
        }
        for (int j = 0; j < g.n_cols; ++j) {
            const double iniX = minB + j * g.w_cell;
            double maxX = iniX + g.w_cell + 6;
            if (iniX >= maxBX - 6) continue;
            if (maxX > maxBX) maxX = maxBX;
            for (int x = (int)iniX + 3; x < (int)maxX - 3; ++x) cellx[x] = (int16_t)j;
        }
        // a cell narrower/lower than 7 px yields nothing in cv::FAST; the ranges above are then empty.
        // octree roots (ref :640-642)
        g.nodes_ini = cv_round((double)(maxBX - minB) / (maxBY - minB));
        if (g.nodes_ini < 1) return mcs_fail(MCS_ERR_UNSUPPORTED, "portrait images narrower than half their height");
        g.hX = (double)(maxBX - minB) / g.nodes_ini;
        g.sel_cap = std::max(g.quota + 3, 4 * g.nodes_ini);
        g.sel_off = sel_off; sel_off += g.sel_cap;
        // raw corner capacity: a cell of w_c x h_c pixels holds at most ceil(w_c / 2) * ceil(h_c / 2) strict maxima (one per 2x2
        // block, the per-cell NMS does not look across cells); the cells form a grid, so the sum over the cells factors per axis
        auto half_cells = [](const std::vector<int16_t>& cell) {
            int s = 0, run = 0;
            for (size_t i = 0; i <= cell.size(); ++i) {
                if (i < cell.size() && cell[i] >= 0 && (run == 0 || cell[i] == cell[i - 1])) { ++run; continue; }
                s += (run + 1) / 2;
                run = (i < cell.size() && cell[i] >= 0) ? 1 : 0;
            }
            return s;
        };
        g.raw_cap = half_cells(cellx) * half_cells(celly);
        g.raw_off = raw_off; raw_off += (size_t)((g.raw_cap + 3) & ~3);
        auto put = [&](const std::vector<int16_t>& v) { size_t o = blob.size(); blob.insert(blob.end(), v.begin(), v.end()); while (blob.size() & 7) blob.push_back(0); return o; };
        off[l] = {put(xofs), put(xa0), put(xa1), put(yofs), put(yb0), put(yb1), put(cellx), put(celly), put(mx), put(my)};
    }
    G.sel_total = sel_off; G.raw_total = raw_off; G.cap = ex->capacity;
    G.tiles_total = 0;
    for (int l = 0; l < L; ++l) { G.lv[l].tile_off = G.tiles_total; G.tiles_total += G.lv[l].tiles_x * G.lv[l].tiles_y; }
    // DistributeOctTree (ref :640-854) divides every one of its nodes_ini roots in its first pass, whatever the quota N: up to
    // 4 nodes_ini nodes.  Every later pass starts below N and adds at most 3 nodes per division, so it ends below N + 3.  K2's
    // node table holds the larger of the two (quota + 8 as before); the output slots are fixed at mcs_extractor_create, before
    // the image size is known, so a geometry whose worst case exceeds them is refused here, before any launch.
    int nodes = 0, most = 0;
    for (int l = 0; l < L; ++l) {
        const LevelGeom& g = G.lv[l];
        nodes = std::max(nodes, std::max(g.quota + 8, 4 * g.nodes_ini));
        most += std::max(g.quota + 2, 4 * g.nodes_ini);
    }
    G.node_cap = (nodes + 31) & ~31;
    if (G.node_cap > kMaxNodes) return mcs_fail(MCS_ERR_UNSUPPORTED, "octree roots exceed the node table");
    if (most > ex->capacity)
        return mcs_fail(MCS_ERR_UNSUPPORTED, "image too wide for nfeatures: the octree can return more keypoints than the capacity");
    return MCS_OK;
}

int build_geometry(mcs_extractor* ex, int W, int H, int in_stride) {
    if (ex->geom_w == W && ex->geom_h == H && ex->geom_stride == in_stride) return MCS_OK;
    ex->geom_w = ex->geom_h = ex->geom_stride = 0;      // ex->G is rewritten: a refused size must not leave the previous key on it
    std::vector<int16_t> blob;     // all LUTs, int16
    LutOffsets off[kMaxLevels];
    int rc = plan_geometry(ex, W, H, in_stride, blob, off);
    if (rc) return rc;
    PyramidGeom& G = ex->G;
    const int L = G.nlevels;
    ex->tile_flags_valid = false;
    // kernels of an earlier *_device call on a caller-supplied stream may still read the tables about to be rewritten (a change of the
    // image size is rare: drain the device)
    CUDA_CHECK(cudaDeviceSynchronize());
    CUDA_CHECK(ex->lut_blob.ensure(blob.size() * sizeof(int16_t)));
    CUDA_CHECK(cudaMemcpyAsync(ex->lut_blob.p, blob.data(), blob.size() * sizeof(int16_t), cudaMemcpyHostToDevice, ex->stream));
    const int16_t* base = (const int16_t*)ex->lut_blob.p;
    for (int l = 0; l < L; ++l) {
        LevelGeom& g = G.lv[l];
        g.xofs = base + off[l].xofs; g.xa0 = base + off[l].xa0; g.xa1 = base + off[l].xa1;
        g.yofs = base + off[l].yofs; g.yb0 = base + off[l].yb0; g.yb1 = base + off[l].yb1;
        g.cellx = base + off[l].cellx; g.celly = base + off[l].celly;
        g.mx0 = base + off[l].mx0; g.my0 = base + off[l].my0;
    }
    CUDA_CHECK(ex->G_dev.ensure(1));
    CUDA_CHECK(cudaMemcpyAsync(ex->G_dev.p, &G, sizeof(G), cudaMemcpyHostToDevice, ex->stream));
    CUDA_CHECK(cudaStreamSynchronize(ex->stream));     // blob / G are host temporaries
    ex->geom_w = W; ex->geom_h = H; ex->geom_stride = in_stride;
    ex->B_cap = 0;      // level buffers depend on the geometry
    return MCS_OK;
}

int ensure_batch(mcs_extractor* ex, int B) {
    if (B <= ex->B_cap) return MCS_OK;
    const PyramidGeom& G = ex->G;
    for (int l = 0; l < G.nlevels; ++l) {
        CUDA_CHECK(ex->lvl[l].ensure(G.lv[l].img_bytes * B + 256));
        CUDA_CHECK(ex->blur[l].ensure(G.lv[l].img_bytes * B + 256));
    }
    CUDA_CHECK(ex->raw.ensure(G.raw_total * B));
    CUDA_CHECK(ex->node_of.ensure(G.raw_total * B));
    CUDA_CHECK(ex->raw_count.ensure((size_t)B * G.nlevels));
    CUDA_CHECK(ex->sel_count.ensure((size_t)B * G.nlevels));
    CUDA_CHECK(ex->sel_xys.ensure((size_t)B * G.sel_total));
    CUDA_CHECK(ex->status.ensure(1));
    ex->B_cap = B;
    return MCS_OK;
}

// Small per-call host inputs (masks, camera models, distortion tables, status word).  They travel over the same
// H2D copy engine as the image chunks of the stream call, so they must be enqueued BEFORE any large copy: a 1 MB
// mask upload queued behind 100 MB of images stalls the compute stream for the whole transfer.
int upload_small_inputs(mcs_extractor* ex, int W, int H, const uint8_t* masks, const mcs_ocam* cams, int n_cams, cudaStream_t st) {
    CUDA_CHECK(ex->masks.ensure((size_t)n_cams * W * H));
    CUDA_CHECK(ex->cams.ensure(n_cams));
    // the masks rarely change between calls (static mirror masks): a 1 MB compare is cheaper than a pageable upload
    const size_t mbytes = (size_t)n_cams * W * H;
    if (ex->masks_host.size() != mbytes || std::memcmp(ex->masks_host.data(), masks, mbytes) != 0) {
        CUDA_CHECK(cudaStreamSynchronize(st));                     // a previous call may still read the old masks
        ex->masks_host.assign(masks, masks + mbytes);
        CUDA_CHECK(cudaMemcpyAsync(ex->masks.p, ex->masks_host.data(), mbytes, cudaMemcpyHostToDevice, st));
        ex->tile_flags_valid = false;
    }
    if (!ex->tile_flags_valid) {
        // per camera and K1 tile: does the tile hold a pixel whose (nearest-neighbour chained) mask value is set?
        const PyramidGeom& G = ex->G;
        // 0 = no pixel of the tile is inside the mask (FAST / NMS skipped), 1 = some are, 2 = all are (no per-corner mask lookup)
        std::vector<uint8_t> flags((size_t)n_cams * G.tiles_total, 0), all_in((size_t)n_cams * G.tiles_total, 1);
        for (int c = 0; c < n_cams; ++c) {
            const uint8_t* m0 = ex->masks_host.data() + (size_t)c * W * H;
            for (int l = 0; l < G.nlevels; ++l) {
                const LevelGeom& g = G.lv[l];
                uint8_t* f = flags.data() + (size_t)c * G.tiles_total + g.tile_off;
                uint8_t* a = all_in.data() + (size_t)c * G.tiles_total + g.tile_off;
                for (int y = 0; y < g.h; ++y) {
                    const uint8_t* mrow = m0 + (size_t)ex->h_my[l][y] * W;
                    uint8_t* frow = f + (size_t)(y / kTH) * g.tiles_x;
                    uint8_t* arow = a + (size_t)(y / kTH) * g.tiles_x;
                    for (int x = 0; x < g.w; ++x) {
                        const uint8_t m = mrow[ex->h_mx[l][x]];
                        frow[x / kTW] |= m;
                        if (!m) arow[x / kTW] = 0;
                    }
                }
            }
        }
        for (size_t i = 0; i < flags.size(); ++i) flags[i] = flags[i] ? (all_in[i] ? 2 : 1) : 0;
        CUDA_CHECK(cudaStreamSynchronize(st));                     // a previous call may still read the old flags
        CUDA_CHECK(ex->tile_flags.ensure(flags.size()));
        CUDA_CHECK(cudaMemcpyAsync(ex->tile_flags.p, flags.data(), flags.size(), cudaMemcpyHostToDevice, st));
        CUDA_CHECK(cudaStreamSynchronize(st));                     // `flags` is a host temporary
        ex->tile_flags_valid = true;
    }
    CUDA_CHECK(cudaMemcpyAsync(ex->cams.p, cams, sizeof(mcs_ocam) * n_cams, cudaMemcpyHostToDevice, st));
    if ((ex->p.do_dbrief || ex->p.learn_masks) &&
        ((int)ex->lut_cams.size() != n_cams || std::memcmp(ex->lut_cams.data(), cams, sizeof(mcs_ocam) * n_cams) != 0)) {
        std::vector<double> all;
        std::vector<size_t> offs(n_cams);
        std::vector<int> ns(n_cams);
        for (int c = 0; c < n_cams; ++c) {
            std::vector<double> coef;
            build_distort_lut(cams[c], coef, ns[c]);
            offs[c] = all.size();
            all.insert(all.end(), coef.begin(), coef.end());
        }
        CUDA_CHECK(cudaStreamSynchronize(st));                 // a previous call may still read the old tables
        CUDA_CHECK(ex->lut_coef.ensure(all.size()));
        CUDA_CHECK(ex->luts.ensure(n_cams));
        std::vector<DistortLut> h(n_cams);
        for (int c = 0; c < n_cams; ++c) h[c] = DistortLut{ex->lut_coef.p + offs[c], ns[c], 1.0};
        CUDA_CHECK(cudaMemcpyAsync(ex->lut_coef.p, all.data(), all.size() * sizeof(double), cudaMemcpyHostToDevice, st));
        CUDA_CHECK(cudaMemcpyAsync(ex->luts.p, h.data(), sizeof(DistortLut) * n_cams, cudaMemcpyHostToDevice, st));
        CUDA_CHECK(cudaStreamSynchronize(st));                 // host staging vectors die here
        ex->lut_cams.assign(cams, cams + n_cams);
    }
    CUDA_CHECK(cudaMemsetAsync(ex->status.p, 0, sizeof(int), st));

    return MCS_OK;
}

constexpr int kGraphMaxImages = 16;      // batches up to this size take the per-frame path (pinned staging, CUDA graph)

// K1 (per level) -> K2 -> K3 on `st`: kernel launches and memsets only (no allocation, no host synchronisation, no pageable
// copy), so the sequence can be stream-captured into a CUDA graph.
int enqueue_kernels(mcs_extractor* ex, int n_images, const uint8_t* images_dev, int W, int H, int stride, const int* coi_d,
                    const FeatureView& out, int capacity, cudaStream_t st) {
    const PyramidGeom& G = ex->G;
    ex->coi_last = coi_d;
    CUDA_CHECK(cudaMemsetAsync(ex->raw_count.p, 0, sizeof(int) * n_images * G.nlevels, st));
    if (ex->profiling) CUDA_CHECK(cudaEventRecord(ex->ev[0], st));
    for (int l = 0; l < G.nlevels; ++l) {
        const uint8_t* src = l ? ex->lvl[l - 1].p : images_dev;
        const size_t src_bytes = l ? G.lv[l - 1].img_bytes : (size_t)stride * H;
        CUDA_CHECK(launch_pyr_fast(G, l, n_images, src, src_bytes, ex->lvl[l].p, ex->blur[l].p, ex->masks.p, W, (size_t)W * H,
                                   coi_d, ex->tile_flags.p, ex->raw.p, ex->raw_count.p, st));
    }
    CUDA_CHECK(cudaGetLastError());
    if (ex->profiling) CUDA_CHECK(cudaEventRecord(ex->ev[1], st));
    // (K2 forked per level onto a second stream behind K1 of the same level was slower for the per-frame path: the per-level
    // launches serialise on that stream, while the single launch runs its 8 x n CTAs side by side)
    CUDA_CHECK(launch_octree(G, ex->G_dev.p, n_images, ex->raw.p, ex->raw_count.p, ex->node_of.p, ex->sel_xys.p, ex->sel_count.p,
                             ex->status.p, st));
    CUDA_CHECK(cudaGetLastError());
    if (ex->profiling) CUDA_CHECK(cudaEventRecord(ex->ev[2], st));
    DescribeArgs a;
    for (int l = 0; l < kMaxLevels; ++l) { a.lvl[l] = ex->lvl[l].p; a.blur[l] = ex->blur[l].p; }
    a.tier_stats = ex->tier_on ? ex->tier.p : nullptr;
    CUDA_CHECK(launch_describe(G, ex->G_dev.p, n_images, a, ex->cams.p, ex->luts.p, coi_d, ex->sel_xys.p, ex->sel_count.p,
                               out.kps, out.desc, out.dmask, out.counts, capacity, st));
    if (ex->profiling) CUDA_CHECK(cudaEventRecord(ex->ev[3], st));
    ex->last_n_images = n_images;
    return MCS_OK;
}

// Validation, geometry, buffer growth and the small host inputs of one call (everything that may allocate, synchronise or read
// pageable host memory).  `batch_images` sizes the per-launch buffers; the camera-of-image table (`n_coi` entries, one per image
// of the call) goes to ex->cam_of_image, which every launch of the call reads from its first image on.
int prepare_inputs(mcs_extractor* ex, int batch_images, int W, int H, int stride, const uint8_t* masks, const mcs_ocam* cams, int n_cams,
                   const int* cam_of_image, int n_coi, cudaStream_t st) {
    if (n_cams < 1 || n_cams > 64) return mcs_fail(MCS_ERR_INVALID, "n_cams must be in [1,64]");
    for (int i = 0; i < n_coi; ++i)
        if (cam_of_image[i] < 0 || cam_of_image[i] >= n_cams) return mcs_fail(MCS_ERR_INVALID, "cam_of_image out of range");
    int rc = build_geometry(ex, W, H, stride);
    if (rc) return rc;
    rc = ensure_batch(ex, batch_images);
    if (rc) return rc;
    CUDA_CHECK(ex->cam_of_image.ensure(n_coi));
    rc = upload_small_inputs(ex, W, H, masks, cams, n_cams, st);
    if (rc) return rc;
    CUDA_CHECK(cudaMemcpyAsync(ex->cam_of_image.p, cam_of_image, sizeof(int) * n_coi, cudaMemcpyHostToDevice, st));
    ex->sf_valid = false;            // shared state (camera table, masks, tables) may now differ from what the cached graph assumes
    return MCS_OK;
}

// the overflow flags K1 / K2 leave in the status word
int status_error(int s) {
    if (s & 1) return mcs_fail(MCS_ERR_CAPACITY, "raw corner list overflow");
    if (s & 2) return mcs_fail(MCS_ERR_CAPACITY, "octree node table overflow");
    if (s & 4) return mcs_fail(MCS_ERR_CAPACITY, "selected keypoint slots overflow");
    return MCS_OK;
}

int check_status(mcs_extractor* ex, cudaStream_t st) {
    int s = 0;
    CUDA_CHECK(cudaMemcpyAsync(&s, ex->status.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    return status_error(s);
}

// the checks every extract entry point makes after its own null-argument list (`count`: images, or frames of the stream calls)
int check_extract_args(const mcs_extractor* ex, int count, int W, int H, int stride, int capacity, const void* dmask) {
    if (count < 1 || W < 1 || H < 1 || stride < W) return mcs_fail(MCS_ERR_INVALID, "bad image geometry");
    if (capacity < ex->capacity) return mcs_fail(MCS_ERR_CAPACITY, "capacity below mcs_extractor_info.capacity");
    if (ex->p.learn_masks && !dmask) return mcs_fail(MCS_ERR_INVALID, "dmask buffer required when learn_masks is set");
    return MCS_OK;
}

// the extractor's own feature buffers, grown to n images
int own_features(mcs_extractor* ex, int n, int capacity, FeatureView* v) {
    const size_t slots = (size_t)n * capacity, bytes = slots * ex->p.desc_size;
    CUDA_CHECK(ex->kps.ensure(slots));
    CUDA_CHECK(ex->desc.ensure(bytes));
    CUDA_CHECK(ex->dmask.ensure(bytes));
    CUDA_CHECK(ex->counts.ensure(n));
    *v = FeatureView{ex->counts.p, ex->kps.p, ex->desc.p, ex->dmask.p};
    return MCS_OK;
}

// device -> host copies of n images' counts, keypoints, descriptors and, when `with_dmask`, descriptor masks
int copy_features(const FeatureView& dst, const FeatureView& src, int n, int capacity, int ds, bool with_dmask, cudaStream_t st) {
    const size_t slots = (size_t)n * capacity;
    CUDA_CHECK(cudaMemcpyAsync(dst.counts, src.counts, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaMemcpyAsync(dst.kps, src.kps, sizeof(mcs_keypoint) * slots, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaMemcpyAsync(dst.desc, src.desc, slots * ds, cudaMemcpyDeviceToHost, st));
    if (with_dmask) CUDA_CHECK(cudaMemcpyAsync(dst.dmask, src.dmask, slots * ds, cudaMemcpyDeviceToHost, st));
    return MCS_OK;
}

bool g_consts_uploaded[64] = {};
std::mutex g_mu;

int upload_consts_once(int dev) {
    std::lock_guard<std::mutex> lk(g_mu);
    if (dev < 64 && g_consts_uploaded[dev]) return MCS_OK;
    // the 845 offsets of the IC_Angle disc, umax as in ref :187-202
    int umax[kHalfPatch + 1];
    const int vmax = cv_floor(kHalfPatch * std::sqrt(2.f) / 2 + 1);
    const int vmin = cv_ceil(kHalfPatch * std::sqrt(2.f) / 2);
    for (int v = 0; v <= vmax; ++v) umax[v] = cv_round(std::sqrt((double)kHalfPatch * kHalfPatch - v * v));
    for (int v = kHalfPatch, v0 = 0; v >= vmin; --v) {
        while (umax[v0] == umax[v0 + 1]) ++v0;
        umax[v] = v0;
        ++v0;
    }
    // the disc is symmetric in u and v, so umax[] gives both the row widths and the column heights
    signed char du[848] = {0}, dv[848] = {0};
    int n = 0;
    for (int v = -kHalfPatch; v <= kHalfPatch; ++v) n += 2 * (v == 0 ? kHalfPatch : umax[std::abs(v)]) + 1;
    if (n != 845) return mcs_fail(MCS_ERR_INVALID, "disc table size");
    for (int v = 0; v <= kHalfPatch; ++v) {
        du[v] = (signed char)(v == 0 ? kHalfPatch : umax[v]);
        // symmetry check: column |u| = v must hold rows |v'| <= umax[v]
        for (int w = 0; w <= kHalfPatch; ++w)
            if ((w <= (v == 0 ? kHalfPatch : umax[v])) != (v <= (w == 0 ? kHalfPatch : umax[w])))
                return mcs_fail(MCS_ERR_INVALID, "IC_Angle disc is not symmetric");
    }
    CUDA_CHECK(upload_constants(kPairs, du, dv));
    if (dev < 64) g_consts_uploaded[dev] = true;
    return MCS_OK;
}

}  // namespace

// ================================================================================================
extern "C" {

const char* mcs_last_error(void) { return g_err.c_str(); }

int mcs_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    int ok = 0;
    for (int i = 0; i < n; ++i) {
        int major = 0;
        if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, i) == cudaSuccess && major == 9) ++ok;
    }
    return ok;
}

void mcs_params_default(mcs_extractor_params* p) {
    if (!p) return;
    *p = mcs_extractor_params{1000, 1.2f, 8, 25, 0, 0, 32, 20, 0, 2, 0, 0, 32};
}

void mcs_cam_world_to_img(const mcs_ocam* cam, double x, double y, double z, double* u, double* v) {
    cam_world_to_img(*cam, x, y, z, *u, *v);
}
void mcs_cam_img_to_world(const mcs_ocam* cam, double u, double v, double* x, double* y, double* z) {
    cam_img_to_world(*cam, u, v, *x, *y, *z);
}
int mcs_cam_mirror_mask(const mcs_ocam* cam, uint8_t* out) {
    if (!cam || !out) return mcs_fail(MCS_ERR_INVALID, "null argument");
    const int w = cam->width, h = cam->height;
    if (cam->mirror_mask != 1) { std::memset(out, 1, (size_t)w * h); return MCS_OK; }
    // ref src/cam_model_omni.cpp:187-188 swaps the names on purpose (SURVEY Appendix C.9)
    const float u0 = (float)cam->v0, v0 = (float)cam->u0;
    for (int i = 0; i < h; ++i)
        for (int j = 0; j < w; ++j) {
            const float a = (float)std::pow(i - u0, 2), b = (float)std::pow(j - v0, 2);
            out[(size_t)i * w + j] = std::sqrt(a + b) < (u0 + 22.0f) ? 255 : 0;
        }
    return MCS_OK;
}

int mcs_extractor_create(const mcs_extractor_params* p, mcs_extractor** out) {
    if (!p || !out) return mcs_fail(MCS_ERR_INVALID, "null argument");
    *out = nullptr;
    std::unique_ptr<mcs_extractor> ex(new mcs_extractor);
    if (int rc = init_tables(ex.get(), p)) return rc;
    int dev = 0;
    {
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) { cudaGetLastError(); return mcs_fail(MCS_ERR_NO_DEVICE, std::string("no CUDA device: ") + cudaGetErrorString(e)); }
        int major = 0;
        cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
        if (major != 9) return mcs_fail(MCS_ERR_NO_DEVICE, "device is not sm_90 (H100); this library has no other code path");
    }
    int rc = upload_consts_once(dev);
    if (rc) return rc;
    ex->device = dev;
    if (cudaStreamCreateWithFlags(&ex->stream, cudaStreamNonBlocking) != cudaSuccess)
        return mcs_fail(MCS_ERR_CUDA, "cudaStreamCreate failed");
    *out = ex.release();
    return MCS_OK;
}

int mcs_extractor_octree_plan(const mcs_extractor_params* p, int32_t width, int32_t height, int32_t* node_table, int32_t* nodes_ini,
                              int32_t* sel_cap, int32_t* capacity) {
    if (!p || !node_table || !nodes_ini || !sel_cap || !capacity) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (width < 1 || height < 1) return mcs_fail(MCS_ERR_INVALID, "bad image geometry");
    mcs_extractor ex;
    if (int rc = init_tables(&ex, p)) return rc;
    std::vector<int16_t> blob;
    LutOffsets off[kMaxLevels];
    const int rc = plan_geometry(&ex, width, height, width, blob, off);
    *node_table = ex.G.node_cap; *capacity = ex.capacity;
    for (int l = 0; l < p->nlevels; ++l) { nodes_ini[l] = ex.G.lv[l].nodes_ini; sel_cap[l] = ex.G.lv[l].sel_cap; }
    return rc;
}

void mcs_extractor_destroy(mcs_extractor* ex) {
    if (!ex) return;
    cudaSetDevice(ex->device);      // the DevBuf members free their memory when `ex` is deleted, on this device
    if (ex->sf_exec) cudaGraphExecDestroy(ex->sf_exec);
    if (ex->pin_in) cudaFreeHost(ex->pin_in);
    if (ex->pin_out) cudaFreeHost(ex->pin_out);
    for (int i = 0; i < 4; ++i) if (ex->ev[i]) cudaEventDestroy(ex->ev[i]);
    if (ex->s_copy) cudaStreamDestroy(ex->s_copy);
    if (ex->s_match) cudaStreamDestroy(ex->s_match);
    if (ex->s_out) cudaStreamDestroy(ex->s_out);
    if (ex->stream) cudaStreamDestroy(ex->stream);
    delete ex;
}

int mcs_extractor_get_info(const mcs_extractor* ex, mcs_extractor_info* info) {
    if (!ex || !info) return mcs_fail(MCS_ERR_INVALID, "null argument");
    std::memset(info, 0, sizeof(*info));
    info->nlevels = ex->p.nlevels; info->capacity = ex->capacity; info->desc_size = ex->p.desc_size;
    for (int l = 0; l < ex->p.nlevels; ++l) {
        info->features_per_level[l] = ex->quota[l];
        info->scale_factor[l] = ex->sf[l];
        info->inv_scale_factor[l] = ex->isf[l];
    }
    return MCS_OK;
}

int mcs_extract_batch_device(mcs_extractor* ex, int32_t n_images, const uint8_t* images_dev, int32_t width, int32_t height,
                             int32_t stride, const uint8_t* masks, const mcs_ocam* cams, int32_t n_cams,
                             const int32_t* cam_of_image, mcs_keypoint* kps_dev, uint8_t* desc_dev, uint8_t* dmask_dev,
                             int32_t* counts_dev, int32_t capacity, void* stream) {
    if (!ex || !images_dev || !masks || !cams || !cam_of_image || !kps_dev || !desc_dev || !counts_dev)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (int rc = check_extract_args(ex, n_images, width, height, stride, capacity, dmask_dev)) return rc;
    CUDA_CHECK(cudaSetDevice(ex->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ex->stream;
    int rc = prepare_inputs(ex, n_images, width, height, stride, masks, cams, n_cams, cam_of_image, n_images, st);
    if (rc == MCS_OK)
        rc = enqueue_kernels(ex, n_images, images_dev, width, height, stride, ex->cam_of_image.p,
                             FeatureView{counts_dev, kps_dev, desc_dev, dmask_dev}, capacity, st);
    if (rc) return rc;
    if (!stream) return check_status(ex, st);
    return MCS_OK;
}

namespace {

int pin_ensure(uint8_t*& p, size_t& cap, size_t need, bool* moved) {
    if (need <= cap) return MCS_OK;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    CUDA_CHECK(cudaMallocHost((void**)&p, need));
    cap = need; *moved = true;
    return MCS_OK;
}

constexpr size_t kStatusHeader = 256;    // pinned output staging: the status word, then the feature sections (mcs_packed_layout)

// copy-in, re-pitch, K1..K3, copy-out of one small call between the extractor's pinned staging buffers: capturable
int enqueue_small(mcs_extractor* ex, int n, int W, int H, int stride, int dpitch, const FeatureView& own, int capacity, bool with_dmask,
                  cudaStream_t st) {
    const int ds = ex->p.desc_size;
    CUDA_CHECK(cudaMemcpyAsync(ex->in_tight.p, ex->pin_in, (size_t)stride * H * n, cudaMemcpyHostToDevice, st));
    launch_repitch(ex->in_tight.p, stride, ex->in_images.p, dpitch, W, (size_t)H * n, st);
    CUDA_CHECK(cudaMemsetAsync(ex->status.p, 0, sizeof(int), st));
    int rc = enqueue_kernels(ex, n, ex->in_images.p, W, H, dpitch, ex->cam_of_image.p, own, capacity, st);
    if (rc) return rc;
    CUDA_CHECK(cudaMemcpyAsync(ex->pin_out, ex->status.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    return copy_features(packed_view(ex->pin_out + kStatusHeader, n, capacity, ds), own, n, capacity, ds, with_dmask, st);
}

// A call of at most kGraphMaxImages host images (what cMultiFrame's constructor issues per frame): pinned staging on both sides,
// and the whole sequence as one graph launch once the inputs repeat.  `own`: the extractor's feature buffers, `out`: the caller's.
int extract_small(mcs_extractor* ex, int n_images, const uint8_t* images, int width, int height, int stride, int dpitch,
                  const uint8_t* masks, const mcs_ocam* cams, int n_cams, const int* cam_of_image, const FeatureView& own,
                  const FeatureView& out, int capacity) {
    cudaStream_t st = ex->stream;
    const int ds = ex->p.desc_size;
    const bool dm = out.dmask != nullptr;
    const size_t in_bytes = (size_t)stride * height * n_images, mbytes = (size_t)n_cams * width * height;
    bool moved = false;
    int rc = pin_ensure(ex->pin_in, ex->pin_in_bytes, in_bytes, &moved);
    if (rc) return rc;
    rc = pin_ensure(ex->pin_out, ex->pin_out_bytes, kStatusHeader + mcs_packed_layout(n_images, capacity, ds, nullptr), &moved);
    if (rc) return rc;
    if (moved) ex->sf_valid = false;
    // the caller's last row may hold only `width` valid bytes (a cv::Mat ROI with step > width at the end of its allocation)
    std::memcpy(ex->pin_in, images, in_bytes - (size_t)(stride - width));
    const mcs_extractor::SfKey& k = ex->sf_key;
    bool hit = ex->sf_valid && ex->sf_exec && k.n == n_images && k.w == width && k.h == height && k.stride == stride &&
               k.capacity == capacity && k.dm == dm && (int)k.cams.size() == n_cams &&
               std::memcmp(k.coi.data(), cam_of_image, sizeof(int) * n_images) == 0 &&
               std::memcmp(k.cams.data(), cams, sizeof(mcs_ocam) * n_cams) == 0 && ex->masks_host.size() == mbytes;
    if (hit) {
        // the graph goes first and the 1 MB mask comparison runs while the GPU works; if the masks did change the result
        // is thrown away and the call starts over on the eager path (which uploads the new masks)
        CUDA_CHECK(cudaGraphLaunch(ex->sf_exec, st));
        if (std::memcmp(ex->masks_host.data(), masks, mbytes) != 0) {
            CUDA_CHECK(cudaStreamSynchronize(st));
            hit = false;
        } else {
            ++ex->sf_replays;
        }
    }
    if (!hit) {
        rc = prepare_inputs(ex, n_images, width, height, dpitch /* K1 reads the re-pitched copy */, masks, cams, n_cams, cam_of_image,
                            n_images, st);
        if (rc) return rc;
        rc = enqueue_small(ex, n_images, width, height, stride, dpitch, own, capacity, dm, st);
        if (rc) return rc;
        // record the same sequence for the next call with these inputs (capture executes nothing)
        if (ex->sf_exec) { cudaGraphExecDestroy(ex->sf_exec); ex->sf_exec = nullptr; }
        cudaGraph_t graph = nullptr;
        if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
            const int crc = enqueue_small(ex, n_images, width, height, stride, dpitch, own, capacity, dm, st);
            const cudaError_t ce = cudaStreamEndCapture(st, &graph);
            if (crc == MCS_OK && ce == cudaSuccess && graph && cudaGraphInstantiate(&ex->sf_exec, graph, 0) == cudaSuccess) {
                mcs_extractor::SfKey& nk = ex->sf_key;
                nk.n = n_images; nk.w = width; nk.h = height; nk.stride = stride; nk.capacity = capacity;
                nk.coi.assign(cam_of_image, cam_of_image + n_images);
                nk.cams.assign(cams, cams + n_cams);
                nk.dm = dm;
                ex->sf_valid = true;
            } else {
                ex->sf_exec = nullptr;
                cudaGetLastError();          // a failed capture only costs the shortcut
            }
            if (graph) cudaGraphDestroy(graph);
        } else {
            cudaGetLastError();
        }
    }
    CUDA_CHECK(cudaStreamSynchronize(st));
    rc = status_error(*(const int*)ex->pin_out);
    if (rc) return rc;
    const FeatureView pin = packed_view(ex->pin_out + kStatusHeader, n_images, capacity, ds);
    for (int i = 0; i < n_images; ++i) {
        const size_t nused = (size_t)std::min(std::max(pin.counts[i], 0), capacity);
        const FeatureView s = feature_at(pin, i, capacity, ds), d = feature_at(out, i, capacity, ds);
        out.counts[i] = pin.counts[i];
        std::memcpy(d.kps, s.kps, nused * sizeof(mcs_keypoint));
        std::memcpy(d.desc, s.desc, nused * ds);
        if (dm) std::memcpy(d.dmask, s.dmask, nused * ds);
    }
    return MCS_OK;
}

}  // namespace

int mcs_extract_batch(mcs_extractor* ex, int32_t n_images, const uint8_t* images, int32_t width, int32_t height, int32_t stride,
                      const uint8_t* masks, const mcs_ocam* cams, int32_t n_cams, const int32_t* cam_of_image,
                      mcs_keypoint* kps_out, uint8_t* desc_out, uint8_t* dmask_out, int32_t* counts_out, int32_t capacity) {
    if (!ex || !images || !masks || !cams || !cam_of_image || !kps_out || !desc_out || !counts_out)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (int rc = check_extract_args(ex, n_images, width, height, stride, capacity, dmask_out)) return rc;
    CUDA_CHECK(cudaSetDevice(ex->device));
    cudaStream_t st = ex->stream;
    // device staging with a 64-byte-aligned pitch so that K1 can use 128-bit loads
    const int dpitch = (width + 63) & ~63;
    const size_t img_bytes = (size_t)dpitch * height;
    const void* before[6] = {ex->in_images.p, ex->kps.p, ex->desc.p, ex->dmask.p, ex->counts.p, ex->in_tight.p};
    CUDA_CHECK(ex->in_images.ensure(img_bytes * n_images + 256));
    FeatureView own;
    int rc = own_features(ex, n_images, capacity, &own);
    if (rc) return rc;
    // linear H2D + device re-pitch (a 2-D DMA of short rows is several times slower)
    CUDA_CHECK(ex->in_tight.ensure((size_t)stride * height * n_images + 256));
    const void* after[6] = {ex->in_images.p, ex->kps.p, ex->desc.p, ex->dmask.p, ex->counts.p, ex->in_tight.p};
    if (std::memcmp(before, after, sizeof(before)) != 0) ex->sf_valid = false;     // the cached graph reads these buffers
    const FeatureView out{counts_out, kps_out, desc_out, dmask_out};
    if (n_images <= kGraphMaxImages && !ex->profiling && !ex->tier_on)
        return extract_small(ex, n_images, images, width, height, stride, dpitch, masks, cams, n_cams, cam_of_image, own, out, capacity);

    CUDA_CHECK(cudaMemcpyAsync(ex->in_tight.p, images, (size_t)stride * height * n_images - (size_t)(stride - width), cudaMemcpyHostToDevice, st));
    launch_repitch(ex->in_tight.p, stride, ex->in_images.p, dpitch, width, (size_t)height * n_images, st);
    rc = prepare_inputs(ex, n_images, width, height, dpitch, masks, cams, n_cams, cam_of_image, n_images, st);
    if (rc == MCS_OK) rc = enqueue_kernels(ex, n_images, ex->in_images.p, width, height, dpitch, ex->cam_of_image.p, own, capacity, st);
    if (rc == MCS_OK) rc = copy_features(out, own, n_images, capacity, ex->p.desc_size, dmask_out != nullptr, st);
    if (rc) return rc;
    return check_status(ex, st);
}

int mcs_extract(mcs_extractor* ex, const uint8_t* image, int32_t width, int32_t height, int32_t stride, const uint8_t* mask,
                int32_t mask_stride, const mcs_ocam* cam, mcs_keypoint* kps_out, uint8_t* desc_out, uint8_t* dmask_out,
                int32_t capacity, int32_t* n_out) {
    if (!ex || !n_out) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (!image) return MCS_OK;   // empty image: silent return, outputs untouched (ref :1252-1253)
    if (!mask || !cam) return mcs_fail(MCS_ERR_INVALID, "a mask and a camera model are mandatory (ref :913-917 throws on an empty mask)");
    std::vector<uint8_t> packed;
    const uint8_t* m = mask;
    if (mask_stride != width) {
        packed.resize((size_t)width * height);
        for (int y = 0; y < height; ++y) std::memcpy(packed.data() + (size_t)y * width, mask + (size_t)y * mask_stride, width);
        m = packed.data();
    }
    const int zero = 0;
    int count = 0;
    // the batch entry point writes `capacity` slots per image; here slot 0 is the caller's buffer
    int rc = mcs_extract_batch(ex, 1, image, width, height, stride, m, cam, 1, &zero, kps_out, desc_out, dmask_out, &count, capacity);
    if (rc) return rc;
    *n_out = count;
    return MCS_OK;
}

int mcs_extractor_debug_read(mcs_extractor* ex, int32_t image_index, int32_t level, int32_t what, void* out, size_t out_bytes,
                             int32_t* w_out, int32_t* h_out) {
    if (!ex || !out || !w_out || !h_out) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (level < 0 || level >= ex->G.nlevels || image_index < 0 || image_index >= ex->last_n_images)
        return mcs_fail(MCS_ERR_INVALID, "bad level / image index");
    CUDA_CHECK(cudaSetDevice(ex->device));
    const LevelGeom& g = ex->G.lv[level];
    const int L = ex->G.nlevels;
    if (what == 0 || what == 1) {
        *w_out = g.w; *h_out = g.h;
        if (out_bytes < (size_t)g.w * g.h) return mcs_fail(MCS_ERR_CAPACITY, "buffer too small");
        const uint8_t* src = (what == 0 ? ex->lvl[level].p : ex->blur[level].p) + (size_t)image_index * g.img_bytes;
        CUDA_CHECK(cudaMemcpy2D(out, g.w, src, g.pitch, g.w, g.h, cudaMemcpyDeviceToHost));
        return MCS_OK;
    }
    if (what == 2) {   // the mask pyramid is never materialised: evaluate the composed nearest-neighbour maps
        *w_out = g.w; *h_out = g.h;
        if (out_bytes < (size_t)g.w * g.h) return mcs_fail(MCS_ERR_CAPACITY, "buffer too small");
        std::vector<int16_t> mx(g.w), my(g.h);
        std::vector<int> coi(ex->last_n_images);
        CUDA_CHECK(cudaMemcpy(mx.data(), g.mx0, g.w * 2, cudaMemcpyDeviceToHost));
        CUDA_CHECK(cudaMemcpy(my.data(), g.my0, g.h * 2, cudaMemcpyDeviceToHost));
        CUDA_CHECK(cudaMemcpy(coi.data(), ex->coi_last, sizeof(int) * ex->last_n_images, cudaMemcpyDeviceToHost));
        std::vector<uint8_t> m0((size_t)ex->G.width * ex->G.height);
        CUDA_CHECK(cudaMemcpy(m0.data(), ex->masks.p + (size_t)coi[image_index] * m0.size(), m0.size(), cudaMemcpyDeviceToHost));
        for (int y = 0; y < g.h; ++y)
            for (int x = 0; x < g.w; ++x) ((uint8_t*)out)[(size_t)y * g.w + x] = m0[(size_t)my[y] * ex->G.width + mx[x]];
        return MCS_OK;
    }
    if (what == 3) {   // raw corners, sorted into the reference order (cell-row-major, then pixel-row-major)
        int n = 0;
        CUDA_CHECK(cudaMemcpy(&n, ex->raw_count.p + (size_t)image_index * L + level, sizeof(int), cudaMemcpyDeviceToHost));
        n = std::min(n, g.raw_cap);
        *w_out = n; *h_out = 3;
        if (out_bytes < (size_t)n * 12) return mcs_fail(MCS_ERR_CAPACITY, "buffer too small");
        std::vector<uint32_t> c(n);
        CUDA_CHECK(cudaMemcpy(c.data(), ex->raw.p + (size_t)image_index * ex->G.raw_total + g.raw_off, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost));
        auto key = [&](uint32_t v) {
            const int x = corner_x(v) - kEdge, y = corner_y(v) - kEdge;
            const int cj = x / g.w_cell, ci = y / g.h_cell;
            return (long long)(ci * g.n_cols + cj) * g.w_cell * g.h_cell + (y - ci * g.h_cell) * g.w_cell + (x - cj * g.w_cell);
        };
        std::sort(c.begin(), c.end(), [&](uint32_t a, uint32_t b) { return key(a) < key(b); });
        int32_t* o = (int32_t*)out;
        for (int i = 0; i < n; ++i) { o[3 * i] = corner_x(c[i]); o[3 * i + 1] = corner_y(c[i]); o[3 * i + 2] = corner_s(c[i]); }
        return MCS_OK;
    }
    return mcs_fail(MCS_ERR_INVALID, "unknown `what`");
}

int mcs_extractor_set_profiling(mcs_extractor* ex, int32_t enable) {
    if (!ex) return mcs_fail(MCS_ERR_INVALID, "null argument");
    CUDA_CHECK(cudaSetDevice(ex->device));
    if (enable) for (int i = 0; i < 4; ++i) if (!ex->ev[i]) CUDA_CHECK(cudaEventCreate(&ex->ev[i]));
    ex->profiling = enable != 0;
    return MCS_OK;
}

int mcs_extractor_tier_stats(mcs_extractor* ex, int32_t enable, int64_t* counts4) {
    if (!ex) return mcs_fail(MCS_ERR_INVALID, "null extractor");
    CUDA_CHECK(cudaSetDevice(ex->device));
    CUDA_CHECK(cudaDeviceSynchronize());
    if (counts4) {
        counts4[0] = counts4[1] = counts4[2] = counts4[3] = 0;
        if (ex->tier_on) CUDA_CHECK(cudaMemcpy(counts4, ex->tier.p, 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    }
    if (enable && !ex->tier_on) {
        CUDA_CHECK(ex->tier.ensure(4));
        CUDA_CHECK(cudaMemset(ex->tier.p, 0, 4 * sizeof(unsigned long long)));
    }
    ex->tier_on = enable != 0;
    return MCS_OK;
}

int mcs_extractor_check_status(mcs_extractor* ex, void* stream) {
    if (!ex) return mcs_fail(MCS_ERR_INVALID, "null extractor");
    if (!ex->status.p) return MCS_OK;                       // nothing has run yet
    CUDA_CHECK(cudaSetDevice(ex->device));
    return check_status(ex, stream ? (cudaStream_t)stream : ex->stream);
}

int mcs_cam_distort_table(const mcs_ocam* cam, double* rows_out, int32_t max_rows, int32_t* n_rows, int32_t* row_doubles) {
    if (!cam || !n_rows || !row_doubles) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (rows_out && max_rows < 0) return mcs_fail(MCS_ERR_INVALID, "negative max_rows");
    std::vector<double> coef;
    int n = 0;
    build_distort_lut(*cam, coef, n);
    *n_rows = n;
    *row_doubles = n > 0 ? (int32_t)(coef.size() / (size_t)n) : 0;
    if (rows_out && n > 0) std::memcpy(rows_out, coef.data(), sizeof(double) * (size_t)std::min(n, (int)max_rows) * (size_t)*row_doubles);
    return MCS_OK;
}

int mcs_extractor_graph_replays(mcs_extractor* ex, int64_t* n) {
    if (!ex || !n) return mcs_fail(MCS_ERR_INVALID, "null argument");
    *n = ex->sf_replays;
    return MCS_OK;
}

int mcs_extractor_get_timings(mcs_extractor* ex, float* ms3) {
    if (!ex || !ms3) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (!ex->profiling || !ex->ev[3]) return mcs_fail(MCS_ERR_INVALID, "profiling is not enabled");
    CUDA_CHECK(cudaEventSynchronize(ex->ev[3]));
    for (int i = 0; i < 3; ++i) CUDA_CHECK(cudaEventElapsedTime(&ms3[i], ex->ev[i], ex->ev[i + 1]));
    return MCS_OK;
}

}  // extern "C"

static int extract_match_stream_impl(mcs_extractor* ex, int32_t n_frames, int32_t n_cams, const uint8_t* images, int32_t width,
                             int32_t height, int32_t stride, const uint8_t* masks, const mcs_ocam* cams, mcs_keypoint* kps_out,
                             uint8_t* desc_out, uint8_t* dmask_out, int32_t* counts_out, int32_t capacity, int32_t K,
                             int32_t* match_idx_out, int32_t* match_dist_out, void* packed_dev, int32_t th_low = 0, double nnratio = 0.0,
                             int32_t* matches12_out = nullptr, int32_t* nmatches_out = nullptr, int32_t* redo_out = nullptr) {
    if (!ex || !images || !masks || !cams || !kps_out || !desc_out || !counts_out || !match_idx_out || !match_dist_out)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    // both n_frames and n_cams must be positive
    if (int rc = check_extract_args(ex, std::min(n_frames, n_cams), width, height, stride, capacity, dmask_out)) return rc;
    if (K < 1 || K > 8) return mcs_fail(MCS_ERR_INVALID, "K must be 1..8");
    const bool replay = matches12_out != nullptr;
    if (replay && (!nmatches_out || !redo_out)) return mcs_fail(MCS_ERR_INVALID, "the greedy acceptance needs all three outputs");
    CUDA_CHECK(cudaSetDevice(ex->device));
    cudaStream_t st = ex->stream;
    if (!ex->s_copy) CUDA_CHECK(cudaStreamCreateWithFlags(&ex->s_copy, cudaStreamNonBlocking));
    if (!ex->s_out) CUDA_CHECK(cudaStreamCreateWithFlags(&ex->s_out, cudaStreamNonBlocking));
    if (!ex->s_match) CUDA_CHECK(cudaStreamCreateWithFlags(&ex->s_match, cudaStreamNonBlocking));
    const int n_images = n_frames * n_cams, ds = ex->p.desc_size;
    const int dpitch = (width + 63) & ~63;
    // Software pipeline over chunks of frames: H2D (copy stream) | re-pitch + K1..K3 + matching (compute stream) |
    // D2H (output stream).  The chunk inputs are copied linearly and re-pitched on the device.
    // Chunk plan: at most 4 chunks of >= 8 frames (every kernel stays above one wave); with >= 32 frames the first chunk is
    // a short one (1/16 of the stream) so that the un-overlapped head -- its H2D copy -- is short too.
    std::vector<int> chunk_lo;                                        // first frame of every chunk, + n_frames
    if (n_frames >= 32) {
        const int first = std::max(4, n_frames / 16), rest = n_frames - first, each = (rest + 2) / 3;
        chunk_lo = {0, first, std::min(first + each, n_frames), std::min(first + 2 * each, n_frames), n_frames};
    } else {
        const int nc = std::min(std::max(n_frames / 8, 1), 4), each = (n_frames + nc - 1) / nc;
        for (int c = 0; c <= nc; ++c) chunk_lo.push_back(std::min(c * each, n_frames));
    }
    const int n_chunks = (int)chunk_lo.size() - 1;
    int fpc = 0;
    for (int c = 0; c < n_chunks; ++c) fpc = std::max(fpc, chunk_lo[c + 1] - chunk_lo[c]);
    const int ipc = fpc * n_cams;                                     // images in the largest chunk
    const size_t tight_img = (size_t)stride * height, pitched_img = (size_t)dpitch * height;
    std::vector<int> coi(n_images);
    for (int i = 0; i < n_images; ++i) coi[i] = i % n_cams;
    // validated before the stream's own buffers grow (a refused call leaves the cached per-frame graph usable), uploaded before
    // the first image copy (see upload_small_inputs)
    if (int rc = prepare_inputs(ex, ipc, width, height, dpitch, masks, cams, n_cams, coi.data(), n_images, st)) return rc;
    CUDA_CHECK(ex->in_tight.ensure(2 * tight_img * ipc + 256));
    CUDA_CHECK(ex->in_images.ensure(pitched_img * ipc + 256));
    // feature buffers: the extractor's own, or the caller's packed exchange buffer (mcs_packed_layout) when one is given
    FeatureView feat;
    if (packed_dev) feat = packed_view(packed_dev, n_images, capacity, ds);
    else if (int rc = own_features(ex, n_images, capacity, &feat)) return rc;
    const FeatureView host{counts_out, kps_out, desc_out, dmask_out};
    CUDA_CHECK(ex->match_idx.ensure((size_t)n_images * capacity * K));
    CUDA_CHECK(ex->match_dist.ensure((size_t)n_images * capacity * K));
    if (replay) {
        CUDA_CHECK(ex->m12.ensure((size_t)n_images * capacity)); CUDA_CHECK(ex->nmat.ensure(n_images)); CUDA_CHECK(ex->redo.ensure(n_images));
    }
    struct Events {                       // destroyed on every path out of this function
        std::vector<cudaEvent_t> v;
        ~Events() { for (cudaEvent_t e : v) cudaEventDestroy(e); }
        cudaError_t add(cudaEvent_t* out, unsigned flags) {
            cudaError_t e = cudaEventCreateWithFlags(out, flags);
            if (e == cudaSuccess) v.push_back(*out);
            return e;
        }
    } events;
    std::vector<cudaEvent_t> ev_in(n_chunks), ev_free(n_chunks), ev_feat(n_chunks), ev_done(n_chunks);
    for (int c = 0; c < n_chunks; ++c) {
        CUDA_CHECK(events.add(&ev_in[c], cudaEventDisableTiming));
        CUDA_CHECK(events.add(&ev_free[c], cudaEventDisableTiming));
        CUDA_CHECK(events.add(&ev_feat[c], cudaEventDisableTiming));
        CUDA_CHECK(events.add(&ev_done[c], cudaEventDisableTiming));
    }
    // The chunks' copies and launches happen inside enqueue(); whatever it returns, the three streams are drained before this
    // function returns, because the copies read and write caller memory.
    auto enqueue = [&]() -> int {
    int rc = MCS_OK;
    const uint8_t* dmask_for_match = ex->p.learn_masks ? feat.dmask : nullptr;
    for (int c = 0; c < n_chunks && rc == MCS_OK; ++c) {
        const int img_lo = chunk_lo[c] * n_cams, nimg = (chunk_lo[c + 1] - chunk_lo[c]) * n_cams;
        if (nimg <= 0) continue;
        uint8_t* tight = ex->in_tight.p + (size_t)(c & 1) * tight_img * ipc;
        if (c >= 2) CUDA_CHECK(cudaStreamWaitEvent(ex->s_copy, ev_free[c - 2], 0));          // staging buffer consumed
        CUDA_CHECK(cudaMemcpyAsync(tight, images + (size_t)img_lo * tight_img, tight_img * nimg - (c == n_chunks - 1 ? (size_t)(stride - width) : 0),
                                   cudaMemcpyHostToDevice, ex->s_copy));
        CUDA_CHECK(cudaEventRecord(ev_in[c], ex->s_copy));
        CUDA_CHECK(cudaStreamWaitEvent(st, ev_in[c], 0));
        launch_repitch(tight, stride, ex->in_images.p, dpitch, width, (size_t)height * nimg, st);
        CUDA_CHECK(cudaEventRecord(ev_free[c], st));
        const FeatureView chunk = feature_at(feat, img_lo, capacity, ds);
        rc = enqueue_kernels(ex, nimg, ex->in_images.p, width, height, dpitch, ex->cam_of_image.p + img_lo, chunk, capacity, st);
        if (rc) break;
        CUDA_CHECK(cudaEventRecord(ev_feat[c], st));                              // features of the chunk are final: their D2H overlaps the matching
        // the matching of chunk c runs on its own stream, so that K1..K3 of chunk c+1 (on `st`) fill the SMs behind its tail;
        // it reads descriptors of this chunk and of the last frame of the previous one, both final at ev_feat[c]
        CUDA_CHECK(cudaStreamWaitEvent(ex->s_match, ev_feat[c], 0));
        // with the greedy acceptance on the device the lists only need the entries that can influence it (kernels.h: greedy_dist_bound)
        CUDA_CHECK(launch_hamming_stream(feat.desc, dmask_for_match, feat.counts, img_lo, nimg, n_cams, capacity, ds, K,
                                         replay ? greedy_dist_bound(th_low, nnratio) : 0xFFFFFFFFu, ex->match_idx.p, ex->match_dist.p, ex->s_match));
        if (replay)     // greedy acceptance of SearchByBoW(KF1, KF2) over the lists of this chunk, still on the device
            CUDA_CHECK(launch_stream_replay(ex->match_idx.p, ex->match_dist.p, feat.counts, feat.desc, dmask_for_match, ds, img_lo, nimg, n_cams,
                                            capacity, K, th_low, nnratio, ex->m12.p, ex->nmat.p, ex->redo.p, ex->s_match));
        CUDA_CHECK(cudaEventRecord(ev_done[c], ex->s_match));
        cudaStream_t so = ex->s_out;
        CUDA_CHECK(cudaStreamWaitEvent(so, ev_feat[c], 0));
        rc = copy_features(feature_at(host, img_lo, capacity, ds), chunk, nimg, capacity, ds, dmask_out != nullptr, so);
        if (rc) break;
        CUDA_CHECK(cudaStreamWaitEvent(so, ev_done[c], 0));
        CUDA_CHECK(cudaMemcpyAsync(match_idx_out + (size_t)img_lo * capacity * K, ex->match_idx.p + (size_t)img_lo * capacity * K,
                                   sizeof(int) * (size_t)nimg * capacity * K, cudaMemcpyDeviceToHost, so));
        CUDA_CHECK(cudaMemcpyAsync(match_dist_out + (size_t)img_lo * capacity * K, ex->match_dist.p + (size_t)img_lo * capacity * K,
                                   sizeof(int) * (size_t)nimg * capacity * K, cudaMemcpyDeviceToHost, so));
        if (replay) {
            CUDA_CHECK(cudaMemcpyAsync(matches12_out + (size_t)img_lo * capacity, ex->m12.p + (size_t)img_lo * capacity, sizeof(int) * (size_t)nimg * capacity,
                                       cudaMemcpyDeviceToHost, so));
            CUDA_CHECK(cudaMemcpyAsync(nmatches_out + img_lo, ex->nmat.p + img_lo, sizeof(int) * nimg, cudaMemcpyDeviceToHost, so));
            CUDA_CHECK(cudaMemcpyAsync(redo_out + img_lo, ex->redo.p + img_lo, sizeof(int) * nimg, cudaMemcpyDeviceToHost, so));
        }
    }
    return rc;
    };
    const int rc = enqueue();
    cudaError_t e1 = cudaStreamSynchronize(ex->s_copy), e2 = cudaStreamSynchronize(st), e3 = cudaStreamSynchronize(ex->s_out);
    { const cudaError_t e4 = cudaStreamSynchronize(ex->s_match); if (e2 == cudaSuccess) e2 = e4; }
    if (rc) return rc;
    CUDA_CHECK(e1); CUDA_CHECK(e2); CUDA_CHECK(e3);
    ex->last_n_images = (chunk_lo[n_chunks] - chunk_lo[n_chunks - 1]) * n_cams;
    return check_status(ex, st);
}

extern "C" {

int mcs_extract_match_stream(mcs_extractor* ex, int32_t n_frames, int32_t n_cams, const uint8_t* images, int32_t width,
                             int32_t height, int32_t stride, const uint8_t* masks, const mcs_ocam* cams, mcs_keypoint* kps_out,
                             uint8_t* desc_out, uint8_t* dmask_out, int32_t* counts_out, int32_t capacity, int32_t K,
                             int32_t* match_idx_out, int32_t* match_dist_out) {
    return extract_match_stream_impl(ex, n_frames, n_cams, images, width, height, stride, masks, cams, kps_out, desc_out, dmask_out,
                                     counts_out, capacity, K, match_idx_out, match_dist_out, nullptr);
}

int mcs_extract_match_stream_packed(mcs_extractor* ex, int32_t n_frames, int32_t n_cams, const uint8_t* images, int32_t width,
                                    int32_t height, int32_t stride, const uint8_t* masks, const mcs_ocam* cams, mcs_keypoint* kps_out,
                                    uint8_t* desc_out, uint8_t* dmask_out, int32_t* counts_out, int32_t capacity, int32_t K,
                                    int32_t* match_idx_out, int32_t* match_dist_out, void* packed_dev, int32_t th_low, double nnratio,
                                    int32_t* matches12_out, int32_t* nmatches_out, int32_t* redo_out) {
    return extract_match_stream_impl(ex, n_frames, n_cams, images, width, height, stride, masks, cams, kps_out, desc_out, dmask_out,
                                     counts_out, capacity, K, match_idx_out, match_dist_out, packed_dev, th_low, nnratio, matches12_out,
                                     nmatches_out, redo_out);
}

int mcs_extract_batch_packed_device(mcs_extractor* ex, int32_t n_images, const uint8_t* images_dev, int32_t width, int32_t height,
                                    int32_t stride, const uint8_t* masks, const mcs_ocam* cams, int32_t n_cams,
                                    const int32_t* cam_of_image, void* packed_dev, int32_t capacity, void* stream) {
    if (!ex || !packed_dev) return mcs_fail(MCS_ERR_INVALID, "null argument");
    const FeatureView v = packed_view(packed_dev, n_images, capacity, ex->p.desc_size);
    return mcs_extract_batch_device(ex, n_images, images_dev, width, height, stride, masks, cams, n_cams, cam_of_image, v.kps, v.desc,
                                    v.dmask, v.counts, capacity, stream);
}

}  // extern "C"
