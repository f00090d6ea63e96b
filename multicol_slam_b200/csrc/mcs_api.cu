// mcs_api.cu -- C-ABI host layer of libmcs_b200.so (see include/mcs_b200.h).
//
// Host responsibilities only: parameter tables of the extractor constructor (ref
// src/mdBRIEFextractorOct.cpp:134-203), per-image-size geometry / look-up tables, device buffers,
// kernel launches, and the order-dependent bookkeeping of the matchers (greedy assignment rules of
// ref src/cORBmatcher.cpp:67-166, :579-726, :885-966) replayed over GPU-computed distances.
// There is no CPU implementation of the image or distance arithmetic in this library: without a CUDA
// device every compute entry point fails with MCS_ERR_NO_DEVICE.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "cam_model.cuh"
#include "kernels.h"
#include "mcs_common.cuh"

using namespace mcs;

namespace {

thread_local std::string g_err;
int fail(int code, const std::string& msg) { g_err = msg; return code; }

#define CK(expr)                                                                                       \
    do {                                                                                               \
        cudaError_t e__ = (expr);                                                                      \
        if (e__ != cudaSuccess) {                                                                      \
            cudaGetLastError();                                                                        \
            return fail(e__ == cudaErrorNoDevice || e__ == cudaErrorInsufficientDriver ? MCS_ERR_NO_DEVICE : MCS_ERR_CUDA, \
                        std::string(#expr) + ": " + cudaGetErrorString(e__));                          \
        }                                                                                              \
    } while (0)

static const signed char kPairs[2048] = {
#include "brief_pairs_64.inc"
};

inline int cv_round(double v) { return (int)lrint(v); }
inline int cv_floor(double v) { int i = (int)v; return i - (i > v); }
inline int cv_ceil(double v) { int i = (int)v; return i + (i < v); }
inline short sat_short_round(float v) { int i = (int)lrintf(v); return (short)std::min(std::max(i, -32768), 32767); }

template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
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
    void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
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
    DevBuf<int> cam_of_image, coi_all;
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

// ---- geometry: everything that depends only on (width, height, params) ------------------------
int build_geometry(mcs_extractor* ex, int W, int H, int in_stride) {
    if (ex->geom_w == W && ex->geom_h == H && ex->geom_stride == in_stride) return MCS_OK;
    PyramidGeom& G = ex->G;
    std::memset(&G, 0, sizeof(G));
    const int L = ex->p.nlevels;
    G.nlevels = L; G.width = W; G.height = H;
    G.fast_threshold = ex->p.fast_threshold; G.desc_size = ex->p.desc_size;
    G.do_dbrief = ex->p.do_dbrief; G.learn_masks = ex->p.learn_masks;
    if (W >= 4096 || H >= 4096) return fail(MCS_ERR_UNSUPPORTED, "images larger than 4095 px are not supported");

    std::vector<int16_t> blob;     // all LUTs, int16
    struct Off { size_t xofs, xa0, xa1, yofs, yb0, yb1, cellx, celly, mx0, my0; } off[kMaxLevels];
    std::vector<int16_t> pmx, pmy;
    size_t raw_off = 0;
    int sel_off = 0;
    for (int l = 0; l < L; ++l) {
        LevelGeom& g = G.lv[l];
        g.w = cv_round((double)W * ex->isf[l]);
        g.h = cv_round((double)H * ex->isf[l]);
        if (g.w < 2 * kEdge + 8 || g.h < 2 * kEdge + 8)
            return fail(MCS_ERR_UNSUPPORTED, "pyramid level smaller than 58 px");
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
            // the staged source region of a 72x40 tile must fit 176 x 88 bytes: (72*s + 17) <= 176, (40*s + 2) <= 88
            if (scale_x > 2.08 || scale_y > 2.08) return fail(MCS_ERR_UNSUPPORTED, "scale factors above 2 are not supported");
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
        }
        // FAST cell grid (ref :876-949, SURVEY Appendix A.6)
        std::vector<int16_t> cellx(g.w, -1), celly(g.h, -1);
        const int minB = kEdge - 3, maxBX = g.w - kEdge + 3, maxBY = g.h - kEdge + 3;
        const double width = maxBX - minB, height = maxBY - minB;
        g.n_cols = (int)(width / 30.0); g.n_rows = (int)(height / 30.0);
        if (g.n_cols < 1 || g.n_rows < 1) return fail(MCS_ERR_UNSUPPORTED, "level too small for the 30 px cell grid");
        g.w_cell = (int)std::ceil(width / g.n_cols); g.h_cell = (int)std::ceil(height / g.n_rows);
        if ((long long)g.n_cols * g.n_rows * g.w_cell * g.h_cell >= (1 << 24))
            return fail(MCS_ERR_UNSUPPORTED, "cell-order key overflow");
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
        if (g.nodes_ini < 1) return fail(MCS_ERR_UNSUPPORTED, "portrait images narrower than half their height");
        g.hX = (double)(maxBX - minB) / g.nodes_ini;
        g.sel_cap = std::max(g.quota + 3, 4 * g.nodes_ini);
        g.sel_off = sel_off; sel_off += g.sel_cap;
        g.raw_cap = ((g.w - 2 * kEdge + 1) / 2 + 1) * ((g.h - 2 * kEdge + 1) / 2 + 1);
        g.raw_off = raw_off; raw_off += (size_t)((g.raw_cap + 3) & ~3);
        auto put = [&](const std::vector<int16_t>& v) { size_t o = blob.size(); blob.insert(blob.end(), v.begin(), v.end()); while (blob.size() & 7) blob.push_back(0); return o; };
        off[l] = {put(xofs), put(xa0), put(xa1), put(yofs), put(yb0), put(yb1), put(cellx), put(celly), put(mx), put(my)};
    }
    G.sel_total = sel_off; G.raw_total = raw_off; G.cap = ex->capacity;
    G.tiles_total = 0;
    for (int l = 0; l < L; ++l) { G.lv[l].tile_off = G.tiles_total; G.tiles_total += G.lv[l].tiles_x * G.lv[l].tiles_y; }
    ex->tile_flags_valid = false;
    // kernels of an earlier *_device call on a caller-supplied stream may still read the tables about to be rewritten (a change of the
    // image size is rare: drain the device)
    CK(cudaDeviceSynchronize());
    CK(ex->lut_blob.ensure(blob.size() * sizeof(int16_t)));
    CK(cudaMemcpyAsync(ex->lut_blob.p, blob.data(), blob.size() * sizeof(int16_t), cudaMemcpyHostToDevice, ex->stream));
    const int16_t* base = (const int16_t*)ex->lut_blob.p;
    for (int l = 0; l < L; ++l) {
        LevelGeom& g = G.lv[l];
        g.xofs = base + off[l].xofs; g.xa0 = base + off[l].xa0; g.xa1 = base + off[l].xa1;
        g.yofs = base + off[l].yofs; g.yb0 = base + off[l].yb0; g.yb1 = base + off[l].yb1;
        g.cellx = base + off[l].cellx; g.celly = base + off[l].celly;
        g.mx0 = base + off[l].mx0; g.my0 = base + off[l].my0;
    }
    CK(ex->G_dev.ensure(1));
    CK(cudaMemcpyAsync(ex->G_dev.p, &G, sizeof(G), cudaMemcpyHostToDevice, ex->stream));
    CK(cudaStreamSynchronize(ex->stream));     // blob / G are host temporaries
    ex->geom_w = W; ex->geom_h = H; ex->geom_stride = in_stride;
    ex->B_cap = 0;      // level buffers depend on the geometry
    return MCS_OK;
}

int ensure_batch(mcs_extractor* ex, int B) {
    if (B <= ex->B_cap) return MCS_OK;
    const PyramidGeom& G = ex->G;
    for (int l = 0; l < G.nlevels; ++l) {
        CK(ex->lvl[l].ensure(G.lv[l].img_bytes * B + 256));
        CK(ex->blur[l].ensure(G.lv[l].img_bytes * B + 256));
    }
    CK(ex->cam_of_image.ensure(B));
    CK(ex->raw.ensure(G.raw_total * B));
    CK(ex->node_of.ensure(G.raw_total * B));
    CK(ex->raw_count.ensure((size_t)B * G.nlevels));
    CK(ex->sel_count.ensure((size_t)B * G.nlevels));
    CK(ex->sel_xys.ensure((size_t)B * G.sel_total));
    CK(ex->status.ensure(1));
    ex->B_cap = B;
    return MCS_OK;
}

// Small per-call host inputs (masks, camera models, distortion tables, status word).  They travel over the same
// H2D copy engine as the image chunks of the stream call, so they must be enqueued BEFORE any large copy: a 1 MB
// mask upload queued behind 100 MB of images stalls the compute stream for the whole transfer.
int upload_small_inputs(mcs_extractor* ex, int W, int H, const uint8_t* masks, const mcs_ocam* cams, int n_cams, cudaStream_t st) {
    CK(ex->masks.ensure((size_t)n_cams * W * H));
    CK(ex->cams.ensure(n_cams));
    // the masks rarely change between calls (static mirror masks): a 1 MB compare is cheaper than a pageable upload
    const size_t mbytes = (size_t)n_cams * W * H;
    if (ex->masks_host.size() != mbytes || std::memcmp(ex->masks_host.data(), masks, mbytes) != 0) {
        CK(cudaStreamSynchronize(st));                     // a previous call may still read the old masks
        ex->masks_host.assign(masks, masks + mbytes);
        CK(cudaMemcpyAsync(ex->masks.p, ex->masks_host.data(), mbytes, cudaMemcpyHostToDevice, st));
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
        CK(cudaStreamSynchronize(st));                     // a previous call may still read the old flags
        CK(ex->tile_flags.ensure(flags.size()));
        CK(cudaMemcpyAsync(ex->tile_flags.p, flags.data(), flags.size(), cudaMemcpyHostToDevice, st));
        CK(cudaStreamSynchronize(st));                     // `flags` is a host temporary
        ex->tile_flags_valid = true;
    }
    CK(cudaMemcpyAsync(ex->cams.p, cams, sizeof(mcs_ocam) * n_cams, cudaMemcpyHostToDevice, st));
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
        CK(cudaStreamSynchronize(st));                 // a previous call may still read the old tables
        CK(ex->lut_coef.ensure(all.size()));
        CK(ex->luts.ensure(n_cams));
        std::vector<DistortLut> h(n_cams);
        for (int c = 0; c < n_cams; ++c) h[c] = DistortLut{ex->lut_coef.p + offs[c], ns[c], 1.0};
        CK(cudaMemcpyAsync(ex->lut_coef.p, all.data(), all.size() * sizeof(double), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(ex->luts.p, h.data(), sizeof(DistortLut) * n_cams, cudaMemcpyHostToDevice, st));
        CK(cudaStreamSynchronize(st));                 // host staging vectors die here
        ex->lut_cams.assign(cams, cams + n_cams);
    }
    CK(cudaMemsetAsync(ex->status.p, 0, sizeof(int), st));

    return MCS_OK;
}

constexpr int kGraphMaxImages = 16;      // batches up to this size take the per-frame path (pinned staging, CUDA graph)

// K1 (per level) -> K2 -> K3 on `st`: kernel launches and memsets only (no allocation, no host synchronisation, no pageable
// copy), so the sequence can be stream-captured into a CUDA graph.
int enqueue_kernels(mcs_extractor* ex, int n_images, const uint8_t* images_dev, int W, int H, int stride, const int* coi_d,
                    mcs_keypoint* kps_dev, uint8_t* desc_dev, uint8_t* dmask_dev, int* counts_dev, int capacity, cudaStream_t st) {
    const PyramidGeom& G = ex->G;
    ex->coi_last = coi_d;
    CK(cudaMemsetAsync(ex->raw_count.p, 0, sizeof(int) * n_images * G.nlevels, st));
    if (ex->profiling) CK(cudaEventRecord(ex->ev[0], st));
    for (int l = 0; l < G.nlevels; ++l) {
        const uint8_t* src = l ? ex->lvl[l - 1].p : images_dev;
        const size_t src_bytes = l ? G.lv[l - 1].img_bytes : (size_t)stride * H;
        launch_pyr_fast(G, l, n_images, src, src_bytes, ex->lvl[l].p, ex->blur[l].p, ex->masks.p, W, (size_t)W * H,
                        coi_d, ex->tile_flags.p, ex->raw.p, ex->raw_count.p, st);
    }
    CK(cudaGetLastError());
    if (ex->profiling) CK(cudaEventRecord(ex->ev[1], st));
    // (K2 forked per level onto a second stream behind K1 of the same level was slower for the per-frame path: the per-level
    // launches serialise on that stream, while the single launch runs its 8 x n CTAs side by side)
    CK(launch_octree(G, ex->G_dev.p, n_images, ex->raw.p, ex->raw_count.p, ex->node_of.p, ex->sel_xys.p, ex->sel_count.p,
                     ex->status.p, st));
    CK(cudaGetLastError());
    if (ex->profiling) CK(cudaEventRecord(ex->ev[2], st));
    DescribeArgs a;
    for (int l = 0; l < kMaxLevels; ++l) { a.lvl[l] = ex->lvl[l].p; a.blur[l] = ex->blur[l].p; }
    a.tier_stats = ex->tier_on ? ex->tier.p : nullptr;
    CK(launch_describe(G, ex->G_dev.p, n_images, a, ex->cams.p, ex->luts.p, coi_d, ex->sel_xys.p, ex->sel_count.p,
                       kps_dev, desc_dev, dmask_dev, counts_dev, capacity, st));
    if (ex->profiling) CK(cudaEventRecord(ex->ev[3], st));
    ex->last_n_images = n_images;
    return MCS_OK;
}

// Validation, geometry, buffer growth and the small host inputs of one call (everything that may allocate, synchronise or read
// pageable host memory); *coi_d receives the device camera-of-image table the kernels should use.
int prepare_inputs(mcs_extractor* ex, int n_images, int W, int H, int stride, const uint8_t* masks, const mcs_ocam* cams, int n_cams,
                   const int* cam_of_image, cudaStream_t st, bool first_chunk, const int* coi_dev, const int** coi_d) {
    if (n_cams < 1 || n_cams > 64) return fail(MCS_ERR_INVALID, "n_cams must be in [1,64]");
    for (int i = 0; i < n_images; ++i)
        if (cam_of_image[i] < 0 || cam_of_image[i] >= n_cams) return fail(MCS_ERR_INVALID, "cam_of_image out of range");
    int rc = build_geometry(ex, W, H, stride);
    if (rc) return rc;
    rc = ensure_batch(ex, n_images);
    if (rc) return rc;
    if (first_chunk) {
        rc = upload_small_inputs(ex, W, H, masks, cams, n_cams, st);
        if (rc) return rc;
    }
    *coi_d = coi_dev;
    if (!coi_dev) {
        CK(cudaMemcpyAsync(ex->cam_of_image.p, cam_of_image, sizeof(int) * n_images, cudaMemcpyHostToDevice, st));
        *coi_d = ex->cam_of_image.p;
    }
    ex->sf_valid = false;            // shared state (camera table, masks, tables) may now differ from what the cached graph assumes
    return MCS_OK;
}

int run_pipeline(mcs_extractor* ex, int n_images, const uint8_t* images_dev, int W, int H, int stride,
                 const uint8_t* masks, const mcs_ocam* cams, int n_cams, const int* cam_of_image,
                 mcs_keypoint* kps_dev, uint8_t* desc_dev, uint8_t* dmask_dev, int* counts_dev, int capacity,
                 cudaStream_t st, bool first_chunk = true, const int* coi_dev = nullptr) {
    const int* coi_d = nullptr;
    int rc = prepare_inputs(ex, n_images, W, H, stride, masks, cams, n_cams, cam_of_image, st, first_chunk, coi_dev, &coi_d);
    if (rc) return rc;
    return enqueue_kernels(ex, n_images, images_dev, W, H, stride, coi_d, kps_dev, desc_dev, dmask_dev, counts_dev, capacity, st);
}

int check_status(mcs_extractor* ex, cudaStream_t st) {
    int s = 0;
    CK(cudaMemcpyAsync(&s, ex->status.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (s & 1) return fail(MCS_ERR_CAPACITY, "raw corner list overflow");
    if (s & 2) return fail(MCS_ERR_CAPACITY, "octree node table overflow");
    if (s & 4) return fail(MCS_ERR_CAPACITY, "selected keypoint slots overflow");
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
    if (n != 845) return fail(MCS_ERR_INVALID, "disc table size");
    for (int v = 0; v <= kHalfPatch; ++v) {
        du[v] = (signed char)(v == 0 ? kHalfPatch : umax[v]);
        // symmetry check: column |u| = v must hold rows |v'| <= umax[v]
        for (int w = 0; w <= kHalfPatch; ++w)
            if ((w <= (v == 0 ? kHalfPatch : umax[v])) != (v <= (w == 0 ? kHalfPatch : umax[w])))
                return fail(MCS_ERR_INVALID, "IC_Angle disc is not symmetric");
    }
    CK(upload_constants(kPairs, du, dv));
    if (dev < 64) g_consts_uploaded[dev] = true;
    return MCS_OK;
}

}  // namespace

void mcs_set_error_(const std::string& msg) { g_err = msg; }

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
    if (!cam || !out) return fail(MCS_ERR_INVALID, "null argument");
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
    if (!p || !out) return fail(MCS_ERR_INVALID, "null argument");
    *out = nullptr;
    if (p->use_agast) return fail(MCS_ERR_UNSUPPORTED, "AGAST detector is not built (north star: FAST-9)");
    if (p->fast_agast_type != 2) return fail(MCS_ERR_UNSUPPORTED, "only FastFeatureDetector::TYPE_9_16 (type 2) is built");
    if (p->nlevels < 1 || p->nlevels > kMaxLevels) return fail(MCS_ERR_INVALID, "nlevels must be in [1,16]");
    if (p->desc_size != 16 && p->desc_size != 32 && p->desc_size != 64) return fail(MCS_ERR_INVALID, "desc_size must be 16, 32 or 64");
    if (p->nfeatures < 1 || !(p->scale_factor > 1.0f) || p->fast_threshold < 1 || p->fast_threshold > 254)
        return fail(MCS_ERR_INVALID, "bad nfeatures / scale_factor / fast_threshold");
    int dev = 0;
    {
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) { cudaGetLastError(); return fail(MCS_ERR_NO_DEVICE, std::string("no CUDA device: ") + cudaGetErrorString(e)); }
        int major = 0;
        cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
        if (major != 9) return fail(MCS_ERR_NO_DEVICE, "device is not sm_90 (H100); this library has no other code path");
    }
    int rc = upload_consts_once(dev);
    if (rc) return rc;
    mcs_extractor* ex = new mcs_extractor;
    ex->p = *p; ex->device = dev;
    // ref :151-179
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
        if (ex->quota[l] + 8 > kMaxNodes) { delete ex; return fail(MCS_ERR_UNSUPPORTED, "nfeatures too large for the octree node table"); }
        ex->capacity += std::max(ex->quota[l] + 2, 16);
    }
    if (cudaStreamCreateWithFlags(&ex->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete ex;
        return fail(MCS_ERR_CUDA, "cudaStreamCreate failed");
    }
    *out = ex;
    return MCS_OK;
}

void mcs_extractor_destroy(mcs_extractor* ex) {
    if (!ex) return;
    cudaSetDevice(ex->device);
    ex->lut_blob.release(); ex->G_dev.release(); ex->in_images.release();
    for (int l = 0; l < kMaxLevels; ++l) { ex->lvl[l].release(); ex->blur[l].release(); }
    ex->masks.release(); ex->cams.release(); ex->cam_of_image.release(); ex->coi_all.release(); ex->raw.release(); ex->node_of.release();
    ex->raw_count.release(); ex->sel_count.release(); ex->status.release(); ex->counts.release(); ex->sel_xys.release();
    ex->kps.release(); ex->desc.release(); ex->dmask.release();
    if (ex->sf_exec) cudaGraphExecDestroy(ex->sf_exec);
    if (ex->pin_in) cudaFreeHost(ex->pin_in);
    if (ex->pin_out) cudaFreeHost(ex->pin_out);
    ex->match_idx.release(); ex->match_dist.release(); ex->m12.release(); ex->nmat.release(); ex->redo.release(); ex->lut_coef.release(); ex->luts.release(); ex->tier.release(); ex->tile_flags.release();
    for (int i = 0; i < 4; ++i) if (ex->ev[i]) cudaEventDestroy(ex->ev[i]);
    ex->in_tight.release();
    if (ex->s_copy) cudaStreamDestroy(ex->s_copy);
    if (ex->s_match) cudaStreamDestroy(ex->s_match);
    if (ex->s_out) cudaStreamDestroy(ex->s_out);
    if (ex->stream) cudaStreamDestroy(ex->stream);
    delete ex;
}

int mcs_extractor_get_info(const mcs_extractor* ex, mcs_extractor_info* info) {
    if (!ex || !info) return fail(MCS_ERR_INVALID, "null argument");
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
        return fail(MCS_ERR_INVALID, "null argument");
    if (n_images < 1 || width < 1 || height < 1 || stride < width) return fail(MCS_ERR_INVALID, "bad image geometry");
    if (capacity < ex->capacity) return fail(MCS_ERR_CAPACITY, "capacity below mcs_extractor_info.capacity");
    if (ex->p.learn_masks && !dmask_dev) return fail(MCS_ERR_INVALID, "dmask buffer required when learn_masks is set");
    CK(cudaSetDevice(ex->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ex->stream;
    int rc = run_pipeline(ex, n_images, images_dev, width, height, stride, masks, cams, n_cams, cam_of_image, kps_dev, desc_dev,
                          dmask_dev, counts_dev, capacity, st);
    if (rc) return rc;
    if (!stream) return check_status(ex, st);
    return MCS_OK;
}

namespace {

int pin_ensure(uint8_t*& p, size_t& cap, size_t need, bool* moved) {
    if (need <= cap) return MCS_OK;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    CK(cudaMallocHost((void**)&p, need));
    cap = need; *moved = true;
    return MCS_OK;
}

struct SmallOut { size_t status, counts, kps, desc, dmask, total; };
SmallOut small_out_layout(int n, int capacity, int ds) {
    SmallOut o;
    auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
    o.status = 0; o.counts = 256;
    o.kps = o.counts + up(sizeof(int) * n);
    o.desc = o.kps + up(sizeof(mcs_keypoint) * n * capacity);
    o.dmask = o.desc + up((size_t)n * capacity * ds);
    o.total = o.dmask + up((size_t)n * capacity * ds);
    return o;
}

// copy-in, re-pitch, K1..K3, copy-out of one small call between the extractor's pinned staging buffers: capturable
int enqueue_small(mcs_extractor* ex, int n, int W, int H, int stride, int dpitch, const int* coi_d, int capacity, bool with_dmask, cudaStream_t st) {
    const int ds = ex->p.desc_size;
    const SmallOut o = small_out_layout(n, capacity, ds);
    CK(cudaMemcpyAsync(ex->in_tight.p, ex->pin_in, (size_t)stride * H * n, cudaMemcpyHostToDevice, st));
    launch_repitch(ex->in_tight.p, stride, ex->in_images.p, dpitch, W, (size_t)H * n, st);
    CK(cudaMemsetAsync(ex->status.p, 0, sizeof(int), st));
    int rc = enqueue_kernels(ex, n, ex->in_images.p, W, H, dpitch, coi_d, ex->kps.p, ex->desc.p, ex->dmask.p, ex->counts.p, capacity, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(ex->pin_out + o.status, ex->status.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(ex->pin_out + o.counts, ex->counts.p, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(ex->pin_out + o.kps, ex->kps.p, sizeof(mcs_keypoint) * n * capacity, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(ex->pin_out + o.desc, ex->desc.p, (size_t)n * capacity * ds, cudaMemcpyDeviceToHost, st));
    if (with_dmask) CK(cudaMemcpyAsync(ex->pin_out + o.dmask, ex->dmask.p, (size_t)n * capacity * ds, cudaMemcpyDeviceToHost, st));
    return MCS_OK;
}

}  // namespace

int mcs_extract_batch(mcs_extractor* ex, int32_t n_images, const uint8_t* images, int32_t width, int32_t height, int32_t stride,
                      const uint8_t* masks, const mcs_ocam* cams, int32_t n_cams, const int32_t* cam_of_image,
                      mcs_keypoint* kps_out, uint8_t* desc_out, uint8_t* dmask_out, int32_t* counts_out, int32_t capacity) {
    if (!ex || !images || !masks || !cams || !cam_of_image || !kps_out || !desc_out || !counts_out)
        return fail(MCS_ERR_INVALID, "null argument");
    if (n_images < 1 || width < 1 || height < 1 || stride < width) return fail(MCS_ERR_INVALID, "bad image geometry");
    if (capacity < ex->capacity) return fail(MCS_ERR_CAPACITY, "capacity below mcs_extractor_info.capacity");
    if (ex->p.learn_masks && !dmask_out) return fail(MCS_ERR_INVALID, "dmask buffer required when learn_masks is set");
    CK(cudaSetDevice(ex->device));
    cudaStream_t st = ex->stream;
    const int ds = ex->p.desc_size;
    // device staging with a 64-byte-aligned pitch so that K1 can use 128-bit loads
    const int dpitch = (width + 63) & ~63;
    const size_t img_bytes = (size_t)dpitch * height;
    const void* before[6] = {ex->in_images.p, ex->kps.p, ex->desc.p, ex->dmask.p, ex->counts.p, ex->in_tight.p};
    CK(ex->in_images.ensure(img_bytes * n_images + 256));
    CK(ex->kps.ensure((size_t)n_images * capacity));
    CK(ex->desc.ensure((size_t)n_images * capacity * ds));
    CK(ex->dmask.ensure((size_t)n_images * capacity * ds));
    CK(ex->counts.ensure(n_images));
    // linear H2D + device re-pitch (a 2-D DMA of short rows is several times slower)
    CK(ex->in_tight.ensure((size_t)stride * height * n_images + 256));
    const void* after[6] = {ex->in_images.p, ex->kps.p, ex->desc.p, ex->dmask.p, ex->counts.p, ex->in_tight.p};
    bool moved = std::memcmp(before, after, sizeof(before)) != 0;

    if (n_images <= kGraphMaxImages && !ex->profiling && !ex->tier_on) {
        // ---- per-frame call: pinned staging + the whole sequence as one graph launch once the inputs repeat ----
        if (n_cams < 1 || n_cams > 64) return fail(MCS_ERR_INVALID, "n_cams must be in [1,64]");
        const size_t in_bytes = (size_t)stride * height * n_images, mbytes = (size_t)n_cams * width * height;
        const SmallOut o = small_out_layout(n_images, capacity, ds);
        int rc = pin_ensure(ex->pin_in, ex->pin_in_bytes, in_bytes, &moved);
        if (rc) return rc;
        rc = pin_ensure(ex->pin_out, ex->pin_out_bytes, o.total, &moved);
        if (rc) return rc;
        if (moved) ex->sf_valid = false;
        // the caller's last row may hold only `width` valid bytes (a cv::Mat ROI with step > width at the end of its allocation)
        std::memcpy(ex->pin_in, images, in_bytes - (size_t)(stride - width));
        const mcs_extractor::SfKey& k = ex->sf_key;
        bool hit = ex->sf_valid && ex->sf_exec && k.n == n_images && k.w == width && k.h == height && k.stride == stride &&
                   k.capacity == capacity && k.dm == (dmask_out != nullptr) && (int)k.cams.size() == n_cams &&
                   std::memcmp(k.coi.data(), cam_of_image, sizeof(int) * n_images) == 0 &&
                   std::memcmp(k.cams.data(), cams, sizeof(mcs_ocam) * n_cams) == 0 && ex->masks_host.size() == mbytes;
        if (hit) {
            // the graph goes first and the 1 MB mask comparison runs while the GPU works; if the masks did change the result
            // is thrown away and the call starts over on the eager path (which uploads the new masks)
            CK(cudaGraphLaunch(ex->sf_exec, st));
            if (std::memcmp(ex->masks_host.data(), masks, mbytes) != 0) {
                CK(cudaStreamSynchronize(st));
                hit = false;
            } else {
                ++ex->sf_replays;
            }
        }
        if (!hit) {
            const int* coi_d = nullptr;
            rc = prepare_inputs(ex, n_images, width, height, dpitch /* K1 reads the re-pitched copy */, masks, cams, n_cams, cam_of_image, st, true, nullptr, &coi_d);
            if (rc) return rc;
            rc = enqueue_small(ex, n_images, width, height, stride, dpitch, coi_d, capacity, dmask_out != nullptr, st);
            if (rc) return rc;
            // record the same sequence for the next call with these inputs (capture executes nothing)
            if (ex->sf_exec) { cudaGraphExecDestroy(ex->sf_exec); ex->sf_exec = nullptr; }
            cudaGraph_t graph = nullptr;
            if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
                const int crc = enqueue_small(ex, n_images, width, height, stride, dpitch, coi_d, capacity, dmask_out != nullptr, st);
                const cudaError_t ce = cudaStreamEndCapture(st, &graph);
                if (crc == MCS_OK && ce == cudaSuccess && graph && cudaGraphInstantiate(&ex->sf_exec, graph, 0) == cudaSuccess) {
                    mcs_extractor::SfKey& nk = ex->sf_key;
                    nk.n = n_images; nk.w = width; nk.h = height; nk.stride = stride; nk.capacity = capacity;
                    nk.coi.assign(cam_of_image, cam_of_image + n_images);
                    nk.cams.assign(cams, cams + n_cams);
                    nk.dm = dmask_out != nullptr;
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
        CK(cudaStreamSynchronize(st));
        const int status = *(const int*)(ex->pin_out + o.status);
        if (status & 1) return fail(MCS_ERR_CAPACITY, "raw corner list overflow");
        if (status & 2) return fail(MCS_ERR_CAPACITY, "octree node table overflow");
        if (status & 4) return fail(MCS_ERR_CAPACITY, "selected keypoint slots overflow");
        const int* cnt = (const int*)(ex->pin_out + o.counts);
        for (int i = 0; i < n_images; ++i) {
            const size_t nused = (size_t)std::min(std::max(cnt[i], 0), capacity), row = (size_t)i * capacity;
            counts_out[i] = cnt[i];
            std::memcpy(kps_out + row, ex->pin_out + o.kps + row * sizeof(mcs_keypoint), nused * sizeof(mcs_keypoint));
            std::memcpy(desc_out + row * ds, ex->pin_out + o.desc + row * ds, nused * ds);
            if (dmask_out) std::memcpy(dmask_out + row * ds, ex->pin_out + o.dmask + row * ds, nused * ds);
        }
        return MCS_OK;
    }

    CK(cudaMemcpyAsync(ex->in_tight.p, images, (size_t)stride * height * n_images - (size_t)(stride - width), cudaMemcpyHostToDevice, st));
    launch_repitch(ex->in_tight.p, stride, ex->in_images.p, dpitch, width, (size_t)height * n_images, st);
    int rc = run_pipeline(ex, n_images, ex->in_images.p, width, height, dpitch, masks, cams, n_cams, cam_of_image, ex->kps.p,
                          ex->desc.p, ex->dmask.p, ex->counts.p, capacity, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(counts_out, ex->counts.p, sizeof(int) * n_images, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(kps_out, ex->kps.p, sizeof(mcs_keypoint) * n_images * capacity, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(desc_out, ex->desc.p, (size_t)n_images * capacity * ds, cudaMemcpyDeviceToHost, st));
    if (dmask_out) CK(cudaMemcpyAsync(dmask_out, ex->dmask.p, (size_t)n_images * capacity * ds, cudaMemcpyDeviceToHost, st));
    return check_status(ex, st);
}

int mcs_extract(mcs_extractor* ex, const uint8_t* image, int32_t width, int32_t height, int32_t stride, const uint8_t* mask,
                int32_t mask_stride, const mcs_ocam* cam, mcs_keypoint* kps_out, uint8_t* desc_out, uint8_t* dmask_out,
                int32_t capacity, int32_t* n_out) {
    if (!ex || !n_out) return fail(MCS_ERR_INVALID, "null argument");
    if (!image) return MCS_OK;   // empty image: silent return, outputs untouched (ref :1252-1253)
    if (!mask || !cam) return fail(MCS_ERR_INVALID, "a mask and a camera model are mandatory (ref :913-917 throws on an empty mask)");
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
    if (!ex || !out || !w_out || !h_out) return fail(MCS_ERR_INVALID, "null argument");
    if (level < 0 || level >= ex->G.nlevels || image_index < 0 || image_index >= ex->last_n_images)
        return fail(MCS_ERR_INVALID, "bad level / image index");
    CK(cudaSetDevice(ex->device));
    const LevelGeom& g = ex->G.lv[level];
    const int L = ex->G.nlevels;
    if (what == 0 || what == 1) {
        *w_out = g.w; *h_out = g.h;
        if (out_bytes < (size_t)g.w * g.h) return fail(MCS_ERR_CAPACITY, "buffer too small");
        const uint8_t* src = (what == 0 ? ex->lvl[level].p : ex->blur[level].p) + (size_t)image_index * g.img_bytes;
        CK(cudaMemcpy2D(out, g.w, src, g.pitch, g.w, g.h, cudaMemcpyDeviceToHost));
        return MCS_OK;
    }
    if (what == 2) {   // the mask pyramid is never materialised: evaluate the composed nearest-neighbour maps
        *w_out = g.w; *h_out = g.h;
        if (out_bytes < (size_t)g.w * g.h) return fail(MCS_ERR_CAPACITY, "buffer too small");
        std::vector<int16_t> mx(g.w), my(g.h);
        std::vector<int> coi(ex->last_n_images);
        CK(cudaMemcpy(mx.data(), g.mx0, g.w * 2, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(my.data(), g.my0, g.h * 2, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(coi.data(), ex->coi_last, sizeof(int) * ex->last_n_images, cudaMemcpyDeviceToHost));
        std::vector<uint8_t> m0((size_t)ex->G.width * ex->G.height);
        CK(cudaMemcpy(m0.data(), ex->masks.p + (size_t)coi[image_index] * m0.size(), m0.size(), cudaMemcpyDeviceToHost));
        for (int y = 0; y < g.h; ++y)
            for (int x = 0; x < g.w; ++x) ((uint8_t*)out)[(size_t)y * g.w + x] = m0[(size_t)my[y] * ex->G.width + mx[x]];
        return MCS_OK;
    }
    if (what == 3) {   // raw corners, sorted into the reference order (cell-row-major, then pixel-row-major)
        int n = 0;
        CK(cudaMemcpy(&n, ex->raw_count.p + (size_t)image_index * L + level, sizeof(int), cudaMemcpyDeviceToHost));
        n = std::min(n, g.raw_cap);
        *w_out = n; *h_out = 3;
        if (out_bytes < (size_t)n * 12) return fail(MCS_ERR_CAPACITY, "buffer too small");
        std::vector<uint32_t> c(n);
        CK(cudaMemcpy(c.data(), ex->raw.p + (size_t)image_index * ex->G.raw_total + g.raw_off, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost));
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
    return fail(MCS_ERR_INVALID, "unknown `what`");
}

int mcs_extractor_set_profiling(mcs_extractor* ex, int32_t enable) {
    if (!ex) return fail(MCS_ERR_INVALID, "null argument");
    CK(cudaSetDevice(ex->device));
    if (enable) for (int i = 0; i < 4; ++i) if (!ex->ev[i]) CK(cudaEventCreate(&ex->ev[i]));
    ex->profiling = enable != 0;
    return MCS_OK;
}

int mcs_extractor_tier_stats(mcs_extractor* ex, int32_t enable, int64_t* counts4) {
    if (!ex) return fail(MCS_ERR_INVALID, "null extractor");
    CK(cudaSetDevice(ex->device));
    CK(cudaDeviceSynchronize());
    if (counts4) {
        counts4[0] = counts4[1] = counts4[2] = counts4[3] = 0;
        if (ex->tier_on) CK(cudaMemcpy(counts4, ex->tier.p, 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    }
    if (enable && !ex->tier_on) {
        CK(ex->tier.ensure(4));
        CK(cudaMemset(ex->tier.p, 0, 4 * sizeof(unsigned long long)));
    }
    ex->tier_on = enable != 0;
    return MCS_OK;
}

int mcs_extractor_check_status(mcs_extractor* ex, void* stream) {
    if (!ex) return fail(MCS_ERR_INVALID, "null extractor");
    if (!ex->status.p) return MCS_OK;                       // nothing has run yet
    CK(cudaSetDevice(ex->device));
    return check_status(ex, stream ? (cudaStream_t)stream : ex->stream);
}

int mcs_cam_distort_table(const mcs_ocam* cam, double* rows_out, int32_t max_rows, int32_t* n_rows, int32_t* row_doubles) {
    if (!cam || !n_rows || !row_doubles) return fail(MCS_ERR_INVALID, "null argument");
    if (rows_out && max_rows < 0) return fail(MCS_ERR_INVALID, "negative max_rows");
    std::vector<double> coef;
    int n = 0;
    build_distort_lut(*cam, coef, n);
    *n_rows = n;
    *row_doubles = n > 0 ? (int32_t)(coef.size() / (size_t)n) : 0;
    if (rows_out && n > 0) std::memcpy(rows_out, coef.data(), sizeof(double) * (size_t)std::min(n, (int)max_rows) * (size_t)*row_doubles);
    return MCS_OK;
}

int mcs_extractor_graph_replays(mcs_extractor* ex, int64_t* n) {
    if (!ex || !n) return fail(MCS_ERR_INVALID, "null argument");
    *n = ex->sf_replays;
    return MCS_OK;
}

int mcs_extractor_get_timings(mcs_extractor* ex, float* ms3) {
    if (!ex || !ms3) return fail(MCS_ERR_INVALID, "null argument");
    if (!ex->profiling || !ex->ev[3]) return fail(MCS_ERR_INVALID, "profiling is not enabled");
    CK(cudaEventSynchronize(ex->ev[3]));
    for (int i = 0; i < 3; ++i) CK(cudaEventElapsedTime(&ms3[i], ex->ev[i], ex->ev[i + 1]));
    return MCS_OK;
}

int mcs_match_stream_device(const uint8_t* desc_dev, const uint8_t* dmask_dev, const int32_t* counts_dev, int32_t n_frames,
                            int32_t n_cams, int32_t capacity, int32_t dim, int32_t K, int32_t* match_idx_dev,
                            int32_t* match_dist_dev, void* stream) {
    if (!desc_dev || !counts_dev || !match_idx_dev || !match_dist_dev) return fail(MCS_ERR_INVALID, "null argument");
    if (n_frames < 1 || n_cams < 1 || capacity < 1 || K < 1 || K > 8) return fail(MCS_ERR_INVALID, "bad sizes (K must be 1..8)");
    if (dim != 16 && dim != 32 && dim != 64) return fail(MCS_ERR_INVALID, "dim must be 16, 32 or 64");
    cudaStream_t st = (cudaStream_t)stream;
    CK(launch_hamming_stream(desc_dev, dmask_dev, counts_dev, 0, n_frames * n_cams, n_cams, capacity, dim, K, 0xFFFFFFFFu, match_idx_dev, match_dist_dev, st));
    return MCS_OK;
}

int mcs_match_stream_greedy_device(const uint8_t* desc_dev, const uint8_t* dmask_dev, const int32_t* counts_dev, int32_t n_frames,
                                   int32_t n_cams, int32_t capacity, int32_t dim, int32_t th_low, double nnratio,
                                   int32_t* matches12_dev, int32_t* nmatches_dev, void* stream) {
    if (!desc_dev || !counts_dev || !matches12_dev || !nmatches_dev) return fail(MCS_ERR_INVALID, "null argument");
    if (n_frames < 1 || n_cams < 1 || capacity < 1 || capacity > 65535) return fail(MCS_ERR_INVALID, "bad sizes (capacity must be 1..65535)");
    if (dim != 16 && dim != 32 && dim != 64) return fail(MCS_ERR_INVALID, "dim must be 16, 32 or 64");
    cudaStream_t st = (cudaStream_t)stream;
    // K-best list length (the acceptance is exact for any K; K only sets how often the replay rescans).  H100 80GB HBM3, 400 W limit, bench.py config 2, 2 alternating runs:
    // K = 8 16.08 / 16.15 ms per 384-image step (47.9 Mfeatures/s) against 16.85 / 16.79 ms with K = 4.
    constexpr int K = 8;
    const size_t n = (size_t)n_frames * n_cams * capacity;
    int *li = nullptr, *ld = nullptr, *redo = nullptr;
    CK(keep_pool_memory());
    CK(cudaMallocAsync((void**)&li, n * K * sizeof(int), st));
    CK(cudaMallocAsync((void**)&ld, n * K * sizeof(int), st));
    CK(cudaMallocAsync((void**)&redo, (size_t)n_frames * n_cams * sizeof(int), st));
    cudaError_t e = launch_hamming_stream(desc_dev, dmask_dev, counts_dev, 0, n_frames * n_cams, n_cams, capacity, dim, K,
                                          greedy_dist_bound(th_low, nnratio), li, ld, st);
    if (e == cudaSuccess)
        e = launch_stream_replay(li, ld, counts_dev, desc_dev, dmask_dev, dim, 0, n_frames * n_cams, n_cams, capacity, K, th_low, nnratio,
                                 matches12_dev, nmatches_dev, redo, st);
    cudaFreeAsync(li, st); cudaFreeAsync(ld, st); cudaFreeAsync(redo, st);
    CK(e);
    return MCS_OK;
}

int mcs_match_stream_replay_device(const int32_t* match_idx_dev, const int32_t* match_dist_dev, const int32_t* counts_dev,
                                   const uint8_t* desc_dev, const uint8_t* dmask_dev, int32_t n_frames, int32_t n_cams, int32_t capacity,
                                   int32_t dim, int32_t K, int32_t th_low, double nnratio, int32_t* matches12_dev, int32_t* nmatches_dev,
                                   int32_t* redo_dev, void* stream) {
    if (!match_idx_dev || !match_dist_dev || !counts_dev || !desc_dev || !matches12_dev || !nmatches_dev || !redo_dev)
        return fail(MCS_ERR_INVALID, "null argument");
    if (n_frames < 1 || n_cams < 1 || capacity < 1 || capacity > 65535 || K < 1 || K > 8) return fail(MCS_ERR_INVALID, "bad sizes (K must be 1..8)");
    if (dim != 16 && dim != 32 && dim != 64) return fail(MCS_ERR_INVALID, "dim must be 16, 32 or 64");
    CK(launch_stream_replay(match_idx_dev, match_dist_dev, counts_dev, desc_dev, dmask_dev, dim, 0, n_frames * n_cams, n_cams, capacity, K,
                            th_low, nnratio, matches12_dev, nmatches_dev, redo_dev, (cudaStream_t)stream));
    return MCS_OK;
}

}  // extern "C"

static int extract_match_stream_impl(mcs_extractor* ex, int32_t n_frames, int32_t n_cams, const uint8_t* images, int32_t width,
                             int32_t height, int32_t stride, const uint8_t* masks, const mcs_ocam* cams, mcs_keypoint* kps_out,
                             uint8_t* desc_out, uint8_t* dmask_out, int32_t* counts_out, int32_t capacity, int32_t K,
                             int32_t* match_idx_out, int32_t* match_dist_out, void* packed_dev, int32_t th_low = 0, double nnratio = 0.0,
                             int32_t* matches12_out = nullptr, int32_t* nmatches_out = nullptr, int32_t* redo_out = nullptr) {
    if (!ex || !images || !masks || !cams || !kps_out || !desc_out || !counts_out || !match_idx_out || !match_dist_out)
        return fail(MCS_ERR_INVALID, "null argument");
    if (n_frames < 1 || n_cams < 1 || width < 1 || height < 1 || stride < width) return fail(MCS_ERR_INVALID, "bad geometry");
    if (capacity < ex->capacity) return fail(MCS_ERR_CAPACITY, "capacity below mcs_extractor_info.capacity");
    if (ex->p.learn_masks && !dmask_out) return fail(MCS_ERR_INVALID, "dmask buffer required when learn_masks is set");
    if (K < 1 || K > 8) return fail(MCS_ERR_INVALID, "K must be 1..8");
    CK(cudaSetDevice(ex->device));
    cudaStream_t st = ex->stream;
    if (!ex->s_copy) CK(cudaStreamCreateWithFlags(&ex->s_copy, cudaStreamNonBlocking));
    if (!ex->s_out) CK(cudaStreamCreateWithFlags(&ex->s_out, cudaStreamNonBlocking));
    if (!ex->s_match) CK(cudaStreamCreateWithFlags(&ex->s_match, cudaStreamNonBlocking));
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
#ifdef MCS_DEBUG_KNOBS                                                  // experiment knobs exist only in -DMCS_DEBUG_KNOBS builds
    if (const char* plan = getenv("MCS_STREAM_CHUNKS")) {               // comma-separated frames per chunk
        std::vector<int> lo(1, 0);
        for (const char* q = plan; *q && lo.back() < n_frames;) {
            lo.push_back(std::min(n_frames, lo.back() + std::max(1, atoi(q))));
            while (*q && *q != ',') ++q;
            if (*q == ',') ++q;
        }
        if (lo.back() < n_frames) lo.push_back(n_frames);
        chunk_lo = lo;
    }
#endif
    const int n_chunks = (int)chunk_lo.size() - 1;
    int fpc = 0;
    for (int c = 0; c < n_chunks; ++c) fpc = std::max(fpc, chunk_lo[c + 1] - chunk_lo[c]);
    const int ipc = fpc * n_cams;                                     // images in the largest chunk
    const size_t tight_img = (size_t)stride * height, pitched_img = (size_t)dpitch * height;
    std::vector<int> coi(n_images);
    for (int i = 0; i < n_images; ++i) coi[i] = i % n_cams;
    CK(ex->in_tight.ensure(2 * tight_img * ipc + 256));
    CK(ex->in_images.ensure(pitched_img * ipc + 256));
    // feature buffers: the extractor's own, or the caller's packed exchange buffer (mcs_packed_layout) when one is given
    mcs_keypoint* kps_d; uint8_t* desc_d; uint8_t* dmask_d; int* counts_d;
    if (packed_dev) {
        size_t off[4];
        mcs_packed_layout(n_images, capacity, ds, off);
        uint8_t* base = (uint8_t*)packed_dev;
        counts_d = (int*)(base + off[0]); kps_d = (mcs_keypoint*)(base + off[1]); desc_d = base + off[2]; dmask_d = base + off[3];
    } else {
        CK(ex->kps.ensure((size_t)n_images * capacity));
        CK(ex->desc.ensure((size_t)n_images * capacity * ds));
        CK(ex->dmask.ensure((size_t)n_images * capacity * ds));
        CK(ex->counts.ensure(n_images));
        kps_d = ex->kps.p; desc_d = ex->desc.p; dmask_d = ex->dmask.p; counts_d = ex->counts.p;
    }
    CK(ex->match_idx.ensure((size_t)n_images * capacity * K));
    CK(ex->match_dist.ensure((size_t)n_images * capacity * K));
    const bool replay = matches12_out != nullptr;
    if (replay) {
        if (!nmatches_out || !redo_out) return fail(MCS_ERR_INVALID, "the greedy acceptance needs all three outputs");
        CK(ex->m12.ensure((size_t)n_images * capacity)); CK(ex->nmat.ensure(n_images)); CK(ex->redo.ensure(n_images));
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
    std::vector<cudaEvent_t> ev_in(n_chunks), ev_free(n_chunks), ev_feat(n_chunks), ev_done(n_chunks), tev;
    for (int c = 0; c < n_chunks; ++c) {
        CK(events.add(&ev_in[c], cudaEventDisableTiming));
        CK(events.add(&ev_free[c], cudaEventDisableTiming));
        CK(events.add(&ev_feat[c], cudaEventDisableTiming));
        CK(events.add(&ev_done[c], cudaEventDisableTiming));
    }
#ifdef MCS_DEBUG_KNOBS
    static const bool trace = getenv("MCS_TRACE_STREAM") != nullptr;    // per-chunk timeline on stderr
#else
    constexpr bool trace = false;
#endif
    // Everything asynchronous happens inside enqueue(); whatever it returns, the three streams are drained before this
    // function returns, because the copies read caller memory and the local cam-of-image table.
    auto enqueue = [&]() -> int {
    int rc = build_geometry(ex, width, height, dpitch);
    if (rc == MCS_OK) rc = ensure_batch(ex, ipc);
    if (rc == MCS_OK) rc = upload_small_inputs(ex, width, height, masks, cams, n_cams, st);     // before the first image copy, see there
    if (rc) return rc;
    CK(ex->coi_all.ensure(n_images));
    CK(cudaMemcpyAsync(ex->coi_all.p, coi.data(), sizeof(int) * n_images, cudaMemcpyHostToDevice, st));
    const uint8_t* dmask_for_match = ex->p.learn_masks ? dmask_d : nullptr;
    // MCS_TRACE_STREAM=1: per-chunk timeline on stderr (H2D begin/end, compute begin/features/end, D2H end), ms from the first H2D
    auto mark = [&](cudaStream_t s_) { if (trace) { cudaEvent_t e; if (events.add(&e, cudaEventDefault) == cudaSuccess) { cudaEventRecord(e, s_); tev.push_back(e); } } };
    for (int c = 0; c < n_chunks && rc == MCS_OK; ++c) {
        const int img_lo = chunk_lo[c] * n_cams, nimg = (chunk_lo[c + 1] - chunk_lo[c]) * n_cams;
        if (nimg <= 0) continue;
        uint8_t* tight = ex->in_tight.p + (size_t)(c & 1) * tight_img * ipc;
        if (c >= 2) CK(cudaStreamWaitEvent(ex->s_copy, ev_free[c - 2], 0));          // staging buffer consumed
        mark(ex->s_copy);
        CK(cudaMemcpyAsync(tight, images + (size_t)img_lo * tight_img, tight_img * nimg - (c == n_chunks - 1 ? (size_t)(stride - width) : 0),
                           cudaMemcpyHostToDevice, ex->s_copy));
        mark(ex->s_copy);
        CK(cudaEventRecord(ev_in[c], ex->s_copy));
        CK(cudaStreamWaitEvent(st, ev_in[c], 0));
        mark(st);
        launch_repitch(tight, stride, ex->in_images.p, dpitch, width, (size_t)height * nimg, st);
        CK(cudaEventRecord(ev_free[c], st));
        rc = run_pipeline(ex, nimg, ex->in_images.p, width, height, dpitch, masks, cams, n_cams, coi.data() + img_lo,
                          kps_d + (size_t)img_lo * capacity, desc_d + (size_t)img_lo * capacity * ds,
                          dmask_d + (size_t)img_lo * capacity * ds, counts_d + img_lo, capacity, st, false, ex->coi_all.p + img_lo);
        if (rc) break;
        mark(st);
        CK(cudaEventRecord(ev_feat[c], st));                              // features of the chunk are final: their D2H overlaps the matching
        // the matching of chunk c runs on its own stream, so that K1..K3 of chunk c+1 (on `st`) fill the SMs behind its tail;
        // it reads descriptors of this chunk and of the last frame of the previous one, both final at ev_feat[c]
        CK(cudaStreamWaitEvent(ex->s_match, ev_feat[c], 0));
        // with the greedy acceptance on the device the lists only need the entries that can influence it (kernels.h: greedy_dist_bound)
        CK(launch_hamming_stream(desc_d, dmask_for_match, counts_d, img_lo, nimg, n_cams, capacity, ds, K,
                                 replay ? greedy_dist_bound(th_low, nnratio) : 0xFFFFFFFFu, ex->match_idx.p, ex->match_dist.p, ex->s_match));
        if (replay)     // greedy acceptance of SearchByBoW(KF1, KF2) over the lists of this chunk, still on the device
            CK(launch_stream_replay(ex->match_idx.p, ex->match_dist.p, counts_d, desc_d, dmask_for_match, ds, img_lo, nimg, n_cams, capacity, K,
                                    th_low, nnratio, ex->m12.p, ex->nmat.p, ex->redo.p, ex->s_match));
        mark(ex->s_match);
        CK(cudaEventRecord(ev_done[c], ex->s_match));
        cudaStream_t so = ex->s_out;
        CK(cudaStreamWaitEvent(so, ev_feat[c], 0));
        CK(cudaMemcpyAsync(counts_out + img_lo, counts_d + img_lo, sizeof(int) * nimg, cudaMemcpyDeviceToHost, so));
        CK(cudaMemcpyAsync(kps_out + (size_t)img_lo * capacity, kps_d + (size_t)img_lo * capacity,
                           sizeof(mcs_keypoint) * (size_t)nimg * capacity, cudaMemcpyDeviceToHost, so));
        CK(cudaMemcpyAsync(desc_out + (size_t)img_lo * capacity * ds, desc_d + (size_t)img_lo * capacity * ds,
                           (size_t)nimg * capacity * ds, cudaMemcpyDeviceToHost, so));
        if (dmask_out)
            CK(cudaMemcpyAsync(dmask_out + (size_t)img_lo * capacity * ds, dmask_d + (size_t)img_lo * capacity * ds,
                               (size_t)nimg * capacity * ds, cudaMemcpyDeviceToHost, so));
        CK(cudaStreamWaitEvent(so, ev_done[c], 0));
        CK(cudaMemcpyAsync(match_idx_out + (size_t)img_lo * capacity * K, ex->match_idx.p + (size_t)img_lo * capacity * K,
                           sizeof(int) * (size_t)nimg * capacity * K, cudaMemcpyDeviceToHost, so));
        CK(cudaMemcpyAsync(match_dist_out + (size_t)img_lo * capacity * K, ex->match_dist.p + (size_t)img_lo * capacity * K,
                           sizeof(int) * (size_t)nimg * capacity * K, cudaMemcpyDeviceToHost, so));
        if (replay) {
            CK(cudaMemcpyAsync(matches12_out + (size_t)img_lo * capacity, ex->m12.p + (size_t)img_lo * capacity, sizeof(int) * (size_t)nimg * capacity,
                               cudaMemcpyDeviceToHost, so));
            CK(cudaMemcpyAsync(nmatches_out + img_lo, ex->nmat.p + img_lo, sizeof(int) * nimg, cudaMemcpyDeviceToHost, so));
            CK(cudaMemcpyAsync(redo_out + img_lo, ex->redo.p + img_lo, sizeof(int) * nimg, cudaMemcpyDeviceToHost, so));
        }
        mark(so);
    }
    return rc;
    };
    const int rc = enqueue();
    cudaError_t e1 = cudaStreamSynchronize(ex->s_copy), e2 = cudaStreamSynchronize(st), e3 = cudaStreamSynchronize(ex->s_out);
    { const cudaError_t e4 = cudaStreamSynchronize(ex->s_match); if (e2 == cudaSuccess) e2 = e4; }
    if (trace && !tev.empty()) {
        for (size_t i = 0; i + 5 < tev.size(); i += 6) {
            float t[6];
            for (int k = 0; k < 6 && i + k < tev.size(); ++k) cudaEventElapsedTime(&t[k], tev[0], tev[i + k]);
            fprintf(stderr, "[mcs stream] chunk %zu: h2d %.2f-%.2f  compute %.2f  features %.2f  matched %.2f  d2h done %.2f ms\n", i / 6,
                    t[0], t[1], t[2], t[3], t[4], t[5]);
        }
    }
    if (rc) return rc;
    CK(e1); CK(e2); CK(e3);
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
    if (!ex || !packed_dev) return fail(MCS_ERR_INVALID, "null argument");
    size_t off[4];
    mcs_packed_layout(n_images, capacity, ex->p.desc_size, off);
    uint8_t* base = (uint8_t*)packed_dev;
    return mcs_extract_batch_device(ex, n_images, images_dev, width, height, stride, masks, cams, n_cams, cam_of_image,
                                    (mcs_keypoint*)(base + off[1]), base + off[2], base + off[3], (int32_t*)(base + off[0]), capacity, stream);
}

}  // extern "C"
