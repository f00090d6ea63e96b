// mcs_match_api.cu -- C-ABI host layer of the matcher entry points (include/mcs_b200.h).
//
// The GPU evaluates every Hamming distance and every grid-window candidate search; the host code here
// only (a) flattens the caller's frame into the CSR grid of cMultiFrame (ref src/cMultiFrame.cpp:168-184,
// :342-353) and (b) replays the reference's order-dependent greedy bookkeeping over the GPU results
// (ref src/cORBmatcher.cpp:121-164, :627-682, :922-961).
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "api_check.h"
#include "cam_model.cuh"
#include "kernels.h"
#include "dev_scratch.h"
#include "mcs_common.cuh"
#include "packed_frame.h"

using namespace mcs;

namespace {

// a frame's keypoints on the device, sorted into the CSR grid of cMultiFrame
struct FrameGrid {
    Dev keys, key_cam, cams, cell, cursor;                      // inputs and scratch of launch_frame_prepare
    Dev kx, ky, koct, cell_start, cell_items, winv, hinv;
};

// Uploads the keypoints, their cameras and the camera records, and enqueues the grid build on `st`: SoA copies of the keypoints,
// the grid cell of every keypoint, the CSR grid and, when `rays` is given, the keypoint bearing vectors.  The caller synchronises
// `st` before it reads the results or `g` dies.
int build_frame_grid(const mcs_keypoint* keys, const int* key_cam, int n, const mcs_ocam* cams, int nc, FrameGrid& g, Dev* rays,
                     cudaStream_t st) {
    for (int i = 0; i < n; ++i)
        if (key_cam[i] < 0 || key_cam[i] >= nc) return mcs_fail(MCS_ERR_INVALID, "key_cam out of range");
    const int ncell = nc * MCS_FRAME_GRID_COLS * MCS_FRAME_GRID_ROWS;
    const size_t m = (size_t)std::max(n, 1);
    CUDA_CHECK(g.keys.upload_async(keys, (size_t)n * sizeof(mcs_keypoint), st));
    CUDA_CHECK(g.key_cam.upload_async(key_cam, (size_t)n * 4, st));
    CUDA_CHECK(g.cams.upload_async(cams, nc * sizeof(mcs_ocam), st));
    CUDA_CHECK(g.cell.alloc(m * 4)); CUDA_CHECK(g.cursor.alloc((size_t)ncell * 4));
    CUDA_CHECK(g.kx.alloc(m * 4)); CUDA_CHECK(g.ky.alloc(m * 4)); CUDA_CHECK(g.koct.alloc(m * 4));
    CUDA_CHECK(g.cell_start.alloc((size_t)(ncell + 1) * 4)); CUDA_CHECK(g.cell_items.alloc(m * 4));
    CUDA_CHECK(g.winv.alloc(nc * 8)); CUDA_CHECK(g.hinv.alloc(nc * 8));
    if (rays) CUDA_CHECK(rays->alloc(m * 24));
    CUDA_CHECK(launch_frame_prepare(g.keys.as<mcs_keypoint>(), g.key_cam.as<int>(), n, g.cams.as<mcs_ocam>(), nc, g.kx.as<float>(),
                                    g.ky.as<float>(), g.koct.as<int>(), rays ? rays->as<double>() : nullptr, g.cell.as<int>(),
                                    g.cursor.as<int>(), g.cell_start.as<int>(), g.cell_items.as<int>(), g.winv.as<double>(),
                                    g.hinv.as<double>(), st));
    return MCS_OK;
}

// frame uploaded for window searches
struct FrameDev {
    FrameGrid grid;
    Dev desc, dmask, cam_first;
    WindowFrameDev view;
};

int upload_frame(const mcs_frame_view* f, FrameDev& d, cudaStream_t st) {
    // keypoints go up as they are; the window searches need only the image size of each camera
    const int n = f->n_keys, nc = f->n_cams;
    std::vector<mcs_ocam> cams(nc);
    std::memset(cams.data(), 0, sizeof(mcs_ocam) * nc);
    for (int c = 0; c < nc; ++c) { cams[c].width = f->cam_width[c]; cams[c].height = f->cam_height[c]; }
    const int rc = build_frame_grid(f->keys, f->key_cam, n, cams.data(), nc, d.grid, nullptr, st);
    if (rc) return rc;
    const size_t db = (size_t)n * f->dim;
    CUDA_CHECK(d.desc.upload_async(f->desc, db, st));
    if (f->dmask) CUDA_CHECK(d.dmask.upload_async(f->dmask, db, st));
    CUDA_CHECK(cudaStreamSynchronize(st));    // `cams` is a host temporary
    FrameGrid& g = d.grid;
    d.view = WindowFrameDev{nc, n, f->dim, g.kx.as<float>(), g.ky.as<float>(), g.koct.as<int>(), d.desc.as<uint8_t>(),
                            f->dmask ? d.dmask.as<uint8_t>() : nullptr, g.cell_start.as<int>(), g.cell_items.as<int>(),
                            g.winv.as<double>(), g.hinv.as<double>()};
    return MCS_OK;
}

// Runs the window-search kernel for host-side queries and returns the candidates as ONE dense array in query order: candidates
// of query q are cidx / cdist [coff[q] .. coff[q + 1]), in the kernel's visiting order.  Only the counts and the candidates that
// exist cross PCIe.  The first pass keeps max_cand candidates per query; a longer list runs the search once more.
int window_search_compact(const FrameDev& fd, const mcs_window_query* qs, const int nq, const uint8_t* qdesc, const uint8_t* qmask,
                          size_t qdesc_rows, int dim, int max_cand, std::vector<int>& cidx, std::vector<int>& cdist, std::vector<int>& coff,
                          cudaStream_t st) {
    coff.assign(nq + 1, 0);
    cidx.clear(); cdist.clear();
    if (nq == 0) return MCS_OK;
    Dev dq, dqd, dqm, dc, doff;
    CUDA_CHECK(dq.upload_async(qs, sizeof(mcs_window_query) * nq, st));
    CUDA_CHECK(dqd.upload_async(qdesc, qdesc_rows * dim, st));
    CUDA_CHECK(dc.alloc((size_t)nq * 4)); CUDA_CHECK(doff.alloc((size_t)nq * 4));
    const bool masked = qmask && fd.view.dmask;
    if (masked) CUDA_CHECK(dqm.upload_async(qmask, qdesc_rows * dim, st));
    std::vector<int> count(nq);
    for (;;) {
        Dev di, dd;
        CUDA_CHECK(di.alloc((size_t)nq * max_cand * 4)); CUDA_CHECK(dd.alloc((size_t)nq * max_cand * 4));
        CUDA_CHECK(launch_window_search(fd.view, dq.as<mcs_window_query>(), nq, dqd.as<uint8_t>(), masked ? dqm.as<uint8_t>() : nullptr,
                                        max_cand, di.as<int>(), dd.as<int>(), dc.as<int>(), st));
        CUDA_CHECK(cudaMemcpyAsync(count.data(), dc.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        const int mx = *std::max_element(count.begin(), count.end());
        if (mx > max_cand) { max_cand = (mx + 31) & ~31; continue; }        // a list overflowed: once more with room for the longest
        for (int q = 0; q < nq; ++q) coff[q + 1] = coff[q] + count[q];
        const int total = coff[nq];
        if (total == 0) return MCS_OK;
        Dev doi, dod;
        CUDA_CHECK(doi.alloc((size_t)total * 4)); CUDA_CHECK(dod.alloc((size_t)total * 4));
        CUDA_CHECK(cudaMemcpyAsync(doff.p, coff.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, st));
        CUDA_CHECK(launch_compact_lists(di.as<int>(), dd.as<int>(), dc.as<int>(), doff.as<int>(), nq, max_cand, doi.as<int>(), dod.as<int>(), st));
        cidx.resize(total); cdist.resize(total);
        CUDA_CHECK(cudaMemcpyAsync(cidx.data(), doi.p, (size_t)total * 4, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaMemcpyAsync(cdist.data(), dod.p, (size_t)total * 4, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        return MCS_OK;
    }
}

// The PsFrameArgs fields the four device searches fill alike: the frame searched (`cams`: its slots in the packed buffer), its
// camera sizes, the acceptance threshold and the outputs.  n_levels and sf stay 0 / NULL for the searches that read no scale factor.
void set_searched_frame(PsFrameArgs& a, const std::vector<PsCamSlots>& cams, int capacity, int dim, const int* cam_w, const int* cam_h,
                        int th_high, int having_masks, int* frame_mp, int* nmatches, int* status, int* diag) {
    a.n_cams = (int)cams.size(); a.capacity = capacity; a.dim = dim;
    a.cams = cams.data(); a.cam_w = cam_w; a.cam_h = cam_h;
    a.th_high = th_high; a.masked = having_masks != 0;
    a.frame_mp = frame_mp; a.nmatches = nmatches; a.status = status; a.diag = diag;
}

// the image sizes of camera models, as the width and height arrays PsFrameArgs and check_cam_sizes read
struct CamSizes {
    std::vector<int> w, h;
    CamSizes(const mcs_ocam* cams, int n) : w(n), h(n) {
        for (int c = 0; c < n; ++c) { w[c] = cams[c].width; h[c] = cams[c].height; }
    }
};

}  // namespace

extern "C" {

int mcs_descriptor_distance64(const uint64_t* a, const uint64_t* b, int32_t dim) {   // ref :2438-2450
    uint64_t d = 0;
    for (int i = 0; i < dim / 8; ++i) d += (uint64_t)__builtin_popcountll(a[i] ^ b[i]);
    return (int)d;
}

int mcs_descriptor_distance64_masked(const uint64_t* a, const uint64_t* b, const uint64_t* ma, const uint64_t* mb,
                                     int32_t dim) {   // ref :2452-2474
    uint64_t d = 0;
    for (int i = 0; i < dim / 8; ++i) {
        const uint64_t x = a[i] ^ b[i];
        d += (uint64_t)__builtin_popcountll(x & ma[i]);
        d += (uint64_t)__builtin_popcountll(x & mb[i]);
    }
    return (int)(d / 2);
}

int mcs_hamming_topk_device(const uint8_t* q_dev, const uint8_t* qmask_dev, int32_t nq, const uint8_t* d_dev,
                            const uint8_t* dmask_dev, int32_t nd, const uint8_t* db_skip_dev, int32_t dim, int32_t K,
                            int32_t* topk_idx_dev, int32_t* topk_dist_dev, void* stream) {
    if (!q_dev || !d_dev || !topk_idx_dev || !topk_dist_dev) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (nq < 0 || nd < 0 || K < 1 || K > 8) return mcs_fail(MCS_ERR_INVALID, "bad sizes (K must be 1..8)");
    if (int rc = check_desc_dim(dim)) return rc;
    if (nd >= (1 << 21)) return mcs_fail(MCS_ERR_UNSUPPORTED, "more than 2^21 - 1 database descriptors in one call (split the database)");
    CUDA_CHECK(launch_hamming_topk(q_dev, qmask_dev, nq, d_dev, dmask_dev, nd, db_skip_dev, dim, K, 0xFFFFFFFFu, topk_idx_dev, topk_dist_dev,
                                   (cudaStream_t)stream));
    return MCS_OK;
}

int mcs_hamming_topk(const uint8_t* q, const uint8_t* qmask, int32_t nq, const uint8_t* d, const uint8_t* dmask, int32_t nd,
                     const uint8_t* db_skip, int32_t dim, int32_t K, int32_t* topk_idx, int32_t* topk_dist) {
    if (!q || !d || !topk_idx || !topk_dist) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (nq <= 0) return MCS_OK;
    const bool masked = qmask && dmask;
    Dev dq, dqm, dd, ddm, ds, di, dt;
    CUDA_CHECK(dq.upload(q, (size_t)nq * dim)); CUDA_CHECK(dd.upload(d, (size_t)nd * dim));
    CUDA_CHECK(di.alloc((size_t)nq * K * 4)); CUDA_CHECK(dt.alloc((size_t)nq * K * 4));
    if (masked) { CUDA_CHECK(dqm.upload(qmask, (size_t)nq * dim)); CUDA_CHECK(ddm.upload(dmask, (size_t)nd * dim)); }
    if (db_skip) CUDA_CHECK(ds.upload(db_skip, nd));
    int rc = mcs_hamming_topk_device(dq.as<uint8_t>(), masked ? dqm.as<uint8_t>() : nullptr, nq, dd.as<uint8_t>(),
                                     masked ? ddm.as<uint8_t>() : nullptr, nd, db_skip ? ds.as<uint8_t>() : nullptr, dim, K,
                                     di.as<int>(), dt.as<int>(), nullptr);
    if (rc) return rc;
    CUDA_CHECK(cudaMemcpy(topk_idx, di.p, (size_t)nq * K * 4, cudaMemcpyDeviceToHost));
    CUDA_CHECK(cudaMemcpy(topk_dist, dt.p, (size_t)nq * K * 4, cudaMemcpyDeviceToHost));
    return MCS_OK;
}

int mcs_match_stream_device(const uint8_t* desc_dev, const uint8_t* dmask_dev, const int32_t* counts_dev, int32_t n_frames,
                            int32_t n_cams, int32_t capacity, int32_t dim, int32_t K, int32_t* match_idx_dev,
                            int32_t* match_dist_dev, void* stream) {
    if (!desc_dev || !counts_dev || !match_idx_dev || !match_dist_dev) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (n_frames < 1 || n_cams < 1 || capacity < 1 || K < 1 || K > 8) return mcs_fail(MCS_ERR_INVALID, "bad sizes (K must be 1..8)");
    if (int rc = check_desc_dim(dim)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    CUDA_CHECK(launch_hamming_stream(desc_dev, dmask_dev, counts_dev, 0, n_frames * n_cams, n_cams, capacity, dim, K, 0xFFFFFFFFu, match_idx_dev, match_dist_dev, st));
    return MCS_OK;
}

int mcs_match_stream_greedy_device(const uint8_t* desc_dev, const uint8_t* dmask_dev, const int32_t* counts_dev, int32_t n_frames,
                                   int32_t n_cams, int32_t capacity, int32_t dim, int32_t th_low, double nnratio,
                                   int32_t* matches12_dev, int32_t* nmatches_dev, void* stream) {
    if (!desc_dev || !counts_dev || !matches12_dev || !nmatches_dev) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (n_frames < 1 || n_cams < 1 || capacity < 1 || capacity > 65535) return mcs_fail(MCS_ERR_INVALID, "bad sizes (capacity must be 1..65535)");
    if (int rc = check_desc_dim(dim)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    // K-best list length (the acceptance is exact for any K; K only sets how often the replay rescans).  H100 80GB HBM3, 400 W limit, bench.py config 2, 2 alternating runs:
    // K = 8 16.08 / 16.15 ms per 384-image step (47.9 Mfeatures/s) against 16.85 / 16.79 ms with K = 4.
    constexpr int K = 8;
    const int n_images = n_frames * n_cams;
    const size_t list_bytes = (size_t)n_images * capacity * K * sizeof(int);
    StreamScratch sc;
    cudaError_t e = sc.alloc({list_bytes, list_bytes, n_images * sizeof(int)}, st);      // list indices, list distances, redo
    if (e == cudaSuccess)
        e = launch_hamming_stream(desc_dev, dmask_dev, counts_dev, 0, n_images, n_cams, capacity, dim, K, greedy_dist_bound(th_low, nnratio),
                                  sc.at<int>(0), sc.at<int>(1), st);
    if (e == cudaSuccess)
        e = launch_stream_replay(sc.at<int>(0), sc.at<int>(1), counts_dev, desc_dev, dmask_dev, dim, 0, n_images, n_cams, capacity, K, th_low,
                                 nnratio, matches12_dev, nmatches_dev, sc.at<int>(2), st);
    CUDA_CHECK(sc.release(e));
    return MCS_OK;
}

int mcs_match_stream_replay_device(const int32_t* match_idx_dev, const int32_t* match_dist_dev, const int32_t* counts_dev,
                                   const uint8_t* desc_dev, const uint8_t* dmask_dev, int32_t n_frames, int32_t n_cams, int32_t capacity,
                                   int32_t dim, int32_t K, int32_t th_low, double nnratio, int32_t* matches12_dev, int32_t* nmatches_dev,
                                   int32_t* redo_dev, void* stream) {
    if (!match_idx_dev || !match_dist_dev || !counts_dev || !desc_dev || !matches12_dev || !nmatches_dev || !redo_dev)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (n_frames < 1 || n_cams < 1 || capacity < 1 || capacity > 65535 || K < 1 || K > 8) return mcs_fail(MCS_ERR_INVALID, "bad sizes (K must be 1..8)");
    if (int rc = check_desc_dim(dim)) return rc;
    CUDA_CHECK(launch_stream_replay(match_idx_dev, match_dist_dev, counts_dev, desc_dev, dmask_dev, dim, 0, n_frames * n_cams, n_cams, capacity, K,
                                    th_low, nnratio, matches12_dev, nmatches_dev, redo_dev, (cudaStream_t)stream));
    return MCS_OK;
}

// SearchByBoW(KF1, KF2) (ref :885-966) with the descriptors already on the device: K best unmatched database entries per query
// on the GPU, sequential greedy replay on the host, further rounds for queries whose list was used up by earlier matches
static thread_local int g_bf_rounds = 0;
int mcs_last_bruteforce_rounds(void) { return g_bf_rounds; }

// seg[0..n_seg]: query segments (e.g. the key frames of a batch) whose "database entry already matched" state is independent, as
// it is between separate SearchByBoW(KF1, KF2) calls of the reference; seg == nullptr: one segment [0, nq).  One K-best launch
// serves all queries of all segments (they start from the same database state); the ordered acceptance (ref :899-961) then runs
// on the device as well, one CTA per segment (bruteforce_replay_kernel): a query whose list was used up by matches accepted
// earlier in its segment is rescanned exactly inside the kernel.  The host only moves the small validity / offset arrays in and
// the matches out.
static int bruteforce_core(const uint8_t* q_dev, const uint8_t* qm_dev, const uint8_t* valid1, int nq, const uint8_t* d_dev,
                           const uint8_t* dm_dev, const uint8_t* valid2, int nd, int dim, int th_low, double nnratio, int* matches12,
                           int* nmatches, cudaStream_t st, const int* seg = nullptr, int n_seg = 1) {
    const bool masked = qm_dev && dm_dev;
    // K = 8: with the relevance bound only entries that matter are ever inserted, so long lists cost nothing in the distance loop
    // and leave few queries to rescan (BASELINE config 4: 207 of 4000 per key frame at K = 4, 60 at K = 8)
    constexpr int K = 8;
    const int one_seg[2] = {0, nq};
    if (!seg) { seg = one_seg; n_seg = 1; }
    // the acceptance kernel keeps one bit per database entry in shared memory (kernels.h: bruteforce_replay_smem): at most
    // 1 622 016 entries.  Checked here so that a larger database is refused before anything is launched.
    if (nd > bruteforce_max_nd(K))
        return mcs_fail(MCS_ERR_UNSUPPORTED, "more than " + std::to_string(bruteforce_max_nd(K)) + " database descriptors in one call");
    std::vector<uint8_t> skip(nd, 0);
    if (valid2) for (int i = 0; i < nd; ++i) skip[i] = valid2[i] ? 0 : 1;
    g_bf_rounds = 1;
    Dev ds, di, dt, dv1, dseg, dm12, dnm;
    CUDA_CHECK(ds.upload_async(skip.data(), nd, st));
    CUDA_CHECK(di.alloc((size_t)nq * K * 4)); CUDA_CHECK(dt.alloc((size_t)nq * K * 4)); CUDA_CHECK(dv1.alloc(nq));
    if (valid1) CUDA_CHECK(cudaMemcpyAsync(dv1.p, valid1, nq, cudaMemcpyHostToDevice, st));
    CUDA_CHECK(dseg.upload_async(seg, (size_t)(n_seg + 1) * 4, st));
    CUDA_CHECK(dm12.alloc((size_t)nq * 4)); CUDA_CHECK(dnm.alloc((size_t)n_seg * 4));
    // Entries at or beyond the relevance bound of (th_low, nnratio) stay out of the lists: a list shorter than K then means "every
    // entry that can influence the decision is here".
    CUDA_CHECK(launch_hamming_topk(q_dev, masked ? qm_dev : nullptr, nq, d_dev, masked ? dm_dev : nullptr, nd, ds.as<uint8_t>(), dim, K,
                                   greedy_dist_bound(th_low, nnratio), di.as<int>(), dt.as<int>(), st));
    // the replay kernel wants "valid" bytes for the database (1 = usable): reuse the skip buffer inverted on the fly is not worth a
    // kernel -- upload the caller's array when there is one
    Dev dv2;
    if (valid2) CUDA_CHECK(dv2.upload_async(valid2, nd, st));
    CUDA_CHECK(launch_bruteforce_replay(di.as<int>(), dt.as<int>(), K, q_dev, masked ? qm_dev : nullptr, valid1 ? dv1.as<uint8_t>() : nullptr,
                                        dseg.as<int>(), n_seg, nq, d_dev, masked ? dm_dev : nullptr, valid2 ? dv2.as<uint8_t>() : nullptr, nd, dim, th_low,
                                        nnratio, dm12.as<int>(), dnm.as<int>(), st));
    CUDA_CHECK(cudaMemcpyAsync(matches12, dm12.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaMemcpyAsync(nmatches, dnm.p, (size_t)n_seg * 4, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    return MCS_OK;
}

int mcs_match_bruteforce_batch_device(const uint8_t* q_dev, const uint8_t* qmask_dev, const uint8_t* valid1, const int32_t* seg_start,
                                      int32_t n_seg, const uint8_t* d_dev, const uint8_t* dmask_dev, const uint8_t* valid2, int32_t nd,
                                      int32_t dim, int32_t th_low, double nnratio, int32_t* matches12, int32_t* nmatches, void* stream) {
    if (!q_dev || !d_dev || !matches12 || !nmatches || !seg_start) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (int rc = check_desc_dim(dim)) return rc;
    if (n_seg < 1 || seg_start[0] != 0) return mcs_fail(MCS_ERR_INVALID, "seg_start must begin at 0 and hold n_seg + 1 offsets");
    for (int s = 0; s < n_seg; ++s)
        if (seg_start[s + 1] < seg_start[s]) return mcs_fail(MCS_ERR_INVALID, "seg_start must be non-decreasing");
    const int nq = seg_start[n_seg];
    for (int s = 0; s < n_seg; ++s) nmatches[s] = 0;
    for (int i = 0; i < nq; ++i) matches12[i] = -1;
    if (nq <= 0 || nd <= 0) return MCS_OK;
    return bruteforce_core(q_dev, qmask_dev, valid1, nq, d_dev, dmask_dev, valid2, nd, dim, th_low, nnratio, matches12, nmatches,
                           (cudaStream_t)stream, seg_start, n_seg);
}

int mcs_match_bruteforce_device(const uint8_t* q_dev, const uint8_t* qmask_dev, const uint8_t* valid1, int32_t nq, const uint8_t* d_dev,
                                const uint8_t* dmask_dev, const uint8_t* valid2, int32_t nd, int32_t dim, int32_t th_low, double nnratio,
                                int32_t* matches12, int32_t* nmatches, void* stream) {
    if (!q_dev || !d_dev || !matches12 || !nmatches) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (int rc = check_desc_dim(dim)) return rc;
    *nmatches = 0;
    for (int i = 0; i < nq; ++i) matches12[i] = -1;
    if (nq <= 0 || nd <= 0) return MCS_OK;
    return bruteforce_core(q_dev, qmask_dev, valid1, nq, d_dev, dmask_dev, valid2, nd, dim, th_low, nnratio, matches12, nmatches,
                           (cudaStream_t)stream);
}

int mcs_match_bruteforce(const uint8_t* q, const uint8_t* qmask, const uint8_t* valid1, int32_t nq, const uint8_t* d,
                         const uint8_t* dmask, const uint8_t* valid2, int32_t nd, int32_t dim, int32_t th_low, double nnratio,
                         int32_t* matches12, int32_t* nmatches) {
    if (!q || !d || !matches12 || !nmatches) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (int rc = check_desc_dim(dim)) return rc;
    *nmatches = 0;
    for (int i = 0; i < nq; ++i) matches12[i] = -1;
    if (nq <= 0 || nd <= 0) return MCS_OK;
    const bool masked = qmask && dmask;
    Dev dq, dqm, dd, ddm;
    CUDA_CHECK(dq.upload(q, (size_t)nq * dim)); CUDA_CHECK(dd.upload(d, (size_t)nd * dim));
    if (masked) { CUDA_CHECK(dqm.upload(qmask, (size_t)nq * dim)); CUDA_CHECK(ddm.upload(dmask, (size_t)nd * dim)); }
    return bruteforce_core(dq.as<uint8_t>(), masked ? dqm.as<uint8_t>() : nullptr, valid1, nq, dd.as<uint8_t>(),
                           masked ? ddm.as<uint8_t>() : nullptr, valid2, nd, dim, th_low, nnratio, matches12, nmatches, nullptr);
}

int mcs_search_for_triangulation(const uint8_t* desc1, const uint8_t* mask1, const int32_t* cam1, const uint8_t* free1,
                                 const double* rays1, int32_t n1, const uint8_t* desc2, const uint8_t* mask2, const int32_t* cam2,
                                 const uint8_t* free2, const double* rays2, int32_t n2, int32_t dim, int32_t th_low, const double* E,
                                 int32_t n_cams, double epi_thresh, int32_t* matches12, int32_t* nmatches) {
    if (!desc1 || !cam1 || !free1 || !rays1 || !desc2 || !cam2 || !free2 || !rays2 || !E || !matches12 || !nmatches)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (int rc = check_desc_dim(dim)) return rc;
    *nmatches = 0;
    for (int i = 0; i < n1; ++i) matches12[i] = -1;
    if (n1 <= 0 || n2 <= 0) return MCS_OK;
    const bool masked = mask1 && mask2;
    constexpr int K = 8;
    Dev dd, ddm, ds;
    CUDA_CHECK(dd.upload(desc2, (size_t)n2 * dim)); CUDA_CHECK(ds.alloc(n2));
    if (masked) CUDA_CHECK(ddm.upload(mask2, (size_t)n2 * dim));
    std::vector<uint8_t> matched2(n2, 0), skip(n2);
    int nm = 0;
    for (int c = 0; c < n_cams; ++c) {                 // queries of camera c only ever see database entries of camera c (ref :1043-1045)
        std::vector<int> q_idx;
        for (int i = 0; i < n1; ++i) if (cam1[i] == c && free1[i]) q_idx.push_back(i);
        if (q_idx.empty()) continue;
        const int nq = (int)q_idx.size();
        std::vector<uint8_t> qd((size_t)nq * dim), qmk(masked ? (size_t)nq * dim : 0);
        for (int k = 0; k < nq; ++k) {
            std::memcpy(&qd[(size_t)k * dim], desc1 + (size_t)q_idx[k] * dim, dim);
            if (masked) std::memcpy(&qmk[(size_t)k * dim], mask1 + (size_t)q_idx[k] * dim, dim);
        }
        Dev dq, dqm, di, dt;
        CUDA_CHECK(dq.upload(qd.data(), (size_t)nq * dim)); CUDA_CHECK(di.alloc((size_t)nq * K * 4)); CUDA_CHECK(dt.alloc((size_t)nq * K * 4));
        if (masked) CUDA_CHECK(dqm.upload(qmk.data(), (size_t)nq * dim));
        std::vector<int> tidx((size_t)nq * K), tdist((size_t)nq * K);
        const double* Ecc = E + ((size_t)c * n_cams + c) * 9;
        // one GPU pass: the K best database entries (distance, index) of every query under the skip state at the start
        for (int i = 0; i < n2; ++i) skip[i] = (matched2[i] || !free2[i] || cam2[i] != c) ? 1 : 0;
        CUDA_CHECK(cudaMemcpy(ds.p, skip.data(), n2, cudaMemcpyHostToDevice));
        int rc = mcs_hamming_topk_device(dq.as<uint8_t>(), masked ? dqm.as<uint8_t>() : nullptr, nq, dd.as<uint8_t>(),
                                         masked ? ddm.as<uint8_t>() : nullptr, n2, ds.as<uint8_t>(), dim, K, di.as<int>(), dt.as<int>(), nullptr);
        if (rc) return rc;
        CUDA_CHECK(cudaMemcpy(tidx.data(), di.p, (size_t)nq * K * 4, cudaMemcpyDeviceToHost));
        CUDA_CHECK(cudaMemcpy(tdist.data(), dt.p, (size_t)nq * K * 4, cudaMemcpyDeviceToHost));
        std::vector<int> pi(K), pd(K), marked;
        for (int k = 0; k < nq; ++k) {                   // sequential replay (ref :1015-1107)
            const double* r1 = rays1 + 3 * (size_t)q_idx[k];
            const int* li = &tidx[(size_t)k * K];
            const int* ld = &tdist[(size_t)k * K];
            int best = -1, dist_th = 0, found = -1;
            bool done = false;
            auto walk = [&](const int* idx, const int* dst) {      // returns true when the list was consumed without a decision
                for (int e = 0; e < K; ++e) {
                    if (idx[e] < 0 || dst[e] > th_low) { done = true; return false; }     // no candidate with dist <= TH_LOW_ left
                    if (matched2[idx[e]]) continue;                                       // taken by an earlier query of this pass
                    if (best < 0) { best = dst[e]; dist_th = (int)lrint(2.0 * best); }
                    if (dst[e] > dist_th) { done = true; return false; }
                    if (cam_epipolar_ok(r1, rays2 + 3 * (size_t)idx[e], Ecc, epi_thresh)) { found = idx[e]; done = true; return false; }
                    skip[idx[e]] = 2; marked.push_back(idx[e]);                           // examined by this query (paging only)
                }
                return true;
            };
            if (walk(li, ld)) {
                // more than K candidates inside both thresholds: page through the rest for this one query on the GPU
                std::vector<uint8_t> sk(n2);
                while (!done) {
                    for (int i = 0; i < n2; ++i) sk[i] = (matched2[i] || !free2[i] || cam2[i] != c || skip[i] == 2) ? 1 : 0;
                    CUDA_CHECK(cudaMemcpy(ds.p, sk.data(), n2, cudaMemcpyHostToDevice));
                    rc = mcs_hamming_topk_device(dq.as<uint8_t>() + (size_t)k * dim, masked ? dqm.as<uint8_t>() + (size_t)k * dim : nullptr, 1,
                                                 dd.as<uint8_t>(), masked ? ddm.as<uint8_t>() : nullptr, n2, ds.as<uint8_t>(), dim, K,
                                                 di.as<int>(), dt.as<int>(), nullptr);
                    if (rc) return rc;
                    CUDA_CHECK(cudaMemcpy(pi.data(), di.p, K * 4, cudaMemcpyDeviceToHost));
                    CUDA_CHECK(cudaMemcpy(pd.data(), dt.p, K * 4, cudaMemcpyDeviceToHost));
                    if (!walk(pi.data(), pd.data())) break;
                }
            }
            for (int e : marked) skip[e] = 0;                                             // clear this query's paging marks
            marked.clear();
            if (found >= 0) { matches12[q_idx[k]] = found; matched2[found] = 1; ++nm; }
        }
    }
    *nmatches = nm;
    return MCS_OK;
}

int mcs_window_search(const mcs_frame_view* frame, const mcs_window_query* queries, int32_t nq, const uint8_t* qdesc,
                      const uint8_t* qmask, int32_t max_cand, int32_t* cand_idx, int32_t* cand_dist, int32_t* cand_count) {
    if (!frame || !queries || !qdesc || !cand_idx || !cand_dist || !cand_count || max_cand < 1)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (nq <= 0) return MCS_OK;
    FrameDev fd;
    int rc = upload_frame(frame, fd, nullptr);
    if (rc) return rc;
    int rows = 0;
    for (int i = 0; i < nq; ++i) {
        if (queries[i].cam < 0 || queries[i].cam >= frame->n_cams) return mcs_fail(MCS_ERR_INVALID, "query camera out of range");
        if (queries[i].desc_index < 0) return mcs_fail(MCS_ERR_INVALID, "negative query descriptor index");
        rows = std::max(rows, queries[i].desc_index + 1);
    }
    std::vector<int> ci, cd, co;
    rc = window_search_compact(fd, queries, nq, qdesc, qmask, rows, frame->dim, max_cand, ci, cd, co, nullptr);
    if (rc) return rc;
    // the kernel stores a candidate at its visiting position, so the first max_cand of a longer list are what a list of
    // max_cand slots would hold
    bool overflow = false;
    for (int q = 0; q < nq; ++q) {
        const int count = co[q + 1] - co[q], n = std::min(count, max_cand);
        int32_t* idx = cand_idx + (size_t)q * max_cand;
        int32_t* dist = cand_dist + (size_t)q * max_cand;
        std::copy(ci.begin() + co[q], ci.begin() + co[q] + n, idx);
        std::copy(cd.begin() + co[q], cd.begin() + co[q] + n, dist);
        std::fill(idx + n, idx + max_cand, -1);
        std::fill(dist + n, dist + max_cand, 0);
        cand_count[q] = count;
        overflow |= count > max_cand;
    }
    if (overflow) return mcs_fail(MCS_ERR_CAPACITY, "max_cand too small for at least one query");
    return MCS_OK;
}

int mcs_frame_prepare(const mcs_keypoint* keys, const int32_t* key_cam, int32_t n_keys, const mcs_ocam* cams, int32_t n_cams,
                      double* rays_out, int32_t* cell_start_out, int32_t* cell_items_out, int32_t* n_in_grid) {
    if (!keys || !key_cam || !cams || !rays_out || !cell_start_out || !cell_items_out || !n_in_grid)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (n_keys < 0 || n_cams < 1) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    FrameGrid g;
    Dev rays;
    const int rc = build_frame_grid(keys, key_cam, n_keys, cams, n_cams, g, &rays, nullptr);
    if (rc) return rc;
    const int ncell = n_cams * MCS_FRAME_GRID_COLS * MCS_FRAME_GRID_ROWS;
    CUDA_CHECK(cudaMemcpy(rays_out, rays.p, (size_t)n_keys * 24, cudaMemcpyDeviceToHost));
    CUDA_CHECK(cudaMemcpy(cell_start_out, g.cell_start.p, (size_t)(ncell + 1) * 4, cudaMemcpyDeviceToHost));
    CUDA_CHECK(cudaMemcpy(cell_items_out, g.cell_items.p, (size_t)n_keys * 4, cudaMemcpyDeviceToHost));
    *n_in_grid = cell_start_out[ncell];
    return MCS_OK;
}

int mcs_project_mappoints(int32_t n_cams, const double* mtmc_inv, const double* mtmc, const mcs_ocam* cams, const uint8_t* masks,
                          int32_t n_points, const double* world_pos, const double* normal, const double* min_dist,
                          const double* max_dist, const double* scale_factors, int32_t n_levels, uint8_t* in_view, int32_t* level,
                          double* proj_x, double* proj_y, double* view_cos) {
    if (!mtmc_inv || !mtmc || !cams || !masks || !world_pos || !normal || !min_dist || !max_dist || !scale_factors || !in_view ||
        !level || !proj_x || !proj_y || !view_cos)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (n_cams < 1 || n_points < 0 || n_levels < 1) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    if (n_points == 0) return MCS_OK;
    size_t mask_bytes = 0;
    for (int c = 0; c < n_cams; ++c) {
        if (cams[c].width != cams[0].width || cams[c].height != cams[0].height)
            return mcs_fail(MCS_ERR_UNSUPPORTED, "cameras of different image sizes");
        mask_bytes += (size_t)cams[c].width * cams[c].height;
    }
    const size_t n = (size_t)n_points * n_cams;
    Dev dmi, dm, dc, dk, dp, dn, dmn, dmx, dsf, div, dlv, dpx, dpy, dvc;
    CUDA_CHECK(dmi.upload(mtmc_inv, n_cams * 128)); CUDA_CHECK(dm.upload(mtmc, n_cams * 128));
    CUDA_CHECK(dc.upload(cams, n_cams * sizeof(mcs_ocam))); CUDA_CHECK(dk.upload(masks, mask_bytes));
    CUDA_CHECK(dp.upload(world_pos, (size_t)n_points * 24)); CUDA_CHECK(dn.upload(normal, (size_t)n_points * 24));
    CUDA_CHECK(dmn.upload(min_dist, (size_t)n_points * 8)); CUDA_CHECK(dmx.upload(max_dist, (size_t)n_points * 8));
    CUDA_CHECK(dsf.upload(scale_factors, n_levels * 8));
    CUDA_CHECK(div.alloc(n)); CUDA_CHECK(dlv.alloc(n * 4)); CUDA_CHECK(dpx.alloc(n * 8)); CUDA_CHECK(dpy.alloc(n * 8)); CUDA_CHECK(dvc.alloc(n * 8));
    CUDA_CHECK(launch_frustum(n_cams, dmi.as<double>(), dm.as<double>(), dc.as<mcs_ocam>(), dk.as<uint8_t>(), n_points, dp.as<double>(),
                              dn.as<double>(), dmn.as<double>(), dmx.as<double>(), dsf.as<double>(), n_levels, div.as<uint8_t>(),
                              dlv.as<int>(), dpx.as<double>(), dpy.as<double>(), dvc.as<double>(), nullptr, nullptr));
    CUDA_CHECK(cudaMemcpy(in_view, div.p, n, cudaMemcpyDeviceToHost));
    CUDA_CHECK(cudaMemcpy(level, dlv.p, n * 4, cudaMemcpyDeviceToHost));
    CUDA_CHECK(cudaMemcpy(proj_x, dpx.p, n * 8, cudaMemcpyDeviceToHost));
    CUDA_CHECK(cudaMemcpy(proj_y, dpy.p, n * 8, cudaMemcpyDeviceToHost));
    CUDA_CHECK(cudaMemcpy(view_cos, dvc.p, n * 8, cudaMemcpyDeviceToHost));
    return MCS_OK;
}

int mcs_search_windows(const mcs_frame_view* f, const mcs_window_query* queries, int32_t nq, const uint8_t* qdesc,
                       const uint8_t* qmask, const int32_t* query_tag, int32_t rule, double nnratio, int32_t threshold,
                       int32_t* assigned, int32_t* nmatches) {
    if (!f || !queries || !qdesc || !query_tag || !assigned || !nmatches) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (rule < 0 || rule > MCS_RULE_SCW) return mcs_fail(MCS_ERR_INVALID, "unknown rule");
    *nmatches = 0;
    if (nq <= 0) return MCS_OK;
    int rows = 0;
    for (int i = 0; i < nq; ++i) {
        if (queries[i].cam < 0 || queries[i].cam >= f->n_cams) return mcs_fail(MCS_ERR_INVALID, "query camera out of range");
        if (query_tag[i] < 0) return mcs_fail(MCS_ERR_INVALID, "query tags must be >= 0");
        if (queries[i].desc_index < 0) return mcs_fail(MCS_ERR_INVALID, "negative query descriptor index");
        rows = std::max(rows, queries[i].desc_index + 1);
    }
    FrameDev fd;
    int rc = upload_frame(f, fd, nullptr);
    if (rc) return rc;
    if (rule == MCS_RULE_SCW) {
        // descriptor row of candidate idx for a query of camera c = row idx of camera c's matrix (ref :2367,2372): needs the
        // camera-major keypoint order of src/cMultiFrame.cpp:168-184
        std::vector<int> first(f->n_cams + 1, 0);
        for (int i = 0; i < f->n_keys; ++i) {
            if (i && f->key_cam[i] < f->key_cam[i - 1]) return mcs_fail(MCS_ERR_INVALID, "MCS_RULE_SCW needs camera-major keypoint order");
            ++first[f->key_cam[i] + 1];
        }
        for (int c = 0; c < f->n_cams; ++c) first[c + 1] += first[c];
        CUDA_CHECK(fd.cam_first.upload(first.data(), first.size() * 4));
        fd.view.cam_first = fd.cam_first.as<int>();
    }
    std::vector<int> ci, cd, co;
    rc = window_search_compact(fd, queries, nq, qdesc, qmask, rows, f->dim, 32, ci, cd, co, nullptr);
    if (rc) return rc;
    int nm = 0;
    for (int qi = 0; qi < nq; ++qi) {       // sequential greedy replay over the GPU-computed candidate lists
        const int n = co[qi + 1] - co[qi];
        const bool stateless = rule == MCS_RULE_BEST_FREE || rule == MCS_RULE_FIRST_FREE;
        if (n == 0) { if (stateless) assigned[qi] = -1; continue; }
        if (rule == MCS_RULE_FIRST_FREE) {
            // Fuse(pKF, vpMapPoints, th) computes the distance and throws it away (ref :1506-1514: `dist` stays 0), so the first
            // candidate that passes the level filter wins with distance 0 <= TH_LOW_
            assigned[qi] = 0 <= threshold ? ci[co[qi]] : -1;
            nm += assigned[qi] >= 0;
            continue;
        }
        int bestDist = INT_MAX, bestLevel = -1, bestDist2 = INT_MAX, bestLevel2 = -1, bestIdx = -1;
        for (int k = 0; k < n; ++k) {
            const int idx = ci[co[qi] + k];
            if (!stateless && assigned[idx] >= 0) continue;
            const int dist = cd[co[qi] + k];
            if (dist < bestDist) {
                bestDist2 = bestDist; bestDist = dist; bestLevel2 = bestLevel;
                bestLevel = f->keys[idx].octave; bestIdx = idx;
            } else if (dist < bestDist2) {
                bestLevel2 = f->keys[idx].octave; bestDist2 = dist;
            }
        }
        if (rule == MCS_RULE_BEST_FREE) {          // stateless: the answer of query qi
            const bool hit = bestIdx >= 0 && bestDist <= threshold;
            assigned[qi] = hit ? bestIdx : -1;
            nm += hit;
            continue;
        }
        bool ok;
        if (rule == MCS_RULE_RATIO) ok = (double)bestDist <= (double)bestDist2 * nnratio && bestDist <= threshold;
        else if (rule == MCS_RULE_BEST) ok = bestDist <= threshold;
        else if (rule == MCS_RULE_SCW) ok = bestDist <= threshold && bestIdx > 0;          // `bestIdx > 0` as written at ref :2385
        else ok = bestDist <= threshold && !(bestLevel == bestLevel2 && bestDist > nnratio * bestDist2);
        if (ok && bestIdx >= 0) {
            assigned[bestIdx] = query_tag[qi];
            ++nm;
        }
    }
    *nmatches = nm;
    return MCS_OK;
}

int mcs_search_by_projection(const mcs_frame_view* f, const mcs_mappoint_view* mps, double th, double nnratio, int32_t th_high,
                             int32_t having_masks, int32_t* frame_mp, int32_t* nmatches) {
    if (!f || !mps || !frame_mp || !nmatches) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (having_masks && (!f->dmask || !mps->dmask)) return mcs_fail(MCS_ERR_INVALID, "masks requested but not supplied");
    *nmatches = 0;
    // queries in the reference's visiting order: map point outer, camera inner (ref :74-98)
    std::vector<mcs_window_query> qs;
    std::vector<int> tags;
    {
        size_t n_view = 0;
        const size_t n_all = (size_t)mps->n_points * f->n_cams;
        for (size_t k = 0; k < n_all; ++k) n_view += mps->in_view[k] != 0;
        qs.reserve(n_view); tags.reserve(n_view);
    }
    const bool bFactor = th != 1.0;
    for (int i = 0; i < mps->n_points; ++i) {
        if (mps->bad && mps->bad[i]) continue;
        for (int cam = 0; cam < f->n_cams; ++cam) {
            const size_t k = (size_t)i * f->n_cams + cam;
            if (!mps->in_view[k]) continue;
            const int lvl = mps->level[k];
            if (lvl < 0 || lvl >= f->n_levels) return mcs_fail(MCS_ERR_INVALID, "map point scale level out of range");
            double r = mps->view_cos[k] > 0.998 ? 2.5 : 4.0;   // RadiusByViewingCos (ref :169-175)
            if (bFactor) r *= th;
            mcs_window_query q;
            q.cam = cam; q.min_level = lvl - 1; q.max_level = lvl; q.desc_index = i;
            q.x = mps->proj_x[k]; q.y = mps->proj_y[k]; q.r = r * f->scale_factors[lvl];
            qs.push_back(q);
            tags.push_back(i);
        }
    }
    if (qs.empty()) return MCS_OK;
    mcs_frame_view fv = *f;
    if (!having_masks) fv.dmask = nullptr;
    return mcs_search_windows(&fv, qs.data(), (int)qs.size(), mps->desc, having_masks ? mps->dmask : nullptr, tags.data(),
                              MCS_RULE_LEVEL_RATIO, nnratio, th_high, frame_mp, nmatches);
}

int mcs_project_mappoints_device(int32_t n_cams, const double* mtmc_inv, const double* mtmc, const mcs_ocam* cams, const uint8_t* masks_dev,
                                 int32_t n_points, const double* world_pos_dev, const double* normal_dev, const double* min_dist_dev,
                                 const double* max_dist_dev, const double* scale_factors, int32_t n_levels, const uint8_t* skip_dev,
                                 uint8_t* in_view_dev, int32_t* level_dev, double* proj_x_dev, double* proj_y_dev, double* view_cos_dev,
                                 void* stream) {
    if (!mtmc_inv || !mtmc || !cams || !masks_dev || !world_pos_dev || !normal_dev || !min_dist_dev || !max_dist_dev || !scale_factors ||
        !in_view_dev || !level_dev || !proj_x_dev || !proj_y_dev || !view_cos_dev)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (n_cams < 1 || n_points < 0 || n_levels < 1 || n_levels > MCS_MAX_LEVELS) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    for (int c = 0; c < n_cams; ++c)
        if (cams[c].width != cams[0].width || cams[c].height != cams[0].height)
            return mcs_fail(MCS_ERR_UNSUPPORTED, "cameras of different image sizes");
    cudaStream_t st = (cudaStream_t)stream;
    // poses, camera models and scale factors: one scratch block, staged in stream order
    StreamScratch sc;
    const double *d_mtmc_inv, *d_mtmc, *d_sf;
    const mcs_ocam* d_cams;
    cudaError_t e = open_scratch(sc, {}, st, host_in(d_mtmc_inv, mtmc_inv, 16 * (size_t)n_cams), host_in(d_mtmc, mtmc, 16 * (size_t)n_cams),
                                 host_in(d_cams, cams, n_cams), host_in(d_sf, scale_factors, n_levels));
    if (e == cudaSuccess)
        e = launch_frustum(n_cams, d_mtmc_inv, d_mtmc, d_cams, masks_dev, n_points, world_pos_dev, normal_dev, min_dist_dev, max_dist_dev, d_sf,
                           n_levels, in_view_dev, level_dev, proj_x_dev, proj_y_dev, view_cos_dev, skip_dev, st);
    CUDA_CHECK(sc.release(e));
    return sync_if_null_stream(stream);
}

int mcs_search_by_projection_max_rounds(void) { return proj_search_max_rounds(); }

int mcs_search_by_projection_device(const void* packed_dev, int32_t n_parts, int32_t part_images, int32_t first_image, int32_t n_cams,
                                    int32_t capacity, int32_t dim, const int32_t* cam_width, const int32_t* cam_height, int32_t n_levels,
                                    const double* scale_factors, const mcs_mappoint_dev_view* mps, double th, double nnratio, int32_t th_high,
                                    int32_t having_masks, int32_t* frame_mp_dev, int32_t* nmatches_dev, int32_t* status_dev, int32_t* diag_dev,
                                    void* stream) {
    if (!packed_dev || !cam_width || !cam_height || !scale_factors || !mps || !frame_mp_dev || !nmatches_dev || !status_dev)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    const mcs_packed_frame frame{packed_dev, n_parts, part_images, first_image};
    if (n_levels < 1 || n_levels > MCS_MAX_LEVELS) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    if (int rc = check_packed_frames(n_cams, capacity, dim, &frame, nullptr)) return rc;
    if (mps->n_points < 0) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    if (!mps->in_view || !mps->level || !mps->proj_x || !mps->proj_y || !mps->view_cos || !mps->desc)
        return mcs_fail(MCS_ERR_INVALID, "null map-point array");
    if (having_masks && !mps->dmask) return mcs_fail(MCS_ERR_INVALID, "masks requested but not supplied");
    if (int rc = check_cam_sizes(n_cams, cam_width, cam_height, false)) return rc;
    if (int rc = check_query_bound((long long)mps->n_points * n_cams, "more than 2^24 - 1 (map point, camera) entries in one call")) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const std::vector<PsCamSlots> slots = packed_slots(frame, n_cams, capacity, dim);
    ProjSearchArgs a{};
    set_searched_frame(a, slots, capacity, dim, cam_width, cam_height, th_high, having_masks, frame_mp_dev, nmatches_dev, status_dev, diag_dev);
    a.n_levels = n_levels; a.sf = scale_factors; a.n_points = mps->n_points;
    a.bad = mps->bad; a.in_view = mps->in_view; a.level = mps->level; a.px = mps->proj_x; a.py = mps->proj_y; a.vcos = mps->view_cos;
    a.mp_desc = mps->desc; a.mp_dmask = having_masks ? mps->dmask : nullptr;
    a.th = th; a.nnratio = nnratio;
    CUDA_CHECK(launch_search_by_projection(a, st));
    return sync_if_null_stream(stream);
}

int mcs_search_by_projection_last_device(const mcs_packed_frame* cur, const mcs_packed_frame* last, int32_t n_cams, int32_t capacity,
                                         int32_t dim, const mcs_ocam* cams, const uint8_t* masks_dev, int32_t n_levels,
                                         const double* scale_factors, const double* mtmc_inv, const int32_t* last_mp_dev,
                                         const uint8_t* last_outlier_dev, int32_t n_points, const double* world_pos_dev, const uint8_t* bad_dev,
                                         double th, int32_t th_high, int32_t having_masks, int32_t* cur_mp_dev, int32_t* nmatches_dev,
                                         int32_t* status_dev, int32_t* diag_dev, void* stream) {
    if (!cur || !last || !cams || !masks_dev || !scale_factors || !mtmc_inv || !last_mp_dev || !world_pos_dev || !cur_mp_dev ||
        !nmatches_dev || !status_dev)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (n_levels < 1 || n_levels > MCS_MAX_LEVELS) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    if (int rc = check_packed_frames(n_cams, capacity, dim, cur, last)) return rc;
    if (n_points < 0) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    const CamSizes cz(cams, n_cams);
    if (int rc = check_cam_sizes(n_cams, cz.w.data(), cz.h.data(), true)) return rc;
    if (int rc = check_query_bound((long long)n_cams * capacity, "n_cams * capacity must stay below 2^24")) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const std::vector<PsCamSlots> cs = packed_slots(*cur, n_cams, capacity, dim), ls = packed_slots(*last, n_cams, capacity, dim);
    ProjSearchLastArgs a{};
    set_searched_frame(a, cs, capacity, dim, cz.w.data(), cz.h.data(), th_high, having_masks, cur_mp_dev, nmatches_dev, status_dev, diag_dev);
    a.n_levels = n_levels; a.sf = scale_factors;
    a.last = ls.data(); a.n_points = n_points; a.last_mp = last_mp_dev; a.bad = bad_dev;
    a.models = cams; a.mtmc_inv = mtmc_inv; a.masks = masks_dev; a.world_pos = world_pos_dev;
    a.last_outlier = last_outlier_dev; a.th = th;
    CUDA_CHECK(launch_search_by_projection_last(a, st));
    return sync_if_null_stream(stream);
}

int mcs_window_search_device(const mcs_packed_frame* cur, const mcs_packed_frame* last, int32_t n_cams, int32_t capacity, int32_t dim,
                             const int32_t* cam_width, const int32_t* cam_height, const int32_t* last_mp_dev, int32_t n_points,
                             const uint8_t* bad_dev, int32_t window, int32_t min_level, int32_t max_level, double nnratio, int32_t th_high,
                             int32_t having_masks, int32_t* cur_mp_dev, int32_t* nmatches_dev, int32_t* status_dev, int32_t* diag_dev,
                             void* stream) {
    if (!cur || !last || !cam_width || !cam_height || !last_mp_dev || !cur_mp_dev || !nmatches_dev || !status_dev)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (int rc = check_packed_frames(n_cams, capacity, dim, cur, last)) return rc;
    if (n_points < 0) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    if (int rc = check_cam_sizes(n_cams, cam_width, cam_height, false)) return rc;
    if (int rc = check_query_bound((long long)n_cams * capacity, "n_cams * capacity must stay below 2^24")) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const std::vector<PsCamSlots> cs = packed_slots(*cur, n_cams, capacity, dim), ls = packed_slots(*last, n_cams, capacity, dim);
    WindowSearchDevArgs a{};
    set_searched_frame(a, cs, capacity, dim, cam_width, cam_height, th_high, having_masks, cur_mp_dev, nmatches_dev, status_dev, diag_dev);
    a.last = ls.data(); a.n_points = n_points; a.last_mp = last_mp_dev; a.bad = bad_dev;
    a.window = window; a.nnratio = nnratio; a.min_level = min_level; a.max_level = max_level;
    CUDA_CHECK(launch_window_search_device(a, st));
    return sync_if_null_stream(stream);
}

int mcs_search_by_projection_frames_device(const mcs_packed_frame* cur, const mcs_packed_frame* last, int32_t n_cams, int32_t capacity,
                                           int32_t dim, const mcs_ocam* cams, const uint8_t* masks_dev, const double* mtmc_inv,
                                           const int32_t* last_mp_dev, int32_t n_points, const double* world_pos_dev, const uint8_t* bad_dev,
                                           int32_t window, double nnratio, int32_t th_high, int32_t having_masks, int32_t* cur_mp_dev,
                                           int32_t* nmatches_dev, int32_t* status_dev, int32_t* diag_dev, void* stream) {
    if (!cur || !last || !cams || !masks_dev || !mtmc_inv || !last_mp_dev || !world_pos_dev || !cur_mp_dev || !nmatches_dev || !status_dev)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (int rc = check_packed_frames(n_cams, capacity, dim, cur, last)) return rc;
    if (n_points < 0) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    const CamSizes cz(cams, n_cams);
    if (int rc = check_cam_sizes(n_cams, cz.w.data(), cz.h.data(), true)) return rc;
    // one query per (last-frame slot, camera)
    if (int rc = check_query_bound((long long)n_cams * n_cams * capacity, "n_cams * n_cams * capacity must stay below 2^24")) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const std::vector<PsCamSlots> cs = packed_slots(*cur, n_cams, capacity, dim), ls = packed_slots(*last, n_cams, capacity, dim);
    SearchFramesDevArgs a{};
    set_searched_frame(a, cs, capacity, dim, cz.w.data(), cz.h.data(), th_high, having_masks, cur_mp_dev, nmatches_dev, status_dev, diag_dev);
    a.last = ls.data(); a.n_points = n_points; a.last_mp = last_mp_dev; a.bad = bad_dev;
    a.models = cams; a.mtmc_inv = mtmc_inv; a.masks = masks_dev; a.world_pos = world_pos_dev;
    a.window = window; a.nnratio = nnratio;
    CUDA_CHECK(launch_search_by_projection_frames(a, st));
    return sync_if_null_stream(stream);
}

int mcs_search_for_initialization_device(const mcs_packed_frame* f1, const mcs_packed_frame* f2, int32_t n_cams, int32_t capacity,
                                         int32_t dim, const int32_t* cam_width, const int32_t* cam_height, double* prev_matched_dev,
                                         int32_t window_size, double nnratio, int32_t th_low, int32_t having_masks,
                                         int32_t* matches12_dev, int32_t* nmatches_dev, int32_t* diag_dev, void* stream) {
    if (!f1 || !f2 || !cam_width || !cam_height || !prev_matched_dev || !matches12_dev || !nmatches_dev)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (int rc = check_packed_frames(n_cams, capacity, dim, f2, f1)) return rc;
    if (int rc = check_cam_sizes(n_cams, cam_width, cam_height, false)) return rc;
    // the front end's query and slot indices (one query per F1 slot)
    if (int rc = check_query_bound((long long)n_cams * capacity, "n_cams * capacity must stay below 2^24")) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const std::vector<PsCamSlots> s2 = packed_slots(*f2, n_cams, capacity, dim), s1 = packed_slots(*f1, n_cams, capacity, dim);
    InitSearchDevArgs a{};
    set_searched_frame(a, s2, capacity, dim, cam_width, cam_height, th_low, having_masks, nullptr, nmatches_dev, nullptr, diag_dev);
    a.last = s1.data();
    a.prev = prev_matched_dev; a.matches12 = matches12_dev; a.window = window_size; a.nnratio = nnratio;
    CUDA_CHECK(launch_search_for_initialization(a, st));
    return sync_if_null_stream(stream);
}

int mcs_search_for_initialization_seed_device(const mcs_packed_frame* f1, int32_t n_cams, int32_t capacity, int32_t dim,
                                              double* prev_matched_dev, void* stream) {
    if (!f1 || !prev_matched_dev) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (int rc = check_packed_frames(n_cams, capacity, dim, f1, nullptr)) return rc;
    if (int rc = check_query_bound((long long)n_cams * capacity, "n_cams * capacity must stay below 2^24")) return rc;
    const std::vector<PsCamSlots> s1 = packed_slots(*f1, n_cams, capacity, dim);
    CUDA_CHECK(launch_search_for_initialization_seed(s1.data(), n_cams, capacity, prev_matched_dev, (cudaStream_t)stream));
    return sync_if_null_stream(stream);
}

int mcs_fuse_device(const mcs_fuse_target* kfs, int32_t n_kf, int32_t n_cams, int32_t capacity, int32_t dim, const mcs_ocam* cams,
                    const uint8_t* masks_dev, int32_t n_levels, const double* scale_factors, int32_t variant, const int32_t* query_mp_dev,
                    int32_t n_q, int32_t n_points, const double* world_pos_dev, const double* min_dist_dev, const double* max_dist_dev,
                    const uint8_t* desc_dev, const uint8_t* dmask_dev, const uint8_t* bad_dev, double th, int32_t th_low,
                    int32_t having_masks, int32_t* hits_dev, int32_t max_hits, int32_t* n_hits_dev, int32_t* status_dev, void* stream) {
    // query_mp_dev / hits_dev may be NULL only when they have no entry (an empty tensor has no address)
    if (!kfs || !cams || !masks_dev || !scale_factors || (!query_mp_dev && n_q > 0) || !world_pos_dev || !min_dist_dev || !max_dist_dev ||
        !desc_dev || (!hits_dev && max_hits > 0) || !n_hits_dev || !status_dev)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (having_masks && !dmask_dev) return mcs_fail(MCS_ERR_INVALID, "masks requested but not supplied");
    if (n_kf <= 0 || n_q < 0 || n_points < 0 || max_hits < 0 || n_levels < 1 || n_levels > MCS_MAX_LEVELS)
        return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    if (variant < MCS_FUSE_NEIGHBOUR || variant > MCS_FUSE_SIM3) return mcs_fail(MCS_ERR_INVALID, "unknown Fuse variant");
    for (int k = 0; k < n_kf; ++k) {
        if (int rc = check_packed_frames(n_cams, capacity, dim, &kfs[k].frame, nullptr)) return rc;
        if (!kfs[k].mtmc_inv) return mcs_fail(MCS_ERR_INVALID, "null argument");
    }
    const CamSizes cz(cams, n_cams);
    if (int rc = check_cam_sizes(n_cams, cz.w.data(), cz.h.data(), true)) return rc;
    // the front end's slot and query indices: one image per (key frame, camera), one entry per (key frame, query, camera)
    if (int rc = check_query_bound((long long)n_kf * n_cams * capacity, "n_kf * n_cams * capacity must stay below 2^24")) return rc;
    if (int rc = check_query_bound((long long)n_kf * n_q * n_cams, "n_kf * n_q * n_cams must stay below 2^24")) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int NI = n_kf * n_cams;
    std::vector<PsCamSlots> slots;
    std::vector<const int*> kf_mp(n_kf);
    std::vector<double> mtmc_inv(16 * (size_t)NI), ow(3 * (size_t)n_kf);
    for (int k = 0; k < n_kf; ++k) {
        append_slots(slots, kfs[k].frame, n_cams, capacity, dim);
        kf_mp[k] = kfs[k].mp_dev;
        std::memcpy(&mtmc_inv[16 * (size_t)k * n_cams], kfs[k].mtmc_inv, 128ull * n_cams);
        for (int i = 0; i < 3; ++i) ow[3 * k + i] = kfs[k].ow[i];
    }
    FuseDevArgs a{};                                     // the camera table is the models' (cam_w / cam_h unread)
    set_searched_frame(a, slots, capacity, dim, nullptr, nullptr, th_low, having_masks, nullptr, nullptr, status_dev, nullptr);
    a.n_levels = n_levels; a.sf = scale_factors;
    a.n_kf = n_kf; a.n_kf_cams = n_cams; a.variant = variant; a.n_q = n_q;
    a.kf_mp = kf_mp.data(); a.mtmc_inv = mtmc_inv.data(); a.ow = ow.data(); a.query_mp = query_mp_dev;
    a.pts = {n_points, world_pos_dev, min_dist_dev, max_dist_dev, desc_dev, having_masks ? dmask_dev : nullptr, bad_dev, cams, masks_dev};
    a.th = th; a.hits = hits_dev; a.max_hits = max_hits; a.n_hits = n_hits_dev;
    CUDA_CHECK(launch_fuse_device(a, st));
    return sync_if_null_stream(stream);
}

int mcs_search_by_bow_keyframes_device(const mcs_packed_frame* kf1, const int32_t* mp1_dev, const mcs_packed_frame* kfs,
                                       const int32_t* const* mp_dev, int32_t n_kf, int32_t n_cams, int32_t capacity, int32_t dim,
                                       int32_t n_points, const uint8_t* bad_dev, int32_t th_low, double nnratio, int32_t having_masks,
                                       int32_t* matches12_dev, int32_t* match_slot_dev, int32_t* nmatches_dev, int32_t* status_dev,
                                       void* stream) {
    if (n_kf < 0) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    if (n_kf == 0) return MCS_OK;
    if (!kf1 || !mp1_dev || !kfs || !mp_dev || !matches12_dev || !nmatches_dev || !status_dev) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (n_points < 0) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    if (int rc = check_packed_frames(n_cams, capacity, dim, kf1, nullptr)) return rc;
    for (int k = 0; k < n_kf; ++k) {
        if (!packed_frame_ok(&kfs[k], n_cams))
            return mcs_fail(MCS_ERR_INVALID, "candidate " + std::to_string(k) + ": no buffer, or first_image + n_cams exceeds its images");
        if (!mp_dev[k]) return mcs_fail(MCS_ERR_INVALID, "candidate " + std::to_string(k) + ": null map-point array");
    }
    // one "taken" bit per database slot in the acceptance CTA's shared memory (K-best lists of 8), compact indices in 21 bits
    const long long ns = (long long)n_cams * capacity;
    if (ns > bruteforce_max_nd(8)) return mcs_fail(MCS_ERR_UNSUPPORTED, "n_cams * capacity above " + std::to_string(bruteforce_max_nd(8)));
    if (int rc = check_query_bound(ns, "n_cams * capacity must stay below 2^24")) return rc;
    if (ns * n_kf >= (1LL << 31)) return mcs_fail(MCS_ERR_UNSUPPORTED, "n_kf * n_cams * capacity must stay below 2^31 (split the candidates)");
    std::vector<PsCamSlots> cams = packed_slots(*kf1, n_cams, capacity, dim);
    std::vector<const int*> mp(1, mp1_dev);
    for (int k = 0; k < n_kf; ++k) {
        append_slots(cams, kfs[k], n_cams, capacity, dim);
        mp.push_back(mp_dev[k]);
    }
    BowKfSearchDevArgs a{};
    a.n_kf = n_kf; a.n_cams = n_cams; a.capacity = capacity; a.dim = dim; a.n_points = n_points; a.th_low = th_low;
    a.nnratio = nnratio; a.masked = having_masks != 0;
    a.cams = cams.data(); a.mp = mp.data(); a.bad = bad_dev;
    a.matches12 = matches12_dev; a.match_slot = match_slot_dev; a.nmatches = nmatches_dev; a.status = status_dev;
    CUDA_CHECK(launch_search_by_bow_keyframes(a, (cudaStream_t)stream));
    return sync_if_null_stream(stream);
}

int mcs_search_for_triangulation_device(const mcs_packed_frame* kf1, const int32_t* mp1_dev, const mcs_packed_frame* kf2,
                                        const int32_t* mp2_dev, int32_t n_cams, int32_t capacity, int32_t dim, const mcs_ocam* cams,
                                        const double* E, double epi_thresh, int32_t th_low, int32_t having_masks,
                                        int32_t* matches12_dev, int32_t* nmatches_dev, int32_t* diag_dev, void* stream) {
    if (!kf1 || !mp1_dev || !kf2 || !mp2_dev || !cams || !E || !matches12_dev || !nmatches_dev)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    // a camera's rows, and the index of a list entry or rescan key inside its segment, fit 16 bits
    if (capacity > 65535) return mcs_fail(MCS_ERR_UNSUPPORTED, "capacity above 65535");
    if (int rc = check_packed_frames(n_cams, capacity, dim, kf1, kf2)) return rc;
    if (int rc = check_query_bound((long long)n_cams * capacity, "n_cams * capacity must stay below 2^24")) return rc;
    std::vector<PsCamSlots> slots = packed_slots(*kf1, n_cams, capacity, dim);
    append_slots(slots, *kf2, n_cams, capacity, dim);
    std::vector<double> e_diag((size_t)n_cams * 9);                  // only E[c][c] is read: a query sees its own camera only
    for (int c = 0; c < n_cams; ++c) std::memcpy(&e_diag[(size_t)c * 9], E + ((size_t)c * n_cams + c) * 9, 9 * sizeof(double));
    TriSearchDevArgs a{};
    a.n_cams = n_cams; a.capacity = capacity; a.dim = dim; a.th_low = th_low;
    a.masked = having_masks != 0; a.epi_thresh = epi_thresh;
    a.cams = slots.data(); a.mp[0] = mp1_dev; a.mp[1] = mp2_dev; a.models = cams; a.E = e_diag.data();
    a.matches12 = matches12_dev; a.nmatches = nmatches_dev; a.diag = diag_dev;
    CUDA_CHECK(launch_search_for_triangulation(a, (cudaStream_t)stream));
    return sync_if_null_stream(stream);
}

int mcs_search_by_sim3_device(const mcs_packed_frame* kf1, const mcs_packed_frame* kf2, int32_t n_cams, int32_t capacity, int32_t dim,
                              const mcs_ocam* cams, const uint8_t* masks_dev, int32_t n_levels, const double* scale_factors, const double* t1w,
                              const double* t2w, const double* mc_inv, double s12, const double* r12, const double* t12, double th,
                              const int32_t* mp1_dev, const int32_t* mp2_dev, int32_t n_points, const double* world_pos_dev,
                              const double* min_dist_dev, const double* max_dist_dev, const uint8_t* desc_dev, const uint8_t* dmask_dev,
                              const uint8_t* bad_dev, const uint8_t* already2_dev, int32_t th_high, int32_t having_masks,
                              int32_t* matches12_dev, int32_t* nfound_dev, int32_t* status_dev, void* stream) {
    if (!kf1 || !kf2 || !cams || !masks_dev || !scale_factors || !t1w || !t2w || !mc_inv || !r12 || !t12 || !mp1_dev || !mp2_dev ||
        !world_pos_dev || !min_dist_dev || !max_dist_dev || !desc_dev || !matches12_dev || !nfound_dev || !status_dev)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (having_masks && !dmask_dev) return mcs_fail(MCS_ERR_INVALID, "masks requested but not supplied");
    if (n_levels < 1 || n_levels > MCS_MAX_LEVELS || n_points < 0) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    if (!(s12 != 0.0)) return mcs_fail(MCS_ERR_INVALID, "s12 must be non-zero");
    if (int rc = check_packed_frames(n_cams, capacity, dim, kf2, kf1)) return rc;
    const CamSizes cz(cams, n_cams);
    if (int rc = check_cam_sizes(n_cams, cz.w.data(), cz.h.data(), true)) return rc;
    // one query per slot of the key frame carried over, in each direction
    if (int rc = check_query_bound((long long)n_cams * capacity, "n_cams * capacity must stay below 2^24")) return rc;
    // sR12 = s12 * R12, sR21 = (1 / s12) * R12^T, t21 = -sR21 * t12 (ref :1741-1743), cv::Matx order: s = 0; s += a(i,k) * b(k) ...
    double xf[48];
    auto rig = [&](double* d, const double* T) {         // Hom2R / Hom2T of a row-major 4x4
        for (int i = 0; i < 3; ++i) { for (int k = 0; k < 3; ++k) d[3 * i + k] = T[4 * i + k]; d[9 + i] = T[4 * i + 3]; }
    };
    rig(xf, t1w);
    rig(xf + 24, t2w);
    const double inv_s = 1.0 / s12;
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k) {
            xf[12 + 3 * i + k] = inv_s * r12[3 * k + i];     // direction 1: sR21
            xf[36 + 3 * i + k] = s12 * r12[3 * i + k];       // direction 2: sR12
        }
    for (int i = 0; i < 3; ++i) {
        double acc = 0.0;
        for (int k = 0; k < 3; ++k) acc += -xf[12 + 3 * i + k] * t12[k];
        xf[21 + i] = acc;                                    // t21
        xf[45 + i] = t12[i];
    }
    cudaStream_t st = (cudaStream_t)stream;
    const std::vector<PsCamSlots> s2 = packed_slots(*kf2, n_cams, capacity, dim), s1 = packed_slots(*kf1, n_cams, capacity, dim);
    Sim3SearchDevArgs a{};
    set_searched_frame(a, s2, capacity, dim, cz.w.data(), cz.h.data(), th_high, having_masks, nullptr, nfound_dev, status_dev, nullptr);
    a.n_levels = n_levels; a.sf = scale_factors;
    a.kf1 = s1.data(); a.xf = xf; a.mc_inv = mc_inv; a.th = th;
    a.pts = {n_points, world_pos_dev, min_dist_dev, max_dist_dev, desc_dev, having_masks ? dmask_dev : nullptr, bad_dev, cams, masks_dev};
    a.mp1 = mp1_dev; a.mp2 = mp2_dev; a.already2 = already2_dev; a.matches12 = matches12_dev;
    CUDA_CHECK(launch_search_by_sim3(a, st));
    return sync_if_null_stream(stream);
}

int mcs_search_by_projection_scw_device(const mcs_packed_frame* kf, int32_t n_cams, int32_t capacity, int32_t dim, const mcs_ocam* cams,
                                        const uint8_t* masks_dev, int32_t n_levels, const double* scale_factors, const double* mtmc_inv,
                                        const double* ow, const int32_t* points_dev, int32_t n_q, int32_t n_points,
                                        const double* world_pos_dev, const double* min_dist_dev, const double* max_dist_dev,
                                        const uint8_t* desc_dev, const uint8_t* dmask_dev, const uint8_t* bad_dev, int32_t th, int32_t th_low,
                                        int32_t having_masks, int32_t* matched_dev, int32_t* nmatches_dev, int32_t* status_dev,
                                        int32_t* diag_dev, void* stream) {
    // points_dev may be NULL only when it has no entry (an empty tensor has no address)
    if (!kf || !cams || !masks_dev || !scale_factors || !mtmc_inv || !ow || (!points_dev && n_q > 0) || !world_pos_dev || !min_dist_dev ||
        !max_dist_dev || !desc_dev || !matched_dev || !nmatches_dev || !status_dev)
        return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (having_masks && !dmask_dev) return mcs_fail(MCS_ERR_INVALID, "masks requested but not supplied");
    if (n_levels < 1 || n_levels > MCS_MAX_LEVELS || n_q < 0 || n_points < 0) return mcs_fail(MCS_ERR_INVALID, "bad sizes");
    if (int rc = check_packed_frames(n_cams, capacity, dim, kf, nullptr)) return rc;
    const CamSizes cz(cams, n_cams);
    if (int rc = check_cam_sizes(n_cams, cz.w.data(), cz.h.data(), true)) return rc;
    // the front end's slot and query indices: one image per camera, one query per entry of vpPoints
    if (int rc = check_query_bound((long long)n_cams * capacity, "n_cams * capacity must stay below 2^24")) return rc;
    if (int rc = check_query_bound(n_q, "n_q must stay below 2^24")) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const std::vector<PsCamSlots> slots = packed_slots(*kf, n_cams, capacity, dim);
    ScwSearchDevArgs a{};
    set_searched_frame(a, slots, capacity, dim, cz.w.data(), cz.h.data(), th_low, having_masks, matched_dev, nmatches_dev, status_dev, diag_dev);
    a.n_levels = n_levels; a.sf = scale_factors;
    a.mtmc_inv = mtmc_inv; a.ow = ow; a.n_q = n_q; a.points = points_dev;
    a.pts = {n_points, world_pos_dev, min_dist_dev, max_dist_dev, desc_dev, having_masks ? dmask_dev : nullptr, bad_dev, cams, masks_dev};
    a.th = th;
    CUDA_CHECK(launch_search_by_projection_scw(a, st));
    return sync_if_null_stream(stream);
}

int mcs_search_for_initialization(const mcs_frame_view* f1, const mcs_frame_view* f2, double* prev_matched, int32_t window_size,
                                  double nnratio, int32_t th_low, int32_t having_masks, int32_t* matches12, int32_t* nmatches) {
    if (!f1 || !f2 || !prev_matched || !matches12 || !nmatches) return mcs_fail(MCS_ERR_INVALID, "null argument");
    if (f1->dim != f2->dim) return mcs_fail(MCS_ERR_INVALID, "descriptor sizes differ");
    if (having_masks && (!f1->dmask || !f2->dmask)) return mcs_fail(MCS_ERR_INVALID, "masks requested but not supplied");
    *nmatches = 0;
    const int n1 = f1->n_keys;
    for (int i = 0; i < n1; ++i) matches12[i] = -1;
    if (n1 == 0 || f2->n_keys == 0) return MCS_OK;
    std::vector<mcs_window_query> qs(n1);
    for (int i1 = 0; i1 < n1; ++i1) {
        mcs_window_query& q = qs[i1];
        q.cam = f1->key_cam[i1];
        if (q.cam < 0 || q.cam >= f2->n_cams) return mcs_fail(MCS_ERR_INVALID, "key_cam out of range");
        q.min_level = q.max_level = f1->keys[i1].octave;
        q.desc_index = i1;
        q.x = prev_matched[2 * i1]; q.y = prev_matched[2 * i1 + 1]; q.r = (double)window_size;
    }
    FrameDev fd;
    int rc = upload_frame(f2, fd, nullptr);
    if (rc) return rc;
    std::vector<int> ci, cd, co;
    rc = window_search_compact(fd, qs.data(), n1, f1->desc, having_masks ? f1->dmask : nullptr, n1, f1->dim, 32, ci, cd, co, nullptr);
    if (rc) return rc;
    int nm = 0;
    std::vector<int> matchedDist(f2->n_keys, INT_MAX), matches21(f2->n_keys, -1);
    for (int i1 = 0; i1 < n1; ++i1) {            // ref :599-682
        const int n = co[i1 + 1] - co[i1];
        if (n == 0) continue;
        int bestDist = INT_MAX, bestDist2 = INT_MAX, bestIdx2 = -1;
        for (int k = 0; k < n; ++k) {
            const int i2 = ci[co[i1] + k], dist = cd[co[i1] + k];
            if (matchedDist[i2] <= dist) continue;
            if (dist < bestDist) { bestDist2 = bestDist; bestDist = dist; bestIdx2 = i2; }
            else if (dist < bestDist2) bestDist2 = dist;
        }
        if (bestDist <= th_low && bestDist < (double)bestDist2 * nnratio) {
            if (matches21[bestIdx2] >= 0) { matches12[matches21[bestIdx2]] = -1; --nm; }
            matches12[i1] = bestIdx2;
            matches21[bestIdx2] = i1;
            matchedDist[bestIdx2] = bestDist;
            ++nm;
        }
    }
    for (int i1 = 0; i1 < n1; ++i1)              // ref :717-720
        if (matches12[i1] >= 0) {
            prev_matched[2 * i1] = f2->keys[matches12[i1]].x;
            prev_matched[2 * i1 + 1] = f2->keys[matches12[i1]].y;
        }
    *nmatches = nm;
    return MCS_OK;
}

}  // extern "C"
