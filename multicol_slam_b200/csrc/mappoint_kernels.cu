// mappoint_kernels.cu -- cMapPoint::ComputeDistinctiveDescriptors (ref src/cMapPoint.cpp:294-388) and UpdateNormalAndDepth
// (:449-492) for many map points in one launch, from the key frames' packed feature buffers to the device map-point tables the
// device searches read (desc / dmask, normal, GetMin/MaxDistanceInvariance).
//
//   mp_update_kernel    one warp per listed point.  Every point depends only on its own observations, so there are no rounds and
//                       no walk: the warp checks the point's observation list, then
//                       - descriptor: for each row i of the non-bad key frames' rows (list order), the rank-floor(len / 2)
//                         element of {D(i, j) : j > i} from a shared histogram over [0, 8 * dim] (no sort, no scratch that grows
//                         with the number of observations); the first strictly smallest median wins;
//                       - normal and depth: lane 0 sums the per-key-frame unit vectors in list order, in the reference's
//                         operation order (OpenCV's Vec / scalar is a multiplication by the rounded reciprocal).
#include <climits>

#include "mappoint_kernels.h"

namespace mcs {

namespace {

constexpr int kMpWarps = 4;                      // warps per block: one listed point each
constexpr unsigned kFull = 0xffffffffu;

struct MpDev {                                   // MpUpdateArgs with the host tables replaced by their staged copies
    int n_kf, n_cams, capacity, n_levels, what;
    const PsCamSlots* slots; const int* kf_bad; const double* kf_ow; const double* sf;
    const int* ids; int n_upd, n_points;
    const int* obs_off; const int* obs_kf; const int* obs_slot;
    const int* ref_kf; const uint8_t* bad; const double* world_pos;
    uint8_t* desc; uint8_t* dmask; double* normal; double* min_dist; double* max_dist;
    int* status;
};

// the image slot of observation e: camera c = slot / capacity of key frame k, keypoint j
struct MpRow { const PsCamSlots* cam; int j; };
__device__ __forceinline__ MpRow mp_row(const MpDev& a, const int k, const int slot) {
    const int c = slot / a.capacity;
    return MpRow{a.slots + (size_t)k * a.n_cams + c, slot - c * a.capacity};
}

// DescriptorDistance64 / DescriptorDistance64Masked (ref src/cORBmatcher.cpp:2438-2474) in 32-bit words, as ps_list_kernel
// evaluates them: the masked sum of both halves is halved once at the end
template <int WORDS, bool MASKED>
__device__ __forceinline__ unsigned mp_dist(const uint32_t (&qw)[WORDS], const uint32_t (&qm)[WORDS], const uint32_t* dd,
                                            const uint32_t* mm) {
    unsigned dist = 0;
    if (MASKED) {
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
    return dist;
}

// The checks of one point (all lanes agree on the result): offsets ordered, every observation's key frame in [0, n_kf) and slot
// below its camera's count, each key frame's observations adjacent.
__device__ bool mp_obs_ok(const MpDev& a, const int o0, const int o1) {
    bool ok = o0 >= 0 && o1 >= o0;
    if (ok)
        for (int e = o0 + (int)(threadIdx.x & 31); e < o1; e += 32) {
            const int k = a.obs_kf[e], s = a.obs_slot[e];
            if (k < 0 || k >= a.n_kf || s < 0 || s >= a.n_cams * a.capacity) { ok = false; break; }
            const MpRow r = mp_row(a, k, s);
            if (r.j >= *r.cam->count) { ok = false; break; }
            if (e > o0 && a.obs_kf[e - 1] != k)              // a run of k starts here: no earlier run of k
                for (int f = o0; f < e - 1; ++f)
                    if (a.obs_kf[f] == k) { ok = false; break; }
        }
    return __all_sync(kFull, ok);
}

// A NaN as the reference computes it on x86-64: SSE arithmetic yields the default NaN 0xFFF8000000000000 (sign set), sm_90 the
// canonical 0x7FFFFFFFFFFFFFFF
__device__ __forceinline__ double nan_x86(const double v) {
    return isnan(v) ? __longlong_as_double((long long)0xFFF8000000000000ull) : v;
}

template <int WORDS, bool MASKED>
__global__ void __launch_bounds__(32 * kMpWarps) mp_update_kernel(const MpDev a) {
    constexpr int kBins = 32 * WORDS + 1;                // distances lie in [0, 8 * dim]
    constexpr int kPer = (kBins + 31) / 32;              // bins per lane in the rank search
    __shared__ unsigned hist_all[kMpWarps][kBins];
    const int lane = threadIdx.x & 31, u = blockIdx.x * kMpWarps + (threadIdx.x >> 5);
    if (u >= a.n_upd) return;                            // whole warps
    unsigned* hist = hist_all[threadIdx.x >> 5];
    const int id = a.ids[u];
    if (id < 0 || id >= a.n_points) {
        if (lane == 0) *a.status = MCS_ERR_INVALID;
        return;
    }
    if (a.bad && a.bad[id]) return;                      // a bad point: nothing changes (ref :306-307, :457-458)
    const int o0 = a.obs_off[id], o1 = a.obs_off[id + 1];
    bool ok = mp_obs_ok(a, o0, o1);
    const bool nd = (a.what & MCS_MP_NORMAL_DEPTH) != 0;
    int ref = 0, level = 1;                              // level 1 when the ref key frame does not observe the point (:479-481)
    if (ok && nd) {
        ref = a.ref_kf[id];
        ok = ref >= 0 && ref < a.n_kf;
        if (ok) {
            for (int base = o0; base < o1; base += 32) {  // its first observation: observations[pRefKF][0]
                const int e = base + lane;
                const unsigned m = __ballot_sync(kFull, e < o1 && a.obs_kf[e] == ref);
                if (m) {
                    const int f = base + __ffs(m) - 1;
                    const MpRow r = mp_row(a, ref, a.obs_slot[f]);
                    level = r.cam->kps[r.j].octave;
                    break;
                }
            }
            ok = level >= 0 && level < a.n_levels;
        }
    }
    if (!ok) {
        if (lane == 0) *a.status = MCS_ERR_INVALID;
        return;
    }

    if (a.what & MCS_MP_DESCRIPTOR) {
        // rows: the observations of non-bad key frames in list order (:313-330); N <= 2 keeps row 0 (:366-383)
        int best_e = -1, best_med = INT_MAX;
        for (int ei = o0; ei < o1; ++ei) {
            const int ki = a.obs_kf[ei];
            if (a.kf_bad[ki]) continue;
            if (best_e < 0) best_e = ei;
            const MpRow ri = mp_row(a, ki, a.obs_slot[ei]);
            uint32_t qw[WORDS], qm[WORDS];
            const uint32_t* qd = (const uint32_t*)(ri.cam->desc) + (size_t)ri.j * WORDS;
            const uint32_t* qmp = MASKED ? (const uint32_t*)(ri.cam->dmask) + (size_t)ri.j * WORDS : nullptr;
#pragma unroll
            for (int k = 0; k < WORDS; ++k) { qw[k] = qd[k]; qm[k] = MASKED ? qmp[k] : 0u; }
            for (int b = lane; b < kBins; b += 32) hist[b] = 0;
            __syncwarp();
            int len = 0;                                 // |{j > i}|: the rows after row i
            for (int base = ei + 1; base < o1; base += 32) {
                const int e = base + lane;
                int k = 0;
                const bool live = e < o1 && !a.kf_bad[k = a.obs_kf[e]];
                if (live) {
                    const MpRow rj = mp_row(a, k, a.obs_slot[e]);
                    const uint32_t* dd = (const uint32_t*)(rj.cam->desc) + (size_t)rj.j * WORDS;
                    const uint32_t* mm = MASKED ? (const uint32_t*)(rj.cam->dmask) + (size_t)rj.j * WORDS : nullptr;
                    atomicAdd(&hist[mp_dist<WORDS, MASKED>(qw, qm, dd, mm)], 1u);
                }
                len += __popc(__ballot_sync(kFull, live));
            }
            if (len == 0) break;                         // the last row has no upper part and cannot win
            __syncwarp();
            // misc.h:96-104 median: nth_element at size / 2, the element of rank floor(len / 2)
            const unsigned r = (unsigned)len >> 1;
            unsigned cnt = 0;
#pragma unroll
            for (int t = 0; t < kPer; ++t) {
                const int b = lane * kPer + t;
                if (b < kBins) cnt += hist[b];
            }
            unsigned incl = cnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned y = __shfl_up_sync(kFull, incl, o);
                if (lane >= o) incl += y;
            }
            const unsigned excl = incl - cnt;
            int med = INT_MAX;
            if (excl <= r && r < incl) {                 // exactly one lane holds rank r
                unsigned acc = excl;
                for (int t = 0; t < kPer; ++t) {
                    acc += hist[lane * kPer + t];
                    if (acc > r) { med = lane * kPer + t; break; }
                }
            }
            const unsigned owner = __ballot_sync(kFull, med != INT_MAX);
            med = __shfl_sync(kFull, med, __ffs(owner) - 1);
            if (med < best_med) { best_med = med; best_e = ei; }
            __syncwarp();                                // the next row clears the histogram
        }
        if (best_e >= 0) {                               // no row: nothing changes (:335-336)
            const MpRow rb = mp_row(a, a.obs_kf[best_e], a.obs_slot[best_e]);
            const uint32_t* src = (const uint32_t*)(rb.cam->desc) + (size_t)rb.j * WORDS;
            uint32_t* dst = (uint32_t*)a.desc + (size_t)id * WORDS;
            for (int k = lane; k < WORDS; k += 32) dst[k] = src[k];
            if (MASKED) {                                // mDescriptorMask only when havingMasks (:385-386)
                const uint32_t* msrc = (const uint32_t*)(rb.cam->dmask) + (size_t)rb.j * WORDS;
                uint32_t* mdst = (uint32_t*)a.dmask + (size_t)id * WORDS;
                for (int k = lane; k < WORDS; k += 32) mdst[k] = msrc[k];
            }
        }
    }

    if (nd && lane == 0) {
        const double X0 = a.world_pos[3 * (size_t)id], X1 = a.world_pos[3 * (size_t)id + 1], X2 = a.world_pos[3 * (size_t)id + 2];
        double n0 = 0.0, n1 = 0.0, n2 = 0.0;
        int n = 0, prev = -1;
        for (int e = o0; e < o1; ++e) {                  // one term per key frame, bad ones included (:466-474)
            const int k = a.obs_kf[e];
            if (k == prev) continue;
            prev = k;
            const double d0 = X0 - a.kf_ow[3 * k], d1 = X1 - a.kf_ow[3 * k + 1], d2 = X2 - a.kf_ow[3 * k + 2];
            const double inv = 1.0 / sqrt((d0 * d0 + d1 * d1) + d2 * d2);   // normali / cv::norm(normali)
            n0 = n0 + d0 * inv; n1 = n1 + d1 * inv; n2 = n2 + d2 * inv;
            ++n;
        }
        const double p0 = X0 - a.kf_ow[3 * ref], p1 = X1 - a.kf_ow[3 * ref + 1], p2 = X2 - a.kf_ow[3 * ref + 2];
        const double dist = sqrt((p0 * p0 + p1 * p1) + p2 * p2);
        const double s = a.sf[level];
        const double mn = ((1.0 / s) * dist) / s;                       // :487
        const double mx = (s * dist) * a.sf[a.n_levels - 1 - level];    // :489
        const double inv_n = 1.0 / (double)n;                           // normal / n: 0 * (1. / 0) = NaN without observations
        double* nrm = a.normal + 3 * (size_t)id;
        nrm[0] = nan_x86(n0 * inv_n); nrm[1] = nan_x86(n1 * inv_n); nrm[2] = nan_x86(n2 * inv_n);
        a.min_dist[id] = nan_x86(0.8 * mn);                             // GetMinDistanceInvariance (:494-498)
        a.max_dist[id] = nan_x86(1.2 * mx);                             // GetMaxDistanceInvariance (:500-504)
    }
}

}  // namespace

cudaError_t launch_update_mappoints(const MpUpdateArgs& a, cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(a.status, 0, 4, st);
    if (e != cudaSuccess || a.n_upd == 0) return e;
    MpDev d{a.n_kf, a.n_cams, a.capacity, a.n_levels, a.what, nullptr, nullptr, nullptr, nullptr,
            a.ids, a.n_upd, a.n_points, a.obs_off, a.obs_kf, a.obs_slot, a.ref_kf, a.bad, a.world_pos,
            a.desc, a.dmask, a.normal, a.min_dist, a.max_dist, a.status};
    StreamScratch sc;
    e = open_scratch(sc, {}, st, host_in(d.slots, a.slots, (size_t)a.n_kf * a.n_cams), host_in(d.kf_bad, a.kf_bad, a.n_kf),
                     host_in(d.kf_ow, a.kf_ow, 3 * (size_t)a.n_kf), host_in(d.sf, a.sf, a.n_levels));
    if (e == cudaSuccess) {
        const unsigned blocks = (unsigned)((a.n_upd + kMpWarps - 1) / kMpWarps);
        with_desc_width(a.dim, a.masked, [&](auto W, auto M) {
            mp_update_kernel<decltype(W)::value, decltype(M)::value><<<blocks, 32 * kMpWarps, 0, st>>>(d);
        });
        e = cudaGetLastError();
    }
    return sc.release(e);
}

}  // namespace mcs
