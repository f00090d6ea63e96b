// extract_kernels.cu -- sm_90a kernels of the extractor half of the hot path.
//
//   (K1, fused pyramid + blur + FAST, lives in pyr_fast_kernel.cu)
//   K2 octree_kernel     : DistributeOctTree, one CTA per (image, level)   (ref :569-861)
//   (K3, orientation + descriptor, lives in describe_kernel.cu)
//
// Everything is integer / exactly-rounded arithmetic; compile with -fmad=false so that no float or
// double expression is contracted (the CPU oracle is built with -ffp-contract=off).
#include "mcs_common.cuh"
#include "cam_model.cuh"
#include "kernels.h"

namespace mcs {

// ------------------------------------------------------------------------------------------------
// K2  octree  (ref src/mdBRIEFextractorOct.cpp:569-861)
// ------------------------------------------------------------------------------------------------
// One CTA owns one (image, level).  The std::list<ExtractorNode> of the reference is kept as a dense
// array in LIST ORDER (index == position from the front); each pass rebuilds the array:
//   new list = [children created this pass, in reverse creation order] ++ [surviving nodes, old order]
// which is exactly what push_front of n1..n4 + erase(parent) produce.  Corners carry the list position
// of their node (node_of[]) and are re-labelled through a per-pass remap table.
//   pass A ("full"): every node with more than one corner is divided, in list order (ref :693-765).
//   pass B ("sorted"): the children created by the previous pass that hold >1 corner are divided
//        largest-first, ties by later creation first (deterministic stand-in for the pointer order of
//        the reference's sort, :782), stopping as soon as the list holds >= N nodes (ref :775-851).
// The best corner of a node is the first maximum of `response` in raw-list (= reference) order; raw lists
// are unordered on the device, so the order is carried by an analytic key (cell-row-major, then
// pixel-row-major inside the cell -- ref :892-949).
struct OctNode {
    short x0, y0, x1, y1;     // UL.x, UL.y, BR.x, BR.y  (cell-grid coordinates)
    int count;
    unsigned seq;             // creation sequence number | bit31: created in the last pass (pass-B candidate)
};
constexpr unsigned kNewFlag = 0x80000000u;

constexpr int kOctThreads = 512;
constexpr int kChunk = kMaxNodes / kOctThreads;   // list positions owned by one thread in the scans

// kOctThreads-wide exclusive scan; every thread of the CTA must call.
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_warp, int& total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    __syncthreads();
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        int w = lane < kOctThreads / 32 ? s_warp[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += t;
        }
        if (lane < kOctThreads / 32) s_warp[lane] = w;
    }
    __syncthreads();
    total = s_warp[kOctThreads / 32 - 1];
    const int r = inc - v + (wid ? s_warp[wid - 1] : 0);
    __syncthreads();
    return r;
}

__device__ __forceinline__ int quadrant(const OctNode& n, int x, int y) {
    // DivideNode (ref :575-619): halfX = ceil((UR.x-UL.x)/2);  n1 | n2 / n3 | n4
    const int mx = n.x0 + ((n.x1 - n.x0 + 1) >> 1);
    const int my = n.y0 + ((n.y1 - n.y0 + 1) >> 1);
    return (x < mx ? 0 : 1) + (y < my ? 0 : 2);
}
__device__ __forceinline__ int nonempty4(const int* c) { return (c[0] > 0) + (c[1] > 0) + (c[2] > 0) + (c[3] > 0); }

size_t octree_smem_bytes(int cap) { return (size_t)cap * (8 + 2 * sizeof(OctNode) + 16 + 2) + 64; }

__global__ void __launch_bounds__(kOctThreads)
octree_kernel(const PyramidGeom* __restrict__ geom, const int cap /* node capacity, <= kMaxNodes */,
              const uint32_t* __restrict__ raw, const size_t raw_img_stride,
              const int* __restrict__ raw_count, uint16_t* __restrict__ node_of_all,
              uint32_t* __restrict__ sel_xys /* [B][sel_total] packed corner */, int* __restrict__ sel_count /* [B][L] */,
              int* __restrict__ status, const int level_lo) {
    extern __shared__ __align__(16) unsigned char oct_smem[];
    unsigned long long* s_key = (unsigned long long*)oct_smem;          // pass-B sort keys / scan scratch / best-corner keys
    OctNode* s_nodes0 = (OctNode*)(s_key + cap);
    OctNode* s_nodes1 = s_nodes0 + cap;
    int (*s_child)[4] = (int (*)[4])(s_nodes1 + cap);                   // corner count per child, then new position per child
    short* s_rank = (short*)(s_child + cap);                            // processing rank of a divided node, -1 = survives
    __shared__ int s_warp[kOctThreads / 32];
    __shared__ int s_nn, s_cut;
    __shared__ unsigned s_seq;

    const int level = level_lo + blockIdx.x, b = blockIdx.y;
    const LevelGeom& g = geom->lv[level];
    const int L = geom->nlevels;
    const int tid = threadIdx.x;
    const int n_all = raw_count[b * L + level];
    const int n = min(n_all, g.raw_cap);
    const uint32_t* corners = raw + (size_t)b * raw_img_stride + g.raw_off;
    uint16_t* node_of = node_of_all + (size_t)b * raw_img_stride + g.raw_off;
    uint32_t* out = sel_xys + (size_t)b * geom->sel_total + g.sel_off;
    const int N = g.quota;

    if (n == 0) { if (tid == 0) sel_count[b * L + level] = 0; return; }
    if (n_all > g.raw_cap && tid == 0) atomicOr(status, 1);

    const int minB = kEdge - 3;
    // ---- roots (ref :640-679) ----
    const int nIni = g.nodes_ini;
    // s_child / s_rank hold one entry per root (the host sizes cap >= 4 nIni, what the first pass can create)
    if (nIni > cap) { if (tid == 0) { sel_count[b * L + level] = 0; atomicOr(status, 2); } return; }
    for (int i = tid; i < nIni; i += kOctThreads) s_child[i][0] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += kOctThreads) {
        const int x = corner_x(corners[i]) - minB;
        const int r = min((int)((double)(float)x / g.hX), nIni - 1);
        node_of[i] = (uint16_t)r;
        atomicAdd(&s_child[r][0], 1);
    }
    __syncthreads();
    if (tid == 0) {
        int k = 0;
        for (int i = 0; i < nIni; ++i) {
            s_rank[i] = -1;
            if (s_child[i][0] == 0) continue;
            OctNode nd;
            nd.x0 = (short)(int)(g.hX * (double)i); nd.x1 = (short)(int)(g.hX * (double)(i + 1));
            nd.y0 = 0; nd.y1 = (short)(g.h - kEdge + 3 - minB);
            nd.count = s_child[i][0]; nd.seq = (unsigned)i;
            s_rank[i] = (short)k;
            s_nodes0[k++] = nd;
        }
        s_nn = k; s_seq = (unsigned)nIni;
    }
    __syncthreads();
    for (int i = tid; i < n; i += kOctThreads) node_of[i] = (uint16_t)s_rank[node_of[i]];
    __syncthreads();

    int cur = 0;
    bool finish = false, pass_b = false;
    while (!finish) {
        const int nn = s_nn;
        OctNode* nodes = cur ? s_nodes1 : s_nodes0;
        OctNode* nnodes = cur ? s_nodes0 : s_nodes1;
        // 1. corner counts per child of every node that may be divided in this pass
        for (int i = tid; i < nn * 4; i += kOctThreads) (&s_child[0][0])[i] = 0;
        __syncthreads();
        for (int i = tid; i < n; i += kOctThreads) {
            const int p = node_of[i];
            const OctNode nd = nodes[p];
            if (nd.count > 1 && (!pass_b || (nd.seq & kNewFlag))) {
                const uint32_t c = corners[i];
                atomicAdd(&s_child[p][quadrant(nd, corner_x(c) - minB, corner_y(c) - minB)], 1);
            }
        }
        __syncthreads();
        // 2. s_rank[p] = processing rank among the divided nodes (-1: survives), ndiv = how many
        int ndiv;
        if (!pass_b) {          // list order (ref :693-765)
            int flag[kChunk], sum = 0;
#pragma unroll
            for (int k = 0; k < kChunk; ++k) {
                const int p = tid * kChunk + k;
                flag[k] = (p < nn && nodes[p].count > 1) ? 1 : 0;
                sum += flag[k];
            }
            int base = block_exclusive_scan(sum, s_warp, ndiv);
#pragma unroll
            for (int k = 0; k < kChunk; ++k) {
                const int p = tid * kChunk + k;
                if (p < nn) s_rank[p] = flag[k] ? (short)base : (short)-1;
                base += flag[k];
            }
            __syncthreads();
        } else {                // largest first, later-created first among equals (ref :782-786)
            for (int p = tid; p < nn; p += kOctThreads) {
                const OctNode nd = nodes[p];
                s_key[p] = (nd.count > 1 && (nd.seq & kNewFlag))
                               ? (((unsigned long long)(unsigned)nd.count << 32) | (nd.seq & ~kNewFlag)) : 0ull;
            }
            __syncthreads();
            int mine = 0;
            for (int p = tid; p < nn; p += kOctThreads) {
                const unsigned long long kp = s_key[p];
                int r = -1;
                if (kp) { r = 0; for (int q = 0; q < nn; ++q) r += (s_key[q] > kp); ++mine; }
                s_rank[p] = (short)r;
            }
            int ncand;
            block_exclusive_scan(mine, s_warp, ncand);
            // growth of the list per candidate, in processing order; cut after the divide reaching N (ref :848-849)
            for (int p = tid; p < nn; p += kOctThreads) {
                const int r = s_rank[p];
                if (r >= 0) s_key[r] = (unsigned long long)(nonempty4(s_child[p]) - 1);
            }
            __syncthreads();
            if (tid == 0) {
                int size = nn, cut = ncand;
                for (int r = 0; r < ncand; ++r) {
                    size += (int)s_key[r];
                    if (size >= N) { cut = r + 1; break; }
                }
                s_cut = cut;
            }
            __syncthreads();
            ndiv = s_cut;
            for (int p = tid; p < nn; p += kOctThreads)
                if (s_rank[p] >= ndiv) s_rank[p] = -1;
            __syncthreads();
        }
        // 3. creation index of the first child of rank r  (children of rank r follow all children of ranks < r)
        for (int p = tid; p < nn; p += kOctThreads) {
            const int r = s_rank[p];
            if (r >= 0) s_key[r] = (unsigned long long)nonempty4(s_child[p]);
        }
        __syncthreads();
        int K;                  // number of nodes created by this pass
        {
            int loc[kChunk], sum = 0;
#pragma unroll
            for (int k = 0; k < kChunk; ++k) {
                const int r = tid * kChunk + k;
                loc[k] = r < ndiv ? (int)s_key[r] : 0;
                sum += loc[k];
            }
            int base = block_exclusive_scan(sum, s_warp, K);
#pragma unroll
            for (int k = 0; k < kChunk; ++k) {
                const int r = tid * kChunk + k;
                if (r < ndiv) s_key[r] = (unsigned long long)base;
                base += loc[k];
            }
            __syncthreads();
        }
        // 4. new list = [new children, reverse creation order] ++ [survivors, old order]
        int nsurv;
        {
            int loc[kChunk], sum = 0;
#pragma unroll
            for (int k = 0; k < kChunk; ++k) {
                const int p = tid * kChunk + k;
                loc[k] = (p < nn && s_rank[p] < 0) ? 1 : 0;
                sum += loc[k];
            }
            int base = block_exclusive_scan(sum, s_warp, nsurv);
            const unsigned seq0 = s_seq;
#pragma unroll
            for (int k = 0; k < kChunk; ++k) {
                const int p = tid * kChunk + k;
                if (p >= nn) continue;
                const OctNode nd = nodes[p];
                if (loc[k]) {
                    const int np = K + base;
                    OctNode c = nd; c.seq &= ~kNewFlag;
                    if (np < cap) nnodes[np] = c;
                    s_child[p][0] = s_child[p][1] = s_child[p][2] = s_child[p][3] = np;
                    ++base;
                } else {
                    int t = (int)s_key[s_rank[p]];
                    const int mx = nd.x0 + ((nd.x1 - nd.x0 + 1) >> 1);
                    const int my = nd.y0 + ((nd.y1 - nd.y0 + 1) >> 1);
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int cnt = s_child[p][q];
                        if (cnt == 0) { s_child[p][q] = 0; continue; }
                        OctNode c;
                        c.x0 = (q & 1) ? (short)mx : nd.x0; c.x1 = (q & 1) ? nd.x1 : (short)mx;
                        c.y0 = (q & 2) ? (short)my : nd.y0; c.y1 = (q & 2) ? nd.y1 : (short)my;
                        c.count = cnt; c.seq = (seq0 + (unsigned)t) | kNewFlag;
                        const int np = K - 1 - t;
                        if (np < cap) nnodes[np] = c;
                        s_child[p][q] = np;
                        ++t;
                    }
                }
            }
        }
        __syncthreads();
        const int new_nn = K + nsurv;
        // 5. relabel the corners
        for (int i = tid; i < n; i += kOctThreads) {
            const int p = node_of[i];
            int q = 0;
            if (s_rank[p] >= 0) {
                const uint32_t c = corners[i];
                q = quadrant(nodes[p], corner_x(c) - minB, corner_y(c) - minB);
            }
            node_of[i] = (uint16_t)s_child[p][q];
        }
        // 6. loop control (ref :767-775, :851-854)
        int n_to_expand;
        {
            int cnt = 0;
            for (int p = tid; p < min(K, cap); p += kOctThreads) cnt += (nnodes[p].count > 1);
            block_exclusive_scan(cnt, s_warp, n_to_expand);
        }
        if (tid == 0) { s_nn = min(new_nn, cap); s_seq += (unsigned)K; }
        cur ^= 1;
        if (new_nn > cap) { if (tid == 0) atomicOr(status, 2); finish = true; }
        if (new_nn >= N || new_nn == nn) finish = true;
        else if (!pass_b && new_nn + 3 * n_to_expand > N) pass_b = true;
        __syncthreads();
    }

    // ---- best corner per node: first maximum of response in reference raw order (ref :857-874) ----
    const int nn = s_nn;
    for (int p = tid; p < nn; p += kOctThreads) s_key[p] = 0ull;
    __syncthreads();
    const int cell_area = g.w_cell * g.h_cell;
    for (int i = tid; i < n; i += kOctThreads) {
        const uint32_t c = corners[i];
        const int x = corner_x(c) - kEdge, y = corner_y(c) - kEdge;       // relative to the first cell interior
        const int cj = x / g.w_cell, ci = y / g.h_cell;
        const unsigned order = (unsigned)((ci * g.n_cols + cj) * cell_area + (y - ci * g.h_cell) * g.w_cell + (x - cj * g.w_cell));
        const unsigned long long key = ((unsigned long long)corner_s(c) << 56) | ((unsigned long long)(0xFFFFFFu - order) << 32) | c;
        atomicMax(&s_key[node_of[i]], key);
    }
    __syncthreads();
    for (int p = tid; p < nn; p += kOctThreads)
        if (p < g.sel_cap) out[p] = (uint32_t)(s_key[p] & 0xFFFFFFFFull);
    if (tid == 0) {
        sel_count[b * L + level] = min(nn, g.sel_cap);
        if (nn > g.sel_cap) atomicOr(status, 4);
    }
}

// ------------------------------------------------------------------------------------------------
// host-callable launchers
// ------------------------------------------------------------------------------------------------
cudaError_t launch_octree(const PyramidGeom& G, const PyramidGeom* G_dev, int n_images, const uint32_t* raw,
                          const int* raw_count, uint16_t* node_of, uint32_t* sel_xys, int* sel_count, int* status,
                          cudaStream_t st, int level_lo, int level_count) {
    const int cap = G.node_cap;
    if (cap > kMaxNodes) return cudaErrorInvalidValue;
    const size_t smem = octree_smem_bytes(cap);
    // the attribute is per device and there may be one extractor per device / thread: set it on every launch (a cheap
    // driver call next to a kernel that runs once per batch) instead of caching a process-wide high-water mark
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(octree_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    if (level_count < 0) level_count = G.nlevels - level_lo;
    dim3 grid(level_count, n_images);
    octree_kernel<<<grid, kOctThreads, smem, st>>>(G_dev, cap, raw, G.raw_total, raw_count, node_of, sel_xys, sel_count, status, level_lo);
    return cudaSuccess;
}

}  // namespace mcs
