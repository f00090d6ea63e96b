// Repro + workarounds for a ptxas 12.9 (-O1 and above) miscompile, seen when targeting sm_100a, while writing the FAST
// score: max(a, max(b, -c)) is folded into VIMNMX3 and the negation is lost.  Variants 1-3 are correct; the
// original scalar form (removed) was wrong on the device and right on the host / with -Xptxas -O0.
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <algorithm>
#include <cuda_runtime.h>
constexpr int S = 76;
__host__ __device__ inline bool has_arc9(uint32_t m) { m |= m << 16; uint32_t r = m & (m >> 1); r &= r >> 2; r &= r >> 4; r &= m >> 8; return (r & 0xFFFFu) != 0; }
#define LOAD_RING \
    int r[16]; \
    r[0] = p[3 * S];       r[1] = p[3 * S + 1];   r[2] = p[2 * S + 2];   r[3] = p[S + 3]; \
    r[4] = p[3];           r[5] = p[-S + 3];      r[6] = p[-2 * S + 2];  r[7] = p[-3 * S + 1]; \
    r[8] = p[-3 * S];      r[9] = p[-3 * S - 1];  r[10] = p[-2 * S - 2]; r[11] = p[-S - 3]; \
    r[12] = p[-3];         r[13] = p[S - 3];      r[14] = p[2 * S - 2];  r[15] = p[3 * S - 1]; \
    uint32_t bm = 0, dm = 0; \
    _Pragma("unroll") for (int k = 0; k < 16; ++k) { bm |= (uint32_t)(r[k] > v + t) << k; dm |= (uint32_t)(r[k] < v - t) << k; } \
    if (!has_arc9(bm) && !has_arc9(dm)) return 0;

int h_score(const uint8_t* p, int t) {
    const int v = p[0];
    LOAD_RING
    int best = t;
    for (int s = 0; s < 16; ++s) { int a = 1000, b = -1000; for (int i = 0; i < 9; ++i) { int d = v - r[(s + i) & 15]; a = std::min(a, d); b = std::max(b, d); } best = std::max(best, std::max(a, -b)); }
    return best - 1;
}
// V1: two min trees, no negation of a max
__device__ int score_v1(const uint8_t* p, int t) {
    const int v = p[0];
    LOAD_RING
    int d[16], e[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) { d[k] = v - r[k]; e[k] = r[k] - v; }
    int d2[16], e2[16], d4[16], e4[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) { d2[k] = min(d[k], d[(k + 1) & 15]); e2[k] = min(e[k], e[(k + 1) & 15]); }
#pragma unroll
    for (int k = 0; k < 16; ++k) { d4[k] = min(d2[k], d2[(k + 2) & 15]); e4[k] = min(e2[k], e2[(k + 2) & 15]); }
    int best = t;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        const int d9 = min(min(d4[k], d4[(k + 4) & 15]), d[(k + 8) & 15]);
        const int e9 = min(min(e4[k], e4[(k + 4) & 15]), e[(k + 8) & 15]);
        best = max(best, max(d9, e9));
    }
    return best - 1;
}
// V3: packed s16x2 lanes: lo = v - r (dark margin), hi = r - v (bright margin); one min tree
__device__ int score_v3(const uint8_t* p, int t) {
    const int v = p[0];
    LOAD_RING
    unsigned q[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) { const int d = v - r[k]; q[k] = ((unsigned)d & 0xFFFFu) | ((unsigned)(-d) << 16); }
    unsigned q2[16], q4[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) q2[k] = __vmins2(q[k], q[(k + 1) & 15]);
#pragma unroll
    for (int k = 0; k < 16; ++k) q4[k] = __vmins2(q2[k], q2[(k + 2) & 15]);
    unsigned m = __vmins2(__vmins2(q4[0], q4[4]), q[8]);
#pragma unroll
    for (int k = 1; k < 16; ++k) m = __vmaxs2(m, __vmins2(__vmins2(q4[k], q4[(k + 4) & 15]), q[(k + 8) & 15]));
    const int lo = (int)(short)(m & 0xFFFFu), hi = (int)(short)(m >> 16);
    return max(t, max(lo, hi)) - 1;
}
// V2: original with an optimisation barrier before the negation
__device__ int score_v2(const uint8_t* p, int t) {
    const int v = p[0];
    LOAD_RING
    int d[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) d[k] = v - r[k];
    int mn2[16], mx2[16], mn4[16], mx4[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) { mn2[k] = min(d[k], d[(k + 1) & 15]); mx2[k] = max(d[k], d[(k + 1) & 15]); }
#pragma unroll
    for (int k = 0; k < 16; ++k) { mn4[k] = min(mn2[k], mn2[(k + 2) & 15]); mx4[k] = max(mx2[k], mx2[(k + 2) & 15]); }
    int bd = t, bb = 1000;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        bd = max(bd, min(min(mn4[k], mn4[(k + 4) & 15]), d[(k + 8) & 15]));
        bb = min(bb, max(max(mx4[k], mx4[(k + 4) & 15]), d[(k + 8) & 15]));
    }
    asm volatile("" : "+r"(bb));
    return max(bd, -bb) - 1;
}
template <int V> __global__ void k(const uint8_t* img, int* out, int t) {
    __shared__ uint8_t tile[40 * S];
    for (int i = threadIdx.x; i < 40 * S; i += blockDim.x) tile[i] = img[i];
    __syncthreads();
    for (int i = threadIdx.x; i < 34 * 66; i += blockDim.x) {
        int y = i / 66, x = i % 66;
        const uint8_t* p = tile + (y + 3) * S + x + 3;
        out[i] = V == 1 ? score_v1(p, t) : V == 2 ? score_v2(p, t) : score_v3(p, t);
    }
}
int main() {
    static uint8_t h[40 * S];
    uint8_t* d; int* o; cudaMalloc(&d, sizeof(h)); cudaMalloc(&o, 34 * 66 * 4);
    static int ho[34 * 66];
    for (int V = 1; V <= 3; ++V) {
        srand(3);
        int bad = 0, tot = 0;
        for (int it = 0; it < 50; ++it) {
            for (auto& v : h) v = (rand() % 3 == 0) ? rand() % 256 : (rand() % 2 ? 0 : 100 + rand() % 40);
            cudaMemcpy(d, h, sizeof(h), cudaMemcpyHostToDevice);
            if (V == 1) k<1><<<1, 256>>>(d, o, 20); else if (V == 2) k<2><<<1, 256>>>(d, o, 20); else k<3><<<1, 256>>>(d, o, 20);
            cudaMemcpy(ho, o, sizeof(ho), cudaMemcpyDeviceToHost);
            for (int i = 0; i < 34 * 66; ++i) {
                int y = i / 66, x = i % 66;
                int e = h_score(h + (y + 3) * S + x + 3, 20);
                tot += e > 0;
                if (e != ho[i]) { if (bad < 3) printf("V%d mismatch (%d,%d): host %d dev %d\n", V, x, y, e, ho[i]); ++bad; }
            }
        }
        printf("variant %d: corners %d mismatches %d (%s)\n", V, tot, bad, cudaGetErrorString(cudaGetLastError()));
    }
}
