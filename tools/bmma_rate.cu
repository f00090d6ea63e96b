// bmma_rate.cu -- issue rate of the binary tensor-core MMA (mma.sync m16n8k256 .b1 AND.POPC, SASS BMMA.168256.AND.POPC) per SM.
//
// One CTA per SM; every warp runs CHAINS independent accumulator chains of back-to-back BMMAs on register operands, and
// thread 0 of each CTA reads the SM clock around the loop.  Reports BMMAs per clock per SM (and, for the masked 32-byte
// Hamming distance, which needs 4 BMMAs per 16x8 tile of 128 pairs, the implied pairs per clock per SM) for several warp
// counts and chain depths.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o bmma_rate tools/bmma_rate.cu && ./bmma_rate
#include <cstdio>
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { std::printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); return 1; } } while (0)

template <int CHAINS>
__global__ void bmma_loop(const uint32_t* __restrict__ seed, const int iters, int* __restrict__ sink, long long* __restrict__ cycles) {
    uint32_t a[4], b[2];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = seed[(threadIdx.x + i) & 63];
#pragma unroll
    for (int i = 0; i < 2; ++i) b[i] = seed[(threadIdx.x + 7 * i + 3) & 63];
    int acc[CHAINS][4];
#pragma unroll
    for (int c = 0; c < CHAINS; ++c)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[c][i] = 0;
    __syncthreads();
    long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int c = 0; c < CHAINS; ++c)
            asm volatile("mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+r"(acc[c][0]), "+r"(acc[c][1]), "+r"(acc[c][2]), "+r"(acc[c][3])
                         : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    }
    __syncthreads();
    long long t1 = clock64();
    int s = 0;
#pragma unroll
    for (int c = 0; c < CHAINS; ++c) s += acc[c][0] + acc[c][1] + acc[c][2] + acc[c][3];
    if (s == 0x12345678) sink[0] = s;          // keeps the chains alive
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int CHAINS>
static int run(int sms, int warps, const uint32_t* seed, int* sink, long long* d_cycles) {
    const int iters = 4096;
    bmma_loop<CHAINS><<<sms, warps * 32>>>(seed, iters, sink, d_cycles);      // warm-up
    CK(cudaGetLastError());
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    bmma_loop<CHAINS><<<sms, warps * 32>>>(seed, iters, sink, d_cycles);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    std::vector<long long> cyc(sms);
    CK(cudaMemcpy(cyc.data(), d_cycles, sizeof(long long) * sms, cudaMemcpyDeviceToHost));
    long long cmax = 0;
    double csum = 0;
    for (long long c : cyc) { cmax = c > cmax ? c : cmax; csum += (double)c; }
    const double per_sm = (double)warps * iters * CHAINS;                 // BMMAs issued on one SM
    const double rate = per_sm / (csum / sms);
    std::printf("{\"warps\": %d, \"chains\": %d, \"bmma_per_clk_per_sm\": %.4f, \"masked32_pairs_per_clk_per_sm\": %.2f, "
                "\"max_cycles\": %lld, \"ms\": %.3f, \"bmma_per_s\": %.4e}\n",
                warps, CHAINS, rate, rate * 32.0, cmax, ms, per_sm * sms / (ms * 1e-3));
    CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1));
    return 0;
}

int main() {
    int dev = 0, sms = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    cudaDeviceProp p;
    CK(cudaGetDeviceProperties(&p, dev));
    std::printf("# %s, %d SMs\n", p.name, sms);
    std::vector<uint32_t> h(64);
    for (int i = 0; i < 64; ++i) h[i] = 0x9E3779B9u * (uint32_t)(i + 1);
    uint32_t* seed; int* sink; long long* cyc;
    CK(cudaMalloc(&seed, 64 * 4)); CK(cudaMalloc(&sink, 4)); CK(cudaMalloc(&cyc, sizeof(long long) * sms));
    CK(cudaMemcpy(seed, h.data(), 64 * 4, cudaMemcpyHostToDevice));
    for (int warps : {1, 4, 8, 16}) {
        if (run<1>(sms, warps, seed, sink, cyc)) return 1;
        if (run<4>(sms, warps, seed, sink, cyc)) return 1;
        if (run<8>(sms, warps, seed, sink, cyc)) return 1;
    }
    CK(cudaFree(seed)); CK(cudaFree(sink)); CK(cudaFree(cyc));
    return 0;
}
