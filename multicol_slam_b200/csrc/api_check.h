// api_check.h -- the error path of the C-ABI host layer: the message mcs_last_error() returns, the MCS_ERR_* code of a failed
// CUDA call, and the argument checks that several entry points share.
#pragma once
#include <cuda_runtime.h>
#include <string>
#include "../../include/mcs_b200.h"
#include "mcs_common.cuh"

// records `msg` for mcs_last_error() on the calling thread and returns `code` (mcs_api.cu)
int mcs_fail(int code, const std::string& msg);

// a failed CUDA call: no device or no usable driver -> MCS_ERR_NO_DEVICE, any other error -> MCS_ERR_CUDA, with the message
// "<what>: <cudaGetErrorString>".  The error is cleared, so that the next call does not see it.
inline int mcs_cuda_fail(cudaError_t e, const std::string& what) {
    cudaGetLastError();
    return mcs_fail(e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver ? MCS_ERR_NO_DEVICE : MCS_ERR_CUDA,
                    what + ": " + cudaGetErrorString(e));
}

// returns from the calling entry point when the CUDA call `expr` fails
#define CUDA_CHECK(expr)                                                   \
    do {                                                                   \
        const cudaError_t e__ = (expr);                                    \
        if (e__ != cudaSuccess) return mcs_cuda_fail(e__, #expr);          \
    } while (0)

// descriptor widths (bytes) the matchers are built for: MCS_OK, or MCS_ERR_INVALID with the message set
inline int check_desc_dim(int dim) {
    return mcs::desc_width_ok(dim) ? MCS_OK : mcs_fail(MCS_ERR_INVALID, "dim must be 16, 32 or 64");
}
