// mcs_comm.cu -- the one exchange step of the path (SURVEY.md 8e): every GPU of a rig extracts its camera(s) into ONE packed
// feature buffer, a single ncclAllGather over NVLink / NVSwitch gives every rank the buffers of all ranks in rank order -- the
// device-side counterpart of the camera-order concatenation of cMultiFrame (ref src/cMultiFrame.cpp:168-184).
//
// NCCL is reached through dlopen: a host program that already carries an NCCL (PyTorch bundles its own libnccl.so.2) must not
// get a second copy with clashing symbols, and a single-GPU user of this library needs no NCCL at all.  The library that is
// already mapped wins (RTLD_NOLOAD), otherwise the system libnccl.so.2 is loaded.
#include <dlfcn.h>

#include <cstring>
#include <mutex>
#include <string>

#include "api_check.h"
#include "kernels.h"
#include "mcs_common.cuh"

namespace {

// the slice of nccl.h this file needs (NCCL 2.x ABI)
struct NcclUniqueId { char internal[128]; };
typedef void* NcclComm;
constexpr int kNcclUint8 = 1;                     // ncclDataType_t: ncclUint8
struct Nccl {
    void* handle = nullptr;
    int (*GetUniqueId)(NcclUniqueId*) = nullptr;
    int (*CommInitRank)(NcclComm*, int, NcclUniqueId, int) = nullptr;
    int (*CommDestroy)(NcclComm) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, NcclComm, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    int (*GetVersion)(int*) = nullptr;
    std::string why;
};
Nccl& nccl() {
    static Nccl n;
    static std::once_flag once;
    std::call_once(once, [] {
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_LOCAL);
        if (!h) { n.why = std::string("libnccl.so.2 not found: ") + (dlerror() ? dlerror() : ""); return; }
        n.handle = h;
        n.GetUniqueId = (int (*)(NcclUniqueId*))dlsym(h, "ncclGetUniqueId");
        n.CommInitRank = (int (*)(NcclComm*, int, NcclUniqueId, int))dlsym(h, "ncclCommInitRank");
        n.CommDestroy = (int (*)(NcclComm))dlsym(h, "ncclCommDestroy");
        n.AllGather = (int (*)(const void*, void*, size_t, int, NcclComm, cudaStream_t))dlsym(h, "ncclAllGather");
        n.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
        n.GetVersion = (int (*)(int*))dlsym(h, "ncclGetVersion");
        if (!n.GetUniqueId || !n.CommInitRank || !n.CommDestroy || !n.AllGather) { n.why = "libnccl.so.2 lacks the NCCL 2 entry points"; n.handle = nullptr; }
    });
    return n;
}
std::string nccl_err(int rc) {
    Nccl& n = nccl();
    return std::string("NCCL error ") + std::to_string(rc) + (n.GetErrorString ? std::string(": ") + n.GetErrorString(rc) : "");
}
}  // namespace

struct mcs_comm {
    NcclComm comm = nullptr;
    int rank = 0, world = 1, device = 0;
};

extern "C" {

int mcs_comm_unique_id(uint8_t* id128) {
    if (!id128) return mcs_fail(MCS_ERR_INVALID, "null argument");
    Nccl& n = nccl();
    if (!n.handle) return mcs_fail(MCS_ERR_UNSUPPORTED, n.why);
    NcclUniqueId id;
    const int rc = n.GetUniqueId(&id);
    if (rc) return mcs_fail(MCS_ERR_CUDA, nccl_err(rc));
    std::memcpy(id128, id.internal, 128);
    return MCS_OK;
}

int mcs_comm_create(const uint8_t* id128, int32_t rank, int32_t world, mcs_comm** out) {
    if (!id128 || !out || world < 1 || rank < 0 || rank >= world) return mcs_fail(MCS_ERR_INVALID, "bad communicator arguments");
    Nccl& n = nccl();
    if (!n.handle) return mcs_fail(MCS_ERR_UNSUPPORTED, n.why);
    mcs_comm* c = new mcs_comm();
    c->rank = rank; c->world = world;
    cudaError_t e = cudaGetDevice(&c->device);
    if (e != cudaSuccess) { delete c; return mcs_fail(MCS_ERR_NO_DEVICE, cudaGetErrorString(e)); }
    NcclUniqueId id;
    std::memcpy(id.internal, id128, 128);
    const int rc = n.CommInitRank(&c->comm, world, id, rank);        // collective: every rank of the rig calls it
    if (rc) { delete c; return mcs_fail(MCS_ERR_CUDA, nccl_err(rc)); }
    *out = c;
    return MCS_OK;
}

void mcs_comm_destroy(mcs_comm* c) {
    if (!c) return;
    if (c->comm && nccl().CommDestroy) nccl().CommDestroy(c->comm);
    delete c;
}

int mcs_comm_info(const mcs_comm* c, int32_t* rank, int32_t* world, int32_t* nccl_version) {
    if (!c) return mcs_fail(MCS_ERR_INVALID, "null communicator");
    if (rank) *rank = c->rank;
    if (world) *world = c->world;
    if (nccl_version) { int v = 0; if (nccl().GetVersion) nccl().GetVersion(&v); *nccl_version = v; }
    return MCS_OK;
}

size_t mcs_packed_layout(int32_t n_images, int32_t capacity, int32_t dim, size_t* offsets4) {
    // [counts int32[n_images] | mcs_keypoint[n_images][capacity] | desc u8[n_images][capacity][dim] | dmask (same)], every
    // section starting on a 256-byte boundary: the buffers K3 writes through four pointers, contiguous for the exchange
    const size_t sizes[4] = {(size_t)n_images * 4, (size_t)n_images * capacity * sizeof(mcs_keypoint), (size_t)n_images * capacity * dim,
                             (size_t)n_images * capacity * dim};
    size_t o = 0;
    for (int k = 0; k < 4; ++k) {
        if (offsets4) offsets4[k] = o;
        o += (sizes[k] + 255) & ~(size_t)255;
    }
    return o;
}

size_t mcs_slot_bytes(int32_t capacity, int32_t dim) { return mcs_packed_layout(1, capacity, dim, nullptr); }

int mcs_allgather_features(mcs_comm* c, const void* packed_dev, size_t bytes, void* gathered_dev, void* stream) {
    if (!c || !packed_dev || !gathered_dev || bytes == 0) return mcs_fail(MCS_ERR_INVALID, "null argument");
    int dev = -1;
    cudaGetDevice(&dev);
    if (dev != c->device) return mcs_fail(MCS_ERR_INVALID, "the communicator belongs to another CUDA device than the current one");
    const int rc = nccl().AllGather(packed_dev, gathered_dev, bytes, kNcclUint8, c->comm, (cudaStream_t)stream);
    if (rc) return mcs_fail(MCS_ERR_CUDA, nccl_err(rc));
    return MCS_OK;
}

}  // extern "C"
