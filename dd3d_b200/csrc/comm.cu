// Multi-GPU boundary of the DD3D path: ONE NCCL all-gather of the packed detections per evaluated batch.
//
// Replaces detectron2 comm.gather of pickled prediction lists in the reference evaluators
// (tridet/evaluators/kitti_3d_evaluator.py:152-164, nuscenes_evaluator.py:255): every rank contributes its fixed-stride
// buffer  [B][out_cap] dd3d_det | counts[B] | flags[1]  (dd3d_packed_bytes; NuscenesDD3D appends the pred_boxes3d_global
// rows [B][out_cap][10] of its sample aggregation, dd3d_packed_bytes_global) and receives all ranks' buffers.  Images are
// independent (eval BN, per-image NMS), so this is the only exchange of the path (SURVEY.md 8e); 295 KB per rank at
// B = 32 -- latency, not bandwidth, so it is issued on a side stream and overlaps the next batch's forward.
//
// NCCL is resolved at run time (dlopen of the libnccl.so.2 already loaded by the host framework, or the system one): the
// library has no link-time dependency on it and single-GPU users never touch it.
#include <dlfcn.h>
#include <stdint.h>
#include <string.h>

#include <string>

#include "../../include/dd3d_b200.h"
#include <cuda_runtime.h>

namespace {

typedef struct { char internal[128]; } nccl_unique_id;  // ncclUniqueId (NCCL_UNIQUE_ID_BYTES = 128)
typedef void* nccl_comm_t;
typedef int nccl_result_t;  // ncclSuccess = 0
constexpr int kNcclInt8 = 0;  // ncclInt8 / ncclChar

struct NcclApi {
    void* lib = nullptr;
    nccl_result_t (*GetUniqueId)(nccl_unique_id*) = nullptr;
    nccl_result_t (*CommInitRank)(nccl_comm_t*, int, nccl_unique_id, int) = nullptr;
    nccl_result_t (*CommDestroy)(nccl_comm_t) = nullptr;
    nccl_result_t (*AllGather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(nccl_result_t) = nullptr;
    nccl_result_t (*GetVersion)(int*) = nullptr;
};

thread_local std::string g_comm_error;

NcclApi* nccl() {
    static NcclApi api;
    static bool tried = false;
    if (!tried) {
        tried = true;
        const char* override_path = getenv("DD3D_NCCL_LIB");
        const char* names[] = {override_path, "libnccl.so.2", "libnccl.so"};
        for (const char* n : names) {
            if (n == nullptr) continue;
            api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.lib) break;
        }
        if (api.lib) {
            api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(api.lib, "ncclGetUniqueId"));
            api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(api.lib, "ncclCommInitRank"));
            api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(api.lib, "ncclCommDestroy"));
            api.AllGather = reinterpret_cast<decltype(api.AllGather)>(dlsym(api.lib, "ncclAllGather"));
            api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(api.lib, "ncclGetErrorString"));
            api.GetVersion = reinterpret_cast<decltype(api.GetVersion)>(dlsym(api.lib, "ncclGetVersion"));
        }
    }
    if (!api.lib || !api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllGather) {
        g_comm_error = "NCCL not available (dlopen libnccl.so.2 failed or symbols missing); set DD3D_NCCL_LIB";
        return nullptr;
    }
    return &api;
}

int nccl_fail(NcclApi* a, nccl_result_t r, const char* what) {
    g_comm_error = std::string(what) + ": " + ((a && a->GetErrorString) ? a->GetErrorString(r) : "NCCL error") + " (" +
                   std::to_string(r) + ")";
    return DD3D_ERR_CUDA;
}

}  // namespace

struct dd3d_comm_s {
    nccl_comm_t comm = nullptr;
    int rank = 0, world = 1, device = 0;
    bool owned = true;
};

extern "C" {

int64_t dd3d_packed_bytes(int B, int out_cap) {
    if (B < 1 || out_cap < 1) return DD3D_ERR_INVALID;
    const int64_t dets = static_cast<int64_t>(B) * out_cap * static_cast<int64_t>(sizeof(dd3d_det));
    const int64_t tail = (static_cast<int64_t>(B + 1) * 4 + 255) / 256 * 256;  // counts[B] + flags[1], padded
    return dets + tail;
}

int64_t dd3d_packed_bytes_global(int B, int out_cap) {
    const int64_t head = dd3d_packed_bytes(B, out_cap);
    if (head < 0) return head;
    const int64_t global = (static_cast<int64_t>(B) * out_cap * 10 * 4 + 255) / 256 * 256;  // float [B][out_cap][10], padded
    return head + global;
}

const char* dd3d_comm_last_error(void) { return g_comm_error.c_str(); }

int dd3d_comm_unique_id(uint8_t* h_id128) {
    if (!h_id128) return DD3D_ERR_INVALID;
    NcclApi* a = nccl();
    if (!a) return DD3D_ERR_CUDA;
    nccl_unique_id id;
    nccl_result_t r = a->GetUniqueId(&id);
    if (r != 0) return nccl_fail(a, r, "ncclGetUniqueId");
    memcpy(h_id128, id.internal, 128);
    return DD3D_OK;
}

int dd3d_comm_create(const uint8_t* h_id128, int rank, int world, dd3d_comm* out) {
    if (!h_id128 || !out || world < 1 || rank < 0 || rank >= world) return DD3D_ERR_INVALID;
    *out = nullptr;
    NcclApi* a = nccl();
    if (!a) return DD3D_ERR_CUDA;
    nccl_unique_id id;
    memcpy(id.internal, h_id128, 128);
    dd3d_comm_s* c = new dd3d_comm_s();
    c->rank = rank;
    c->world = world;
    if (cudaGetDevice(&c->device) != cudaSuccess) {
        delete c;
        g_comm_error = "cudaGetDevice failed";
        return DD3D_ERR_CUDA;
    }
    nccl_result_t r = a->CommInitRank(&c->comm, world, id, rank);  // collective over all ranks
    if (r != 0) {
        delete c;
        return nccl_fail(a, r, "ncclCommInitRank");
    }
    *out = c;
    return DD3D_OK;
}

int dd3d_comm_from_nccl(void* nccl_comm, int rank, int world, dd3d_comm* out) {
    if (!nccl_comm || !out || world < 1 || rank < 0 || rank >= world) return DD3D_ERR_INVALID;
    if (!nccl()) return DD3D_ERR_CUDA;
    dd3d_comm_s* c = new dd3d_comm_s();
    c->comm = nccl_comm;
    c->rank = rank;
    c->world = world;
    c->owned = false;
    cudaGetDevice(&c->device);
    *out = c;
    return DD3D_OK;
}

void dd3d_comm_destroy(dd3d_comm c) {
    if (!c) return;
    NcclApi* a = nccl();
    if (a && c->owned && c->comm) a->CommDestroy(c->comm);
    delete c;
}

int dd3d_comm_world(dd3d_comm c) { return c ? c->world : DD3D_ERR_INVALID; }

int dd3d_allgather(dd3d_comm c, const void* d_send, void* d_recv, int64_t bytes_per_rank, dd3d_stream stream) {
    if (!c || !d_send || !d_recv || bytes_per_rank < 1) return DD3D_ERR_INVALID;
    NcclApi* a = nccl();
    if (!a) return DD3D_ERR_CUDA;
    cudaSetDevice(c->device);
    nccl_result_t r = a->AllGather(d_send, d_recv, static_cast<size_t>(bytes_per_rank), kNcclInt8, c->comm,
                                   static_cast<cudaStream_t>(stream));
    if (r != 0) return nccl_fail(a, r, "ncclAllGather");
    return DD3D_OK;
}

}  // extern "C"
