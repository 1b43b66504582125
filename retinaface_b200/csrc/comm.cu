// comm.cu -- multi-GPU exchange of the final detections behind the C ABI (SURVEY.md 8e: images are independent, the batch is
// sharded over one process per GPU, the only exchange is an all-gather of the fixed-size per-image detection records).
//
// The reference has no multi-GPU path (single default device everywhere, RetinaFace.h:89 `ctx_id` unused).  Here the
// all-gather is FUSED into the NMS: every rank owns a gather window in device memory, exported to its peers through CUDA
// IPC; the CTA that finishes an image's NMS (postproc_dev.cuh nms_image -- the stand-alone k_nms or the last-block NMS of
// the tile chains) stores the kept records straight into the window of EVERY rank over NVLink / NVSwitch peer mappings and
// then raises that image's flag there.  No collective kernel, no extra launch on the producing side; a consumer orders its
// reads behind one tiny kernel that waits for the step's flags (k_comm_wait_p, the last node of the forward graph).
//
// Window of one rank: [ring][world][max_batch] x {max_faces records, count, flag}.  A step with sequence number q uses slot
// q % ring of every window.  Flow control needs no acknowledgements: a rank can only run RF_PIPELINE_DEPTH + `streams`
// steps ahead of the slowest rank (its own results need that rank's records), which is less than `ring` = 32.
#include <dlfcn.h>
#include <unistd.h>

#include "engine_internal.cuh"

namespace rf_eng {

namespace {

constexpr uint32_t COMM_MAGIC = 0x52464331;   // "RFC1"
constexpr int COMM_RING = 32;

struct CommBlob {                // RF_COMM_BLOB_BYTES = 128
    uint32_t magic;
    int32_t rank, world, pid, device, max_batch, max_faces, ring;
    uint64_t ptr, bytes;
    cudaIpcMemHandle_t ipc;      // 64 bytes
    char pad[128 - 8 * 4 - 2 * 8 - 64];
};
static_assert(sizeof(CommBlob) == RF_COMM_BLOB_BYTES, "blob layout");

size_t dets_bytes(rf_handle h, int world) { return sizeof(rf_det) * (size_t)COMM_RING * world * h->cfg.max_batch * h->cfg.max_faces; }
size_t words(rf_handle h, int world) { return (size_t)COMM_RING * world * h->cfg.max_batch; }

// The consumer side: one tiny kernel that waits for the step's flags of every rank, as the LAST NODE of the forward graph.
// Sequence number and slot come from the run parameters in device memory (0 = this run has no exchange: return at once), so
// one captured graph serves every step; a peer that never delivers is reported (err), not waited for forever
__global__ void __launch_bounds__(1024) k_comm_wait_p(const unsigned *flags, const PostParams *__restrict__ params, int world, int max_batch, int n, unsigned *err) {
    const unsigned seq = params->comm_seq;
    if (!seq) return;
    const size_t base = (size_t)params->comm_slot * world * max_batch;
    for (int t = threadIdx.x; t < world * n; t += blockDim.x) {
        const int r = t / n, i = t - r * n;
        const volatile unsigned *f = flags + base + (size_t)r * max_batch + i;
        unsigned spins = 0;
        while (*f != seq) {
            if (++spins > (1u << 25)) { atomicMax(err, 1u + (unsigned)r); break; }
            __nanosleep(200);
        }
    }
    __threadfence_system();
}

}  // namespace

void comm_release(rf_handle h) {
    Comm &c = h->comm;
    for (int p = 0; p < c.world; p++)
        if (c.opened[p] && c.peer[p]) cudaIpcCloseMemHandle(c.peer[p]);
    cudaFree(c.window);
    cudaFree(c.d_err);
    cudaFreeHost(c.h_err);
    for (auto &sl : c.slots) { cudaFreeHost(sl.h_dets); cudaFreeHost(sl.h_counts); }
    c = Comm{};
}

// Orders `s` behind the arrival of every rank's records of the step the run parameters name.
void comm_wait_in_graph(rf_handle h, const Ctx &x, int n, cudaStream_t s) {
    Comm &c = h->comm;
    const unsigned *flags = reinterpret_cast<const unsigned *>(c.window + dets_bytes(h, c.world) + words(h, c.world) * 4);
    const int threads = std::min(1024, std::max(32, c.world * n));
    k_comm_wait_p<<<1, threads, 0, s>>>(flags, x.d_params, c.world, h->cfg.max_batch, n, c.d_err);
    CK(cudaGetLastError());
}

}  // namespace rf_eng

extern "C" {

int rf_comm_export(rf_handle h, int rank, int world, void *blob) {
    if (!h || !blob) return fail(h, RF_ERR_INVALID_ARG, "rf_comm_export: NULL argument");
    if (world < 1 || world > RF_COMM_MAX_WORLD || rank < 0 || rank >= world) return fail(h, RF_ERR_INVALID_ARG, fmt("rf_comm_export: rank %d of %d (world <= %d)", rank, world, RF_COMM_MAX_WORLD));
    try {
        CK(cudaSetDevice(h->device));
        CK(rf_synchronize(h) == RF_OK ? cudaSuccess : cudaErrorUnknown);
        comm_release(h);
        Comm &c = h->comm;
        c.rank = rank; c.world = world; c.ring = COMM_RING;
        c.bytes = dets_bytes(h, world) + 2 * words(h, world) * 4;
        CK(cudaMalloc(&c.window, c.bytes));
        CK(cudaMemset(c.window, 0, c.bytes));
        CK(cudaMalloc(&c.d_err, 4));
        CK(cudaMemset(c.d_err, 0, 4));
        CK(cudaHostAlloc(&c.h_err, 4, cudaHostAllocDefault));
        CommBlob b{};
        b.magic = COMM_MAGIC; b.rank = rank; b.world = world; b.pid = (int)getpid(); b.device = h->device;
        b.max_batch = h->cfg.max_batch; b.max_faces = h->cfg.max_faces; b.ring = COMM_RING;
        b.ptr = (uint64_t)(uintptr_t)c.window; b.bytes = c.bytes;
        CK(cudaIpcGetMemHandle(&b.ipc, c.window));
        memcpy(blob, &b, sizeof b);
        memcpy(&c.blob, &b, sizeof b);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

int rf_comm_init(rf_handle h, const void *blobs) {
    if (!h || !blobs) return fail(h, RF_ERR_INVALID_ARG, "rf_comm_init: NULL argument");
    Comm &c = h->comm;
    if (!c.window) return fail(h, RF_ERR_INVALID_ARG, "rf_comm_init: call rf_comm_export first");
    try {
        CK(cudaSetDevice(h->device));
        const CommBlob *B = reinterpret_cast<const CommBlob *>(blobs);
        for (int p = 0; p < c.world; p++) {
            const CommBlob &b = B[p];
            if (b.magic != COMM_MAGIC || b.rank != p || b.world != c.world || b.max_batch != h->cfg.max_batch || b.max_faces != h->cfg.max_faces || b.ring != c.ring ||
                b.bytes != c.bytes)
                return fail(h, RF_ERR_INVALID_ARG, fmt("rf_comm_init: blob %d does not describe rank %d of %d with max_batch %d, max_faces %d", p, p, c.world,
                                                       h->cfg.max_batch, h->cfg.max_faces));
            if (p == c.rank) { c.peer[p] = c.window; continue; }
            if (b.pid == (int)getpid()) {
                // another handle of this process (tests; one process driving several GPUs): plain peer access
                if (b.device != h->device) {
                    cudaError_t e = cudaDeviceEnablePeerAccess(b.device, 0);
                    if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) throw CudaFail{e, "cudaDeviceEnablePeerAccess", __FILE__, __LINE__};
                    cudaGetLastError();
                }
                c.peer[p] = reinterpret_cast<unsigned char *>((uintptr_t)b.ptr);
            } else {
                void *ptr = nullptr;
                CK(cudaIpcOpenMemHandle(&ptr, b.ipc, cudaIpcMemLazyEnablePeerAccess));
                c.peer[p] = static_cast<unsigned char *>(ptr);
                c.opened[p] = true;
            }
        }
        CommView v{};
        v.world = c.world; v.rank = c.rank; v.ring = c.ring;
        for (int p = 0; p < c.world; p++) {
            v.dets[p] = reinterpret_cast<rf_det *>(c.peer[p]);
            v.counts[p] = reinterpret_cast<int *>(c.peer[p] + dets_bytes(h, c.world));
            v.flags[p] = reinterpret_cast<unsigned *>(c.peer[p] + dets_bytes(h, c.world) + words(h, c.world) * 4);
        }
        // every context's NMS gets the peer view; graphs captured before carry the old (empty) one
        for (Ctx &x : h->ctx) {
            CK(cudaStreamSynchronize(x.stream));
            x.pb.comm = v;
            for (auto &g : x.graphs) cudaGraphExecDestroy(g.second);
            x.graphs.clear();
        }
        c.ready = true;
        c.seq = 0;
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

// ---- bootstrap through NCCL (optional: libnccl.so.2 is opened at run time, the library does not link it) ----------------
namespace {
struct Id128 { char b[128]; };        // ncclUniqueId (passed by value to ncclCommInitRank)
struct NcclApi {
    void *lib = nullptr;
    int (*GetUniqueId)(void *) = nullptr;
    int (*CommInitRank)(void **, int, Id128, int) = nullptr;
    int (*AllGather)(const void *, void *, size_t, int, void *, cudaStream_t) = nullptr;
    int (*CommDestroy)(void *) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
};
NcclApi *nccl_api(std::string &err) {
    static NcclApi api;
    if (api.lib) return &api;
    void *lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) { err = std::string("libnccl.so.2 not found: ") + dlerror(); return nullptr; }
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(lib, "ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(lib, "ncclCommInitRank"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(dlsym(lib, "ncclAllGather"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(lib, "ncclCommDestroy"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(lib, "ncclGetErrorString"));
    if (!api.GetUniqueId || !api.CommInitRank || !api.AllGather || !api.CommDestroy) { err = "libnccl.so.2 lacks the expected symbols"; return nullptr; }
    api.lib = lib;
    return &api;
}
}  // namespace

int rf_comm_nccl_unique_id(void *out128) {
    if (!out128) return fail(nullptr, RF_ERR_INVALID_ARG, "rf_comm_nccl_unique_id: NULL");
    std::string err;
    NcclApi *api = nccl_api(err);
    if (!api) return fail(nullptr, RF_ERR_UNSUPPORTED, err);
    const int rc = api->GetUniqueId(out128);
    if (rc) return fail(nullptr, RF_ERR_CUDA, fmt("ncclGetUniqueId failed (%d)", rc));
    return RF_OK;
}

int rf_comm_init_nccl(rf_handle h, const void *nccl_unique_id, int rank, int world) {
    if (!h || !nccl_unique_id) return fail(h, RF_ERR_INVALID_ARG, "rf_comm_init_nccl: NULL argument");
    std::string err;
    NcclApi *api = nccl_api(err);
    if (!api) return fail(h, RF_ERR_UNSUPPORTED, err);
    CommBlob mine;
    int rc = rf_comm_export(h, rank, world, &mine);
    if (rc) return rc;
    void *comm = nullptr;
    unsigned char *d_send = nullptr, *d_recv = nullptr;
    std::vector<CommBlob> all(world);
    try {
        CK(cudaSetDevice(h->device));
        Id128 id;
        memcpy(&id, nccl_unique_id, 128);
        int nrc = api->CommInitRank(&comm, world, id, rank);
        if (nrc) return fail(h, RF_ERR_CUDA, fmt("ncclCommInitRank failed: %s", api->GetErrorString ? api->GetErrorString(nrc) : "?"));
        CK(cudaMalloc(&d_send, sizeof(CommBlob)));
        CK(cudaMalloc(&d_recv, sizeof(CommBlob) * world));
        cudaStream_t s = h->ctx[0].stream;
        CK(cudaMemcpyAsync(d_send, &mine, sizeof mine, cudaMemcpyHostToDevice, s));
        nrc = api->AllGather(d_send, d_recv, sizeof(CommBlob), /* ncclChar */ 0, comm, s);
        if (nrc) { api->CommDestroy(comm); cudaFree(d_send); cudaFree(d_recv); return fail(h, RF_ERR_CUDA, fmt("ncclAllGather failed: %s", api->GetErrorString ? api->GetErrorString(nrc) : "?")); }
        CK(cudaMemcpyAsync(all.data(), d_recv, sizeof(CommBlob) * world, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        api->CommDestroy(comm);
        cudaFree(d_send); cudaFree(d_recv);
    } catch (const CudaFail &f) {
        if (comm) api->CommDestroy(comm);
        cudaFree(d_send); cudaFree(d_recv);
        return fail_cuda(h, f);
    }
    return rf_comm_init(h, all.data());
}

int rf_comm_info(rf_handle h, int *rank, int *world) {
    if (!h) return RF_ERR_INVALID_ARG;
    if (rank) *rank = h->comm.rank;
    if (world) *world = h->comm.ready ? h->comm.world : 1;
    return RF_OK;
}

}  // extern "C"
