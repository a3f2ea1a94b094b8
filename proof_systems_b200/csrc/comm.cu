// comm.cu — the one exchange step of the path, owned by the library (SURVEY.md §8e): an MSM sharded by points over the GPUs of a
// node ends with ONE collective — an all-gather of every rank's c slice sums (c x 128 bytes) over NVLink — enqueued from C on the
// context's stream right behind the MSM kernels, followed by the cross-rank sum on the device and the O(c) tail.
// The reference's own split is poly-commitment/src/ipa.rs:652-662 (2-way rayon::join) and benches/msm.rs:92-140 (1/2/4/8-way).
//
// NCCL is bound at run time (dlopen of libnccl.so.2: the copy already loaded by the host process — torch's — or the system
// one), so libzkb200.so itself loads on hosts without NCCL; zk_comm_* then fail with ZK_ERR_INVALID.
#include <dlfcn.h>

#include <cstring>
#include <mutex>

#include "../../include/zkb200.h"
#include "ctx.hpp"
#include "host_field.hpp"

using namespace zkb;

namespace {

// the handful of NCCL declarations used here (nccl.h: 143-181 and the collective prototypes); ABI-stable since NCCL 2.0
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;                   // ncclSuccess == 0
constexpr int NCCL_UINT8 = 1;               // ncclDataType_t: ncclInt8 = 0, ncclUint8 = 1

struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};

NcclApi& nccl() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        // RTLD_NOLOAD first: reuse the libnccl the host process already mapped (two NCCL copies in one process do not mix)
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return;
        api.handle = h;
        api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(h, "ncclGetUniqueId");
        api.CommInitRank = (decltype(api.CommInitRank))dlsym(h, "ncclCommInitRank");
        api.CommDestroy = (decltype(api.CommDestroy))dlsym(h, "ncclCommDestroy");
        api.AllGather = (decltype(api.AllGather))dlsym(h, "ncclAllGather");
        api.GetErrorString = (decltype(api.GetErrorString))dlsym(h, "ncclGetErrorString");
        api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.GetErrorString;
    });
    return api;
}

int nccl_check(ncclResult_t r, const char* what) {
    if (r == 0) return ZK_OK;
    zk_set_error("%s: NCCL error %d (%s)", what, r, nccl().GetErrorString ? nccl().GetErrorString(r) : "?");
    return ZK_ERR_CUDA;
}

}  // namespace

struct zk_comm {
    zk_ctx* ctx = nullptr;
    ncclComm_t comm = nullptr;        // NCCL's handle: destroyed explicitly by zk_comm_destroy
    int world = 1, rank = 0;
    zkb::DevScratch slices;           // this rank's slice sums | world x slice sums
    zkb::xyzz_t* d_mine = nullptr;
    zkb::xyzz_t* d_all = nullptr;
    size_t cap_points = 0;
};

extern "C" {

int zk_comm_unique_id(uint8_t out_id[128]) {
    if (!out_id) { zk_set_error("comm_unique_id: null argument"); return ZK_ERR_INVALID; }
    if (!nccl().ok) { zk_set_error("comm: libnccl.so.2 could not be loaded"); return ZK_ERR_INVALID; }
    ncclUniqueId id;
    int rc = nccl_check(nccl().GetUniqueId(&id), "ncclGetUniqueId");
    if (rc) return rc;
    memcpy(out_id, id.internal, 128);
    return ZK_OK;
}

int zk_comm_init_rank(zk_ctx* ctx, const uint8_t id[128], int world, int rank, zk_comm** out) {
    if (!ctx || !id || !out) { zk_set_error("comm_init_rank: null argument"); return ZK_ERR_INVALID; }
    if (world < 1 || rank < 0 || rank >= world) { zk_set_error("comm_init_rank: rank %d outside a world of %d", rank, world); return ZK_ERR_INVALID; }
    if (!nccl().ok) { zk_set_error("comm: libnccl.so.2 could not be loaded"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    auto c = std::make_unique<zk_comm>();
    c->ctx = ctx; c->world = world; c->rank = rank;
    ncclUniqueId uid;
    memcpy(uid.internal, id, 128);
    int rc = nccl_check(nccl().CommInitRank(&c->comm, world, uid, rank), "ncclCommInitRank");
    if (rc) return rc;
    *out = c.release();
    return ZK_OK;
}

void zk_comm_destroy(zk_comm* c) {
    if (!c) return;
    std::lock_guard<std::mutex> lk(c->ctx->mu);
    cudaSetDevice(c->ctx->device);
    cudaStreamSynchronize(c->ctx->stream);
    if (c->comm) nccl().CommDestroy(c->comm);
    delete c;
}

int zk_comm_world(const zk_comm* c) { return c ? c->world : 0; }
int zk_comm_rank(const zk_comm* c) { return c ? c->rank : -1; }

// One MSM over world x n points: this rank's slice [off, off + n) of ITS resident bases with its n scalars; every rank receives
// the full result (identical bits).  All ranks must call it, with bases of the same table window.
int zk_msm_sharded(zk_comm* c, const zk_bases* bases, size_t off, size_t n, const void* scalars, int scalars_are_mont, int window_bits,
                   uint64_t out_xyz[12]) {
    if (!c || !bases || !out_xyz || (!scalars && n)) { zk_set_error("msm_sharded: null argument"); return ZK_ERR_INVALID; }
    zk_ctx* ctx = c->ctx;
    if (ctx_root(bases->ctx) != ctx_root(ctx)) { zk_set_error("msm_sharded: bases belong to another context"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    constexpr size_t MAX_POINTS = 4096;       // groups x c of any supported window
    if (!c->d_mine) {
        if (int rc = c->slices.ensure((1 + (size_t)c->world) * MAX_POINTS * sizeof(xyzz_t))) return rc;
        c->d_mine = c->slices.at<xyzz_t>();
        c->d_all = c->d_mine + MAX_POINTS;
        c->cap_points = MAX_POINTS;
    }
    unsigned cc = 0, groups = 0;
    int rc = ctx_msm_partial(ctx, bases, off, n, scalars, scalars_are_mont, window_bits, c->d_mine, c->cap_points, &cc, &groups);
    if (rc) return rc;
    const size_t cnt = (size_t)cc * groups;
    if (c->world == 1) return ctx_msm_finish_gathered(ctx, bases->b.curve, c->d_mine, 1, cc, groups, out_xyz);
    // the collective rides the context's stream behind the kernels: no host synchronisation between the MSM and the exchange
    rc = nccl_check(nccl().AllGather(c->d_mine, c->d_all, cnt * sizeof(xyzz_t), NCCL_UINT8, c->comm, ctx->stream), "ncclAllGather");
    if (rc) return rc;
    return ctx_msm_finish_gathered(ctx, bases->b.curve, c->d_all, (size_t)c->world, cc, groups, out_xyz);
}

}  // extern "C"
