// filtlong_b200/csrc/fl_comm.cu -- the read set sharded across GPUs (SURVEY 8e): one context per GPU, one
// NCCL communicator behind the C ABI. The reference has nothing to shard with (single thread); what crosses
// ranks here is exactly the coupling of main.cpp:169-261 -- global statistics, the base-weighted score
// histogram, the tie class at the cut-off -- plus one broadcast of the finished 16-mer bitmap.
//
// NCCL is bound at run time (dlopen of libnccl.so.2: the copy a host process already loaded, e.g. torch's,
// else the system one), so the single-GPU library and CLI have no link-time dependency on it.
#include <dlfcn.h>
#include <nccl.h>

#include <mutex>

#include "fl_internal.cuh"

namespace {

struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Broadcast)(const void *, void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    std::string why;
};

NcclApi g_nccl;
std::once_flag g_nccl_once;

template <typename F>
bool bind(void *h, const char *name, F &fn) {
    fn = reinterpret_cast<F>(dlsym(h, name));
    return fn != nullptr;
}

const NcclApi &nccl() {
    std::call_once(g_nccl_once, [] {
        const char *names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char *n : names) {
            g_nccl.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (g_nccl.handle) break;
        }
        if (!g_nccl.handle) { g_nccl.why = std::string("libnccl.so.2 not found: ") + dlerror(); return; }
        void *h = g_nccl.handle;
        if (!(bind(h, "ncclGetUniqueId", g_nccl.GetUniqueId) && bind(h, "ncclCommInitRank", g_nccl.CommInitRank) &&
              bind(h, "ncclCommDestroy", g_nccl.CommDestroy) && bind(h, "ncclAllReduce", g_nccl.AllReduce) &&
              bind(h, "ncclAllGather", g_nccl.AllGather) && bind(h, "ncclBroadcast", g_nccl.Broadcast) &&
              bind(h, "ncclGetErrorString", g_nccl.GetErrorString))) {
            g_nccl.why = "libnccl.so.2 lacks a required symbol";
            g_nccl.handle = nullptr;
        }
    });
    return g_nccl;
}

#define FL_NCCL(ctx, call)                                                                        \
    do {                                                                                          \
        ncclResult_t r__ = (call);                                                                \
        if (r__ != ncclSuccess) {                                                                 \
            (ctx)->set_error(std::string(#call) + ": " + nccl().GetErrorString(r__));            \
            return FL_ECUDA;                                                                      \
        }                                                                                         \
    } while (0)

}  // namespace

extern "C" int fl_comm_unique_id(void *out128) {
    if (!out128) return FL_EINVAL;
    const NcclApi &n = nccl();
    if (!n.handle) return FL_ENODEV;
    ncclUniqueId id;
    if (n.GetUniqueId(&id) != ncclSuccess) return FL_ECUDA;
    memcpy(out128, id.internal, FL_COMM_ID_BYTES);
    return FL_OK;
}

extern "C" int fl_comm_init(fl_ctx *ctx, const void *id128, int rank, int nranks) {
    FL_ENTER(ctx);
    if (!id128 || nranks < 1 || rank < 0 || rank >= nranks) { ctx->set_error("fl_comm_init: bad rank / nranks / id"); return FL_EINVAL; }
    if (ctx->comm) { ctx->set_error("fl_comm_init: the context already has a communicator"); return FL_EINVAL; }
    const NcclApi &n = nccl();
    if (!n.handle) { ctx->set_error(n.why); return FL_ENODEV; }
    ncclUniqueId id;
    memcpy(id.internal, id128, FL_COMM_ID_BYTES);
    ncclComm_t comm = nullptr;
    FL_NCCL(ctx, n.CommInitRank(&comm, nranks, id, rank));
    ctx->comm = comm;
    ctx->comm_rank = rank;
    ctx->comm_nranks = nranks;
    if (!ctx->d_comm) FL_CUDA(ctx, cudaMalloc(&ctx->d_comm, FL_COMM_SCRATCH_BYTES));
    return FL_OK;
}

extern "C" int fl_comm_destroy(fl_ctx *ctx) {
    FL_ENTER(ctx);
    if (ctx->comm) {
        cudaStreamSynchronize(ctx->stream);
        nccl().CommDestroy(static_cast<ncclComm_t>(ctx->comm));
    }
    ctx->comm = nullptr;
    ctx->comm_rank = 0;
    ctx->comm_nranks = 1;
    return FL_OK;
}

extern "C" int fl_comm_info(const fl_ctx *ctx, int *rank, int *nranks) {
    if (!ctx) return FL_EINVAL;
    if (rank) *rank = ctx->comm_rank;
    if (nranks) *nranks = ctx->comm_nranks;
    return FL_OK;
}

// ---- stream-ordered collectives on device buffers, used by fl_select.cu / fl_kmers.cu ----
int fl_comm_allgather(fl_ctx *ctx, const void *send, void *recv, size_t bytes_per_rank) {
    if (!ctx->comm) {
        if (send != recv) FL_CUDA(ctx, cudaMemcpyAsync(recv, send, bytes_per_rank, cudaMemcpyDeviceToDevice, ctx->stream));
        return FL_OK;
    }
    FL_NCCL(ctx, nccl().AllGather(send, recv, bytes_per_rank, ncclUint8, static_cast<ncclComm_t>(ctx->comm), ctx->stream));
    ctx->collectives++;
    return FL_OK;
}

int fl_comm_allreduce_u64(fl_ctx *ctx, unsigned long long *buf, size_t n) {
    if (!ctx->comm) return FL_OK;
    FL_NCCL(ctx, nccl().AllReduce(buf, buf, n, ncclUint64, ncclSum, static_cast<ncclComm_t>(ctx->comm), ctx->stream));
    ctx->collectives++;
    return FL_OK;
}

int fl_comm_broadcast_bytes(fl_ctx *ctx, void *buf, size_t bytes, int root) {
    if (!ctx->comm) return FL_OK;
    FL_NCCL(ctx, nccl().Broadcast(buf, buf, bytes, ncclUint8, root, static_cast<ncclComm_t>(ctx->comm), ctx->stream));
    ctx->collectives++;
    return FL_OK;
}

extern "C" int fl_comm_allreduce_i64_host(fl_ctx *ctx, int64_t *inout, int n) {
    FL_ENTER(ctx);
    if (!inout || n < 0 || (size_t)n * 8 > 256) return FL_EINVAL;
    if (!ctx->comm || n == 0) return FL_OK;
    unsigned long long *d = ctx->d_scalars + 40;               // 24 spare slots of the context's scalar block
    if (n > 24) return FL_ERANGE;
    FL_CUDA(ctx, cudaMemcpyAsync(d, inout, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    FL_TRY(fl_comm_allreduce_u64(ctx, d, (size_t)n));          // two's complement: signed sums come out right
    FL_CUDA(ctx, cudaMemcpyAsync(inout, d, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return FL_OK;
}

// A set replicated across the shards: the finished direct-address bitmap (512 MiB) goes from `root` to every other rank
// over NVLink; each rank then derives its own probe tables from it (fl_kmers_recount).
static int broadcast_set(fl_ctx *ctx, KmerSet &s, int root, const char *entry) {
    if (root < 0 || root >= ctx->comm_nranks) { ctx->set_error(std::string(entry) + ": bad root"); return FL_EINVAL; }
    if (s.k > 16) return fl_ck_broadcast(ctx, s, root);     // every rank configured the same k and size (fl_contam_configure)
    if (ctx->comm_rank == root && (s.stale || (&s == &ctx->ref && ctx->multi_pending))) FL_TRY(fl_kmers_recount(ctx, s));
    FL_TRY(fl_kmers_ensure_bitmap(ctx, s));
    if (!ctx->comm) return FL_OK;
    FL_NCCL(ctx, nccl().Broadcast(s.bitmap, s.bitmap, (size_t)1 << 29, ncclUint8, root, static_cast<ncclComm_t>(ctx->comm),
                                  ctx->stream));
    ctx->collectives++;
    if (ctx->comm_rank != root) s.stale = true;
    return FL_OK;
}

extern "C" int fl_kmers_broadcast(fl_ctx *ctx, int root) {
    FL_ENTER(ctx);
    return broadcast_set(ctx, ctx->ref, root, "fl_kmers_broadcast");
}

// A contaminant set of k > 16 goes as its table's bytes, so every rank must hold one of the same k and size. Two small
// collectives (the root's k and bucket count out, then the sum of the ranks' disagreements) let every rank see a mismatch
// and return FL_EINVAL together, instead of issuing broadcasts of different sizes.
static int check_same_contam(fl_ctx *ctx, int root) {
    if (!ctx->comm) return FL_OK;
    if (root < 0 || root >= ctx->comm_nranks) { ctx->set_error("fl_contam_broadcast: bad root"); return FL_EINVAL; }
    const KmerSet &s = ctx->contam;
    unsigned long long *d = ctx->d_scalars + 48, *h = ctx->h_scalars + 48;
    h[0] = (unsigned long long)s.k;
    h[1] = s.n_buckets;
    FL_CUDA(ctx, cudaMemcpyAsync(d, h, 2 * sizeof(unsigned long long), cudaMemcpyHostToDevice, ctx->stream));
    FL_TRY(fl_comm_broadcast_bytes(ctx, d, 2 * sizeof(unsigned long long), root));
    FL_CUDA(ctx, cudaMemcpyAsync(h + 2, d, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    h[4] = (h[2] != (unsigned long long)s.k || h[3] != s.n_buckets) ? 1ull : 0ull;
    FL_CUDA(ctx, cudaMemcpyAsync(d + 4, h + 4, sizeof(unsigned long long), cudaMemcpyHostToDevice, ctx->stream));
    FL_TRY(fl_comm_allreduce_u64(ctx, d + 4, 1));
    FL_CUDA(ctx, cudaMemcpyAsync(h + 5, d + 4, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (h[5]) {
        ctx->set_error("fl_contam_broadcast: the ranks' contaminant sets differ in k or table size (fl_contam_configure every "
                       "rank with the same k and max_kmers)");
        return FL_EINVAL;
    }
    return FL_OK;
}

extern "C" int fl_contam_broadcast(fl_ctx *ctx, int root) {
    FL_ENTER(ctx);
    FL_TRY(check_same_contam(ctx, root));
    return broadcast_set(ctx, ctx->contam, root, "fl_contam_broadcast");
}

extern "C" uint64_t fl_comm_collective_count(const fl_ctx *ctx) { return ctx ? ctx->collectives : 0; }
