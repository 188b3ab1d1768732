// filtlong_b200/csrc/fl_api.cu -- context management, host packer, batch entry points, result
// download and the deterministic synthetic-workload generators behind the C ABI.
#include <cmath>
#include <cstdlib>

#include "fl_device.cuh"

static std::string g_create_error;
static void drain_timers(fl_ctx *c);

// ---------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------
extern "C" const char *fl_version(void) { return "filtlong-b200 0.1 (Filtlong v0.3.1 semantics, sm_90a)"; }

extern "C" const char *fl_last_error(const fl_ctx *ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

static int validate_params(const fl_params *p, std::string &why) {
    if (!p) { why = "params is NULL"; return FL_EINVAL; }
    if (p->window_size <= 0) { why = "the value for --window_size must be a positive integer"; return FL_EINVAL; }   // arguments.cpp:388-392
    if (p->split_set && p->split <= 0) { why = "the value for --split must be a positive integer"; return FL_EINVAL; }   // arguments.cpp:381-385
    if (p->length_weight < 0.0 || p->mean_q_weight < 0.0 || p->window_q_weight < 0.0) {
        why = "weight values cannot be negative";                                                                      // arguments.cpp:374-378
        return FL_EINVAL;
    }
    if (p->trim_q < 0 || p->trim_q > 93) { why = "the value for --trim_q must be an integer from 1 to 93"; return FL_EINVAL; }
    return FL_OK;     // max_contam is checked where it is used: on a push with a non-empty contaminant set (fl_check_trim_q)
}

extern "C" int fl_device_warmup(int device) {
    if (cudaSetDevice(device) != cudaSuccess) return FL_ENODEV;
    return cudaFree(nullptr) == cudaSuccess ? FL_OK : FL_ENODEV;
}

extern "C" int fl_ctx_create(const fl_params *params, int device, fl_ctx **out) {
    if (!out) return FL_EINVAL;
    *out = nullptr;
    std::string why;
    if (validate_params(params, why) != FL_OK) { g_create_error = why; return FL_EINVAL; }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0 || device < 0 || device >= ndev) {
        g_create_error = std::string("no usable CUDA device (there is no CPU fallback): ") +
                         (e != cudaSuccess ? cudaGetErrorString(e) : "device index out of range");
        return FL_ENODEV;
    }
    if ((e = cudaSetDevice(device)) != cudaSuccess) { g_create_error = cudaGetErrorString(e); return FL_ECUDA; }
    fl_ctx *c = new (std::nothrow) fl_ctx();
    if (!c) return FL_ENOMEM;
    c->device = device;
    c->p = *params;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->sm_count = prop.multiProcessorCount;
    if ((e = cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking)) != cudaSuccess ||
        (e = cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking)) != cudaSuccess ||
        (e = cudaEventCreateWithFlags(&c->ev_copied, cudaEventDisableTiming)) != cudaSuccess ||
        (e = cudaMalloc(&c->d_scalars, 64 * sizeof(unsigned long long))) != cudaSuccess ||
        (e = cudaMemset(c->d_scalars, 0, 64 * sizeof(unsigned long long))) != cudaSuccess ||
        (e = cudaMallocHost(&c->h_scalars, 64 * sizeof(unsigned long long))) != cudaSuccess) {
        g_create_error = cudaGetErrorString(e);
        delete c;
        return FL_ECUDA;
    }
    c->stream = c->own_stream;
    // tuning knobs for profiling runs (DESIGN.md section 4.2)
    if (const char *f = getenv("FL_FILTER")) c->filter_enabled = atoi(f);
    if (const char *f = getenv("FL_ANCHOR")) c->anchor_enabled = atoi(f);
    if (const char *f = getenv("FL_PHRED_MODE")) c->phred_mode = atoi(f);
    if (const char *f = getenv("FL_FASTA_TWO_LINE")) c->fasta_two_line_only = atoi(f) != 0;
    if (const char *f = getenv("FL_PHRED_OCC")) c->phred_occupancy = atoi(f);
    if (const char *f = getenv("FL_FILTER_LOG2_WORDS")) c->filter_log2_words = (unsigned)atoi(f);
    if (const char *f = getenv("FL_FILTER_KIND")) c->filter_kind_request = atoi(f);
    if (const char *f = getenv("FL_FILTER_G4_MAX")) c->filter_group4_max = (uint64_t)atoll(f);
    if (const char *f = getenv("FL_FILTER_PAIR_MAX")) c->filter_pair_max = (uint64_t)atoll(f);
    if (const char *f = getenv("FL_FILTER_MIN_BITS")) c->filter_min_bits_per_key = atoi(f);
    *out = c;
    return FL_OK;
}

extern "C" void fl_ctx_destroy(fl_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    if (c->comm) fl_comm_destroy(c);
    if (c->d_comm) cudaFree(c->d_comm);
    drain_timers(c);
    c->ref.release();
    c->contam.release();
    for (int i = 0; i < 4; ++i) if (c->d_seen[i]) cudaFree(c->d_seen[i]);
    if (c->d_tfirst) cudaFree(c->d_tfirst);
    if (c->d_bittime) cudaFree(c->d_bittime);
    if (c->d_lut) cudaFree(c->d_lut);
    if (c->d_buckets) cudaFree(c->d_buckets);
    if (c->d_scalars) cudaFree(c->d_scalars);
    if (c->h_scalars) cudaFreeHost(c->h_scalars);
    if (c->ev_rows) cudaEventDestroy(c->ev_rows);
    fl_norm_select_free(c);
    for (int i = 0; i < 2; ++i) if (c->stg[i].consumed) cudaEventDestroy(c->stg[i].consumed);
    if (c->ev_copied) cudaEventDestroy(c->ev_copied);
    if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    delete c;
}

extern "C" int fl_ctx_set_stream(fl_ctx *c, void *cuda_stream) {
    FL_ENTER(c);
    FL_CUDA(c, cudaStreamSynchronize(c->stream));
    c->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : c->own_stream;
    return FL_OK;
}

extern "C" int fl_ctx_sync(fl_ctx *c) {
    FL_ENTER(c);
    FL_CUDA(c, cudaStreamSynchronize(c->stream));
    return FL_OK;
}

extern "C" int fl_ctx_set_params(fl_ctx *c, const fl_params *p) {
    FL_ENTER(c);
    std::string why;
    if (validate_params(p, why) != FL_OK) { c->set_error(why); return FL_EINVAL; }
    c->p = *p;
    return FL_OK;
}

extern "C" uint64_t fl_ctx_launch_count(const fl_ctx *c) { return c ? c->launches : 0; }

static void drain_timers(fl_ctx *c) {
    for (auto &t : c->timed) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, t.a, t.b) == cudaSuccess) {
            c->kernel_ms[t.which] += ms;
            c->kernel_launches[t.which]++;
        }
        cudaEventDestroy(t.a);
        cudaEventDestroy(t.b);
    }
    c->timed.clear();
}

extern "C" int fl_ctx_enable_timing(fl_ctx *c, int on) {
    FL_ENTER(c);
    c->timing = on != 0;
    return FL_OK;
}

extern "C" int fl_ctx_reset_timing(fl_ctx *c) {
    FL_ENTER(c);
    FL_CUDA(c, cudaStreamSynchronize(c->stream));
    drain_timers(c);
    for (int i = 0; i < FL_KERNEL_COUNT; ++i) { c->kernel_ms[i] = 0; c->kernel_launches[i] = 0; }
    return FL_OK;
}

extern "C" int fl_ctx_kernel_time(fl_ctx *c, int which, double *total_ms, uint64_t *launches) {
    if (!c || which < 0 || which >= FL_KERNEL_COUNT) return FL_EINVAL;
    FL_ENTER(c);
    FL_CUDA(c, cudaStreamSynchronize(c->stream));
    drain_timers(c);
    if (total_ms) *total_ms = c->kernel_ms[which];
    if (launches) *launches = c->kernel_launches[which];
    return FL_OK;
}

extern "C" int fl_ctx_phred_paths(fl_ctx *c, uint64_t out[9]) {
    if (!c || !out) return FL_EINVAL;
    FL_ENTER(c);
    FL_CUDA(c, cudaStreamSynchronize(c->stream));
    FL_CUDA(c, cudaMemcpy(out, c->d_scalars + FL_SCALAR_PHRED_PATHS, 9 * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    return FL_OK;
}

// ---------------------------------------------------------------------------------------------
// host packer
// ---------------------------------------------------------------------------------------------
extern "C" void fl_anchor_slot_host(uint32_t kmer, uint32_t pos_lo2, uint32_t *word, uint32_t *bit) {
    uint32_t w = 0, b = 0;
    fl_anchor_slot(kmer, 3u - (pos_lo2 & 3u), w, b);
    if (word) *word = w;
    if (bit) *bit = b;
}

extern "C" uint64_t fl_padded_len(int64_t len) {
    if (len <= 0) return 0;
    return ((uint64_t)len + FL_ALIGN_BASES - 1) & ~(uint64_t)(FL_ALIGN_BASES - 1);
}

extern "C" void fl_pack_sequence(const char *seq, const char *qual, int64_t len, uint64_t off, uint32_t *seq2b,
                                 uint8_t *qual_out, uint32_t *nmask) {
    if (qual_out && qual) memcpy(qual_out + off, qual, (size_t)len);
    if (!seq2b && !nmask) return;
    // kmers.cpp:176-196: A/a 0, C/c 1, G/g 2, T/t 3, anything else 0 (and flagged in nmask)
    static const struct Tab {
        uint8_t code[256], other[256];
        Tab() {
            for (int i = 0; i < 256; ++i) { code[i] = 0; other[i] = 1; }
            const char *acgt = "AaCcGgTt";
            for (int i = 0; i < 8; ++i) { code[(unsigned char)acgt[i]] = (uint8_t)(i >> 1); other[(unsigned char)acgt[i]] = 0; }
        }
    } tab;
    const unsigned char *s = reinterpret_cast<const unsigned char *>(seq);
    int64_t i = 0;
    // head up to the next 32-base boundary of the arena, then whole 32-base groups, then the tail
    auto slow = [&](int64_t lo, int64_t hi) {
        for (int64_t k = lo; k < hi; ++k) {
            const uint64_t b = off + (uint64_t)k;
            const uint32_t code = tab.code[s[k]];
            if (seq2b && code) seq2b[b >> 4] |= code << (30 - 2 * (b & 15));
            if (nmask && tab.other[s[k]]) nmask[b >> 5] |= 1u << (b & 31);
        }
    };
    const int64_t head = (int64_t)((32 - (off & 31)) & 31);
    slow(0, head < len ? head : len);
    i = head < len ? head : len;
    for (; i + 32 <= len; i += 32) {
        const uint64_t b = off + (uint64_t)i;
        uint32_t w0 = 0, w1 = 0, m = 0;
        for (int k = 0; k < 16; ++k) {
            w0 = (w0 << 2) | tab.code[s[i + k]];
            w1 = (w1 << 2) | tab.code[s[i + 16 + k]];
            m |= (uint32_t)tab.other[s[i + k]] << k;
            m |= (uint32_t)tab.other[s[i + 16 + k]] << (16 + k);
        }
        if (seq2b) { seq2b[b >> 4] |= w0; seq2b[(b >> 4) + 1] |= w1; }
        if (nmask && m) nmask[b >> 5] |= m;
    }
    slow(i, len);
}

extern "C" void fl_phred_luts(int32_t window_size, double *q256, double *a256) {
    for (int b = 0; b < 256; ++b) {
        int q = (int)(signed char)b - 33;                       // read.cpp:271 (char is signed)
        double v = 1.0 - pow(10.0, -q / 10.0);                  // read.cpp:272, host libm
        if (q256) q256[b] = v;
        if (a256) a256[b] = v / (double)window_size;            // read.cpp:229-230: qualities[i] / window_size
    }
}

// ---------------------------------------------------------------------------------------------
// device-side packer: text -> 2-bit codes (kmers.cpp:176-196: A/a 0, C/c 1, G/g 2, T/t 3, anything else 0)
// and the non-ACGT mask reference sequences need (kmers.cpp:199-219). A pure stream over the arena: one
// thread per 32 bases (two 16-byte loads -> two sequence words + one mask word). Padding bytes produce
// arbitrary codes; no kernel ever forms a 16-mer from bases at or beyond a sequence's length.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_pack_ascii(const uint8_t *__restrict__ ascii, unsigned long long groups,
                                                    uint32_t *__restrict__ seq2b, uint32_t *__restrict__ nmask) {
    const uint4 *in = reinterpret_cast<const uint4 *>(ascii);
    for (unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; g < groups;
         g += (unsigned long long)gridDim.x * blockDim.x) {
        const uint4 a = __ldg(in + 2 * g), b = __ldg(in + 2 * g + 1);
        const uint32_t c[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        uint32_t w[2] = {0u, 0u}, m = 0u;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            uint32_t code8, other4;
            fl_pack4(c[i], code8, other4);
            w[i >> 2] |= code8 << (24 - 8 * (i & 3));
            m |= other4 << (4 * i);
        }
        reinterpret_cast<uint2 *>(seq2b)[g] = make_uint2(w[0], w[1]);
        if (nmask) nmask[g] = m;
    }
}

int fl_pack_ascii_device(fl_ctx *c, const uint8_t *ascii, uint64_t padded_bases, uint32_t *seq2b, uint32_t *nmask, cudaStream_t s) {
    const unsigned long long groups = padded_bases >> 5;
    if (!groups) return FL_OK;
    unsigned blocks = fl_blocks(groups, 256);
    if (blocks > (unsigned)c->sm_count * 16) blocks = (unsigned)c->sm_count * 16;
    k_pack_ascii<<<blocks, 256, 0, s>>>(ascii, groups, seq2b, nmask);
    c->launches++;
    FL_CUDA(c, cudaGetLastError());
    return FL_OK;
}

// ---------------------------------------------------------------------------------------------
// batches
// ---------------------------------------------------------------------------------------------
static int check_batch(fl_ctx *c, const fl_batch *b) {
    if (!b) { c->set_error("batch is NULL"); return FL_EINVAL; }
    if (b->n && (!b->off || !b->len)) { c->set_error("batch.off / batch.len missing"); return FL_EINVAL; }
    if (b->padded_bases % FL_ALIGN_BASES) { c->set_error("batch.padded_bases must be a multiple of 64"); return FL_EINVAL; }
    return FL_OK;
}

static int stage_host_batch(fl_ctx *c, const fl_batch *h, BatchView *v, bool want_seq, bool want_qual, bool want_nmask,
                            int slot, cudaStream_t s) {
    fl_ctx::Staging &S = c->stg[slot];
    const size_t n = h->n;
    FL_CUDA(c, S.off.reserve(n, 0, s));
    FL_CUDA(c, S.len.reserve(n, 0, s));
    FL_CUDA(c, cudaMemcpyAsync(S.off.p, h->off, n * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    FL_CUDA(c, cudaMemcpyAsync(S.len.p, h->len, n * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    v->n = h->n;
    v->padded_bases = h->padded_bases;
    v->off = S.off.p;
    v->len = S.len.p;
    v->seq2b = nullptr; v->qual = nullptr; v->nmask = nullptr; v->ascii = nullptr;
    if (want_seq && h->seq2b) {
        size_t words = (size_t)(h->padded_bases >> 4);
        FL_CUDA(c, S.seq.reserve(words + 4, 0, s));
        FL_CUDA(c, cudaMemcpyAsync(S.seq.p, h->seq2b, words * 4, cudaMemcpyHostToDevice, s));
        v->seq2b = S.seq.p;
    } else if (want_seq && h->ascii) {
        // text hand-off (read.h:32 / kmers.cpp:96-121): copy the bytes, pack on the device
        size_t words = (size_t)(h->padded_bases >> 4);
        FL_CUDA(c, S.ascii.reserve((size_t)h->padded_bases + 64, 0, s));
        FL_CUDA(c, S.seq.reserve(words + 4, 0, s));
        if (want_nmask) FL_CUDA(c, S.nmask.reserve((words >> 1) + 4, 0, s));
        FL_CUDA(c, cudaMemcpyAsync(S.ascii.p, h->ascii, (size_t)h->padded_bases, cudaMemcpyHostToDevice, s));
        v->ascii = S.ascii.p;            // packed by the caller on the COMPUTE stream (stage_pack): the copy stream only copies
    }
    if (want_qual && h->qual) {
        FL_CUDA(c, S.qual.reserve((size_t)h->padded_bases + 64, 0, s));
        FL_CUDA(c, cudaMemcpyAsync(S.qual.p, h->qual, (size_t)h->padded_bases, cudaMemcpyHostToDevice, s));
        v->qual = S.qual.p;
    }
    if (want_nmask && h->nmask && h->seq2b) {
        size_t words = (size_t)(h->padded_bases >> 5);
        FL_CUDA(c, S.nmask.reserve(words + 4, 0, s));
        FL_CUDA(c, cudaMemcpyAsync(S.nmask.p, h->nmask, words * 4, cudaMemcpyHostToDevice, s));
        v->nmask = S.nmask.p;
    }
    return FL_OK;
}

// second half of a text hand-off: 2-bit codes (+ non-ACGT mask) from the staged characters, on the compute stream
static int stage_pack(fl_ctx *c, BatchView *v, bool want_nmask, int slot) {
    if (v->seq2b || !v->ascii) return FL_OK;
    fl_ctx::Staging &S = c->stg[slot];
    FL_TRY(fl_pack_ascii_device(c, v->ascii, v->padded_bases, S.seq.p, want_nmask ? S.nmask.p : nullptr, c->stream));
    v->seq2b = S.seq.p;
    if (want_nmask) v->nmask = S.nmask.p;
    return FL_OK;
}

// waits until no kernel still reads staging slot `slot`
static int staging_acquire(fl_ctx *c, int slot) {
    fl_ctx::Staging &S = c->stg[slot];
    if (!S.consumed) FL_CUDA(c, cudaEventCreateWithFlags(&S.consumed, cudaEventDisableTiming));
    if (S.in_use) FL_CUDA(c, cudaEventSynchronize(S.consumed));
    S.in_use = false;
    return FL_OK;
}

static int view_of_device_batch(fl_ctx *c, const fl_batch *b, bool want_nmask, BatchView *out) {
    BatchView v{};
    v.n = b->n; v.padded_bases = b->padded_bases; v.off = b->off; v.len = b->len;
    v.seq2b = b->seq2b; v.qual = b->qual; v.nmask = b->nmask;
    if (!b->seq2b && b->ascii && b->padded_bases) {            // device-resident text: pack into scratch
        const size_t words = (size_t)(b->padded_bases >> 4);
        FL_CUDA(c, c->sc_pack_seq.reserve(words + 4, 0, c->stream));
        if (want_nmask) FL_CUDA(c, c->sc_pack_nmask.reserve((words >> 1) + 4, 0, c->stream));
        FL_TRY(fl_pack_ascii_device(c, reinterpret_cast<const uint8_t *>(b->ascii), b->padded_bases, c->sc_pack_seq.p,
                                    want_nmask ? c->sc_pack_nmask.p : nullptr, c->stream));
        v.seq2b = c->sc_pack_seq.p;
        v.nmask = want_nmask ? c->sc_pack_nmask.p : nullptr;
    }
    *out = v;
    return FL_OK;
}

static int add_host_batch(fl_ctx *c, KmerSet &set, const fl_batch *h, int multi) {
    FL_TRY(check_batch(c, h));
    if (h->n == 0) return FL_OK;
    BatchView v{};
    FL_TRY(staging_acquire(c, 0));
    FL_TRY(stage_host_batch(c, h, &v, true, false, true, 0, c->stream));
    FL_TRY(stage_pack(c, &v, true, 0));
    FL_TRY(fl_kmers_add_view(c, set, v, multi));
    FL_CUDA(c, cudaStreamSynchronize(c->stream));   // staging buffers are reused by the next call
    return FL_OK;
}

extern "C" int fl_kmers_add_batch(fl_ctx *c, const fl_batch *h, int multi) {
    FL_ENTER(c);
    return add_host_batch(c, c->ref, h, multi);
}

extern "C" int fl_contam_add_batch(fl_ctx *c, const fl_batch *h) {
    FL_ENTER(c);
    FL_TRY(fl_contam_check_order(c));
    return add_host_batch(c, c->contam, h, 0);
}

extern "C" int fl_kmers_add_batch_device(fl_ctx *c, const fl_batch *d, int multi) {
    FL_ENTER(c);
    FL_TRY(check_batch(c, d));
    BatchView v{};
    FL_TRY(view_of_device_batch(c, d, true, &v));
    return fl_kmers_add_view(c, c->ref, v, multi);
}

__global__ void k_sum_len(const int32_t *len, uint32_t n, unsigned long long *out) {
    unsigned long long s = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) s += (unsigned long long)len[i];
#pragma unroll
    for (int d = 16; d; d >>= 1) s += __shfl_down_sync(0xffffffffu, s, d);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(out, s);
}

#define FL_SCALAR_TOTAL_BASES 16   // slot in d_scalars accumulating the lengths of device batches

extern "C" int fl_reads_push(fl_ctx *c, const fl_batch *h) {
    FL_ENTER_NOFLUSH(c);
    FL_TRY(check_batch(c, h));
    if (h->n == 0) return fl_score_complete(c);
    FL_TRY(fl_sets_ready(c));
    FL_TRY(fl_check_trim_q(c));                                  // before anything is staged
    const bool kmer_mode = c->ref.n > 0;
    BatchView v{};
    // double-buffered staging: this batch's host->device copies run on the copy stream while the
    // kernels of the previous batch are still busy on the compute stream
    const int slot = c->stg_next;
    c->stg_next ^= 1;
    FL_TRY(staging_acquire(c, slot));
    FL_TRY(stage_host_batch(c, h, &v, fl_wants_bases(c), !kmer_mode, false, slot, c->copy_stream));
    FL_CUDA(c, cudaEventRecord(c->ev_copied, c->copy_stream));
    // With --trim / --split the previous batch still owes its second half, which starts with a host round trip (its row
    // count). Paying it HERE, with this batch's copy already under way, keeps the copy engine busy during that batch's probe.
    FL_TRY(fl_score_complete(c));
    FL_CUDA(c, cudaStreamWaitEvent(c->stream, c->ev_copied, 0));
    FL_TRY(stage_pack(c, &v, false, slot));
    FL_TRY(fl_score_view(c, v, /*defer=*/true));
    if (c->kmer_pending) c->kmer_pending_slot = slot;            // fl_score_complete releases the slot
    else {
        FL_CUDA(c, cudaEventRecord(c->stg[slot].consumed, c->stream));
        c->stg[slot].in_use = true;
    }
    for (uint32_t i = 0; i < h->n; ++i) c->total_bases += h->len[i];     // main.cpp:89
    FL_CUDA(c, cudaStreamSynchronize(c->copy_stream));   // the caller may reuse its host buffers now
    return FL_OK;
}

extern "C" int fl_reads_push_device(fl_ctx *c, const fl_batch *d) {
    FL_ENTER(c);
    FL_TRY(check_batch(c, d));
    if (d->n == 0) return FL_OK;
    FL_TRY(fl_sets_ready(c));
    BatchView v{};
    {
        fl_batch d2 = *d;
        if (!fl_wants_bases(c)) d2.ascii = nullptr;              // Phred mode never reads the bases (read.cpp:35-39)
        FL_TRY(view_of_device_batch(c, &d2, false, &v));
    }
    FL_TRY(fl_score_view(c, v));
    k_sum_len<<<c->sm_count, 256, 0, c->stream>>>(d->len, d->n, c->d_scalars + FL_SCALAR_TOTAL_BASES);
    c->launches++;
    FL_CUDA(c, cudaGetLastError());
    return FL_OK;
}

extern "C" int fl_reads_reset(fl_ctx *c) {
    FL_ENTER(c);
    FL_CUDA(c, cudaMemsetAsync(c->d_scalars + FL_SCALAR_TOTAL_BASES, 0, sizeof(unsigned long long), c->stream));
    c->n_reads = 0;
    c->n_rows = 0;
    c->total_bases = 0;
    c->finalized = false;
    return FL_OK;
}

static int device_total_bases(fl_ctx *c, int64_t *out) {
    FL_CUDA(c, cudaMemcpyAsync(c->h_scalars + 32, c->d_scalars + FL_SCALAR_TOTAL_BASES, sizeof(unsigned long long),
                               cudaMemcpyDeviceToHost, c->stream));
    FL_CUDA(c, cudaStreamSynchronize(c->stream));
    *out = c->total_bases + (int64_t)c->h_scalars[32];
    return FL_OK;
}

extern "C" int fl_reads_count(fl_ctx *c, uint64_t *n_reads, uint64_t *n_rows, int64_t *total_bases) {
    FL_ENTER(c);
    if (n_reads) *n_reads = c->n_reads;
    if (n_rows) *n_rows = c->n_rows;
    if (total_bases) FL_TRY(device_total_bases(c, total_bases));
    return FL_OK;
}

// ---------------------------------------------------------------------------------------------
// results
// ---------------------------------------------------------------------------------------------
template <typename T>
static int dl(fl_ctx *c, T *host, const T *dev, size_t n) {
    if (!host || !n) return FL_OK;
    FL_CUDA(c, cudaMemcpyAsync(host, dev, n * sizeof(T), cudaMemcpyDeviceToHost, c->stream));
    return FL_OK;
}

static double host_length_score(int length) {              // read.cpp:241-244
    double half = 5000.0;
    return 100.0 * (1.0 + (-half / (length + half)));
}

extern "C" int fl_results_reads(fl_ctx *c, const fl_read_results *o) {
    if (!c || !o) return FL_EINVAL;
    FL_ENTER(c);
    const size_t n = c->n_reads;
    std::vector<int32_t> len_tmp;
    int32_t *len_host = o->length;
    if (o->length_score && !len_host) { len_tmp.resize(n); len_host = len_tmp.data(); }
    FL_TRY(dl(c, len_host, c->r_len.p, n));
    FL_TRY(dl(c, o->mean_q, c->r_mean.p, n));
    FL_TRY(dl(c, o->window_q, c->r_window.p, n));
    FL_TRY(dl(c, o->passed, c->r_passed.p, n));
    FL_TRY(dl(c, o->first_base_in_kmer, c->r_first.p, n));
    FL_TRY(dl(c, o->last_base_in_kmer, c->r_last.p, n));
    FL_TRY(dl(c, o->n_bad, c->r_nbad.p, n));
    FL_TRY(dl(c, o->n_child, c->r_nchild.p, n));
    FL_TRY(dl(c, reinterpret_cast<unsigned long long *>(o->row_start), c->r_rowstart.p, n));
    FL_CUDA(c, cudaStreamSynchronize(c->stream));
    if (o->length_score)
        for (size_t i = 0; i < n; ++i) o->length_score[i] = host_length_score(len_host[i]);
    return FL_OK;
}

extern "C" int fl_results_rows(fl_ctx *c, const fl_row_results *o) {
    if (!c || !o) return FL_EINVAL;
    FL_ENTER(c);
    const size_t n = c->n_rows;
    std::vector<int32_t> s_tmp, e_tmp;
    int32_t *s_host = o->start, *e_host = o->end;
    if (o->length_score) {
        if (!s_host) { s_tmp.resize(n); s_host = s_tmp.data(); }
        if (!e_host) { e_tmp.resize(n); e_host = e_tmp.data(); }
    }
    FL_TRY(dl(c, o->parent, c->w_parent.p, n));
    FL_TRY(dl(c, s_host, c->w_start.p, n));
    FL_TRY(dl(c, e_host, c->w_end.p, n));
    FL_TRY(dl(c, o->mean_q, c->w_mean.p, n));
    FL_TRY(dl(c, o->window_q, c->w_window.p, n));
    FL_TRY(dl(c, o->passed, c->w_passed.p, n));
    if (c->finalized) {
        FL_TRY(dl(c, o->norm_mean, c->w_nmean.p, n));
        FL_TRY(dl(c, o->norm_window, c->w_nwindow.p, n));
        FL_TRY(dl(c, o->final_score, c->w_final.p, n));
        FL_TRY(dl(c, o->passed_final, c->w_pfinal.p, n));
    } else {
        FL_TRY(dl(c, o->passed_final, c->w_passed.p, n));
        if (o->norm_mean) memset(o->norm_mean, 0, n * sizeof(double));
        if (o->norm_window) memset(o->norm_window, 0, n * sizeof(double));
        if (o->final_score) memset(o->final_score, 0, n * sizeof(double));
    }
    FL_CUDA(c, cudaStreamSynchronize(c->stream));
    if (o->length_score)
        for (size_t i = 0; i < n; ++i) o->length_score[i] = host_length_score(e_host[i] - s_host[i]);
    return FL_OK;
}

__global__ void k_contam_count(const uint8_t *__restrict__ removed, const int32_t *__restrict__ len, size_t n_reads,
                               const uint8_t *__restrict__ excl, size_t n_rows, unsigned long long *__restrict__ out) {
    unsigned long long reads = 0, bases = 0, rows = 0;
    const size_t n = n_reads > n_rows ? n_reads : n_rows;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        if (i < n_reads && removed[i]) { ++reads; bases += (unsigned long long)len[i]; }
        if (i < n_rows && excl[i]) ++rows;
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) {
        reads += __shfl_down_sync(0xffffffffu, reads, d);
        bases += __shfl_down_sync(0xffffffffu, bases, d);
        rows += __shfl_down_sync(0xffffffffu, rows, d);
    }
    if ((threadIdx.x & 31) == 0) {
        if (reads) atomicAdd(out, reads);
        if (bases) atomicAdd(out + 1, bases);
        if (rows) atomicAdd(out + 2, rows);
    }
}

extern "C" int fl_results_contam(fl_ctx *c, double *percent, uint8_t *removed, fl_contam_counts *counts) {
    if (!c) return FL_EINVAL;
    FL_ENTER(c);
    const size_t n = c->n_reads;
    if (counts) *counts = fl_contam_counts{};
    if (c->contam.n == 0) {
        if (percent) for (size_t i = 0; i < n; ++i) percent[i] = 0.0;
        if (removed) memset(removed, 0, n);
        return FL_OK;
    }
    FL_TRY(dl(c, percent, c->r_contam.p, n));
    FL_TRY(dl(c, removed, c->r_removed.p, n));
    if (counts && (n || c->n_rows)) {
        unsigned long long *d = c->d_scalars + FL_SCALAR_CONTAM;
        FL_CUDA(c, cudaMemsetAsync(d, 0, 3 * sizeof(unsigned long long), c->stream));
        unsigned blocks = fl_blocks(n > c->n_rows ? n : c->n_rows, 256);
        if (blocks > (unsigned)c->sm_count * 8) blocks = (unsigned)c->sm_count * 8;
        k_contam_count<<<blocks, 256, 0, c->stream>>>(c->r_removed.p, c->r_len.p, n, c->w_excl.p, c->n_rows, d);
        c->launches++;
        FL_CUDA(c, cudaGetLastError());
        FL_CUDA(c, cudaMemcpyAsync(c->h_scalars + FL_SCALAR_CONTAM, d, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
    }
    FL_CUDA(c, cudaStreamSynchronize(c->stream));
    if (counts && (n || c->n_rows)) {
        counts->reads = c->h_scalars[FL_SCALAR_CONTAM];
        counts->bases = (int64_t)c->h_scalars[FL_SCALAR_CONTAM + 1];
        counts->rows = c->h_scalars[FL_SCALAR_CONTAM + 2];
    }
    return FL_OK;
}

extern "C" int fl_results_pass_dev(fl_ctx *c, void **dev_passed_final, uint64_t *n_rows) {
    if (!c || !dev_passed_final) return FL_EINVAL;
    FL_ENTER(c);
    *dev_passed_final = c->finalized ? (void *)c->w_pfinal.p : (void *)c->w_passed.p;
    if (n_rows) *n_rows = c->n_rows;
    return FL_OK;
}

extern "C" int fl_results_pass(fl_ctx *c, uint8_t *host_out, uint64_t cap, uint64_t *n_rows) {
    if (!c || (!host_out && cap)) return FL_EINVAL;
    FL_ENTER(c);
    if (n_rows) *n_rows = c->n_rows;
    size_t n = c->n_rows < cap ? c->n_rows : cap;
    if (n) FL_CUDA(c, cudaMemcpyAsync(host_out, c->finalized ? c->w_pfinal.p : c->w_passed.p, n, cudaMemcpyDeviceToHost, c->stream));
    FL_CUDA(c, cudaStreamSynchronize(c->stream));
    return FL_OK;
}

