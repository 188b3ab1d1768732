// filtlong_b200/csrc/fl_inflate.cu -- ordinary (non-BGZF) gzip input inflated on the device: the two-stage speculative
// scheme of fl_inflate.h, with these kernels behind its steps:
//   k_inf_find     one CTA of 256 threads per chunk; each thread runs the block-start test at one bit offset, 256
//                  offsets per step from the chunk's nominal start, until a step holds a candidate (the lowest wins);
//   k_inf_decode   one thread per chunk, 32 threads per CTA. The thread's Huffman tables and code lengths
//                  (FlInfTables, 2.9 KB) live in shared memory: 92 KB per CTA, two CTAs per SM. Symbols go to the
//                  chunk's slot in global memory; back-references read the slot back through L1/L2;
//   k_inf_walk     one CTA: in chunk order, the 32 KiB window of every chunk from the resolved end of the one before;
//   k_inf_resolve  one CTA per chunk: markers to window bytes, compacted to the round's output;
//   k_inf_crc      one thread per 16 KiB of output: raw CRC-32 of its piece of every member segment, shifted to the
//                  segment's end (fl_bgzf.h) and XORed into the segment's CRC.
// Every device buffer is allocated by the call and freed before it returns.
#include "fl_internal.cuh"
#include "fl_inflate.h"

namespace {

constexpr int INF_FIND_THREADS = 256;
constexpr int INF_DEC_THREADS = 32;
constexpr uint32_t INF_CRC_SLICE = 16384;

__global__ void __launch_bounds__(INF_FIND_THREADS) k_inf_find(const uint8_t *__restrict__ d, unsigned long long n,
                                                              const unsigned long long *__restrict__ lo,
                                                              const unsigned long long *__restrict__ hi,
                                                              unsigned long long *__restrict__ bit, uint32_t *__restrict__ kind) {
    __shared__ unsigned long long best;
    FlInfTables t;
    const unsigned long long a = lo[blockIdx.x], b = hi[blockIdx.x];
    if (threadIdx.x == 0) best = ~0ull;
    __syncthreads();
    for (unsigned long long base = a; base < b; base += INF_FIND_THREADS) {
        const unsigned long long p = base + threadIdx.x;
        if (p < b) {
            const int k = fl_inf_candidate(d, n, p, &t);
            if (k >= 0) atomicMin(&best, p);
        }
        __syncthreads();
        if (best != ~0ull) break;                                 // every thread reads the same value after the barrier
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        bit[blockIdx.x] = best;
        kind[blockIdx.x] = best == ~0ull ? 0xffffffffu : (uint32_t)fl_inf_candidate(d, n, best, &t);
    }
}

__global__ void __launch_bounds__(INF_DEC_THREADS) k_inf_decode(const uint8_t *__restrict__ d, unsigned long long n,
                                                               FlInfChunk *__restrict__ ch, const uint32_t *__restrict__ idx,
                                                               uint32_t m, uint16_t *__restrict__ slots,
                                                               unsigned long long cap, FlInfEvent *__restrict__ ev) {
    extern __shared__ __align__(16) unsigned char sm[];
    const uint32_t i = blockIdx.x * INF_DEC_THREADS + threadIdx.x;
    if (i >= m) return;
    FlInfTables *t = reinterpret_cast<FlInfTables *>(sm) + threadIdx.x;
    const uint32_t k = idx[i];
    FlInfChunk c = ch[k];
    fl_inf_decode(d, n, &c, slots + (size_t)k * cap, cap, ev + (size_t)k * FL_INF_MAXEV, t);
    ch[k] = c;
}

__global__ void __launch_bounds__(1024) k_inf_walk(const uint16_t *__restrict__ slots, unsigned long long cap,
                                                   const FlInfChunk *__restrict__ ch, uint32_t K, uint8_t *__restrict__ win) {
    for (uint32_t k = 0; k < K; ++k) {
        const uint8_t *w = win + (size_t)k * FL_INF_WINDOW;
        uint8_t *nw = win + (size_t)(k + 1) * FL_INF_WINDOW;
        const uint16_t *s = slots + (size_t)k * cap;
        const long long L = (long long)ch[k].out_len;
        for (uint32_t j = threadIdx.x; j < FL_INF_WINDOW; j += blockDim.x) {
            const long long p = L - (long long)FL_INF_WINDOW + j;
            nw[j] = p >= 0 ? fl_inf_resolve(s[p], w) : w[FL_INF_WINDOW + p];
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_inf_resolve(const uint16_t *__restrict__ slots, unsigned long long cap,
                                                     const FlInfChunk *__restrict__ ch, const uint8_t *__restrict__ win,
                                                     const unsigned long long *__restrict__ off,
                                                     const uint32_t *__restrict__ win_lo, uint8_t *__restrict__ out,
                                                     uint32_t *bad) {
    const uint32_t k = blockIdx.x;
    const uint16_t *s = slots + (size_t)k * cap;
    const uint8_t *w = win + (size_t)k * FL_INF_WINDOW;
    const unsigned long long L = ch[k].out_len, o = off[k];
    const uint32_t lo_ok = win_lo[k];
    bool b = false;
    for (unsigned long long i = threadIdx.x; i < L; i += blockDim.x) {
        const uint16_t v = s[i];
        b |= v >= FL_INF_MARKER && v - FL_INF_MARKER < lo_ok;
        out[o + i] = fl_inf_resolve(v, w);
    }
    if (__syncthreads_or(b) && threadIdx.x == 0) atomicOr(bad, 1u);
}

__global__ void __launch_bounds__(256) k_inf_crc(const uint8_t *__restrict__ out, unsigned long long total,
                                                 const unsigned long long *__restrict__ seg_lo,
                                                 const unsigned long long *__restrict__ seg_hi, uint32_t nseg,
                                                 uint32_t *__restrict__ raw) {
    __shared__ uint32_t tab[256];
    tab[threadIdx.x] = fl_crc32_table_entry(threadIdx.x);
    __syncthreads();
    const unsigned long long a = (unsigned long long)(blockIdx.x * blockDim.x + threadIdx.x) * INF_CRC_SLICE;
    if (a >= total) return;
    const unsigned long long b = a + INF_CRC_SLICE < total ? a + INF_CRC_SLICE : total;
    uint32_t lo = 0, hi = nseg;                                    // the first segment that ends after a
    while (lo < hi) {
        const uint32_t mid = (lo + hi) / 2;
        if (seg_hi[mid] <= a) lo = mid + 1; else hi = mid;
    }
    for (uint32_t s = lo; s < nseg && seg_lo[s] < b; ++s) {
        const unsigned long long p = seg_lo[s] > a ? seg_lo[s] : a, q = seg_hi[s] < b ? seg_hi[s] : b;
        if (p >= q) continue;
        uint32_t c = 0;
        for (unsigned long long i = p; i < q; ++i) c = tab[(c ^ out[i]) & 0xffu] ^ (c >> 8);
        atomicXor(&raw[s], fl_gf2_mulmod(c, fl_crc32_shift(seg_hi[s] - q)));
    }
}

template <typename T>
struct DevArr {
    T *p = nullptr;
    size_t n = 0;
    ~DevArr() { if (p) cudaFree(p); }
    bool get(size_t want) {                                        // false: no memory (the error is cleared)
        if (want <= n) return true;
        if (p) cudaFree(p);
        p = nullptr; n = 0;
        if (cudaMalloc(&p, want * sizeof(T)) != cudaSuccess) { p = nullptr; (void)cudaGetLastError(); return false; }
        n = want;
        return true;
    }
};

struct Gpu {
    fl_ctx *c;
    cudaStream_t s;
    const uint8_t *h_in;              // the input on the host, or
    const uint8_t *d_in = nullptr;    // on the device (fl_gzip_inflate_device): then no copy
    bool dev_out = false;             // fetch() copies into device memory
    const uint8_t *src = nullptr;     // the input the kernels read
    uint64_t n;
    uint64_t cap = 0, R = 0;
    cudaError_t err = cudaSuccess;
    const char *what = "";
    DevArr<uint8_t> in, out, win;
    DevArr<uint16_t> slots;
    DevArr<FlInfChunk> ch;
    DevArr<FlInfEvent> ev;
    DevArr<uint32_t> idx, kind, win_lo, raw, bad;
    DevArr<unsigned long long> lo, hi, bit, off, seg_lo, seg_hi;

    bool ok(cudaError_t e, const char *w) { if (e != cudaSuccess && err == cudaSuccess) { err = e; what = w; } return e == cudaSuccess; }
    template <typename T>
    bool h2d(DevArr<T> &a, const T *src, size_t cnt) {
        if (!a.get(cnt ? cnt : 1)) return ok(cudaErrorMemoryAllocation, "cudaMalloc");
        return !cnt || ok(cudaMemcpyAsync(a.p, src, cnt * sizeof(T), cudaMemcpyHostToDevice, s), "cudaMemcpyAsync");
    }
    template <typename T>
    bool d2h(T *dst, const DevArr<T> &a, size_t cnt) {
        return ok(cudaMemcpyAsync(dst, a.p, cnt * sizeof(T), cudaMemcpyDeviceToHost, s), "cudaMemcpyAsync") &&
               ok(cudaStreamSynchronize(s), "cudaStreamSynchronize");
    }
    uint64_t free_bytes() {
        size_t fr = 0, tot = 0;
        if (cudaMemGetInfo(&fr, &tot) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
        const uint64_t margin = 256ull << 20;                       // for the allocator's own granularity
        return fr > margin ? fr - margin : 0;
    }
    int upload() {                                                 // 0: no device memory for the input (the call declines)
        if (d_in) { src = d_in; return 1; }
        if (!in.get(n + 8)) return 0;
        src = in.p;
        return ok(cudaMemcpyAsync(in.p, h_in, n, cudaMemcpyHostToDevice, s), "cudaMemcpyAsync") ? 1 : -1;
    }
    bool alloc(uint64_t r, uint64_t c_) {                            // false: not enough memory (the call declines)
        if (slots.p && r <= R) return true;
        R = r; cap = c_;
        return slots.get(r * c_) && out.get(r * c_) && win.get((r + 1) * FL_INF_WINDOW) && ch.get(r) &&
               ev.get(r * FL_INF_MAXEV) && idx.get(r) && off.get(r) && win_lo.get(r) && bad.get(1) && lo.get(r) &&
               hi.get(r) && bit.get(r) && kind.get(r) && seg_lo.get(r * FL_INF_MAXEV + 1) && seg_hi.get(r * FL_INF_MAXEV + 1) &&
               raw.get(r * FL_INF_MAXEV + 1) &&
               ok(cudaMemsetAsync(win.p, 0, FL_INF_WINDOW, s), "cudaMemsetAsync");
    }
    bool find(uint32_t m, const uint64_t *l, const uint64_t *h, uint64_t *b, uint32_t *k) {
        if (!h2d(lo, (const unsigned long long *)l, m) || !h2d(hi, (const unsigned long long *)h, m)) return false;
        k_inf_find<<<m, INF_FIND_THREADS, 0, s>>>(src, n, lo.p, hi.p, bit.p, kind.p);
        c->launches += 1;
        if (!ok(cudaGetLastError(), "k_inf_find")) return false;
        return d2h((unsigned long long *)b, bit, m) && d2h(k, kind, m);
    }
    bool decode(FlInfChunk *hch, uint32_t K, const uint32_t *hidx, uint32_t m) {
        if (!h2d(ch, hch, K) || !h2d(idx, hidx, m)) return false;
        const size_t smem = INF_DEC_THREADS * sizeof(FlInfTables);
        k_inf_decode<<<(m + INF_DEC_THREADS - 1) / INF_DEC_THREADS, INF_DEC_THREADS, smem, s>>>(src, n, ch.p, idx.p, m,
                                                                                                 slots.p, cap, ev.p);
        c->launches += 1;
        if (!ok(cudaGetLastError(), "k_inf_decode")) return false;
        return d2h(hch, ch, K);
    }
    bool events(uint32_t K, FlInfEvent *dst) { return d2h(dst, ev, (size_t)K * FL_INF_MAXEV); }
    bool resolve(const FlInfChunk *hch, uint32_t K, const uint64_t *hoff, const uint32_t *hlo, uint64_t total, uint8_t *hbad) {
        (void)total;
        if (!h2d(ch, hch, K) || !h2d(off, (const unsigned long long *)hoff, K) || !h2d(win_lo, hlo, K)) return false;
        if (!ok(cudaMemsetAsync(bad.p, 0, sizeof(uint32_t), s), "cudaMemsetAsync")) return false;
        k_inf_walk<<<1, 1024, 0, s>>>(slots.p, cap, ch.p, K, win.p);
        k_inf_resolve<<<K, 256, 0, s>>>(slots.p, cap, ch.p, win.p, off.p, win_lo.p, out.p, bad.p);
        c->launches += 2;
        if (!ok(cudaGetLastError(), "k_inf_resolve")) return false;
        // the last window starts the next round
        if (!ok(cudaMemcpyAsync(win.p, win.p + (size_t)K * FL_INF_WINDOW, FL_INF_WINDOW, cudaMemcpyDeviceToDevice, s), "cudaMemcpyAsync"))
            return false;
        uint32_t b = 0;
        if (!d2h(&b, bad, 1)) return false;
        *hbad = b != 0;
        return true;
    }
    bool crc(uint32_t m, const uint64_t *l, const uint64_t *h, uint32_t *r) {
        // alloc() sized the segment arrays for the most segments a round can have: no allocation here
        if (!h2d(seg_lo, (const unsigned long long *)l, m) || !h2d(seg_hi, (const unsigned long long *)h, m)) return false;
        if (!ok(cudaMemsetAsync(raw.p, 0, m * sizeof(uint32_t), s), "cudaMemsetAsync")) return false;
        const uint64_t total = h[m - 1];
        const uint64_t slices = (total + INF_CRC_SLICE - 1) / INF_CRC_SLICE;
        if (slices) {
            k_inf_crc<<<(unsigned)((slices + 255) / 256), 256, 0, s>>>(out.p, total, seg_lo.p, seg_hi.p, m, raw.p);
            c->launches += 1;
            if (!ok(cudaGetLastError(), "k_inf_crc")) return false;
        }
        return d2h(r, raw, m);
    }
    bool fetch(uint64_t total, uint8_t *dst) {
        if (!dev_out) return d2h(dst, out, total);
        return ok(cudaMemcpyAsync(dst, out.p, total, cudaMemcpyDeviceToDevice, s), "cudaMemcpyAsync") &&
               ok(cudaStreamSynchronize(s), "cudaStreamSynchronize");
    }
};

// in / outp: host memory (device_io == 0) or memory on the context's device (device_io == 1)
int gunzip_run(fl_ctx *c, const void *in, uint64_t n, void *outp, uint64_t cap, uint64_t chunk_bytes, uint64_t max_device_bytes,
               uint64_t *n_out, int *status, fl_gunzip_stats *st, bool device_io) {
    if ((!in && n) || (!outp && cap) || !n_out || !status) { c->set_error("fl_gzip_inflate: NULL argument"); return FL_EINVAL; }
    *status = FL_GUNZIP_DECLINED;
    *n_out = 0;
    if (!c->inflate_attr_set) {
        FL_CUDA(c, cudaFuncSetAttribute(k_inf_decode, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)(INF_DEC_THREADS * sizeof(FlInfTables))));
        c->inflate_attr_set = true;
    }
    uint8_t head[2] = {0, 0};
    if (n >= 2) {
        if (device_io) FL_CUDA(c, cudaMemcpy(head, in, 2, cudaMemcpyDeviceToHost));
        else { head[0] = static_cast<const uint8_t *>(in)[0]; head[1] = static_cast<const uint8_t *>(in)[1]; }
    }
    FlInfStats fs;
    uint64_t got = 0;
    int rc;
    {
        Gpu be;
        be.c = c; be.s = c->stream; be.n = n;
        be.h_in = device_io ? nullptr : static_cast<const uint8_t *>(in);
        be.d_in = device_io ? static_cast<const uint8_t *>(in) : nullptr;
        be.dev_out = device_io;
        rc = fl_inf_run(be, head, n, static_cast<uint8_t *>(outp), cap, chunk_bytes, max_device_bytes, &got, &fs);
        if (rc < 0 || be.err != cudaSuccess) {
            if (be.err == cudaSuccess) be.err = cudaErrorUnknown;
            c->set_error(std::string("fl_gzip_inflate: ") + be.what + ": " + cudaGetErrorString(be.err));
            (void)cudaStreamSynchronize(c->stream);
            return FL_ECUDA;
        }
        FL_CUDA(c, cudaStreamSynchronize(c->stream));               // nothing in flight when the buffers go
    }
    if (st) { st->members = fs.members; st->chunks = fs.chunks; st->redecoded = fs.redecoded; st->rounds = fs.rounds; }
    if (rc == 1) { *status = FL_GUNZIP_OK; *n_out = got; }
    return FL_OK;
}

}  // namespace

extern "C" int fl_gzip_inflate(fl_ctx *c, const void *host_in, uint64_t n, void *host_out, uint64_t cap, uint64_t chunk_bytes,
                               uint64_t max_device_bytes, uint64_t *n_out, int *status, fl_gunzip_stats *st) {
    FL_ENTER(c);
    return gunzip_run(c, host_in, n, host_out, cap, chunk_bytes, max_device_bytes, n_out, status, st, false);
}

extern "C" int fl_gzip_inflate_device(fl_ctx *c, const void *dev_in, uint64_t n, void *dev_out, uint64_t cap,
                                      uint64_t chunk_bytes, uint64_t max_device_bytes, uint64_t *n_out, int *status,
                                      fl_gunzip_stats *st) {
    FL_ENTER(c);
    return gunzip_run(c, dev_in, n, dev_out, cap, chunk_bytes, max_device_bytes, n_out, status, st, true);
}
