"""`--bgzip`'s kernel on its own: device-resident GB/s of FASTQ text compressed as BGZF, the compression ratio, and zlib
level 1 on the same 65,280-byte blocks (its ratio, and its rate on every host core, core count stated). One JSON line.

    python tools/bgzf_bench.py [--bytes 4e9] [--steps 5] [--warmup 2] [--out result.json]

The text is FASTQ with bench.py's C2 read lengths and qualities (fl_synth_qual_host), bases sliced from a uniform random
genome (fl_synth_genome_host) and ONT-style headers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def fastq_text(total_bytes, seed=11):
    """FASTQ text of about total_bytes (uint8 array)."""
    import bench
    from filtlong_b200 import capi
    S = capi.synth_host_lib()
    n_reads = max(int(total_bytes / 20200), 1)
    w = bench.phred_workload(0, n_reads, total_bytes / 2.02, seed=seed)
    qual = np.zeros(w["padded"] + 64, dtype=np.uint8)
    S.fl_synth_qual_host(w["seed"], w["n"], capi.ptr(w["off"]), capi.ptr(w["len"]), capi.ptr(w["qbar"]), 0, capi.ptr(qual))
    g_bases = 1 << 26
    g2b = np.zeros(g_bases // 16 + 8, dtype=np.uint32)
    S.fl_synth_genome_host(seed, g_bases, capi.ptr(g2b))
    genome = np.zeros(g_bases + 64, dtype=np.uint8)
    one = np.zeros(1, dtype=np.uint64)
    S.fl_synth_ascii_host(1, capi.ptr(one), capi.ptr(np.array([g_bases], dtype=np.int32)), capi.ptr(g2b), None, capi.ptr(genome))
    rng = np.random.default_rng(seed)
    n = w["n"]
    starts = rng.integers(0, g_bases - int(w["len"].max()), size=n)
    cols = [rng.integers(0, 1 << 32, size=n)] + [rng.integers(0, 1 << 16, size=n) for _ in range(3)] + [
        rng.integers(0, 1 << 48, size=n), rng.integers(1, 513, size=n), rng.integers(0, 24, size=n),
        rng.integers(0, 60, size=n), rng.integers(0, 60, size=n)]
    heads = [b"@%08x-%04x-%04x-%04x-%012x runid=8e3c7f42a5b1d9e06f2c4d8a1b3e5f7092c4d6e8 read=%d ch=%d "
             b"start_time=2019-03-14T%02d:%02d:%02dZ\n" % (int(a), int(b), int(c), int(d), int(e), i, int(ch), int(hh), int(mm), int(ss))
             for i, (a, b, c, d, e, ch, hh, mm, ss) in enumerate(zip(*cols))]
    L = w["len"].astype(np.int64)
    hl = np.array([len(h) for h in heads], dtype=np.int64)
    at = np.zeros(n + 1, dtype=np.int64)
    at[1:] = np.cumsum(hl + 2 * L + 4)
    text = np.empty(int(at[-1]), dtype=np.uint8)
    for i in range(n):
        o, Li, h = int(at[i]), int(L[i]), int(hl[i])
        text[o:o + h] = np.frombuffer(heads[i], dtype=np.uint8)
        o += h
        text[o:o + Li] = genome[int(starts[i]):int(starts[i]) + Li]
        text[o + Li:o + Li + 3] = (10, 43, 10)
        q = int(w["off"][i])
        text[o + Li + 3:o + 2 * Li + 3] = qual[q:q + Li]
        text[o + 2 * Li + 3] = 10
    return text


def zlib1_all_cores(text, block=65280):
    """zlib level 1 on the same blocks, one thread per host core: (bytes out incl. BGZF framing, seconds, cores)."""
    import zlib
    from concurrent.futures import ThreadPoolExecutor
    cores = os.cpu_count() or 1
    mv = memoryview(text)
    spans = [(lo, min(lo + (64 << 20), len(text))) for lo in range(0, len(text), 64 << 20)]

    def job(span):
        out = 0
        for lo in range(span[0], span[1], block):
            co = zlib.compressobj(1, zlib.DEFLATED, -15)
            out += len(co.compress(mv[lo:min(lo + block, span[1])])) + len(co.flush()) + 26
        return out
    t0 = time.perf_counter()
    with ThreadPoolExecutor(cores) as ex:
        total = sum(ex.map(job, spans))
    return total + 28, time.perf_counter() - t0, cores


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=float, default=4e9)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    from filtlong_b200 import api
    text = fastq_text(a.bytes)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    with api.Context() as ctx:
        d_in = torch.from_numpy(text).cuda()
        cap = int(ctx.L.fl_bgzf_bound(len(text)))
        d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        n_out = None
        for _ in range(max(a.warmup, 1)):
            n_out = ctx.bgzf_compress_device(d_in, len(text), d_out, cap)
        t0 = time.perf_counter()                     # every call ends in a device synchronise (it reads back the size)
        for _ in range(a.steps):
            assert ctx.bgzf_compress_device(d_in, len(text), d_out, cap) == n_out
        ms = (time.perf_counter() - t0) * 1e3 / a.steps
    z_bytes, z_s, cores = zlib1_all_cores(text)
    res = {"gpu": gpu, "input_bytes": len(text), "ms_per_call": ms, "device_GB_per_s": len(text) / ms / 1e6,
           "ratio": n_out / len(text), "zlib1_ratio": z_bytes / len(text), "zlib1_cpu_GB_per_s": len(text) / z_s / 1e9,
           "zlib1_cpu_cores": cores}
    line = json.dumps(res)
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
