"""How the quality bytes reach k_phred_sum and k_phred_win, on config 2's workload (bench.phred_workload, default 2 M
reads / 20 Gbp) and on the same bases cut into reads of 10,000.

Part 1, the library's kernels: ms per step and GB/s of arena bytes of k_phred_sum and k_phred_win with FL_PHRED_OCC =
1..4 blocks per SM (one context per setting, device times from torch.profiler). A time that falls as 1 / occupancy is a
kernel waiting for its loads.

Part 2, load-only probes (tools/phred_loads.cu, compiled here with the library's nvcc flags into a temporary directory,
never linked into the library): the same claim loop, addresses and shared-memory footprint as each kernel, the per-base
work replaced by an XOR. Variants: loads one step ahead in registers; a per-warp shared-memory ring of 2, 4 or 8 tiles
filled by cp.async.bulk or by per-lane cp.async; for k_phred_sum's walk alone, the per-lane slots the kernel uses (2, 3
or 4 steps ahead, a cold start per read); reads taken longest first or in arena order; the next read claimed
and prefetched while this one is walked, or not. Then the chunked walks, with the shared-memory footprint of a
one-pass kernel that would hold both chains' tables (72 KiB, three blocks per SM): each read cut into chunks of 2, 4 or
8 KiB, lane 0 asking L2 for the chunk D = 1 or 2 ahead with cp.async.bulk.prefetch.L2 (D = 0: no prefetch), the loads
one step ahead in registers; k_phred_sum's walk, k_phred_win's walk, and one pass doing both per chunk (the sum's
512-byte steps that start in the chunk, then the window steps that end in it). Times are CUDA events over --launches
launches.

    python tools/phred_loads.py [--scale 1.0] [--steps 3] [--launches 5] [--skip-library] [--skip-probes]

Prints the card name and power limit beside the numbers."""
import argparse
import ctypes
import os
import subprocess
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import bench  # noqa: E402


def workloads(scale):
    n_reads, total = max(int(round(2e6 * scale)), 64), int(round(20e9 * scale))
    w = bench.phred_workload(0, n_reads, total)
    n_fixed = max(total // 10000, 1)
    lengths = np.full(n_fixed, 10000, dtype=np.int32)
    off, padded = bench.layout(lengths)
    fixed = dict(w, n=n_fixed, len=lengths, off=off, padded=padded, bases=int(lengths.sum()),
                 qbar=np.full(n_fixed, 14, dtype=np.uint8))
    return [("C2 lognormal", w), ("every read 10,000", fixed)]


def device_arena(torch, dev, ctx, w):
    from filtlong_b200 import capi
    L = capi.lib()
    t_len = torch.from_numpy(w["len"]).to(dev)
    t_off = torch.from_numpy(w["off"].view(np.int64)).to(dev)
    d_qual = torch.empty(w["padded"] + 64, dtype=torch.uint8, device=dev)
    capi.check(ctx.h, L.fl_synth_qual_device(ctx.h, w["seed"], w["n"], t_off.data_ptr(), t_len.data_ptr(),
                                             torch.from_numpy(w["qbar"]).to(dev).data_ptr(), w["read_base"], d_qual.data_ptr()), "synth_qual")
    return t_len, t_off, d_qual


def library_part(torch, dev, stream, args):
    from torch.profiler import ProfilerActivity, profile

    from filtlong_b200 import api
    print("library kernels, ms per step (GB/s of arena bytes):")
    print("%-20s %4s %24s %24s" % ("lengths", "occ", "k_phred_sum", "k_phred_win"))
    for name, w in workloads(args.scale):
        for occ in (1, 2, 3, 4):
            os.environ["FL_PHRED_OCC"] = str(occ)
            ctx = api.Context(api.make_params(target_bases=int(round(5e9 * args.scale))), device=0)
            ctx.set_stream(stream.cuda_stream)
            t_len, t_off, d_qual = device_arena(torch, dev, ctx, w)
            batch = api.device_batch(w["n"], w["padded"], t_off, t_len, qual=d_qual)

            def step():
                ctx.reset_reads()
                ctx.push_device(batch)
                return ctx.finalize(-1)

            step()
            torch.cuda.synchronize(dev)
            per = defaultdict(float)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    step()
                torch.cuda.synchronize(dev)
            for e in prof.events():
                if e.device_type.name == "CUDA":
                    for k in ("k_phred_sum", "k_phred_win"):
                        if k in e.name:
                            per[k] += e.device_time_total / 1000.0 / args.steps
            cells = ["%8.2f ms (%6.0f GB/s)" % (per[k], w["padded"] / per[k] / 1e6 if per[k] else 0.0) for k in ("k_phred_sum", "k_phred_win")]
            print("%-20s %4d %24s %24s" % (name, occ, cells[0], cells[1]))
            ctx.close()
            del batch, d_qual, t_len, t_off
            torch.cuda.empty_cache()
    os.environ.pop("FL_PHRED_OCC", None)


def build_probes(tmp):
    from filtlong_b200 import build as b
    so = os.path.join(tmp, "phred_loads.so")
    flags = [f for f in b.FLAGS if f not in ("-Xptxas", "-v")]
    cmd = [b.NVCC] + flags + ["-shared", "-o", so, os.path.join(ROOT, "tools", "phred_loads.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed on tools/phred_loads.cu:\n" + r.stdout + r.stderr)
    lib = ctypes.CDLL(so)
    lib.probe_launch.restype = ctypes.c_int
    lib.probe_launch.argtypes = [ctypes.c_int] * 5 + [ctypes.c_void_p] * 4 + [ctypes.c_uint32] + [ctypes.c_void_p] * 2 + [ctypes.c_int, ctypes.c_void_p]
    lib.chunked_launch.restype = ctypes.c_int
    lib.chunked_launch.argtypes = lib.probe_launch.argtypes
    return lib


# (label, mode, depth, two-deep claim, longest first)
VARIANTS = [("registers, one step ahead", 0, 1, 0, 1), ("registers, arena order", 0, 1, 0, 0),
            ("bulk ring 4, cold start per read", 1, 4, 0, 1),
            ("bulk ring 2", 1, 2, 1, 1), ("bulk ring 4", 1, 4, 1, 1), ("bulk ring 8", 1, 8, 1, 1),
            ("bulk ring 4, arena order", 1, 4, 1, 0),
            ("cp.async ring 2", 2, 2, 1, 1), ("cp.async ring 4", 2, 4, 1, 1), ("cp.async ring 8", 2, 8, 1, 1),
            ("per-lane slots 2 (k_phred_sum's only)", 3, 2, 0, 1), ("per-lane slots 3", 3, 3, 0, 1),
            ("per-lane slots 4", 3, 4, 0, 1)]


def probe_part(torch, dev, stream, args):
    from filtlong_b200 import api
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_probes(tmp)
        print("load-only probes, ms per launch (GB/s of arena bytes) [blocks per SM that ran]:")
        print("%-20s %-34s %28s %28s" % ("lengths", "variant", "k_phred_sum's walk", "k_phred_win's walk"))
        for name, w in workloads(args.scale):
            ctx = api.Context(api.make_params(), device=0)
            ctx.set_stream(stream.cuda_stream)
            t_len, t_off, d_qual = device_arena(torch, dev, ctx, w)
            ctx.close()
            longest = torch.argsort(t_len, descending=True, stable=True).to(torch.int32)
            arena = torch.arange(w["n"], dtype=torch.int32, device=dev)
            work = torch.zeros(1, dtype=torch.int64, device=dev)
            out = torch.zeros(w["n"], dtype=torch.int32, device=dev)
            for label, mode, depth, deep, by_length in VARIANTS:
                order = longest if by_length else arena
                cells = []
                for kind in (0, 1):
                    if mode == 3 and kind == 1:
                        cells.append("-")
                        continue

                    def launch():
                        rc = lib.probe_launch(kind, mode, depth, deep, 4, d_qual.data_ptr(), t_off.data_ptr(), t_len.data_ptr(),
                                              order.data_ptr(), w["n"], work.data_ptr(), out.data_ptr(), sms, stream.cuda_stream)
                        if rc > -100:
                            raise RuntimeError("probe %s kind %d: error %d" % (label, kind, rc))
                        return -rc - 100
                    occ = launch()
                    torch.cuda.synchronize(dev)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    for _ in range(args.launches):
                        launch()
                    e1.record(stream)
                    torch.cuda.synchronize(dev)
                    ms = e0.elapsed_time(e1) / args.launches
                    cells.append("%7.2f ms (%6.0f GB/s) [%d]" % (ms, w["padded"] / ms / 1e6, occ))
                print("%-20s %-34s %28s %28s" % (name, label, cells[0], cells[1]))
            chunked_part(torch, dev, stream, args, lib, sms, name, w, d_qual, t_off, t_len, longest, work, out)
            del d_qual, t_len, t_off, longest, arena, out
            torch.cuda.empty_cache()


# Dynamic shared memory of the one-pass kernel's tables: the sum's (32 KiB), the window filter's (32 KiB) and the
# window's grid table in 4 copies (8 KiB). Three blocks of 256 threads fit an SM.
CHAIN_SMEM = 73728


def chunked_part(torch, dev, stream, args, lib, sms, name, w, d_qual, t_off, t_len, order, work, out):
    """Chunked walks, register loads plus a bulk L2 prefetch D chunks ahead (D = 0: none), longest first, with the
    one-pass kernel's shared-memory footprint and three blocks per SM."""
    print("chunked walks, %d B of tables, ms per launch (GB/s of arena bytes) [blocks per SM that ran]:" % CHAIN_SMEM)
    print("%-20s %6s %2s %28s %28s %28s" % ("lengths", "chunk", "D", "k_phred_sum's walk", "k_phred_win's walk", "one pass, both"))
    for ch in (2048, 4096, 8192):
        for depth in (0, 1, 2):
            cells = []
            for kind in (0, 1, 2):
                def launch():
                    rc = lib.chunked_launch(kind, ch, depth, CHAIN_SMEM, 3, d_qual.data_ptr(), t_off.data_ptr(), t_len.data_ptr(),
                                            order.data_ptr(), w["n"], work.data_ptr(), out.data_ptr(), sms, stream.cuda_stream)
                    if rc > -100:
                        raise RuntimeError("chunked probe %d/%d/%d: error %d" % (kind, ch, depth, rc))
                    return -rc - 100
                occ = launch()
                torch.cuda.synchronize(dev)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(args.launches):
                    launch()
                e1.record(stream)
                torch.cuda.synchronize(dev)
                ms = e0.elapsed_time(e1) / args.launches
                cells.append("%7.2f ms (%6.0f GB/s) [%d]" % (ms, w["padded"] / ms / 1e6, occ))
            print("%-20s %6d %2d %28s %28s %28s" % (name, ch, depth, cells[0], cells[1], cells[2]))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--skip-library", action="store_true")
    ap.add_argument("--skip-probes", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/phred_loads.py measures on a GPU and found none")
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        smi = "nvidia-smi unavailable"
    print("card:", smi)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    if not args.skip_library:
        library_part(torch, dev, stream, args)
    if not args.skip_probes:
        probe_part(torch, dev, stream, args)


if __name__ == "__main__":
    main()
