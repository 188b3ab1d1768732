"""fl_gzip_inflate (ordinary gzip inflated on the GPU) against one zlib thread on the same bytes.

Seed-generated C2-like FASTQ (8 kb reads, ACGT, Phred around Q18), each file one gzip member from one zlib stream:
  * L1: --gb GB of FASTQ at level 1;  * L6: a quarter of that at level 6;
  * the sweep: prefixes of the L1 FASTQ compressed at level 1, about 1 MiB to 256 MiB compressed.
fl_gzip_inflate is timed from host buffers to host buffers (copies included), with the default chunk size and device
memory; one zlib thread is Python's zlib.decompressobj (wbits 31) on the same bytes, in the same call, alternated run by
run. fl_gzip_inflate_device is the same call on device buffers (no copies).
The CLI legs time `filtlong -p 90` end to end (wall-clock, output to /dev/null) on the plain FASTQ, on its gzip with the
GPU inflater (FL_GUNZIP_MIN_BYTES=0) and on its gzip with one host zlib thread (FL_GUNZIP_HOST=1, the path before the GPU
inflater), alternated; the CLI sweep over compressed sizes is what Kmers::kDeviceGunzipMinBytes is taken from.
Prints one JSON line per measurement and the card's name and power limit.
usage: python tools/gunzip_bench.py [--gb 2] [--reps 3] [--tmp DIR]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import zlib

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from filtlong_b200 import capi  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def fastq(seed, n_bytes, read_len=8000):
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    out, total, i = [], 0, 0
    while total < n_bytes:
        seq = acgt[rng.integers(0, 4, size=(256, read_len))]
        qual = np.clip(rng.normal(18, 6, size=(256, read_len)), 1, 50).astype(np.uint8) + 33
        for j in range(256):
            r = b"@%032x runid=c2 read=%d ch=%d\n" % (int(rng.integers(0, 1 << 62)), i, j) + seq[j].tobytes() + b"\n+\n" + \
                qual[j].tobytes() + b"\n"
            out.append(r)
            total += len(r)
            i += 1
    return b"".join(out)


def gz(data, level):
    c = zlib.compressobj(level, zlib.DEFLATED, 31)
    return c.compress(data) + c.flush()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=2.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-api", action="store_true", help="only the CLI legs")
    ap.add_argument("--tmp", default=None, help="directory for the CLI legs' files (default: a temporary one)")
    a = ap.parse_args()
    L = capi.lib()
    ctx = capi.C.c_void_p()
    capi.check(None, L.fl_ctx_create(capi.make_params(), 0, capi.C.byref(ctx)), "fl_ctx_create")
    print(json.dumps({"card": card()}), flush=True)
    t0 = time.time()
    raw = fastq(3, int(a.gb * 1e9))
    print(json.dumps({"generated_bytes": len(raw), "s": round(time.time() - t0, 1)}), flush=True)

    def gpu(blob, n):
        src = np.frombuffer(blob, dtype=np.uint8)
        out = np.empty(n, dtype=np.uint8)
        out[::4096] = 0                                            # fault the pages in before timing
        n_out, status, st = capi.C.c_uint64(0), capi.C.c_int(-1), capi.GunzipStats()
        t = time.perf_counter()
        capi.check(ctx, L.fl_gzip_inflate(ctx, src.ctypes.data, len(blob), out.ctypes.data, n, 0, 0, capi.C.byref(n_out),
                                          capi.C.byref(status), capi.C.byref(st)), "fl_gzip_inflate")
        dt = time.perf_counter() - t
        ok = status.value == 0 and n_out.value == n
        return dt, ok, (st.members, st.chunks, st.redecoded, st.rounds), out

    def host(blob):
        t = time.perf_counter()
        d = zlib.decompressobj(31).decompress(blob)
        return time.perf_counter() - t, d

    def compare(name, data, blob):
        gt, ht = [], []
        same = True
        declined = False
        stats = None
        for _ in range(a.reps):
            dt, ok, stats, out = gpu(blob, len(data))
            declined |= not ok
            same &= ok and out.tobytes() == data
            gt.append(dt)
            del out
            dh, d = host(blob)
            same &= d == data
            ht.append(dh)
            del d
        g, h = min(gt), min(ht)
        print(json.dumps({"file": name, "compressed": len(blob), "inflated": len(data), "identical": same, "declined": declined,
                          "gpu_s": [round(x, 4) for x in gt], "zlib_1thread_s": [round(x, 4) for x in ht],
                          "gpu_GBps_out": round(len(data) / g / 1e9, 3), "zlib_GBps_out": round(len(data) / h / 1e9, 3),
                          "speedup": round(h / g, 2), "stats_members_chunks_redecoded_rounds": stats}), flush=True)

    def device_resident(name, data, blob):
        import torch
        src = torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda()
        out = torch.empty(len(data), dtype=torch.uint8, device="cuda")
        ts, ok = [], True
        for _ in range(a.reps):
            n_out, status, st = capi.C.c_uint64(0), capi.C.c_int(-1), capi.GunzipStats()
            torch.cuda.synchronize()
            t = time.perf_counter()
            capi.check(ctx, L.fl_gzip_inflate_device(ctx, src.data_ptr(), len(blob), out.data_ptr(), len(data), 0, 0,
                                                     capi.C.byref(n_out), capi.C.byref(status), capi.C.byref(st)),
                       "fl_gzip_inflate_device")
            ts.append(time.perf_counter() - t)
            ok &= status.value == 0 and n_out.value == len(data)
        ok &= bytes(out.cpu().numpy()) == data
        print(json.dumps({"file": name, "device_resident": True, "identical": ok, "gpu_s": [round(x, 4) for x in ts],
                          "gpu_GBps_out": round(len(data) / min(ts) / 1e9, 3)}), flush=True)
        del src, out
        torch.cuda.empty_cache()

    blob1 = gz(raw, 1)
    if not a.skip_api:
        compare("L1", raw, blob1)
        device_resident("L1", raw, blob1)
        q = raw[:len(raw) // 4]
        blob6 = gz(q, 6)
        compare("L6", q, blob6)
        device_resident("L6", q, blob6)
        del blob6
    # threshold sweep: compressed sizes from about 1 MiB to 256 MiB
    ratio = len(gz(raw[:8 << 20], 1)) / (8 << 20)
    sweep = []
    for mib in (1, 4, 16, 64, 256):
        n = min(len(raw), int((mib << 20) / ratio))
        n = raw.rfind(b"\n", 0, raw.rfind(b" runid=c2 read=", 0, n)) + 1     # whole records: the CLI scores the prefix
        part = raw[:n]
        b = gz(part, 1)
        if not a.skip_api:
            compare("sweep_%dMiB" % mib, part, b)
        sweep.append((mib, n, b))
    L.fl_ctx_destroy(ctx)

    # ---- the CLI ----
    cli = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "filtlong_b200", "bin", "filtlong")
    tmp = tempfile.TemporaryDirectory(dir=a.tmp)

    def cli_run(path, env_extra):
        env = dict(os.environ, LC_ALL="C", **env_extra)
        with open(os.devnull, "wb") as null:
            t = time.perf_counter()
            p = subprocess.run([cli, "-p", "90", path], stdout=null, stderr=subprocess.PIPE, env=env)
            dt = time.perf_counter() - t
        return dt, p.returncode

    def cli_compare(name, data, blob, with_plain):
        plain = os.path.join(tmp.name, name + ".fastq")
        gzp = plain + ".gz"
        open(gzp, "wb").write(blob)
        if with_plain:
            open(plain, "wb").write(data)
        modes = [("gpu_inflater", gzp, {"FL_GUNZIP_MIN_BYTES": "0"}), ("host_zlib", gzp, {"FL_GUNZIP_HOST": "1"})]
        if with_plain:
            modes.append(("plain", plain, {}))
        times = {m: [] for m, _, _ in modes}
        rcs = set()
        for _ in range(a.reps):
            for m, path, env in modes:
                dt, rc = cli_run(path, env)
                times[m].append(round(dt, 3))
                rcs.add(rc)
        print(json.dumps({"cli": "filtlong -p 90", "file": name, "compressed": len(blob), "inflated": len(data),
                          "exit_codes": sorted(rcs), "wall_s": times,
                          "best_s": {m: min(v) for m, v in times.items()}}), flush=True)
        for p in (plain, gzp):
            if os.path.exists(p):
                os.remove(p)

    cli_compare("L1", raw, blob1, True)
    for mib, n, b in sweep:
        cli_compare("sweep_%dMiB" % mib, raw[:n], b, False)


if __name__ == "__main__":
    main()
