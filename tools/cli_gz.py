#!/usr/bin/env python
"""gzip input through the `filtlong` command line of this repo: the same synthetic FASTQ as a plain file, as ONE gzip
member (what `gzip` / MinKNOW write), and as BGZF blocks (`bgzip`), each to /dev/null with the device feeder, plus the
streaming host reader (FL_GZ_HOST=1: gzread under a kseq-compatible parser, twice -- the reference's structure) for
comparison. Reports wall-clock seconds of the whole process and checks that every variant prints the same bytes.
Measurement infrastructure; writes one JSON line.

    python tools/cli_gz.py [--gbp 1.0] > cli_gz.json
"""
import argparse
import hashlib
import json
import multiprocessing as mp
import os
import struct
import subprocess
import sys
import tempfile
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import cli_e2e  # noqa: E402

OURS = cli_e2e.OURS
PIECE = 32 << 20


def _deflate_piece(job):
    path, lo, n, level = job
    with open(path, "rb") as f:
        f.seek(lo)
        data = f.read(n)
    co = zlib.compressobj(level, zlib.DEFLATED, -15)
    return co.compress(data) + co.flush(zlib.Z_SYNC_FLUSH)


def write_single_member(src, dst, level=1):
    """One gzip member, deflated in parallel the way pigz does it: independent pieces ended with a sync flush are a
    valid deflate stream when concatenated; an empty final block closes it. (The member's CRC-32 is run over the whole
    file afterwards: Python does not expose zlib's crc32_combine.)"""
    size = os.path.getsize(src)
    jobs = [(src, lo, min(PIECE, size - lo), level) for lo in range(0, size, PIECE)]
    crc = 0
    with mp.Pool(min(32, os.cpu_count() or 4)) as pool, open(dst, "wb") as out:
        out.write(b"\x1f\x8b\x08\x00\0\0\0\0\x00\xff")
        for body in pool.imap(_deflate_piece, jobs):
            out.write(body)
        out.write(b"\x03\x00")
    with open(src, "rb") as f:
        for blk in iter(lambda: f.read(1 << 26), b""):
            crc = zlib.crc32(blk, crc)
    with open(dst, "ab") as out:
        out.write(struct.pack("<II", crc & 0xffffffff, size & 0xffffffff))


def _bgzf_piece(job):
    path, lo, n, level = job
    with open(path, "rb") as f:
        f.seek(lo)
        data = f.read(n)
    out = []
    for o in range(0, len(data), 0xff00):
        chunk = data[o:o + 0xff00]
        co = zlib.compressobj(level, zlib.DEFLATED, -15)
        body = co.compress(chunk) + co.flush()
        out.append(b"\x1f\x8b\x08\x04\0\0\0\0\x00\xff" + struct.pack("<H", 6) + b"BC" + struct.pack("<HH", 2, 12 + 6 + len(body) + 8 - 1)
                   + body + struct.pack("<II", zlib.crc32(chunk) & 0xffffffff, len(chunk)))
    return b"".join(out)


def write_bgzf(src, dst, level=1):
    size = os.path.getsize(src)
    piece = 0xff00 * 512
    jobs = [(src, lo, min(piece, size - lo), level) for lo in range(0, size, piece)]
    with mp.Pool(min(32, os.cpu_count() or 4)) as pool, open(dst, "wb") as out:
        for body in pool.imap(_bgzf_piece, jobs):
            out.write(body)
        out.write(bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000"))   # the empty end-of-file block


def run(args, env_extra, out_path):
    r = cli_e2e.run([OURS] + args, out_path, env_extra)
    return r


def gz_cases(a, td, res):
    fq = os.path.join(td, "reads.fastq")
    bases = cli_e2e.write_random_fastq(fq, a.gbp * 1e9, 21, fast=True)
    t = time.time()
    write_single_member(fq, fq + ".gz")
    write_bgzf(fq, fq + ".bgz.gz")
    res.update(bases=bases, plain_bytes=os.path.getsize(fq), gz_bytes=os.path.getsize(fq + ".gz"), bgzf_bytes=os.path.getsize(fq + ".bgz.gz"),
               compress_seconds=time.time() - t, host_cpus=os.cpu_count())
    tgt = ["--target_bases", str(bases // 4)]
    runs = [("plain_feeder", fq, {}), ("gz_one_member_feeder", fq + ".gz", {}), ("gz_bgzf_feeder", fq + ".bgz.gz", {}),
            ("gz_bgzf_feeder_1_thread", fq + ".bgz.gz", {"FL_INFLATE_THREADS": "1"}),
            ("gz_one_member_host_reader", fq + ".gz", {"FL_GZ_HOST": "1"})]
    md5 = set()
    for tag, path, env in runs:
        out = os.path.join(td, tag + ".out")
        r = run(tgt + [path], env, out)
        r["gbases_per_s"] = bases / r["seconds"] / 1e9
        md5.add(r.get("md5"))
        res[tag] = r
        os.unlink(out)
    res["all_outputs_identical"] = len(md5) == 1


def reference_cases(a, td, res):
    import numpy as np
    # ---- the -1/-2 reference files: device text (fl_kmers_add_text) against the host reader ----
    if a.short_reads > 0:
        rng = np.random.default_rng(5)
        genome = cli_e2e.ACGT[rng.integers(0, 4, size=10_000_000, dtype=np.uint8)]
        windows = np.lib.stride_tricks.sliding_window_view(genome, 150)
        stride = max(1, len(windows) // max(a.short_reads, 1))
        paths = []
        for mate in (1, 2):
            sp = os.path.join(td, "short_%d.fastq" % mate)
            with open(sp, "wb", buffering=1 << 24) as f:
                for lo in range(0, a.short_reads, 200000):      # fixed-width records "@p0000000/1", filled column-wise
                    n = min(200000, a.short_reads - lo)
                    idx = np.arange(lo, lo + n)
                    rec = np.empty((n, 12 + 150 + 3 + 150 + 1), dtype=np.uint8)
                    rec[:, 0:2] = np.frombuffer(b"@p", np.uint8)
                    for d in range(7):
                        rec[:, 2 + d] = 48 + (idx // 10 ** (6 - d)) % 10
                    rec[:, 9] = ord("/")
                    rec[:, 10] = 48 + mate
                    rec[:, 11] = 10
                    rec[:, 12:162] = windows[(idx * stride + mate) % len(windows)]       # overlapping windows: every 16-mer many times
                    rec[:, 162:165] = np.frombuffer(b"\n+\n", np.uint8)
                    rec[:, 165:315] = ord("I")
                    rec[:, 315] = 10
                    f.write(rec.tobytes())
            paths.append(sp)
        small = os.path.join(td, "few.fastq")
        cli_e2e.write_random_fastq(small, 2e7, 3, fast=True)
        args = ["-1", paths[0], "-2", paths[1], "-p", "90", small]
        ref = {"short_reads_per_file": a.short_reads, "bytes_per_file": os.path.getsize(paths[0])}
        m = set()
        for tag, env in (("device_text", {}), ("host_reader", {"FL_HOST_PARSER": "1"})):
            out = os.path.join(td, "ref_" + tag + ".out")
            r = run(args, env, out)
            m.add(r.get("md5"))
            ref[tag] = r
        ref["outputs_identical"] = len(m) == 1
        res["reference_files"] = ref
        if a.assembly_gbp > 0:
            # ---- -a with a WRAPPED assembly (60 columns): device text (wrapped-FASTA index) against the host reader ----
            fa = os.path.join(td, "assembly.fasta")
            n_contigs = 10
            per = int(a.assembly_gbp * 1e9 / n_contigs) // 60 * 60
            with open(fa, "wb", buffering=1 << 24) as f:
                for ci in range(n_contigs):
                    f.write(b">contig_%d length=%d\n" % (ci, per))
                    for lo in range(0, per, 60 * 500000):
                        nl_ = min(500000, (per - lo) // 60)
                        blk = np.empty((nl_, 61), dtype=np.uint8)
                        blk[:, :60] = cli_e2e.ACGT[rng.integers(0, 4, size=(nl_, 60), dtype=np.uint8)]
                        blk[:, 60] = 10
                        f.write(blk.tobytes())
            asm = {"contigs": n_contigs, "bases": per * n_contigs, "bytes": os.path.getsize(fa)}
            m = set()
            for tag, env in (("device_text", {}), ("host_reader", {"FL_HOST_PARSER": "1"})):
                out = os.path.join(td, "asm_" + tag + ".out")
                r = run(["-a", fa, "-p", "90", small], env, out)
                m.add(r.get("md5"))
                asm[tag] = r
            asm["outputs_identical"] = len(m) == 1
            res["assembly_file"] = asm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbp", type=float, default=1.0, help="reads file of the gzip cases (0: skip them)")
    ap.add_argument("--tmp", default=None)
    ap.add_argument("--assembly-gbp", type=float, default=1.0, help="wrapped FASTA for the -a case (0: skip)")
    ap.add_argument("--short-reads", type=int, default=1000000, help="reads per -1/-2 file (0: skip the reference-file cases)")
    a = ap.parse_args()
    res = {"what": "filtlong CLI: gzip input (one inflate into memory + device parse) and reference files as text, each against the streaming host reader"}
    with tempfile.TemporaryDirectory(prefix="flgz_", dir=a.tmp) as td:
        if a.gbp > 0:
            gz_cases(a, td, res)
        reference_cases(a, td, res)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
