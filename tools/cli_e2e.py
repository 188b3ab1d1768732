#!/usr/bin/env python
"""Text in -> text out: the `filtlong` command line of this repo (GPU) beside the unmodified reference
binary (oracle/_ref/filtlong_ref, CPU) on the same synthetic FASTQ, same arguments, on this box.
Checks that stdout is byte-identical and reports wall-clock seconds and Gbases/s of the whole process
(CUDA start-up included). Test / measurement infrastructure (it executes oracle/_ref); writes one JSON line.

    python tools/cli_e2e.py [--small-gbp 0.5] [--large-gbp 5] [--kmer-gbp 0.1] [--gpus N] > cli_e2e.json

Cases: a small Phred file and a k-mer + --trim --split 500 file through BOTH binaries (byte-identical stdout
required), and a large plain FASTQ through ours only (the reference needs ~26 s per Gbp), once with the device
feeder and once with FL_HOST_PARSER=1 (the kseq-compatible host path) for comparison.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (workload generators)

OURS = os.path.join(ROOT, "filtlong_b200", "bin", "filtlong")
REF = os.path.join(ROOT, "oracle", "_ref", "filtlong_ref")
ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)


def write_random_fastq(path, total_bases, seed, fast=False):
    """Lognormal read lengths (bench.make_lengths), uniform bases, qualities Q1..Q40; ~1 GB/s.
    fast: one random pool re-sliced for every block of reads (I/O experiments only: 5x quicker to write)."""
    rng = np.random.default_rng(seed)
    n = max(int(total_bases // 10000), 16)
    lens = bench.make_lengths(n, int(total_bases), seed)
    pool = None
    with open(path, "wb", buffering=1 << 24) as f:
        for lo in range(0, n, 2000):
            L = lens[lo:lo + 2000]
            tot = int(L.sum())
            if fast:
                if pool is None or len(pool[0]) < tot:
                    m = max(tot, 64 << 20)
                    pool = (ACGT[rng.integers(0, 4, size=m, dtype=np.uint8)].tobytes(), rng.integers(34, 74, size=m, dtype=np.uint8).tobytes())
                sh = int(rng.integers(0, len(pool[0]) - tot + 1))
                seq, qual = pool[0][sh:sh + tot], pool[1][sh:sh + tot]
            else:
                seq = ACGT[rng.integers(0, 4, size=tot, dtype=np.uint8)].tobytes()
                qual = rng.integers(34, 74, size=tot, dtype=np.uint8).tobytes()
            o, parts = 0, []
            for i, l in enumerate(L):
                l = int(l)
                parts += [b"@read_%d len=%d\n" % (lo + i, l), seq[o:o + l], b"\n+\n", qual[o:o + l], b"\n"]
                o += l
            f.write(b"".join(parts))
    return int(lens.sum())


def run(cmd, out_path, env_extra=None, to_null=False):
    env = dict(os.environ, LC_ALL="C", LANG="C", FL_CLI_TIMING="1")
    env.update(env_extra or {})
    t = time.time()
    with open("/dev/null" if to_null else out_path, "wb") as f:
        r = subprocess.run(cmd, stdout=f, stderr=subprocess.PIPE, env=env)
    dt = time.time() - t
    res = dict(seconds=dt, rc=r.returncode)
    if not to_null:
        h = hashlib.md5()
        with open(out_path, "rb") as f:
            for blk in iter(lambda: f.read(1 << 24), b""):
                h.update(blk)
        res.update(md5=h.hexdigest(), bytes=os.path.getsize(out_path))
    err = r.stderr.decode(errors="replace").strip().splitlines()
    res["stderr_tail"] = [x.split("\r")[-1] for x in err if not x.startswith("[timing]")][-4:]
    res["phases"] = [x[9:].strip() for x in err if x.startswith("[timing]")]
    return res


def both(name, fq, bases, extra, td, gpus):
    res = {"case": name, "bases": bases, "args": extra}
    for tag, exe in (("reference_cpu", [REF]), ("ours_gpu", [OURS] + (["--gpus", str(gpus)] if gpus > 1 else []))):
        if not os.path.exists(exe[0]):
            res[tag] = {"error": "missing " + exe[0]}
            continue
        r = run(exe + extra + [fq], os.path.join(td, name + "." + tag + ".out"))
        r["gbases_per_s"] = bases / r["seconds"] / 1e9
        res[tag] = r
    a, b = res.get("reference_cpu", {}), res.get("ours_gpu", {})
    res["stdout_identical"] = bool(a.get("md5") and a.get("md5") == b.get("md5"))
    if a.get("seconds") and b.get("seconds"):
        res["speedup_wall"] = a["seconds"] / b["seconds"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small-gbp", type=float, default=0.5)
    ap.add_argument("--large-gbp", type=float, default=5.0)
    ap.add_argument("--kmer-gbp", type=float, default=0.1)
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--tmp", default=None)
    ap.add_argument("--large-only", action="store_true")
    ap.add_argument("--fast-gen", action="store_true", help="large file from a re-sliced random pool (I/O experiments)")
    ap.add_argument("--large-env", default="", help="extra runs of the large case to /dev/null: tag:ENV=V,ENV=V;tag2:...")
    a = ap.parse_args()
    out = {"what": "filtlong CLI, FASTQ text in -> FASTQ text out, wall clock of the whole process (CUDA start-up included)", "cases": []}
    with tempfile.TemporaryDirectory(prefix="flcli_", dir=a.tmp) as td:
        if not a.large_only:
            fq = os.path.join(td, "small.fastq")
            bases = write_random_fastq(fq, a.small_gbp * 1e9, 11)
            out["cases"].append(both("phred_small_target_25pct", fq, bases, ["--target_bases", str(bases // 4)], td, a.gpus))
            os.unlink(fq)
            wk = bench.kmer_workload(0, 200000, 2 * 10 ** 9, 1, 10 ** 7, 0.03, 0.15, seed=3)
            fa = os.path.join(td, "genome.fasta")
            g = bench.reference_fasta(fa, 1, 10 ** 7, 2, 0)
            fqk = os.path.join(td, "kmer.fastq")
            kb = bench.write_sample_fastq(fqk, wk, max(int(a.kmer_gbp * 1e9 / 10000), 100), genome=g)
            out["cases"].append(both("kmer_assembly_trim_split_500", fqk, kb, ["-a", fa, "--trim", "--split", "500", "-p", "90"], td, a.gpus))
            os.unlink(fqk)
        if a.large_gbp > 0 and os.path.exists(OURS):
            fql = os.path.join(td, "large.fastq")
            t0 = time.time()
            lb = write_random_fastq(fql, a.large_gbp * 1e9, 12, fast=a.fast_gen)
            gen_s = time.time() - t0
            res = {"case": "phred_large_target_25pct", "bases": lb, "file_bytes": os.path.getsize(fql), "generate_seconds": gen_s}
            args = ["--target_bases", str(lb // 4), fql]
            gp = ["--gpus", str(a.gpus)] if a.gpus > 1 else []
            runs = [("ours_gpu_feeder_to_devnull", {}, True), ("ours_gpu_feeder_to_file", {}, False),
                    ("ours_gpu_feeder_to_devnull_again", {}, True)]
            if not a.large_only:
                runs.append(("ours_gpu_host_parser_to_devnull", {"FL_HOST_PARSER": "1"}, True))
            for spec in [x for x in a.large_env.split(";") if x]:
                tag, _, kv = spec.partition(":")
                runs.append(("ours_gpu_feeder_to_devnull_" + tag, dict(e.split("=", 1) for e in kv.split(",") if e), True))
            for tag, envx, null in runs:
                r = run([OURS] + gp + args, os.path.join(td, "large." + tag + ".out"), envx, to_null=null)
                r["gbases_per_s"] = lb / r["seconds"] / 1e9
                res[tag] = r
                if not null:
                    os.unlink(os.path.join(td, "large." + tag + ".out"))
            out["cases"].append(res)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
