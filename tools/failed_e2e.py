"""What `--failed FILE` costs end to end: the `filtlong` command line on C2-like reads (the FASTQ and the unaligned BAM that
tools/bam_e2e.py builds, RG / qs / MM / ML tags on every BAM record) with and without `--failed`, every output to a file.
FASTQ: `-p 90`, plain and with `--bgzip`; BAM: `-p 90 -a <assembly> --trim --split 500` (BAM output is always BGZF). Each
command runs `--repeats` times, alternated with its pair. Reports the wall-clock of every run, the CLI's phases
(FL_CLI_TIMING), the output sizes, whether the paired runs wrote identical stdout (and identical FILEs across repeats),
and the card's name and power limit read in the same call, as one JSON line.

    python tools/failed_e2e.py --gbases 4 --dir /tmp/failed [--repeats 3] [--pairs fastq_p90,...] [--out result.json]
"""
import argparse
import filecmp
import json
import os
import re
import struct
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
CLI = os.path.join(ROOT, "filtlong_b200", "bin", "filtlong")
EOF_MEMBER = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def make_inputs(d, gbases):
    """reads.bam, reads.fastq (its FASTQ equivalent) and asm.fasta, as tools/bam_e2e.py writes them"""
    import bam_e2e
    from filtlong_b200 import api, capi
    bam_path, fq_path, asm_path = (os.path.join(d, x) for x in ("reads.bam", "reads.fastq", "asm.fasta"))
    hdr_text = b"@HD\tVN:1.6\tSO:unknown\n@RG\tID:run1_dorado\tSM:sample\n"
    with open(bam_path, "wb") as fb, open(fq_path, "wb") as ff, api.Context() as ctx:
        fb.write(ctx.bgzf_compress(b"BAM\1" + struct.pack("<I", len(hdr_text)) + hdr_text + struct.pack("<I", 0), append_eof=False))
        left, seed = gbases, 11
        while left > 0:
            raw, fq = bam_e2e.piece(min(left, 2.0), seed)
            fb.write(ctx.bgzf_compress(raw, append_eof=False))
            ff.write(fq)
            del raw, fq
            left -= 2.0
            seed += 1
        fb.write(EOF_MEMBER)
    S = capi.synth_host_lib()
    g_bases = 1 << 26
    g2b = np.zeros(g_bases // 16 + 8, dtype=np.uint32)
    S.fl_synth_genome_host(11, g_bases, capi.ptr(g2b))
    genome = np.zeros(g_bases + 64, dtype=np.uint8)
    one = np.zeros(1, dtype=np.uint64)
    S.fl_synth_ascii_host(1, capi.ptr(one), capi.ptr(np.array([g_bases], dtype=np.int32)), capi.ptr(g2b), None, capi.ptr(genome))
    with open(asm_path, "wb") as f:
        f.write(b">contig_1\n" + genome[:g_bases].tobytes() + b"\n")
    return bam_path, fq_path, asm_path


def timed(args, out_path, failed_path=None):
    env = dict(os.environ, LC_ALL="C", FL_CLI_TIMING="1")
    argv = [CLI] + args[:-1] + (["--failed", failed_path] if failed_path else []) + args[-1:]
    t0 = time.perf_counter()
    with open(out_path, "wb") as f:
        r = subprocess.run(argv, stdout=f, stderr=subprocess.PIPE, env=env)
    dt = time.perf_counter() - t0
    phases = {m.group(1).strip(): float(m.group(2)) for m in re.finditer(r"^\[timing\] (.+?) +([0-9.]+) s$", r.stderr.decode(), re.M)}
    res = dict(seconds=round(dt, 3), rc=r.returncode, output_bytes=os.path.getsize(out_path), phases=phases)
    if failed_path:
        res["failed_bytes"] = os.path.getsize(failed_path)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbases", type=float, default=4.0)
    ap.add_argument("--dir", required=True)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--pairs", default="fastq_p90,fastq_p90_bgzip,bam_p90_asm_trim_split500", help="which commands to time")
    ap.add_argument("--out")
    a = ap.parse_args()
    os.makedirs(a.dir, exist_ok=True)
    t0 = time.time()
    bam_path, fq_path, asm_path = make_inputs(a.dir, a.gbases)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    res = dict(gbases=a.gbases, write_seconds=round(time.time() - t0, 1), bam_bytes=os.path.getsize(bam_path),
               fastq_bytes=os.path.getsize(fq_path), gpu=gpu.strip().splitlines()[0] if gpu.strip() else "unknown",
               host_cpus=os.cpu_count(), repeats=a.repeats)
    out, out2, failed, failed0 = (os.path.join(a.dir, x) for x in ("out", "out2", "failed", "failed0"))
    pairs = [("fastq_p90", ["-p", "90", fq_path]), ("fastq_p90_bgzip", ["-p", "90", "--bgzip", fq_path]),
             ("bam_p90_asm_trim_split500", ["-p", "90", "-a", asm_path, "--trim", "--split", "500", bam_path])]
    pairs = [(tag, args) for tag, args in pairs if tag in a.pairs.split(",")]
    identical = True
    for tag, args in pairs:
        runs = {"without": [], "with": []}
        for k in range(a.repeats):
            runs["without"].append(timed(args, out))
            runs["with"].append(timed(args, out2, failed))
            same = filecmp.cmp(out, out2, shallow=False)              # stdout does not change with --failed
            if k == 0:
                os.replace(failed, failed0)
            else:
                same = same and filecmp.cmp(failed, failed0, shallow=False)
            identical = identical and same
            runs["with"][-1]["identical"] = same
            print(tag, k, runs["without"][-1]["seconds"], runs["with"][-1]["seconds"], same, flush=True)
        res[tag] = runs
        for p in (out, out2, failed, failed0):
            if os.path.exists(p):
                os.remove(p)
    res["outputs_identical"] = identical
    for p in (bam_path, fq_path, asm_path):
        os.remove(p)
    line = json.dumps(res)
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
