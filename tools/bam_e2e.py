"""Unaligned BAM through the `filtlong` command line against its FASTQ equivalent: C2-like reads (bench.py's lengths and
qualities, made by fl_synth with bgzf_bench.py's seeds) written once as uBAM (BGZF compressed on the GPU with
api.bgzf_compress; RG, qs, MM and ML aux fields on every record) and once as the equivalent FASTQ, then `-p 90` and
`-a <assembly> --trim --split 500` on each with FL_CLI_TIMING=1. Reports wall-clock seconds, the CLI's phases, the input
and output sizes and the card's name and power limit, as one JSON line.

    python tools/bam_e2e.py --gbases 10 --dir /tmp/bam [--out result.json]
"""
import argparse
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
CODE = np.zeros(256, dtype=np.uint8)
for i, c in enumerate(b"=ACMGRSVTWYHKDBN"):
    CODE[c] = i
AUX = b"RGZrun1_dorado\0qsf" + struct.pack("<f", 14.0) + b"MMZC+h?,0,3,1;C+m?,0,3,1;\0MLBC" + struct.pack("<I", 6) + bytes(range(6))


def piece(gbases, seed):
    """(uncompressed BAM records, FASTQ equivalent) of about gbases of C2-like reads"""
    import bgzf_bench
    text = bgzf_bench.fastq_text(gbases * 1e9 * 2.02, seed=seed)
    nl = np.flatnonzero(text == 10)
    bam, fq = [], []
    for k in range(0, len(nl) - 3, 4):
        h0 = 1 if k == 0 else int(nl[k - 1]) + 2
        name = text[h0:int(nl[k])].tobytes().split(b" ", 1)[0]
        s0, s1 = int(nl[k]) + 1, int(nl[k + 1])
        seq = text[s0:s1]
        qual = text[int(nl[k + 2]) + 1:int(nl[k + 3])]
        codes = CODE[seq]
        if len(codes) & 1:
            codes = np.append(codes, 0)
        packed = ((codes[0::2] << 4) | codes[1::2]).astype(np.uint8).tobytes()
        body = struct.pack("<iiBBHHHiiii", -1, -1, len(name) + 1, 255, 4680, 0, 4, s1 - s0, -1, -1, 0) + name + b"\0" + packed + \
            (qual - 33).astype(np.uint8).tobytes() + AUX
        bam.append(struct.pack("<I", len(body)) + body)
        fq.append(b"@" + name + b"\n" + seq.tobytes() + b"\n+\n" + qual.tobytes() + b"\n")
    return b"".join(bam), b"".join(fq)


def timed(args, out_path):
    env = dict(os.environ, LC_ALL="C", FL_CLI_TIMING="1")
    t0 = time.perf_counter()
    with open(out_path, "wb") as f:
        r = subprocess.run([CLI] + args, stdout=f, stderr=subprocess.PIPE, env=env)
    dt = time.perf_counter() - t0
    phases = {m.group(1).strip(): float(m.group(2)) for m in re.finditer(r"^\[timing\] (.+?) +([0-9.]+) s$", r.stderr.decode(), re.M)}
    res = dict(seconds=round(dt, 3), rc=r.returncode, output_bytes=os.path.getsize(out_path), phases=phases)
    os.remove(out_path)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbases", type=float, default=10.0)
    ap.add_argument("--dir", required=True)
    ap.add_argument("--out")
    a = ap.parse_args()
    from filtlong_b200 import api, capi
    os.makedirs(a.dir, exist_ok=True)
    bam_path, fq_path, asm_path = (os.path.join(a.dir, x) for x in ("reads.bam", "reads.fastq", "asm.fasta"))
    hdr_text = b"@HD\tVN:1.6\tSO:unknown\n@RG\tID:run1_dorado\tSM:sample\n"
    t0 = time.time()
    with open(bam_path, "wb") as fb, open(fq_path, "wb") as ff, api.Context() as ctx:
        fb.write(ctx.bgzf_compress(b"BAM\1" + struct.pack("<I", len(hdr_text)) + hdr_text + struct.pack("<I", 0), append_eof=False))
        left, seed = a.gbases, 11
        while left > 0:                                     # 2 Gbases per piece, each from its own seed
            raw, fq = piece(min(left, 2.0), seed)
            fb.write(ctx.bgzf_compress(raw, append_eof=False))
            ff.write(fq)
            del raw, fq
            left -= 2.0
            seed += 1
            print("written", ff.tell(), flush=True)
        fb.write(EOF_MEMBER)
    # the assembly: the genome the first piece's reads come from (bgzf_bench.fastq_text, seed 11)
    S = capi.synth_host_lib()
    g_bases = 1 << 26
    g2b = np.zeros(g_bases // 16 + 8, dtype=np.uint32)
    S.fl_synth_genome_host(11, g_bases, capi.ptr(g2b))
    genome = np.zeros(g_bases + 64, dtype=np.uint8)
    one = np.zeros(1, dtype=np.uint64)
    S.fl_synth_ascii_host(1, capi.ptr(one), capi.ptr(np.array([g_bases], dtype=np.int32)), capi.ptr(g2b), None, capi.ptr(genome))
    with open(asm_path, "wb") as f:
        f.write(b">contig_1\n" + genome[:g_bases].tobytes() + b"\n")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    res = dict(gbases=a.gbases, write_seconds=round(time.time() - t0, 1), bam_bytes=os.path.getsize(bam_path), fastq_bytes=os.path.getsize(fq_path),
               gpu=gpu.strip().splitlines()[0] if gpu.strip() else "unknown", host_cpus=os.cpu_count())
    out = os.path.join(a.dir, "out")
    for tag, args in (("p90", ["-p", "90"]), ("asm_trim_split500", ["-a", asm_path, "--trim", "--split", "500"])):
        for kind, path in (("bam", bam_path), ("fastq", fq_path)):
            res["%s_%s" % (tag, kind)] = timed(args + [path], out)
            print(tag, kind, res["%s_%s" % (tag, kind)], flush=True)
    for p in (bam_path, fq_path, asm_path):
        os.remove(p)
    line = json.dumps(res)
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
