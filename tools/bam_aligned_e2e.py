"""Aligned BAM (--aligned) on the GPU: what the reverse-strand gather costs, and the command line end to end.

1. Device time of fl_reads_push_bam_strand (CUDA events around the call on the context's stream: the chunk's copy, the
   gather into the arena and the scoring) over the same seeded chunk of C2-like reads (bench.py's lengths and qualities,
   made by fl_synth), pushed until about --push_gbases have gone through, once with every record forward and once with
   every record reverse, alternating the two --reps times, in Phred mode and in k-mer mode.
2. Wall-clock of `--aligned -p 90` on a seeded coordinate-sorted aligned BAM of about --gbases (half the reads reverse,
   one hard-clipped supplementary record per four reads, Dorado-like RG / qs / MM / ML tags) against `-p 90` on the same
   reads as unaligned BAM, alternating, --reps times each, with FL_CLI_TIMING=1's phases.

The card's name and power limit are read in the same run. One JSON line:

    python tools/bam_aligned_e2e.py --gbases 4 --dir /tmp/aligned [--out result.json]
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
COMP = np.arange(256, dtype=np.uint8)
for a, b in zip(b"ACGTN", b"TGCAN"):
    COMP[a] = b
AUX = b"RGZrun1_dorado\0qsf" + struct.pack("<f", 14.0) + b"MMZC+h?,0,3,1;C+m?,0,3,1;\0MLBC" + struct.pack("<I", 6) + bytes(range(6))
REF_LEN = 1 << 30


def reads_of(gbases, seed):
    """(name, seq, qual) numpy views of about gbases of C2-like reads (bgzf_bench.fastq_text)"""
    import bgzf_bench
    text = bgzf_bench.fastq_text(gbases * 1e9 * 2.02, seed=seed)
    nl = np.flatnonzero(text == 10)
    for k in range(0, len(nl) - 3, 4):
        h0 = 1 if k == 0 else int(nl[k - 1]) + 2
        yield (text[h0:int(nl[k])].tobytes().split(b" ", 1)[0], text[int(nl[k]) + 1:int(nl[k + 1])],
               text[int(nl[k + 2]) + 1:int(nl[k + 3])])


def record(name, seq, qual, flag, cigar=(), ref_id=-1, pos=-1, aux=AUX):
    codes = CODE[seq]
    if len(codes) & 1:
        codes = np.append(codes, 0)
    packed = ((codes[0::2] << 4) | codes[1::2]).astype(np.uint8).tobytes()
    body = struct.pack("<iiBBHHHiiii", ref_id, pos, len(name) + 1, 60 if ref_id >= 0 else 255, 4680, len(cigar), flag, len(seq), -1, -1, 0) + \
        name + b"\0" + b"".join(struct.pack("<I", c) for c in cigar) + packed + (qual - 33).astype(np.uint8).tobytes() + aux
    return struct.pack("<I", len(body)) + body


def piece(gbases, seed, pos0):
    """(aligned records sorted by position, the same reads as unaligned records, positions used) of one seed"""
    rng = np.random.default_rng(seed)
    aligned, unaligned, pos = [], [], pos0
    for i, (name, seq, qual) in enumerate(reads_of(gbases, seed)):
        L = len(seq)
        unaligned.append(record(name, seq, qual, 4))
        rev = i % 2 == 1
        stored, squal = (COMP[seq[::-1]], qual[::-1]) if rev else (seq, qual)
        aligned.append((pos, record(name, stored, squal, 0x10 if rev else 0, (L << 4,), 0, pos)))
        if i % 4 == 0 and L > 200:
            a = int(rng.integers(0, L - 100))
            b = min(L, a + 1000)
            cg = ((a << 4) | 5,) + (((b - a) << 4),) + ((((L - b) << 4) | 5,) if L > b else ())
            spos = pos + int(rng.integers(-50000, 50000))
            aligned.append((max(spos, 0), record(name, stored[a:b], squal[a:b], 0x800 | (0x10 if rev else 0), cg, 0, max(spos, 0),
                                                 aux=b"SAZchr1,1,+,100M,60,0;\0")))
        pos += int(rng.integers(1, 2000))
    aligned.sort(key=lambda x: x[0])
    return b"".join(r for _, r in aligned), b"".join(unaligned), pos


def write_inputs(gbases, d):
    from filtlong_b200 import api
    paths = os.path.join(d, "aligned.bam"), os.path.join(d, "unaligned.bam")
    text = b"@HD\tVN:1.6\tSO:coordinate\n@RG\tID:run1_dorado\tSM:sample\n"
    hdr = [b"BAM\1" + struct.pack("<I", len(t)) + t + struct.pack("<I", n) + (struct.pack("<I", 5) + b"chr1\0" + struct.pack("<I", REF_LEN) if n else b"")
           for t, n in ((text, 1), (text.replace(b"coordinate", b"unknown"), 0))]
    with open(paths[0], "wb") as fa, open(paths[1], "wb") as fu, api.Context() as ctx:
        fa.write(ctx.bgzf_compress(hdr[0], append_eof=False))
        fu.write(ctx.bgzf_compress(hdr[1], append_eof=False))
        left, seed, pos = gbases, 31, 0
        while left > 0:                                    # 1 Gbase per piece, each from its own seed
            al, un, pos = piece(min(left, 1.0), seed, pos)
            fa.write(ctx.bgzf_compress(al, append_eof=False))
            fu.write(ctx.bgzf_compress(un, append_eof=False))
            left -= 1.0
            seed += 1
        fa.write(EOF_MEMBER)
        fu.write(EOF_MEMBER)
    return paths


def push_times(push_gbases, reps):
    """device ms per push of the same chunk, all forward and all reverse, alternating, in Phred and k-mer mode"""
    import torch
    from filtlong_b200 import api, capi
    recs = [record(n, s, q, 0, (len(s) << 4,), 0, 0) for n, s, q in reads_of(0.9, 7)]
    raw = b"".join(recs)
    chunk = torch.empty(len(raw), dtype=torch.uint8, pin_memory=True).numpy()
    chunk[:] = np.frombuffer(raw, np.uint8)
    so, qo, ln, p = [], [], [], 0
    for r in recs:
        l_name, n_cigar, l_seq = r[12], struct.unpack_from("<H", r, 16)[0], struct.unpack_from("<i", r, 20)[0]
        so.append(p + 36 + l_name + 4 * n_cigar)
        qo.append(so[-1] + (l_seq + 1) // 2)
        ln.append(l_seq)
        p += len(r)
    bases = int(sum(ln))
    n_push = max(1, int(round(push_gbases * 1e9 / bases)))
    genome = np.frombuffer(b"ACGT", np.uint8)[np.random.default_rng(5).integers(0, 4, size=4_000_000)].tobytes()
    out = dict(chunk_bytes=len(raw), chunk_bases=bases, pushes_per_measurement=n_push)
    stream = torch.cuda.Stream()
    for mode in ("phred", "kmer"):
        times = {"forward": [], "reverse": []}
        for rep in range(reps + 1):                        # the first round warms up
            for kind in ("forward", "reverse") if rep % 2 == 0 else ("reverse", "forward"):
                ctx = api.Context(api.make_params(keep_percent=90.0))
                if mode == "kmer":
                    ctx.kmers_add([genome], False)
                    ctx.kmers_count()
                capi.check(ctx.h, ctx.L.fl_ctx_set_stream(ctx.h, stream.cuda_stream), "fl_ctx_set_stream")
                rev = np.full(len(ln), 1 if kind == "reverse" else 0, np.uint8)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(n_push):
                    ctx.push_bam(chunk, so, qo, ln, reverse=rev)
                e1.record(stream)
                e1.synchronize()
                if rep:
                    times[kind].append(e0.elapsed_time(e1))
                ctx.close()
        out[mode] = {k: dict(ms=[round(x, 1) for x in v], min=round(min(v), 1), max=round(max(v), 1),
                             gbases_per_s=round(bases * n_push / (min(v) / 1e3) / 1e9, 2)) for k, v in times.items()}
        print(mode, out[mode], flush=True)
    return out


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
    ap.add_argument("--gbases", type=float, default=4.0)
    ap.add_argument("--push_gbases", type=float, default=4.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dir", required=True)
    ap.add_argument("--out")
    a = ap.parse_args()
    os.makedirs(a.dir, exist_ok=True)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    res = dict(gpu=gpu.strip().splitlines()[0] if gpu.strip() else "unknown", host_cpus=os.cpu_count())
    res["push"] = push_times(a.push_gbases, a.reps)
    t0 = time.time()
    aligned, unaligned = write_inputs(a.gbases, a.dir)
    res.update(gbases=a.gbases, write_seconds=round(time.time() - t0, 1), aligned_bytes=os.path.getsize(aligned),
               unaligned_bytes=os.path.getsize(unaligned))
    out = os.path.join(a.dir, "out")
    runs = {"aligned": [], "unaligned": []}
    for rep in range(a.reps):
        order = (("aligned", ["--aligned", "-p", "90", aligned]), ("unaligned", ["-p", "90", unaligned]))
        for tag, args in order if rep % 2 == 0 else order[::-1]:
            runs[tag].append(timed(args, out))
            print(tag, runs[tag][-1], flush=True)
    res["cli"] = {k: dict(seconds=[r["seconds"] for r in v], rc=[r["rc"] for r in v], output_bytes=v[-1]["output_bytes"], phases=v[-1]["phases"])
                  for k, v in runs.items()}
    for p in (aligned, unaligned):
        os.remove(p)
    line = json.dumps(res)
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
