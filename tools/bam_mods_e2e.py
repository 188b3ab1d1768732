"""BAM pass 2 with children built on the device: `-a <64 Mbp> --trim --split 500` on tools/bam_e2e.py's uBAM (RG, qs, MM
and ML on every record), run by a given older build of `filtlong`, by this one without --keep_mods and by this one with
it, alternated, `--rounds` times each, FL_CLI_TIMING=1. Reports wall-clock seconds and the pass-2 phase of each run,
whether the older build and this one wrote the same bytes without the flag, and, from CUDA events on one batch of the
same records (64 MiB of parents, their children at the CLI's rows), the device time of the child builder (fl_bam_build)
and of the BGZF compressor, with the card's name and power limit, as one JSON line.

    python tools/bam_mods_e2e.py --gbases 4 --dir /tmp/bam --old build/parent/filtlong_b200/bin/filtlong [--out result.json]
"""
import argparse
import hashlib
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
import bam_e2e  # noqa: E402

CLI = os.path.join(ROOT, "filtlong_b200", "bin", "filtlong")


def timed(cli, args, out_path):
    env = dict(os.environ, LC_ALL="C", FL_CLI_TIMING="1")
    t0 = time.perf_counter()
    with open(out_path, "wb") as f:
        r = subprocess.run([cli] + args, stdout=f, stderr=subprocess.PIPE, env=env)
    dt = time.perf_counter() - t0
    err = r.stderr.decode()
    phases = {m.group(1).strip(): float(m.group(2)) for m in re.finditer(r"^\[timing\] (.+?) +([0-9.]+) s$", err, re.M)}
    h = hashlib.sha256()
    with open(out_path, "rb") as f:
        for b in iter(lambda: f.read(1 << 24), b""):
            h.update(b)
    mods = re.search(r"modification tags: .*", err)
    os.remove(out_path)
    return dict(seconds=round(dt, 3), rc=r.returncode, pass2=phases.get("pass 2 (slices of the mapped input)"), sha=h.hexdigest()[:16],
                log=mods.group(0) if mods else None)


def device_times(raw, asm_rows=500, reps=5):
    """fl_bam_build and fl_bgzf_compress device milliseconds on 64 MiB of parents, each split into pieces of asm_rows"""
    from filtlong_b200 import api
    items, p = [], 0
    while p < len(raw) and p < (64 << 20):
        bs = struct.unpack_from("<I", raw, p)[0]
        l_seq = struct.unpack_from("<i", raw, p + 20)[0]
        items += [(p, s, min(s + asm_rows, l_seq)) for s in range(0, l_seq, asm_rows + 1)]
        p += 4 + bs
    batch = raw[:p]
    out = {}
    with api.Context() as ctx:
        for keep in (False, True):
            stream, _ = ctx.bam_build(batch, items, keep)
            ctx.enable_timing(True)
            ctx.reset_timing()
            for _ in range(reps):
                ctx.bam_build(batch, items, keep)
            out["build_ms_keep_mods" if keep else "build_ms"] = round(ctx.kernel_time("bam_build")[0] / reps, 3)
            ctx.reset_timing()
            for _ in range(reps):
                ctx.bgzf_compress(stream, append_eof=False)
            out["bgzf_ms_keep_mods" if keep else "bgzf_ms"] = round(ctx.kernel_time("bgzf")[0] / reps, 3)
            out["built_bytes_keep_mods" if keep else "built_bytes"] = len(stream)
            ctx.enable_timing(False)
    out.update(batch_bytes=len(batch), children=len(items))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbases", type=float, default=4.0)
    ap.add_argument("--dir", required=True)
    ap.add_argument("--old", required=True, help="an older build's filtlong binary")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    from filtlong_b200 import api, capi
    os.makedirs(a.dir, exist_ok=True)
    bam_path, asm_path = os.path.join(a.dir, "reads.bam"), os.path.join(a.dir, "asm.fasta")
    hdr_text = b"@HD\tVN:1.6\tSO:unknown\n@RG\tID:run1_dorado\tSM:sample\n"
    first = None
    with open(bam_path, "wb") as fb, api.Context() as ctx:
        fb.write(ctx.bgzf_compress(b"BAM\1" + struct.pack("<I", len(hdr_text)) + hdr_text + struct.pack("<I", 0), append_eof=False))
        left, seed = a.gbases, 11
        while left > 0:
            raw, _ = bam_e2e.piece(min(left, 2.0), seed)
            if first is None:
                first = raw[:80 << 20]
            fb.write(ctx.bgzf_compress(raw, append_eof=False))
            del raw
            left -= 2.0
            seed += 1
        fb.write(bam_e2e.EOF_MEMBER)
    S = capi.synth_host_lib()                                # the genome of the first piece's reads, as bam_e2e.py makes it
    g_bases = 1 << 26
    g2b = np.zeros(g_bases // 16 + 8, dtype=np.uint32)
    S.fl_synth_genome_host(11, g_bases, capi.ptr(g2b))
    genome = np.zeros(g_bases + 64, dtype=np.uint8)
    one = np.zeros(1, dtype=np.uint64)
    S.fl_synth_ascii_host(1, capi.ptr(one), capi.ptr(np.array([g_bases], dtype=np.int32)), capi.ptr(g2b), None, capi.ptr(genome))
    with open(asm_path, "wb") as f:
        f.write(b">contig_1\n" + genome[:g_bases].tobytes() + b"\n")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    res = dict(gbases=a.gbases, bam_bytes=os.path.getsize(bam_path), gpu=gpu.strip().splitlines()[0] if gpu.strip() else "unknown",
               host_cpus=os.cpu_count(), runs={"old": [], "new": [], "new_keep_mods": []})
    args = ["-a", asm_path, "--trim", "--split", "500", bam_path]
    out = os.path.join(a.dir, "out.bam")
    for _ in range(a.rounds):
        for tag, cli, extra in (("old", a.old, []), ("new", CLI, []), ("new_keep_mods", CLI, ["--keep_mods"])):
            r = timed(cli, extra + args, out)
            res["runs"][tag].append(r)
            print(tag, r, flush=True)
    res["same_bytes_without_flag"] = len({r["sha"] for k in ("old", "new") for r in res["runs"][k]}) == 1
    res["device"] = device_times(first)
    for p in (bam_path, asm_path):
        os.remove(p)
    line = json.dumps(res)
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
