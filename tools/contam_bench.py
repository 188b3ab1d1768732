"""What `--contam` costs on the GPU.

Device-resident: scoring + finalise of config-2-shaped Phred reads (bench.py's lengths, qualities from the library's own
generator, uniform random bases) without a contaminant set, and with a 48.5 kbp (lambda-sized) and a 5 Mbp set, each set
once with the position-anchored table (the default) and once probed through the bitmap behind its pre-filter
(FL_ANCHOR=0 on that context). The modes are alternated step by step; reported are the median and min-max ms per step,
the FL_KERNEL_CONTAM event times (contaminant probe, per-read count, per-row exclusion), the device memory each set takes
and the card's name and power limit, read in the same call. Random reads lie almost nowhere in the sets, as most reads of
a real run do.

With --cli_gbases G: `filtlong -p 90` wall-clock on a FASTQ of G Gbases of C2-like reads (bgzf_bench.fastq_text), with
and without `--contam` of a 48.5 kbp FASTA cut from the genome those reads come from, alternated, --cli_runs each.

    python tools/contam_bench.py [--bases 4e9] [--reads 4e5] [--steps 5] [--warmup 2] [--cli_gbases 4 --dir /tmp/c]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
CLI = os.path.join(ROOT, "filtlong_b200", "bin", "filtlong")


def card():
    g = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return g.strip().splitlines()[0] if g.strip() else "unknown"


def device_resident(a):
    import torch
    from filtlong_b200 import api, capi
    from qtrim_bench import workload

    L, off, padded, qbar = workload(int(a.reads), a.bases)
    dev = torch.device("cuda:0")
    t_len, t_off = torch.from_numpy(L).to(dev), torch.from_numpy(off.view(np.int64)).to(dev)
    d_qual = torch.empty(padded + 64, dtype=torch.uint8, device=dev)
    d_seq = torch.randint(-2 ** 31, 2 ** 31 - 1, (padded // 16 + 8,), dtype=torch.int32, device=dev)
    rng = np.random.default_rng(5)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    sets = {"48.5k": acgt[rng.integers(0, 4, 48502)].tobytes(), "5M": acgt[rng.integers(0, 4, 5_000_000)].tobytes()}
    target = int(L.sum()) // 2
    params = api.make_params(target_bases=target, max_contam=50.0)
    ctxs, mem, members = {}, {}, {}
    for mode in ["none", "48.5k", "48.5k_no_anchor", "5M", "5M_no_anchor"]:
        if mode.endswith("_no_anchor"):
            os.environ["FL_ANCHOR"] = "0"
        free0 = torch.cuda.mem_get_info()[0]
        c = api.Context(params)
        os.environ.pop("FL_ANCHOR", None)
        if mode != "none":
            c.contam_add([sets[mode.split("_")[0]]])
            members[mode] = c.contam_count()
            c.sync()
        mem[mode] = round((free0 - torch.cuda.mem_get_info()[0]) / 2 ** 30, 3)
        ctxs[mode] = c
    lib = capi.lib()
    c0 = ctxs["none"]
    capi.check(c0.h, lib.fl_synth_qual_device(c0.h, 1, len(L), t_off.data_ptr(), t_len.data_ptr(),
                                               torch.from_numpy(qbar).to(dev).data_ptr(), 0, d_qual.data_ptr()), "synth_qual")
    torch.cuda.synchronize()
    batch = api.device_batch(len(L), padded, t_off, t_len, seq2b=d_seq, qual=d_qual)

    def step(ctx):
        ctx.reset_reads()
        ctx.push_device(batch)
        return ctx.finalize(-1)

    for _ in range(a.warmup):
        for c in ctxs.values():
            step(c)
    for c in ctxs.values():
        c.enable_timing(True)
        c.reset_timing()
    ms = {k: [] for k in ctxs}
    summ = {}
    for _ in range(a.steps):
        for k, c in ctxs.items():                    # alternated
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            summ[k] = step(c)
            c.sync()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    rec = dict(card=card(), reads=len(L), bases=int(L.sum()), steps=a.steps, set_members=members,
               set_device_gib=mem,
               ms_per_step={k: float(np.median(v)) for k, v in ms.items()},
               ms_per_step_min_max={k: [float(min(v)), float(max(v))] for k, v in ms.items()},
               contam_kernel_ms_per_step={k: c.kernel_time("contam")[0] / a.steps for k, c in ctxs.items()},
               removed={k: int(c.contam_results()[2]["reads"]) for k, c in ctxs.items()},
               keeping={k: int(s.keeping) for k, s in summ.items()})
    for c in ctxs.values():
        c.close()
    return rec


def cli(a):
    import bgzf_bench
    from filtlong_b200 import capi
    os.makedirs(a.dir, exist_ok=True)
    fq, lam, out = (os.path.join(a.dir, x) for x in ("reads.fastq", "lambda.fasta", "out.fastq"))
    with open(fq, "wb") as f:
        left, seed = a.cli_gbases, 11
        while left > 0:
            f.write(bgzf_bench.fastq_text(min(left, 2.0) * 1e9 * 2.02, seed=seed).tobytes())
            left -= 2.0
            seed += 1
    S = capi.synth_host_lib()                          # the genome of seed 11's reads (tools/bam_e2e.py), first 48,502 bases
    g_bases = 1 << 26
    g2b = np.zeros(g_bases // 16 + 8, dtype=np.uint32)
    S.fl_synth_genome_host(11, g_bases, capi.ptr(g2b))
    genome = np.zeros(g_bases + 64, dtype=np.uint8)
    S.fl_synth_ascii_host(1, capi.ptr(np.zeros(1, dtype=np.uint64)), capi.ptr(np.array([g_bases], dtype=np.int32)), capi.ptr(g2b), None,
                          capi.ptr(genome))
    with open(lam, "wb") as f:
        f.write(b">lambda\n" + genome[:48502].tobytes() + b"\n")
    res = dict(card=card(), fastq_bytes=os.path.getsize(fq), runs={"p90": [], "contam_p90": []})
    env = dict(os.environ, LC_ALL="C")
    for _ in range(a.cli_runs):
        for tag, args in (("p90", ["-p", "90", fq]), ("contam_p90", ["--contam", lam, "-p", "90", fq])):
            t0 = time.perf_counter()
            with open(out, "wb") as f:
                r = subprocess.run([CLI] + args, stdout=f, stderr=subprocess.PIPE, env=env)
            res["runs"][tag].append(round(time.perf_counter() - t0, 3))
            if r.returncode:
                raise SystemExit(r.stderr.decode()[-2000:])
            if tag == "contam_p90":
                res["contam_log"] = [l for l in r.stderr.decode().splitlines() if "contaminant 16-mers" in l or "random base" in l]
    for p in (fq, lam, out):
        os.remove(p)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bases", type=float, default=4e9)
    ap.add_argument("--reads", type=float, default=4e5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cli_gbases", type=float, default=0.0)
    ap.add_argument("--cli_runs", type=int, default=3)
    ap.add_argument("--dir", default="/tmp/contam_bench")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rec = {"device_resident": device_resident(a)}
    print(json.dumps(rec), flush=True)
    if a.cli_gbases > 0:
        rec["cli"] = cli(a)
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
