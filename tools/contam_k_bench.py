"""What `--contam_k K` costs on the GPU.

Device-resident: scoring + finalise of config-2-shaped Phred reads (bench.py's lengths, qualities from the library's own
generator) in five modes, alternated step by step: no contaminant set; the 48.5 kbp (lambda-sized) 16-mer set; the same
sequence at K = 31; a 3.1 Gbp random genome at K = 31 with uniform random reads (miss-heavy, like a metagenome); and the
same set with reads cut from that genome (hit-heavy, like a clinical sample). Reported: median and min-max ms per step,
the FL_KERNEL_CONTAM event time per step, the device GiB each set takes, the sectors per look-up from the table's
probe-length distribution (a present k-mer, and an absent one by where it hashes), the removed reads, and the card's name
and power limit, read in the same call. The 3.1 Gbp genome is drawn on the device from a seed.

With --cli_gbases G: the CLI's build of the 3.1 Gbp set from a FASTA and from its gzip (the "Hashing" phase of
FL_CLI_TIMING), and `filtlong -p 90` wall-clock on a FASTQ of G Gbases of C2-like reads (from another genome) plus
--host_reads error-free reads cut from the 3.1 Gbp genome, with and without `--contam big.fa --contam_k 31`, alternated,
--cli_runs each; how many of the genome's reads the runs with the set kept (none should be).

    python tools/contam_k_bench.py [--bases 4e9] [--reads 4e5] [--steps 5] [--warmup 2] [--cli_gbases 4 --dir /tmp/ck]
"""
import argparse
import gzip
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
GENOME_BASES = 3_100_000_000
RECORD_BASES = 100_000_000


def card():
    g = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return g.strip().splitlines()[0] if g.strip() else "unknown"


def genome_records(seed, n_bases=GENOME_BASES, record_bases=RECORD_BASES):
    """(2-bit words on the device, ASCII bytes on the host) per record of a random genome"""
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    acgt = torch.tensor(list(b"ACGT"), dtype=torch.uint8, device="cuda")
    shifts = torch.arange(30, -2, -2, dtype=torch.int32, device="cuda")
    left = n_bases
    while left > 0:
        n = min(left, record_bases)
        words = torch.randint(-2 ** 31, 2 ** 31 - 1, ((n + 15) // 16,), dtype=torch.int32, device="cuda", generator=g)
        codes = ((words[:, None] >> shifts[None, :]) & 3).reshape(-1)[:n]
        yield words, acgt[codes.long()].cpu().numpy().tobytes()
        left -= n


def sectors(hist):
    h = np.asarray(hist, dtype=np.float64)
    return float((h * np.arange(len(h))).sum() / max(h.sum(), 1))


def device_resident(a):
    import torch
    from filtlong_b200 import api, capi
    from qtrim_bench import workload

    L, off, padded, qbar = workload(int(a.reads), a.bases)
    dev = torch.device("cuda:0")
    t_len, t_off = torch.from_numpy(L).to(dev), torch.from_numpy(off.view(np.int64)).to(dev)
    d_qual = torch.empty(padded + 64, dtype=torch.uint8, device=dev)
    d_rand = torch.randint(-2 ** 31, 2 ** 31 - 1, (padded // 16 + 8,), dtype=torch.int32, device=dev)
    rng = np.random.default_rng(5)
    lam = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 48502)].tobytes()
    params = api.make_params(target_bases=int(L.sum()) // 2, max_contam=50.0)
    ctxs, mem, members, probe = {}, {}, {}, {}
    for mode in ["none", "48.5k_k16", "48.5k_k31", "3.1G_k31_random"]:
        free0 = torch.cuda.mem_get_info()[0]
        c = api.Context(params)
        if mode == "48.5k_k16":
            c.contam_add([lam])
        elif mode == "48.5k_k31":
            c.contam_configure(31, len(lam))
            c.contam_add([lam])
        elif mode.startswith("3.1G"):
            c.contam_configure(31, GENOME_BASES)
            parts = []
            t0 = time.perf_counter()
            n_rec = (GENOME_BASES + RECORD_BASES - 1) // RECORD_BASES
            for i, (words, seq) in enumerate(genome_records(1)):
                c.contam_add_text(b">c%d\n%s\n" % (i, seq), fastq=False, is_last=int(i + 1 == n_rec))
                parts.append(words)
            c.sync()
            mem["3.1G_build_s_api"] = round(time.perf_counter() - t0, 2)
            g = torch.cat(parts)                           # reads cut from the genome: its 2-bit words, repeated to the arena
            del parts
            d_hit = g.repeat((d_rand.numel() + g.numel() - 1) // g.numel())[:d_rand.numel()].contiguous()
            del g
        if mode != "none":
            members[mode] = c.contam_count()
        if mode.endswith("k31") or mode.startswith("3.1G"):
            hit, miss = c.contam_probe_lengths(32)
            probe[mode] = dict(present=sectors(hit), absent=sectors(miss), present_hist=[int(x) for x in hit[:8]],
                               absent_hist=[int(x) for x in miss[:8]])
        c.sync()
        mem[mode] = round((free0 - torch.cuda.mem_get_info()[0]) / 2 ** 30, 3)
        ctxs[mode] = c
    lib = capi.lib()
    c0 = ctxs["none"]
    capi.check(c0.h, lib.fl_synth_qual_device(c0.h, 1, len(L), t_off.data_ptr(), t_len.data_ptr(),
                                               torch.from_numpy(qbar).to(dev).data_ptr(), 0, d_qual.data_ptr()), "synth_qual")
    torch.cuda.synchronize()
    rand_batch = api.device_batch(len(L), padded, t_off, t_len, seq2b=d_rand, qual=d_qual)
    hit_batch = api.device_batch(len(L), padded, t_off, t_len, seq2b=d_hit, qual=d_qual)
    modes = [(k, c, rand_batch) for k, c in ctxs.items()] + [("3.1G_k31_sampled", ctxs["3.1G_k31_random"], hit_batch)]

    def step(ctx, batch):
        ctx.reset_reads()
        ctx.push_device(batch)
        return ctx.finalize(-1)

    for _ in range(a.warmup):
        for _, c, b in modes:
            step(c, b)
    ms = {k: [] for k, _, _ in modes}
    kms = {k: 0.0 for k, _, _ in modes}
    summ, removed = {}, {}
    for _ in range(a.steps):
        for k, c, b in modes:                    # alternated
            c.enable_timing(True)
            c.reset_timing()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            summ[k] = step(c, b)
            c.sync()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
            kms[k] += c.kernel_time("contam")[0]
            removed[k] = int(c.contam_results()[2]["reads"])
    rec = dict(card=card(), reads=len(L), bases=int(L.sum()), steps=a.steps, set_members=members, set_device_gib=mem,
               sectors_per_lookup=probe,
               ms_per_step={k: float(np.median(v)) for k, v in ms.items()},
               ms_per_step_min_max={k: [float(min(v)), float(max(v))] for k, v in ms.items()},
               contam_kernel_ms_per_step={k: v / a.steps for k, v in kms.items()},
               removed=removed, keeping={k: int(s.keeping) for k, s in summ.items()})
    for c in ctxs.values():
        c.close()
    return rec


def cli(a):
    import bgzf_bench
    os.makedirs(a.dir, exist_ok=True)
    fq, fa, fgz, out = (os.path.join(a.dir, x) for x in ("reads.fastq", "big.fa", "big.fa.gz", "out.fastq"))
    rng = np.random.default_rng(3)
    host = []                                          # error-free reads cut from the genome: all of them must go
    with open(fa, "wb") as f, gzip.open(fgz, "wb", compresslevel=1) as z:
        for i, (_, seq) in enumerate(genome_records(1)):
            rec = b">c%d\n%s\n" % (i, seq)
            f.write(rec)
            z.write(rec)
            for p in rng.integers(0, len(seq) - 20000, a.host_reads // 31 + 1):
                host.append(seq[p:p + int(rng.integers(1000, 20000))])
    with open(fq, "wb") as f:
        left, seed = a.cli_gbases, 11
        while left > 0:
            f.write(bgzf_bench.fastq_text(min(left, 2.0) * 1e9 * 2.02, seed=seed).tobytes())
            left -= 2.0
            seed += 1
        for i, s in enumerate(host):
            f.write(b"@host_%d\n%s\n+\n%s\n" % (i, s, b"5" * len(s)))
    env = dict(os.environ, LC_ALL="C", FL_CLI_TIMING="1")
    res = dict(card=card(), fastq_bytes=os.path.getsize(fq), fasta_bytes=os.path.getsize(fa), gzip_bytes=os.path.getsize(fgz),
               host_reads=len(host), host_bases=sum(len(s) for s in host), build_s={}, runs={"p90": [], "contam_k31_p90": []},
               host_reads_kept=[])

    def timed(args):
        t0 = time.perf_counter()
        with open(out, "wb") as f:
            r = subprocess.run([CLI] + args, stdout=f, stderr=subprocess.PIPE, env=env)
        if r.returncode:
            raise SystemExit(r.stderr.decode()[-2000:])
        return round(time.perf_counter() - t0, 3), r.stderr.decode()

    for tag, path in (("fasta", fa), ("gzip", fgz)):
        _, err = timed(["--contam", path, "--contam_k", "31", "--min_length", "1000000000", fq])
        res["build_s"][tag] = [l.strip() for l in err.splitlines() if l.startswith("[timing]") and ("reference" in l or "k-mers" in l)]
    for _ in range(a.cli_runs):
        for tag, args in (("p90", ["-p", "90", fq]), ("contam_k31_p90", ["--contam", fa, "--contam_k", "31", "-p", "90", fq])):
            s, err = timed(args)
            res["runs"][tag].append(s)
            if tag != "p90":
                res["contam_log"] = [l for l in err.splitlines() if "31-mers" in l or "random base" in l]
                with open(out, "rb") as f:
                    res["host_reads_kept"].append(sum(1 for line in f if line.startswith(b"@host_")))
    for p in (fq, fa, fgz, out):
        os.remove(p)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bases", type=float, default=4e9)
    ap.add_argument("--reads", type=float, default=4e5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cli_gbases", type=float, default=0.0)
    ap.add_argument("--cli_runs", type=int, default=2)
    ap.add_argument("--host_reads", type=int, default=6000, help="reads cut from the genome, appended to the CLI's FASTQ")
    ap.add_argument("--dir", default="/tmp/contam_k_bench")
    ap.add_argument("--out", default=None)
    ap.add_argument("--no_device", action="store_true", help="only the CLI part")
    a = ap.parse_args()
    rec = {} if a.no_device else {"device_resident": device_resident(a)}
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
