"""What `--trim_q` costs on the GPU: device-resident scoring + finalise of config-2-shaped Phred reads (lognormal lengths,
per-read mean quality ~N(14, 4), qualities from the library's own generator), plain Phred mode beside
`--trim_q Q --trim --split N`, alternated step by step. Reports ms per step of each, the per-kernel event times of the
--trim_q path (quality mask, the row passes, the gather of the children's qualities, the Phred pass over the children,
every Phred kernel together), rows and kept bases, and the card's name and power limit read in the same call, as one
JSON line.

    python tools/qtrim_bench.py [--bases 4e9] [--reads 4e5] [--steps 5] [--warmup 2] [--trim_q 10] [--split 500]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def workload(n_reads, total_bases, seed=1):
    """lengths lognormal(8.517, 1.177) in [200, 1e6] rescaled to the total, 64-aligned arena, per-read mean quality"""
    rng = np.random.default_rng(1000 + seed)
    L = np.clip(np.random.default_rng(seed * 7919).lognormal(8.517, 1.177, size=n_reads), 200, 1_000_000)
    for _ in range(4):
        L = np.clip(L * (total_bases / L.sum()), 200, 1_000_000)
    L = np.floor(L).astype(np.int32)
    padded = (L.astype(np.int64) + 63) & ~63
    off = np.zeros(n_reads, dtype=np.uint64)
    off[1:] = np.cumsum(padded)[:-1].astype(np.uint64)
    qbar = np.clip(np.rint(rng.normal(14, 4, size=n_reads)), 5, 30).astype(np.uint8)
    return L, off, int(padded.sum()), qbar


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bases", type=float, default=4e9)
    ap.add_argument("--reads", type=float, default=4e5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--trim_q", type=int, default=10)
    ap.add_argument("--split", type=int, default=500)
    ap.add_argument("--window_size", type=int, default=250)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from filtlong_b200 import api, capi

    L, off, padded, qbar = workload(int(a.reads), a.bases)
    dev = torch.device("cuda:0")
    t_len, t_off = torch.from_numpy(L).to(dev), torch.from_numpy(off.view(np.int64)).to(dev)
    d_qual = torch.empty(padded + 64, dtype=torch.uint8, device=dev)
    target = int(L.sum()) // 2
    modes = {"plain": api.make_params(target_bases=target, window_size=a.window_size),
             "trim_q": api.make_params(target_bases=target, window_size=a.window_size, trim=True, split=a.split, trim_q=a.trim_q)}
    ctxs = {k: api.Context(p) for k, p in modes.items()}
    lib = capi.lib()
    c0 = ctxs["plain"]
    capi.check(c0.h, lib.fl_synth_qual_device(c0.h, 1, len(L), t_off.data_ptr(), t_len.data_ptr(),
                                               torch.from_numpy(qbar).to(dev).data_ptr(), 0, d_qual.data_ptr()), "synth_qual")
    torch.cuda.synchronize()
    batch = api.device_batch(len(L), padded, t_off, t_len, qual=d_qual)

    def step(ctx):
        ctx.reset_reads()
        ctx.push_device(batch)
        return ctx.finalize(-1)

    for _ in range(a.warmup):
        for c in ctxs.values():
            step(c)
    ms = {k: [] for k in ctxs}
    kernels = ["qual_mask", "row_scan", "qual_gather", "qual_children", "score_phred"]
    ctxs["trim_q"].enable_timing(True)
    ctxs["trim_q"].reset_timing()
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
    kt = {k: ctxs["trim_q"].kernel_time(k)[0] / a.steps for k in kernels}
    counts = {k: c.counts() for k, c in ctxs.items()}
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    rec = {
        "card": gpu.strip().splitlines()[0] if gpu.strip() else torch.cuda.get_device_name(0),
        "reads": len(L), "bases": int(L.sum()), "target_bases": target, "trim_q": a.trim_q, "split": a.split,
        "window_size": a.window_size, "steps": a.steps,
        "ms_per_step": {k: float(np.median(v)) for k, v in ms.items()},
        "ms_per_step_min_max": {k: [float(min(v)), float(max(v))] for k, v in ms.items()},
        "trim_q_kernel_ms_per_step": kt,
        "rows": {k: int(v[1]) for k, v in counts.items()},
        "kept_bases": {k: int(s.keeping) for k, s in summ.items()},
        "summary": {k: dict(status=int(s.status), target=int(s.target), passed_bases=int(s.passed_bases),
                            keeping=int(s.keeping), rows_bases=int(s.rows_bases)) for k, s in summ.items()},
    }
    rec["ratio"] = rec["ms_per_step"]["trim_q"] / rec["ms_per_step"]["plain"]
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    for c in ctxs.values():
        c.close()


if __name__ == "__main__":
    main()
