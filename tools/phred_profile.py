"""Where config 2's step time goes: bench.py's Phred-only workload (bench.phred_workload, default 2 M reads /
20 Gbp, --target_bases 5g), warmed steps under torch.profiler with CUDA activities, the device time of each
kernel per step, and how many reads and bases took each path of k_phred_win (fl_ctx_phred_paths).

    python tools/phred_profile.py [--steps 5] [--warmup 2] [--scale 1.0] [--trace DIR]

Prints the card name and power limit beside the numbers, and writes a Chrome trace to DIR when
--trace is given."""
import argparse
import os
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import bench  # noqa: E402

GROUPS = [("k_phred_first", "k_phred_first"), ("k_phred_sum", "k_phred_sum"), ("k_phred_win", "k_phred_win"),
          ("k_phred_fallback", "k_phred_fallback"), ("order_by_length", "k_bucket"), ("finalize", "")]


def group_of(name):
    for g, key in GROUPS[:-1]:
        if key in name:
            return g
    return "finalize / other"


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--trace", default=None, metavar="DIR", help="also write a Chrome trace there")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from filtlong_b200 import api, capi
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        smi = "nvidia-smi unavailable"
    print("card:", smi)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    n_reads, total = max(int(round(2e6 * args.scale)), 64), int(round(20e9 * args.scale))
    w = bench.phred_workload(0, n_reads, total)
    L = capi.lib()
    ctx = api.Context(api.make_params(target_bases=int(round(5e9 * args.scale))), device=0)
    ctx.set_stream(stream.cuda_stream)
    t_len = torch.from_numpy(w["len"]).to(dev)
    t_off = torch.from_numpy(w["off"].view(np.int64)).to(dev)
    d_qual = torch.empty(w["padded"] + 64, dtype=torch.uint8, device=dev)
    capi.check(ctx.h, L.fl_synth_qual_device(ctx.h, w["seed"], w["n"], t_off.data_ptr(), t_len.data_ptr(),
                                             torch.from_numpy(w["qbar"]).to(dev).data_ptr(), w["read_base"], d_qual.data_ptr()), "synth_qual")
    batch = api.device_batch(w["n"], w["padded"], t_off, t_len, qual=d_qual)

    def step():
        ctx.reset_reads()
        ctx.push_device(batch)
        return ctx.finalize(-1)

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize(dev)
    have_paths = hasattr(ctx, "phred_paths")
    p0 = ctx.phred_paths() if have_paths else None
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize(dev)
    p1 = ctx.phred_paths() if have_paths else None
    per = defaultdict(float)
    names = defaultdict(set)
    for e in prof.events():
        if e.device_type.name == "CUDA" and e.device_time_total > 0 and "Memcpy" not in e.name and "Memset" not in e.name:
            g = group_of(e.name)
            per[g] += e.device_time_total / 1000.0
            names[g].add(e.name.split("(")[0][:60])
    total_ms = sum(per.values()) / args.steps
    print("%d reads, %.3g Gbases, %d timed steps" % (w["n"], w["bases"] / 1e9, args.steps))
    print("%-20s %10s %7s  kernels" % ("group", "ms/step", "share"))
    for g in [g for g, _ in GROUPS[:-1]] + ["finalize / other"]:
        ms = per.get(g, 0.0) / args.steps
        print("%-20s %10.3f %6.1f%%  %s" % (g, ms, 100.0 * ms / total_ms if total_ms else 0.0, ", ".join(sorted(names.get(g, [])))[:120]))
    print("%-20s %10.3f" % ("all kernels", total_ms))
    if have_paths:
        (a0, s0), (a1, s1) = p0, p1
        print("k_phred_win paths per step (reads, bases):")
        for k in a1:
            r, b = (a1[k][0] - a0[k][0]) / args.steps, (a1[k][1] - a0[k][1]) / args.steps
            print("  %-12s %12.0f reads %16.0f bases" % (k, r, b))
        print("  exact steps walked per step: %.0f" % ((s1 - s0) / args.steps))
    else:
        print("k_phred_win paths: not counted by this build")
    if args.trace:
        os.makedirs(args.trace, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.trace, "phred_profile.json"))
    ctx.close()


if __name__ == "__main__":
    main()
