"""Worker of tests/test_nccl_ranks.py: one rank = one process = one GPU = one context with a communicator.
argv: rank nranks workdir. Reads its shard from workdir/input.npz, writes workdir/out_<rank>.npz."""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rank, nranks, wd = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
    from filtlong_b200 import api, sharding
    z = np.load(os.path.join(wd, "input.npz"), allow_pickle=True)
    seqs, quals, assembly, opts = list(z["seqs"]), list(z["quals"]), list(z["assembly"]), z["opts"].item()
    ctx = api.Context(api.make_params(**opts), device=rank)
    idf = os.path.join(wd, "nccl_id")
    if rank == 0:
        with open(idf + ".tmp", "wb") as f:
            f.write(api.Context.comm_unique_id())
        os.rename(idf + ".tmp", idf)
    t0 = time.time()
    while not os.path.exists(idf):
        if time.time() - t0 > 120:
            raise SystemExit("no NCCL id")
        time.sleep(0.05)
    ctx.comm_init(open(idf, "rb").read(), rank, nranks)
    if assembly:
        if rank == 0:
            ctx.kmers_add(assembly, False)          # Kmers built on one rank ...
        ctx.kmers_broadcast(0)                      # ... used by all (main.cpp:53-59 once per run)
    n_k = ctx.kmers_count()
    lo, hi = sharding.shard_by_bases([len(s) for s in seqs], nranks)[rank]
    if hi > lo:
        ctx.push(api.HostBatch(seqs[lo:hi], quals[lo:hi] if not assembly else None, want_seq=bool(assembly)))
    summ = ctx.finalize(-1)                         # collective: NCCL inside
    rows = ctx.row_results()
    np.savez(os.path.join(wd, "out_%d.npz" % rank), lo=lo, hi=hi, n_kmers=n_k, passed_final=rows["passed_final"], start=rows["start"],
             end=rows["end"], final_score=rows["final_score"], mean_q=rows["mean_q"], window_q=rows["window_q"],
             passed=rows["passed"], length_score=rows["length_score"], norm_mean=rows["norm_mean"], norm_window=rows["norm_window"],
             summary=np.array([summ.status, summ.target, summ.keeping, summ.passed_bases, summ.total_bases, summ.rows_bases],
                              dtype=np.int64),
             stats=np.array([summ.min_q, summ.max_q, summ.mean_q, summ.stdev_q, summ.min_z, summ.max_z]),
             collectives=ctx.collective_count())
    ctx.comm_destroy()
    ctx.close()


if __name__ == "__main__":
    main()
