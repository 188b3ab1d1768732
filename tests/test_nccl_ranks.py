"""The sharded path as the product runs it: one process per GPU, one NCCL communicator behind the C ABI
(fl_comm_init / fl_kmers_broadcast / collective fl_finalize). Needs >= 2 GPUs (skipped otherwise):
    python -m pytest tests/test_nccl_ranks.py -m gpu      (on a machine with two or more GPUs)
The union of the ranks' rows must equal what one context computes on the whole read set, and the oracle."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest

from tests import parity, util

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("mode,opts", [("phred", dict(keep_percent=60.0)), ("phred", dict(target_bases=400000, min_length=300)),
                                       ("kmer", dict(keep_percent=70.0, trim=True, split=100))])
def test_nccl_ranks_equal_single_context(mode, opts, tmp_path):
    n = min(_ngpus(), 4)
    if n < 2:
        pytest.skip("needs at least 2 GPUs")
    from filtlong_b200 import api
    from oracle import oracle as orc
    rng = np.random.default_rng(77)
    genome = util.rand_seq(rng, 40000)
    reads = [(s, q) for _, s, q in util.long_reads(rng, genome, 300, max_len=6000)]
    reads = reads + reads[:40]                    # exact ties that can straddle the cut-off and a shard boundary
    assembly = [genome] if mode == "kmer" else []
    np.savez(tmp_path / "input.npz", seqs=np.array([r[0] for r in reads], dtype=object), quals=np.array([r[1] for r in reads], dtype=object),
             assembly=np.array(assembly, dtype=object), opts=np.array(opts, dtype=object))
    ps = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "nccl_worker.py"), str(r), str(n), str(tmp_path)],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(n)]
    outs = [p.communicate(timeout=600)[0] for p in ps]
    assert all(p.returncode == 0 for p in ps), "\n".join(outs)
    z = [np.load(tmp_path / ("out_%d.npz" % r)) for r in range(n)]
    p, op = api.make_params(**opts), orc.make_params(**opts)
    one, summ = api.score_and_filter(reads, p, assembly=assembly or None)
    rows = one.row_results()
    for k in ("start", "end", "passed_final"):
        assert np.array_equal(np.concatenate([x[k] for x in z]), rows[k]), k
    for k in ("mean_q", "window_q"):
        assert np.array_equal(np.concatenate([x[k] for x in z]).view(np.uint64), rows[k].view(np.uint64)), k
    assert np.allclose(np.concatenate([x["final_score"] for x in z]), rows["final_score"], rtol=1e-9, atol=0, equal_nan=True)
    for x in z:
        assert tuple(x["summary"][:4]) == (summ.status, summ.target, summ.keeping, summ.passed_bases)
        assert int(x["summary"][4]) == sum(len(r[0]) for r in reads)
        assert int(x["collectives"]) > 0
    ok = None
    if assembly:
        ok = orc.Kmers()
        ok.add_assembly(assembly)
        assert all(int(x["n_kmers"]) == len(ok) for x in z)
    sc = orc.finalize(orc.score([(s, q if not assembly else None) for s, q in reads], op, ok), op)
    got = [int(v) for v in np.concatenate([x["passed_final"] for x in z])]
    # exact, against the ranks' own statistics and scores (every rank holds the same summary)
    cat = {k: np.concatenate([x[k] for x in z]) for k in ("start", "end", "passed", "passed_final", "mean_q", "window_q",
                                                          "length_score", "norm_mean", "norm_window", "final_score")}
    sv, st = z[0]["summary"], z[0]["stats"]
    s0 = types.SimpleNamespace(status=int(sv[0]), target=int(sv[1]), keeping=int(sv[2]), passed_bases=int(sv[3]),
                               total_bases=int(sv[4]), rows_bases=int(sv[5]), min_q=st[0], max_q=st[1], mean_q=st[2],
                               stdev_q=st[3], min_z=st[4], max_z=st[5])
    parity.check_rescale_exact(cat, s0, p, nranks=n)
    parity.check_selection_exact(cat, s0, p)
    parity.check_selection(got, [r.passed_final for r in sc.rows], [r.final_score for r in sc.rows], [r.length for r in sc.rows])
    one.close()
