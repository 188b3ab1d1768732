"""Committed golden vectors (tests/golden/*.json = outputs of the unmodified reference on seeded
inputs, made by tests/golden/make_golden.py). CPU: the C restatement must reproduce them.
GPU: the CUDA path must reproduce them. Neither needs /root/reference or oracle/_ref at run time."""
import glob
import json
import os

import numpy as np
import pytest

from oracle import oracle as orc
from tests import parity
from tests.golden.make_golden import inputs

GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.json")))


def load(path):
    g = json.load(open(path))
    genome_n, reads, short = inputs(g["case"])
    return g, genome_n, [(s, q) for _, s, q in reads], short


def check_reads(g, get):
    """get(i) -> dict(mean_q, window_q, passed, first, last, children=[(start,end,mean,window,passed)])"""
    for i, r in enumerate(g["reads"]):
        o = get(i)
        assert parity.same(o["mean_q"], float.fromhex(r["mean_q"])), ("mean", i)
        assert parity.same(o["window_q"], float.fromhex(r["window_q"])), ("window", i)
        assert (o["passed"], o["first"], o["last"]) == (r["passed"], r["first"], r["last"]), i
        assert len(o["children"]) == len(r["children"]), i
        for c, k in zip(o["children"], r["children"]):
            assert (c[0], c[1]) == (k["start"], k["end"])
            assert parity.same(c[2], float.fromhex(k["mean_q"])) and parity.same(c[3], float.fromhex(k["window_q"]))
            assert c[4] == k["passed"]


def kmers_checksum(kmers):
    k = np.asarray(kmers, dtype=np.uint64)
    return int(np.bitwise_xor.reduce(k * np.uint64(0x9E3779B97F4A7C15))) if k.size else 0


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p)[:-5] for p in GOLD])
def test_oracle_restatement_reproduces_golden(path):
    g, genome_n, reads, short = load(path)
    p = orc.make_params(**g["case"]["opts"])
    ok = None
    if g["case"]["mode"] == "assembly":
        ok = orc.Kmers(); ok.add_assembly([genome_n])
    elif g["case"]["mode"] == "short":
        ok = orc.Kmers()
        for f in short:
            ok.add_short_reads([r[1] for r in f])
    sc = orc.finalize(orc.score(reads, p, ok), p)
    if ok is not None:
        assert len(ok) == g["n_kmers"] and kmers_checksum(ok.dump()) == g["kmers_checksum"]
    check_reads(g, lambda i: dict(mean_q=sc.parents[i].mean_q, window_q=sc.parents[i].window_q, passed=sc.parents[i].passed,
                                  first=sc.parents[i].first, last=sc.parents[i].last,
                                  children=[(c.start, c.end, c.mean_q, c.window_q, c.passed) for c in sc.children[i]]))
    assert len(sc.rows) == len(g["rows"])
    for r, gr in zip(sc.rows, g["rows"]):
        assert parity.same(r.final_score, float.fromhex(gr["final_score"]))
    parity.check_selection([r.passed_final for r in sc.rows], [gr["passed_final"] for gr in g["rows"]],
                           [float.fromhex(gr["final_score"]) for gr in g["rows"]], [gr["length"] for gr in g["rows"]])
    assert sc.summary.keeping == g["tail"]["keeping"] and sc.summary.status == g["tail"]["status"]


@pytest.mark.gpu
@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p)[:-5] for p in GOLD])
def test_cuda_path_reproduces_golden(path):
    from filtlong_b200 import api
    g, genome_n, reads, short = load(path)
    p = api.make_params(**g["case"]["opts"])
    asm = [genome_n] if g["case"]["mode"] == "assembly" else None
    sh = [[r[1] for r in f] for f in short] if g["case"]["mode"] == "short" else None
    ctx, summ = api.score_and_filter(reads, p, assembly=asm, short_reads=sh)
    if asm or sh:
        assert ctx.kmers_count() == g["n_kmers"] and kmers_checksum(ctx.kmers_export()) == g["kmers_checksum"]
    rr, rw = ctx.read_results(), ctx.row_results()

    def get(i):
        rs = int(rr["row_start"][i])
        kids = [(int(rw["start"][rs + c]), int(rw["end"][rs + c]), rw["mean_q"][rs + c], rw["window_q"][rs + c],
                 int(rw["passed"][rs + c])) for c in range(int(rr["n_child"][i]))]
        return dict(mean_q=rr["mean_q"][i], window_q=rr["window_q"][i], passed=int(rr["passed"][i]),
                    first=int(rr["first_base_in_kmer"][i]), last=int(rr["last_base_in_kmer"][i]), children=kids)
    check_reads(g, get)
    assert len(rw["parent"]) == len(g["rows"])
    for i, gr in enumerate(g["rows"]):
        assert parity.close(rw["final_score"][i], float.fromhex(gr["final_score"]))     # 1e-5 relative (north star)
    parity.check_selection([int(x) for x in rw["passed_final"]], [gr["passed_final"] for gr in g["rows"]],
                           [float.fromhex(gr["final_score"]) for gr in g["rows"]], [gr["length"] for gr in g["rows"]])
    assert summ.keeping == g["tail"]["keeping"] and summ.status == g["tail"]["status"]
    parity.check_rescale_exact(rw, summ, p)
    parity.check_selection_exact(rw, summ, p)
    ctx.close()
