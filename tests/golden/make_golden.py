#!/usr/bin/env python
"""Generates tests/golden/*.json: outputs of the UNMODIFIED reference (oracle/_ref/refdump, i.e.
the reference's own read.o / kmers.o) on seeded synthetic inputs, doubles as C99 hex floats.
Run where oracle/_ref is built (`make -C oracle REF=<Filtlong v0.3.1 source tree>`):

    python tests/golden/make_golden.py

The inputs are regenerated from the seeds by tests (tests/util.py), so only outputs are stored."""
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as orc   # noqa: E402
from tests import util             # noqa: E402

CASES = {
    "phred_seed101": dict(seed=101, mode="phred", opts=dict(keep_percent=70.0, min_length=300)),
    "phred_seed102_ws100": dict(seed=102, mode="phred", opts=dict(target_bases=150000, window_size=100, min_mean_q=75.0)),
    "assembly_seed103_trim_split": dict(seed=103, mode="assembly", opts=dict(keep_percent=80.0, trim=True, split=90)),
    "assembly_seed104_minwin": dict(seed=104, mode="assembly", opts=dict(min_window_q=80.0, split=40)),
    "short_seed105_trim_split": dict(seed=105, mode="short", opts=dict(keep_percent=85.0, trim=True, split=150)),
}


def inputs(case):
    """Deterministic inputs of a golden case (shared with the tests)."""
    rng = np.random.default_rng(case["seed"])
    genome = util.rand_seq(rng, 40000)
    ga = np.frombuffer(genome, dtype=np.uint8).copy()
    ga[500:504] = ord("N")
    genome_n = ga.tobytes()
    reads = util.long_reads(rng, genome, 80, max_len=7000)
    reads.append(("edge15", genome[100:115], b"I" * 15))
    reads.append(("edge16", genome[200:216], b"I" * 16))
    reads.append(("junk", util.rand_seq(rng, 600), b"5" * 600))
    reads.append(("sandwich", util.rand_seq(rng, 40) + genome[3000:3300] + util.rand_seq(rng, 200) + genome[8000:8400], b"7" * 940))
    short = util.short_reads(rng, genome, 6000) if case["mode"] == "short" else None
    return genome_n, reads, short


def h(x):
    return float(x).hex()


def main():
    assert orc.have_ref(), "build oracle/_ref first (make -C oracle REF=<Filtlong v0.3.1 source tree>)"
    os.environ.setdefault("FL_REFERENCE_RECORD", os.devnull)      # live runs of the reference binaries
    out_dir = os.path.dirname(os.path.abspath(__file__))
    for name, case in CASES.items():
        genome_n, reads, short = inputs(case)
        with tempfile.TemporaryDirectory() as td:
            fq = util.write_fastq(os.path.join(td, "r.fastq"), reads)
            cli = orc.params_to_cli(orc.make_params(**case["opts"]))
            if case["mode"] == "assembly":
                cli += ["-a", util.write_fasta(os.path.join(td, "a.fasta"), [("g", genome_n)], width=70)]
            elif case["mode"] == "short":
                cli += ["-1", util.write_fastq(os.path.join(td, "s1.fastq"), short[0]),
                        "-2", util.write_fastq(os.path.join(td, "s2.fastq"), short[1])]
            kout = os.path.join(td, "k.bin")
            ref = orc.run_refdump(cli + [fq], kmers_out=kout)
            kmers = np.fromfile(kout, dtype=np.uint32)
        gold = {
            "case": case, "n_kmers": ref["n_kmers"],
            "kmers_checksum": int(np.bitwise_xor.reduce(kmers.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15))) if kmers.size else 0,
            "reads": [dict(length=r["length"], mean_q=h(r["mean_q"]), window_q=h(r["window_q"]), passed=r["passed"],
                           first=r["first"], last=r["last"], bad=r["bad"],
                           children=[dict(start=c["start"], end=c["end"], mean_q=h(c["mean_q"]), window_q=h(c["window_q"]),
                                          passed=c["passed"]) for c in r["children"]]) for r in ref["reads"]],
            "rows": [dict(name=r["name"], length=r["length"], final_score=h(r["final_score"]), passed_final=r["passed_final"])
                     for r in ref["rows"]],
            "tail": ref["tail"],
        }
        with open(os.path.join(out_dir, name + ".json"), "w") as f:
            json.dump(gold, f, indent=0, separators=(",", ":"))
        print(name, len(gold["reads"]), "reads", len(gold["rows"]), "rows", "kmers", gold["n_kmers"])


if __name__ == "__main__":
    main()
