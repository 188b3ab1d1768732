"""Shared helpers for the test-suite: seeded synthetic inputs and FASTA/FASTQ writers."""
import gzip
import os

import numpy as np

BASES = np.frombuffer(b"ACGT", dtype=np.uint8)
COMP = np.zeros(256, dtype=np.uint8)
for a, b in zip(b"ACGTacgtNn", b"TGCAtgcaNn"):
    COMP[a] = b


def revcomp(seq: bytes) -> bytes:
    a = np.frombuffer(seq, dtype=np.uint8)
    return COMP[a][::-1].tobytes()


def rand_seq(rng, n) -> bytes:
    return BASES[rng.integers(0, 4, size=n)].tobytes()


def mutate(rng, seq: bytes, sub_rate) -> bytes:
    """Substitution-only errors (always to a different base)."""
    a = np.frombuffer(seq, dtype=np.uint8).copy()
    hit = rng.random(a.size) < sub_rate
    idx = np.nonzero(hit)[0]
    code = np.searchsorted(BASES, a[idx])
    a[idx] = BASES[(code + rng.integers(1, 4, size=idx.size)) % 4]
    return a.tobytes()


def rand_qual(rng, n, mean_q=14, sd=4, lo=1, hi=50) -> bytes:
    q = np.clip(np.rint(rng.normal(mean_q, sd, size=n)), lo, hi).astype(np.uint8) + 33
    return q.tobytes()


def long_reads(rng, genome: bytes, n, min_len=200, max_len=20000, junk_frac=0.3, lower_frac=0.05,
               n_frac=0.02):
    """(name, seq, qual) long reads sampled from `genome` on a random strand with per-read
    substitution errors, optional junk blocks (start / middle / end) and a few odd characters."""
    reads = []
    G = len(genome)
    for i in range(n):
        L = int(np.clip(rng.lognormal(8.0, 1.0), min_len, min(max_len, G)))
        s = int(rng.integers(0, G - L + 1))
        seq = genome[s:s + L]
        if rng.random() < 0.5:
            seq = revcomp(seq)
        seq = mutate(rng, seq, rng.uniform(0.0, 0.15))
        if rng.random() < junk_frac:
            parts = []
            if rng.random() < 0.5:
                parts.append(rand_seq(rng, int(rng.integers(1, 120))))
            if rng.random() < 0.5 and L > 400:
                cut = int(rng.integers(100, L - 100))
                parts += [seq[:cut], rand_seq(rng, int(rng.integers(20, 1500))), seq[cut:]]
            else:
                parts.append(seq)
            if rng.random() < 0.5:
                parts.append(rand_seq(rng, int(rng.integers(1, 120))))
            seq = b"".join(parts)
        a = np.frombuffer(seq, dtype=np.uint8).copy()
        if rng.random() < lower_frac:
            a = np.frombuffer(seq.lower(), dtype=np.uint8).copy()
        if rng.random() < n_frac and a.size:
            a[rng.integers(0, a.size, size=3)] = ord("N")
        seq = a.tobytes()
        reads.append(("read_%d" % i, seq, rand_qual(rng, len(seq), mean_q=rng.uniform(5, 30))))
    return reads


def short_reads(rng, genome: bytes, n_pairs, length=100, sub_rate=0.003, insert=300):
    r1, r2 = [], []
    G = len(genome)
    for i in range(n_pairs):
        ins = int(np.clip(rng.normal(insert, 30), length, G))
        s = int(rng.integers(0, G - ins + 1))
        frag = genome[s:s + ins]
        a = mutate(rng, frag[:length], sub_rate)
        b = mutate(rng, revcomp(frag)[:length], sub_rate)
        r1.append(("sr_%d/1" % i, a, b"I" * length))
        r2.append(("sr_%d/2" % i, b, b"I" * length))
    return r1, r2


def _open(path):
    return gzip.open(path, "wb") if str(path).endswith(".gz") else open(path, "wb")


def write_fastq(path, reads):
    with _open(path) as f:
        for name, seq, qual in reads:
            f.write(b"@" + name.encode() + b"\n" + seq + b"\n+\n" + qual + b"\n")
    return str(path)


def write_fasta(path, reads, width=0):
    with _open(path) as f:
        for r in reads:
            name, seq = r[0], r[1]
            f.write(b">" + name.encode() + b"\n")
            if width:
                for i in range(0, len(seq), width):
                    f.write(seq[i:i + width] + b"\n")
            else:
                f.write(seq + b"\n")
    return str(path)


REF_FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_fixtures")


def read_fastx(path):
    """Minimal FASTA/FASTQ reader for the test fixtures (single- or multi-line FASTA, 4-line FASTQ)."""
    op = gzip.open if str(path).endswith(".gz") else open
    recs = []
    with op(path, "rb") as f:
        lines = [l.rstrip(b"\r\n") for l in f]
    i = 0
    while i < len(lines):
        if lines[i].startswith(b"@"):
            recs.append((lines[i][1:].split()[0].decode(), lines[i + 1], lines[i + 3]))
            i += 4
        elif lines[i].startswith(b">"):
            name = lines[i][1:].split()[0].decode()
            i += 1
            seq = []
            while i < len(lines) and not lines[i].startswith(b">"):
                seq.append(lines[i])
                i += 1
            recs.append((name, b"".join(seq), None))
        else:
            i += 1
    return recs


def split_phase_finalize(ctxs, total_bases):
    """Runs the split-phase normalise/select protocol of filtlong_b200/sharding.py over N contexts (rank =
    position in `ctxs`) on ONE GPU, with the all-reduces done by hand on the device buffers (what NCCL does
    between ranks). Returns the per-context summaries."""
    import torch
    from filtlong_b200 import sharding
    world = len(ctxs)
    bks = [sharding.CabiBackend(c) for c in ctxs]
    bufs = [sharding.Buffers(torch, "cuda", world) for _ in ctxs]

    def allreduce(name, op="sum"):
        ts = [getattr(b, name) for b in bufs]
        for c in ctxs:
            c.sync()
        torch.cuda.synchronize()
        st = torch.stack(ts)
        red = st.sum(0) if op == "sum" else (st.min(0).values if op == "min" else st.max(0).values)
        for t in ts:
            t.copy_(red)
        torch.cuda.synchronize()

    for bk, b in zip(bks, bufs):
        bk.norm_partial1(b.sums, b.mn, b.mx)
    allreduce("sums"); allreduce("mn", "min"); allreduce("mx", "max")
    for bk, b in zip(bks, bufs):
        bk.norm_partial2(b.sums, b.mn, b.mx, b.sq)
    allreduce("sq")
    for bk, b in zip(bks, bufs):
        bk.norm_apply(b.sums, b.mn, b.mx, b.sq)
        bk.select_begin(total_bases, b.sums)
    for level in range(8):
        for bk, b in zip(bks, bufs):
            bk.select_hist(level, b.hist)
        allreduce("hist")
        for bk, b in zip(bks, bufs):
            bk.select_pick(level, b.hist)
    for rank, (bk, b) in enumerate(zip(bks, bufs)):
        bk.select_tie_local(b.tie, rank, world)
    allreduce("tie")
    for rank, (bk, b) in enumerate(zip(bks, bufs)):
        bk.select_apply(b.tie, rank, b.keeping)
    allreduce("keeping")
    return [bk.select_summary(b.sums, b.mn, b.mx, b.sq, b.keeping, total_bases) for bk, b in zip(bks, bufs)]
