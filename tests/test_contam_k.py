"""`--contam_k K`: the contaminant set of k-mers of 17 to 32 bases, a device hash set of canonical k-mers.

What these tests check: the argument errors and the help line (no GPU); the numpy model of the set and of c against a
brute-force string version (no GPU); on the GPU, the set's count, members and look-ups against the model on every add
path, c bit-identical to the model on every push path for designed reads, a table filled to within a few percent of its
load limit, the API's refusals, the CLI's stdout against its own run on the model-filtered input, and a human-sized set."""
import gzip
import os
import subprocess
import threading

import numpy as np
import pytest

from tests import bam_util as bu
from tests import contam_k_model as km
from tests import util
from tests.test_cli import CLI, log_lines, need_cli
from tests.test_contam import (_push_all, fastq, filtered_args, gpu_count, io_path, make_inputs, run, wrapped_fasta)

LONG_KS = list(range(17, 33))


# ---- argument errors and help (no GPU) --------------------------------------------------------------------------------
ERRORS = [(["--contam_k", "31", "-p", "90", "FQ"], "Error: --contam_k needs --contam")] + [
    (["--contam", "FA", "--contam_k", v, "-p", "90", "FQ"], "Error: the value for --contam_k must be an integer from 16 to 32")
    for v in ("15", "33", "0", "24.5", "-1", "x")]


@need_cli
@pytest.mark.parametrize("args,message", ERRORS, ids=lambda x: " ".join(x) if isinstance(x, list) else None)
def test_argument_errors(args, message, tmp_path):
    fq = util.write_fastq(tmp_path / "x.fastq", [("r1", b"ACGT" * 10, b"I" * 40)])
    fa = util.write_fasta(tmp_path / "a.fasta", [("c", b"ACGT" * 10)])
    rc, out, err = run([{"FQ": fq, "FA": fa}.get(a, a) for a in args])
    assert (rc, out, err.decode()) == (1, b"", message + "\n")


@need_cli
def test_help_lists_contam_k_after_max_contam():
    rc, out, err = run(["--help"])
    text = err.decode()
    assert rc == 0 and "--contam_k [int]" in text
    assert text.index("contaminant removal:") < text.index("--max_contam [float]") < text.index("--contam_k [int]") \
        < text.index("read manipulation:")


# ---- the model against its definition (no GPU) -------------------------------------------------------------------------
def random_case(rng, k):
    """contaminant records with lowercase, N and IUPAC letters, palindromes (even k) and lengths k - 1, k, k + 1; reads
    with planted contaminant k-mers (either strand) and N"""
    recs = []
    for _ in range(4):
        s = bytearray(util.rand_seq(rng, int(rng.integers(k + 2, 4 * k))))
        for p in rng.integers(0, len(s), 3):
            s[p] = rng.choice(list(b"NRYKMSWBDHVn"))
        lo = int(rng.integers(0, len(s)))
        s[lo:lo + 10] = bytes(s[lo:lo + 10]).lower()
        recs.append(bytes(s))
    for L in (k - 1, k, k + 1):
        recs.append(util.rand_seq(rng, L))
    if k % 2 == 0:
        h = util.rand_seq(rng, k // 2)
        recs.append(util.rand_seq(rng, 5) + h + util.revcomp(h) + util.rand_seq(rng, 3))
    reads = [b"", util.rand_seq(rng, k - 1)]
    for _ in range(8):
        src = recs[int(rng.integers(0, len(recs)))].upper()
        if len(src) < k:
            continue
        p = int(rng.integers(0, len(src) - k + 1))
        w = src[p:p + k]
        if rng.random() < 0.5:
            w = util.revcomp(w)
        pre, post = util.rand_seq(rng, int(rng.integers(0, 40))), util.rand_seq(rng, int(rng.integers(0, 40)))
        r = bytearray(pre + w + post)
        if rng.random() < 0.3:
            r[int(rng.integers(0, len(r)))] = ord("N")
        reads.append(bytes(r))
    return recs, reads


@pytest.mark.parametrize("k", LONG_KS)
def test_model_equals_brute_force(k):
    rng = np.random.default_rng(100 + k)
    pal_seen = 0
    for _ in range(6):
        recs, reads = random_case(rng, k)
        members, m = km.kmer_set(recs, k)
        canon, m_bf = km.brute_set(recs, k)
        assert set(int(x) for x in members) == canon and m == m_bf
        pal_seen += 2 * len(canon) - m_bf
        for r in reads:
            a, b = km.percent(r, members, k), km.brute_percent(r, canon, k)
            assert (np.isnan(a) and np.isnan(b)) or a == b, (r, a, b)
        assert np.array_equal(km.canonical(km.revcomp(members, k), k), members)
    assert (pal_seen > 0) == (k % 2 == 0)


# ---- GPU: the set ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("contam_k")
    genome, contam, reads = make_inputs()
    rng = np.random.default_rng(77)
    c = bytearray(contam)
    for p in rng.integers(0, len(c), 60):                   # IUPAC letters, besides test_contam's lowercase and N runs
        c[p] = rng.choice(list(b"RYKMSWBDHVrykm"))
    records = [bytes(c)] + [util.rand_seq(rng, L) for L in (16, 20, 23, 24, 25, 30, 31, 32, 33)]
    fa = b"".join(wrapped_fasta(b"c%d" % i, s) for i, s in enumerate(records))
    (d / "contam.fa").write_bytes(fa)
    with gzip.open(d / "contam.fa.gz", "wb") as f:
        f.write(fa)
    fq_text = b"".join(b"@c%d\n%s\n+\n%s\n" % (i, s, b"I" * len(s)) for i, s in enumerate(records))
    util.write_fasta(d / "sample.fa", [("chr", genome)], width=80)
    text = fastq(reads)
    (d / "reads.fastq").write_bytes(text)
    with gzip.open(d / "reads.fastq.gz", "wb") as f:
        f.write(text)
    return dict(dir=d, genome=genome, records=records, fa=fa, fq_text=fq_text, reads=reads, text=text,
                cfa=str(d / "contam.fa"), cgz=str(d / "contam.fa.gz"), sample=str(d / "sample.fa"),
                fq=str(d / "reads.fastq"), gz=str(d / "reads.fastq.gz"), bases=sum(len(r[1]) for r in reads), sets={})


def model_set(inputs, k):
    if k not in inputs["sets"]:
        inputs["sets"][k] = km.kmer_set(inputs["records"], k)
    return inputs["sets"][k]


def contam_ctx(inputs, k, how="fasta", params=None):
    from filtlong_b200 import api
    ctx = api.Context(params or api.make_params())
    ctx.contam_configure(k, sum(len(s) for s in inputs["records"]))
    if how == "fasta":
        assert ctx.contam_add_text(inputs["fa"], fastq=False)["status"] == "ok"
    elif how == "fastq":
        assert ctx.contam_add_text(inputs["fq_text"], fastq=True)["status"] == "ok"
    else:
        ctx.contam_add(inputs["records"])
    return ctx


@pytest.mark.gpu
@pytest.mark.parametrize("k", [17, 20, 24, 31, 32])
def test_set_equals_the_model(inputs, k):
    members, m = model_set(inputs, k)
    rng = np.random.default_rng(k)
    for how in ("fasta", "fastq", "batch"):
        with contam_ctx(inputs, k, how) as ctx:
            assert ctx.contam_count() == m, how
            assert np.array_equal(ctx.contam_export64(), members), how
            present = members[rng.integers(0, len(members), 2000)]
            absent = rng.integers(0, 1 << (2 * k), 2000, dtype=np.uint64)
            want_absent = np.isin(km.canonical(absent, k), members)
            assert ctx.contam_contains64(present).all()
            assert ctx.contam_contains64(km.revcomp(present, k)).all()
            assert np.array_equal(ctx.contam_contains64(absent), want_absent)
            assert ctx.kmers_count() == 0


# ---- GPU: percentages -------------------------------------------------------------------------------------------------------
def designed_reads(inputs, k, P):
    """contaminant k-mers planted at every start around lane (32), step (1,024) and tile (8,192) seams, reverse-complement
    plants, a plant with an N inside, reads of k - 1, k and k + 1 bases, and one read with c == P exactly"""
    rng = np.random.default_rng(1000 + k)
    src = inputs["records"][0].upper()
    members = model_set(inputs, k)[0]

    def kmer():
        while True:
            p = int(rng.integers(0, len(src) - k))
            w = src[p:p + k]
            if not w.strip(b"ACGT"):
                return w if rng.random() < 0.5 else util.revcomp(w)

    out = []
    for seam in (32, 1024, 8192, 16384):
        for d in range(-40, 24):
            s = seam + d
            r = bytearray(util.rand_seq(rng, seam + 64))
            r[s:s + k] = kmer()
            out.append(bytes(r))
    for L in (k - 1, k, k + 1):
        w = kmer()
        out.append((w + util.rand_seq(rng, 1))[:L])
    w = bytearray(kmer())
    w[k // 2] = ord("N")
    out.append(util.rand_seq(rng, 50) + bytes(w) + util.rand_seq(rng, 50))
    while True:                                             # c == P exactly: kept (only c > P removes)
        L = int(round(k * 100 / P))
        r = kmer() + util.rand_seq(rng, L - k)
        if km.percent(r, members, k) == P:
            out.append(r)
            break
    return [("designed_%d" % i, s, util.rand_qual(rng, len(s))) for i, s in enumerate(out)]


@pytest.mark.gpu
@pytest.mark.parametrize("how", ["push", "push_text", "push_device", "push_bam"])
@pytest.mark.parametrize("k", [17, 24, 31, 32])
@pytest.mark.parametrize("with_reference", [False, True])
def test_percentages_equal_the_model(inputs, how, k, with_reference):
    from filtlong_b200 import api
    P = 50.0
    reads = [r for r in inputs["reads"] if len(r[1]) > 0] + designed_reads(inputs, k, P)
    if how == "push":
        reads = reads + [("empty", b"", b"")]
    members = model_set(inputs, k)[0]
    c = km.percents([r[1] for r in reads], members, k)
    assert (c == P).sum() >= 1 and (c > P).sum() > 0 and ((c > 0) & (c <= P)).sum() > 0
    with contam_ctx(inputs, k, params=api.make_params(max_contam=P, keep_percent=90)) as ctx:
        if with_reference:
            ctx.kmers_add_text(open(inputs["sample"], "rb").read(), fastq=False)
        _push_all(ctx, reads, how)
        pct, removed, counts = ctx.contam_results()
    ok = ~np.isnan(c)
    assert np.array_equal(np.isnan(pct), np.isnan(c))
    assert np.array_equal(pct.view(np.uint64)[ok], c.view(np.uint64)[ok])
    assert np.array_equal(removed, c > P)
    assert counts["reads"] == int((c > P).sum())


# ---- GPU: a table near its load limit, and the API's refusals ------------------------------------------------------------
@pytest.mark.gpu
def test_full_table_and_refusals():
    from filtlong_b200 import api, capi
    k = 31
    rng = np.random.default_rng(5)
    limit = 4 * 4096 // 5 * 4                  # 2^12 buckets of 4 slots, at most 4/5 of them taken: 13,104 members
    recs = [util.rand_seq(rng, 2000) for _ in range(6)] + [util.rand_seq(rng, 1180 + k - 1)]   # 13,000 windows
    members, m = km.kmer_set(recs, k)
    assert limit - len(members) < 0.02 * limit
    reads = [(b"r%d" % i, s[:600] + util.rand_seq(rng, 300), b"I" * 900) for i, s in enumerate(recs)]
    reads += [(b"x%d" % i, util.rand_seq(rng, 700), b"I" * 700) for i in range(20)]
    with api.Context(api.make_params(max_contam=50.0, keep_percent=90)) as ctx:
        ctx.contam_configure(k, limit)
        ctx.contam_add(recs)
        assert ctx.contam_count() == m and np.array_equal(ctx.contam_export64(), members)
        hits, misses = ctx.contam_probe_lengths(8)
        assert hits.sum() == len(members) and hits[2:].sum() > 0       # chains cross bucket boundaries
        assert misses.sum() == 4096 and misses[2:].sum() > 0
        absent = rng.integers(0, 1 << (2 * k), 5000, dtype=np.uint64)
        assert ctx.contam_contains64(members).all() and ctx.contam_contains64(km.revcomp(members, k)).all()
        assert np.array_equal(ctx.contam_contains64(absent), np.isin(km.canonical(absent, k), members))
        with pytest.raises(capi.FLError, match="reserved for 13104"):
            ctx.contam_add([util.rand_seq(rng, 200)])                   # 170 more windows: beyond the reservation
        assert ctx.contam_count() == m
        with pytest.raises(capi.FLError):
            ctx.contam_configure(24, 100)                                # after an add
        ctx.push(api.HostBatch([r[1] for r in reads], [r[2] for r in reads], want_seq=True))
        pct, _, _ = ctx.contam_results()
        c = km.percents([r[1] for r in reads], members, k)
        assert np.array_equal(pct.view(np.uint64), c.view(np.uint64)) and (c > 50).sum() >= 7
    with api.Context() as ctx:
        for bad in (15, 33):
            with pytest.raises(capi.FLError):
                ctx.contam_configure(bad, 100)
        with pytest.raises(capi.FLError, match="GiB"):
            ctx.contam_configure(31, 1 << 40)
        ctx.contam_configure(31, 100)                                    # still usable after the refusal
        ctx.contam_add([util.rand_seq(rng, 60)])
        assert ctx.contam_count() == 60
        with pytest.raises(capi.FLError):
            ctx.contam_export()                                          # 16-mer export on a long set


# ---- GPU: the CLI ---------------------------------------------------------------------------------------------------------
def strip_k(config):
    out, i = [], 0
    while i < len(config):
        if config[i] == "--contam_k":
            i += 2
        else:
            out, i = out + [config[i]], i + 1
    return out


CONFIGS = [
    ["--contam", "C", "--contam_k", "31", "-p", "90"],
    ["--contam", "C", "--contam_k", "24", "-a", "S", "--trim", "--split", "500", "-p", "70"],
    ["--contam", "C", "--contam_k", "32", "--max_contam", "20", "--trim_q", "10", "--trim", "--split", "500", "-p", "90"],
]


def cli_case(inputs, config, tmp_path):
    k = int(config[config.index("--contam_k") + 1])
    P = float(config[config.index("--max_contam") + 1]) if "--max_contam" in config else 50.0
    members, m = model_set(inputs, k)
    c = km.percents([r[1] for r in inputs["reads"]], members, k)
    kept = [r for r, x in zip(inputs["reads"], c) if not x > P]
    path = tmp_path / "filtered.fastq"
    path.write_bytes(fastq(kept))
    sub = {"C": inputs["cfa"], "S": inputs["sample"]}
    args = [sub.get(a, a) for a in config]
    return k, P, c, m, args, filtered_args(strip_k(args), inputs["bases"]), str(path)


@need_cli
@pytest.mark.gpu
@pytest.mark.parametrize("j", range(len(CONFIGS)))
def test_cli_equals_its_run_on_the_filtered_input(inputs, j, tmp_path):
    k, P, c, m, args, fargs, fpath = cli_case(inputs, CONFIGS[j], tmp_path)
    assert 0 < (c > P).sum() < len(c) and ((c > 0) & ~(c > P)).sum() > 0
    rc, out, err = run(args + [inputs["fq"]])
    assert rc == 0, err[-2000:]
    rc2, want, err2 = run(fargs + [fpath])
    assert rc2 == 0 and out == want and len(out) > 0, err2[-2000:]
    lines = log_lines(err.decode())
    assert "Hashing %d-mers from contaminant sequences" % k in lines
    assert "  %d contigs, %d %d-mers" % (len(inputs["records"]), m, k) in lines
    p = -np.expm1(k * np.log1p(-m / 4.0 ** k))
    assert "  a random base lies in one of them with probability %.3g" % p in lines
    removed_bases = sum(len(r[1]) for r, x in zip(inputs["reads"], c) if x > P)
    assert "  %d reads (%d bp) with more than %g%% of bases in contaminant %d-mers" % ((c > P).sum(), removed_bases, P, k) in lines
    if j:
        return
    variants = [(inputs["gz"], None, None, inputs["cfa"]), ("-", inputs["text"], None, inputs["cfa"]),
                (inputs["fq"], None, {"FL_CHUNK_MB": "1"}, inputs["cfa"]), (inputs["fq"], None, {"FL_HOST_PARSER": "1"}, inputs["cfa"]),
                (inputs["fq"], None, {"FL_HOST_PARSER": "1"}, inputs["cgz"]), (inputs["fq"], None, None, inputs["cgz"])]
    if gpu_count() >= 2:
        variants.append((inputs["fq"], None, {"FL_CHUNK_MB": "1"}, inputs["cfa"], ["--gpus", "2"]))
    for v in variants:
        path, data, env, cont = v[:4]
        extra = v[4] if len(v) > 4 else []
        a = extra + [cont if x == inputs["cfa"] else x for x in args]
        rc, o, e = run(a + [path], data, env)
        assert rc == 0 and o == out, (path, env, cont, e[-2000:])
    rc, z, e = run(["--bgzip"] + args + [inputs["fq"]])
    assert rc == 0 and gzip.decompress(z) == out
    failed = tmp_path / "failed.fastq"
    rc, o, e = run(args + ["--failed", str(failed), inputs["fq"]])
    assert rc == 0 and o == out
    kept = {r[0] for r in util.read_fastx(io_path(tmp_path, out))}
    lost = {r[0] for r in util.read_fastx(str(failed))}
    assert kept | lost == {r[0] for r in inputs["reads"]} and not kept & lost
    assert {r[0] for r, x in zip(inputs["reads"], c) if x > P} <= lost


def run_with_pipe(args, data, env_extra=None):
    """the CLI with `PIPE` in args replaced by /dev/fd/N, the read end of a pipe that a thread fills with data"""
    r, w = os.pipe()

    def feed():
        with os.fdopen(w, "wb") as f:
            try:
                f.write(data)
            except BrokenPipeError:
                pass

    t = threading.Thread(target=feed)
    t.start()
    env = dict(os.environ, LC_ALL="C", **(env_extra or {}))
    env.pop("LANG", None)
    try:
        p = subprocess.run([CLI] + [("/dev/fd/%d" % r) if a == "PIPE" else a for a in args], capture_output=True, env=env,
                           pass_fds=(r,), timeout=300)
    finally:
        os.close(r)
        t.join()
    return p.returncode, p.stdout, p.stderr


@need_cli
@pytest.mark.gpu
def test_cli_reads_a_streamed_contaminant_once(inputs, tmp_path):
    """a contaminant from a pipe, and a gzip one the host reader streams (FL_GZ_HOST=1), is read in one pass and sized
    from its bases: the same set, stdout and log as the mapped FASTA"""
    k, P, c, m, args, fargs, fpath = cli_case(inputs, CONFIGS[0], tmp_path)
    rc, want, err = run(args + [inputs["fq"]])
    assert rc == 0 and len(want) > 0, err[-2000:]
    piped = [("PIPE" if a == inputs["cfa"] else a) for a in args]
    for data, env in ((inputs["fa"], None), (inputs["fa"], {"FL_HOST_PARSER": "1"}), (gzip.compress(inputs["fa"]), None)):
        rc, out, err = run_with_pipe(piped + [inputs["fq"]], data, env)
        assert rc == 0 and out == want, (env, err[-2000:])
        assert "  %d contigs, %d %d-mers" % (len(inputs["records"]), m, k) in log_lines(err.decode())
    gz = [(inputs["cgz"] if a == inputs["cfa"] else a) for a in args]
    for env in ({"FL_GZ_HOST": "1"}, {"FL_GZ_HOST": "1", "FL_HOST_PARSER": "1"}):
        rc, out, err = run(gz + [inputs["fq"]], None, env)
        assert rc == 0 and out == want, (env, err[-2000:])
        assert "  %d contigs, %d %d-mers" % (len(inputs["records"]), m, k) in log_lines(err.decode())


@need_cli
@pytest.mark.gpu
def test_cli_bam_input_gives_its_fastq_equivalent(inputs, tmp_path):
    recs = [(n.encode(), s.upper(), bytes(x - 33 for x in q), b"") for n, s, q in inputs["reads"] if len(s) > 0]
    raw = bu.bam_of(recs, bu.header(refs=[(b"chr1", 150000)]))
    (tmp_path / "r.bam").write_bytes(bu.bgzf(raw))
    (tmp_path / "r.fastq").write_bytes(bu.to_fastq(raw))
    args = cli_case(inputs, CONFIGS[0], tmp_path)[4]
    rc_f, out_f, _ = run(args + [str(tmp_path / "r.fastq")])
    rc_b, out_b, err_b = run(args + [str(tmp_path / "r.bam")])
    assert rc_f == rc_b == 0, err_b[-2000:]
    assert bu.to_fastq(gzip.decompress(out_b)) == out_f and len(out_f) > 0


@need_cli
@pytest.mark.gpu
def test_contam_k_16_is_the_16mer_path(inputs):
    base = ["--contam", inputs["cfa"], "-p", "90", inputs["fq"]]
    assert run(base) == run(base[:2] + ["--contam_k", "16"] + base[2:])


# ---- GPU: a human-sized set --------------------------------------------------------------------------------------------
def random_genome_records(seed, n_bases, record_bases):
    """(2-bit words on the device, ASCII bytes on the host) of each record of a random genome, generated on the GPU"""
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
        del codes
        left -= n


@pytest.mark.gpu
def test_human_sized_set():
    import torch
    from filtlong_b200 import api
    if torch.cuda.mem_get_info()[0] < 70 * 2 ** 30:
        pytest.skip("needs 70 GiB of free device memory")
    k, n_bases, rec_bases = 31, 3_100_000_000, 100_000_000
    rng = np.random.default_rng(31)
    samples, reads = [], []
    with api.Context(api.make_params(max_contam=10.0, keep_percent=90)) as ctx:
        free0 = torch.cuda.mem_get_info()[0]
        ctx.contam_configure(k, n_bases + n_bases // 200)      # the FASTA's bytes bound its bases
        assert free0 - torch.cuda.mem_get_info()[0] <= 32 * 2 ** 30 + 2 ** 26
        n_rec = (n_bases + rec_bases - 1) // rec_bases
        for i, (_, seq) in enumerate(random_genome_records(1, n_bases, rec_bases)):
            r = ctx.contam_add_text(b">c%d\n%s\n" % (i, seq), fastq=False, is_last=int(i + 1 == n_rec))
            assert r["status"] == "ok" and r["n"] == 1
            a = np.frombuffer(seq, np.uint8)
            pos = rng.integers(0, len(a) - k, 10_000_000 // n_rec + 1)
            codes = km.read_codes(seq)
            fwd = np.zeros(len(pos), np.uint64)
            for j in range(k):
                fwd = (fwd << np.uint64(2)) | codes[pos + j]
            samples.append(fwd)
            for p in rng.integers(0, len(a) - 20000, 8):
                reads.append(seq[p:p + int(rng.integers(1000, 20000))])
        m = ctx.contam_count()
        assert 2 * 3.0e9 < m <= 2 * n_bases
        fwd = np.concatenate(samples)
        assert len(fwd) >= 10_000_000
        for i in range(0, len(fwd), 1 << 22):
            assert ctx.contam_contains64(fwd[i:i + (1 << 22)]).all()
        foreign = [s[:int(rng.integers(1000, 20000))] for _, s in random_genome_records(2, 4_000_000, 200_000)]
        push = reads + foreign
        ctx.push(api.HostBatch(push, [b"I" * len(s) for s in push], want_seq=True))
        pct, removed, _ = ctx.contam_results()
    assert (pct[:len(reads)] == 100.0).all()
    assert not removed[len(reads):].any()
