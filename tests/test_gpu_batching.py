"""Results must not depend on how the reads reach the library: cut into batches in many ways (tests/batch_schedule.py),
pushed through every entry point, with results read between batches.

The seams under test: the second half of a batch with --trim / --split, which fl_reads_push defers to the next call
(fl_score_complete), and the contaminant rows it must then mark; the read / row offsets every kernel takes; per-read and
per-row arrays that grow with a kept prefix while scratch buffers are reused; fl_reads_push's two staging slots; the
input's total bases, counted on the host for host batches and on the device for device batches; and a context that is
finalised, takes more reads and is finalised again, or is reset and run again.

Per mode: the one-batch run is judged against the models (the oracle, tests/qtrim_model.py, tests/contam_k_model.py);
every other schedule must give its read, row and contaminant results and its summary bit for bit; whatever a result call
returned mid-stream must be a prefix of the final arrays."""
import numpy as np
import pytest

from filtlong_b200 import api
from oracle import oracle as orc
from tests import bam_util as bu
from tests import batch_schedule as bs
from tests import parity
from tests.test_contam import _push_all, fastq

pytestmark = pytest.mark.gpu

MODES = list(bs.MODES)
SCHEDULES = ["one_per_batch", "grow", "empty", "seams", "alternating"] + ["random_%d" % s for s in bs.SEEDS]
SUMMARY = ("status", "target", "keeping", "total_bases", "passed_bases", "rows_bases")
ROW_KEYS = ("parent", "start", "end", "mean_q", "window_q", "length_score", "passed")     # set before fl_finalize


@pytest.fixture(scope="module")
def data():
    d = bs.read_set()
    d["kmers"] = bs.assembly_kmers(d["genome"])
    d["lengths"] = np.array([len(r[1]) for r in d["reads"]], dtype=np.int64)
    d["models"], d["baselines"] = {}, {}
    return d


def model(data, mode):
    """(the oracle's Scored of the mode without its contaminant set, the contaminant percentages or None, attrs)"""
    if mode not in data["models"]:
        sc = bs.scored(data, mode, data["kmers"])
        k = bs.MODES[mode].get("contam")
        pct = bs.contam_percentages(data, k) if k else None
        data["models"][mode] = (sc, pct, bs.attrs(data, mode, sc, pct))
    return data["models"][mode]


def schedule(data, mode, name):
    return bs.schedules(model(data, mode)[2], bs.paths_of(mode))[name]


# ---- running a schedule -------------------------------------------------------------------------------------------------
def new_ctx(data, mode):
    m = bs.MODES[mode]
    ctx = api.Context(api.make_params(**m["kw"]))
    if m.get("kmer"):
        ctx.kmers_add([data["genome"]], False)
    k = m.get("contam")
    if k:
        if k > 16:
            ctx.contam_configure(k, len(data["contam"]))
        ctx.contam_add([data["contam"]])
    return ctx


def push(ctx, path, reads):
    if path == "push_fasta":
        r = ctx.push_text(b"".join(b">" + n.encode() + b"\n" + s + b"\n" for n, s, _ in reads), fastq=False)
        assert r["status"] == "ok" and r["n"] == len(reads)
    elif reads:
        _push_all(ctx, reads, path)
    elif path == "push":
        ctx.push(api.HostBatch([], []))
    elif path == "push_text":
        assert ctx.push_text(b"")["n"] == 0
    elif path == "push_bam":
        ctx.push_bam(bu.bam_of([]), [], [], [])
    else:
        ctx.push_device(api.device_batch(0, 0, None, None))


OBSERVE = {"counts": lambda c: c.counts(), "read_results": lambda c: c.read_results(), "row_results": lambda c: c.row_results(),
           "contam_results": lambda c: c.contam_results(), "kmers_count": lambda c: c.kmers_count()}


def run(ctx, data, steps):
    """push the schedule's batches, calling its observers; returns [(observer, reads pushed before it, its result)]"""
    seen, done = [], 0
    for st in steps:
        if st[0] == "batch":
            push(ctx, st[1], data["reads"][st[2]:st[3]])
            done = st[3]
        else:
            seen.append((st[1], done, OBSERVE[st[1]](ctx)))
    return seen


def results(ctx):
    pct, removed, cc = ctx.contam_results()
    return dict(reads=ctx.read_results(), rows=ctx.row_results(), contam=dict(percent=pct, removed=removed), contam_counts=cc,
                counts=ctx.counts(), kmers=ctx.kmers_count())


def final(ctx):
    s = ctx.finalize(-1)
    out = results(ctx)
    out["summary"], out["s"] = {f: getattr(s, f) for f in SUMMARY}, s
    return out


def baseline(data, mode):
    """everything in one push batch"""
    if mode not in data["baselines"]:
        with new_ctx(data, mode) as ctx:
            run(ctx, data, schedule(data, mode, "one_batch"))
            data["baselines"][mode] = final(ctx)
    return data["baselines"][mode]


def u8(a):
    return np.ascontiguousarray(a).view(np.uint8)


def assert_same(got, want, what=""):
    for part in ("reads", "rows", "contam"):
        for k in want[part]:
            assert np.array_equal(u8(got[part][k]), u8(want[part][k])), (what, part, k)
    for k in ("contam_counts", "counts", "kmers", "summary"):
        assert got[k] == want[k], (what, k, got[k], want[k])


def check_observed(seen, fin, lengths):
    """each mid-stream result is the prefix of the final arrays that the reads pushed before it own"""
    n = len(lengths)
    row_start, parent = fin["reads"]["row_start"], fin["rows"]["parent"]
    removed = fin["contam"]["removed"]
    for what, done, v in seen:
        rows = int(row_start[done]) if done < n else len(parent)
        if what == "counts":
            assert v == (done, rows, int(lengths[:done].sum())), (v, done, rows)
        elif what == "read_results":
            for k, x in v.items():
                assert len(x) == done and np.array_equal(u8(x), u8(fin["reads"][k][:done])), (what, done, k)
        elif what == "row_results":
            for k in ROW_KEYS:
                assert len(v[k]) == rows and np.array_equal(u8(v[k]), u8(fin["rows"][k][:rows])), (what, done, k)
        elif what == "contam_results":
            pct, rem, cc = v
            assert np.array_equal(u8(pct), u8(fin["contam"]["percent"][:done])) and np.array_equal(rem, removed[:done])
            want = dict(reads=int(removed[:done].sum()), bases=int(lengths[:done][removed[:done]].sum()),
                        rows=int(removed[parent[:rows]].sum()))
            assert cc == want, (done, cc, want)
        else:
            assert v == fin["kmers"]


# ---- the one-batch run against the models ------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_one_batch_equals_the_models(data, mode):
    sc, pct, a = model(data, mode)
    fin = baseline(data, mode)
    rr, rw, s = fin["reads"], fin["rows"], fin["s"]
    p = api.make_params(**bs.MODES[mode]["kw"])
    n, total = len(data["reads"]), int(data["lengths"].sum())
    assert fin["counts"] == (n, len(sc.rows), total) and s.total_bases == total
    assert fin["kmers"] == (len(data["kmers"]) if bs.MODES[mode].get("kmer") else 0)
    parity.check_reads_vs_oracle(rr, sc)
    if pct is None:
        parity.check_rows_vs_oracle(rw, rr, sc, s)
        parity.check_rescale_exact(rw, s, p)
        parity.check_selection_exact(rw, s, p)
        return
    # the contaminant percentages: bit-identical to the model; removed iff above max_contam
    got, removed, cc = fin["contam"]["percent"], fin["contam"]["removed"], fin["contam_counts"]
    nan = np.isnan(pct)
    assert np.array_equal(np.isnan(got), nan) and np.array_equal(u8(got[~nan]), u8(pct[~nan]))
    assert np.array_equal(removed, a["removed"]) and removed.sum() > 0 and (~removed).sum() > 0
    gone = removed[rw["parent"]]
    assert cc == dict(reads=int(removed.sum()), bases=int(data["lengths"][removed].sum()), rows=int(gone.sum()))
    # the rows are the model's; a removed read's rows neither pass nor are kept, and only the others are ranked
    row = 0
    for i, kids in enumerate(sc.children):
        assert rr["row_start"][i] == row
        row += max(len(kids), 1)
    for i, r in enumerate(sc.rows):
        assert (rw["parent"][i], rw["start"][i], rw["end"][i]) == (r.parent, r.start, r.end), i
        assert parity.same(rw["mean_q"][i], r.mean_q) and parity.same(rw["window_q"][i], r.window_q), i
        assert rw["passed"][i] == (r.passed and not gone[i]), i
    assert not rw["passed_final"][gone].any()
    kept = {k: v[~gone] for k, v in rw.items()}
    parity.check_rescale_exact(kept, s, p)
    parity.check_selection_exact(kept, s, p)
    # and the kept rows are the oracle's finalised run on the kept reads alone, over all the input's bases
    keep = ~removed
    sk = orc.Scored([x for x, k in zip(sc.parents, keep) if k], [x for x, k in zip(sc.bad, keep) if k],
                    [x for x, k in zip(sc.children, keep) if k], total_bases=total)
    orc.finalize(sk, orc.make_params(**{k: v for k, v in bs.MODES[mode]["kw"].items() if k != "trim_q"}))
    before = np.concatenate(([0], np.cumsum(gone)))                # removed rows before each row
    rr_kept = {k: v[keep] for k, v in rr.items()}
    rr_kept["row_start"] = rr_kept["row_start"] - before[rr_kept["row_start"].astype(np.int64)]
    parity.check_rows_vs_oracle(kept, rr_kept, sk, s)


# ---- every schedule against the one-batch run --------------------------------------------------------------------------
@pytest.mark.parametrize("name", SCHEDULES)
@pytest.mark.parametrize("mode", MODES)
def test_schedule_equals_one_batch(data, mode, name):
    want = baseline(data, mode)
    with new_ctx(data, mode) as ctx:
        seen = run(ctx, data, schedule(data, mode, name))
        assert ctx.counts()[2] == int(data["lengths"].sum())
        got = final(ctx)
    assert_same(got, want, name)
    check_observed(seen, want, data["lengths"])


# ---- an empty read on each path ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode,path", [("phred", "push_text"), ("phred", "push_bam"), ("phred", "push_device"),
                                       ("kmer_trim_split100_contam16", "push_text"), ("kmer_trim_split100_contam16", "push_fasta"),
                                       ("kmer_trim_split100_contam16", "push_bam"), ("kmer_trim_split100_contam16", "push_device")])
def test_an_empty_read_on_each_path(data, mode, path):
    """Why the schedules send an empty read through push only: a text chunk holding an empty record is handed back to the
    host parser (status fallback) and push_bam refuses a record of length 0, both before scoring anything of the batch;
    push_device scores it as push does"""
    empty = [i for i, r in enumerate(data["reads"]) if len(r[1]) == 0]
    reads = [data["reads"][i] for i in (0, empty[0], 1)]
    with new_ctx(data, mode) as ctx:
        if path in ("push_text", "push_fasta"):
            text = b"".join(b">" + n.encode() + b"\n" + s + b"\n" for n, s, _ in reads) if path == "push_fasta" else fastq(reads)
            r = ctx.push_text(text, fastq=path == "push_text")
            assert r["status"] == "fallback" and ctx.counts() == (0, 0, 0)
            return
        if path == "push_bam":
            with pytest.raises(api.FLError, match="record 1 does not lie inside the chunk"):
                push(ctx, path, reads)
            assert ctx.counts() == (0, 0, 0)
            return
        push(ctx, path, reads)
        got = final(ctx)
    with new_ctx(data, mode) as ctx:
        push(ctx, "push", reads)
        want = final(ctx)
    assert got["counts"][0] == 3 and got["reads"]["length"][1] == 0
    assert_same(got, want, path)


# ---- the context's lifecycle -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_finalize_push_more_and_finalize_again(data, mode):
    """fl_finalize after part of the reads, then the rest, then fl_finalize again: the one-batch result"""
    steps = schedule(data, mode, "random_12")
    at = [i for i, st in enumerate(steps) if st[0] == "batch"]
    cut = at[len(at) // 3]
    with new_ctx(data, mode) as ctx:
        seen = run(ctx, data, steps[:cut])
        done = max([st[3] for st in steps[:cut] if st[0] == "batch"] + [0])
        assert 0 < done < len(data["reads"])
        first = ctx.finalize(-1)
        assert first.total_bases == int(data["lengths"][:done].sum())
        seen += run(ctx, data, steps[cut:])
        got = final(ctx)
    want = baseline(data, mode)
    assert_same(got, want)
    check_observed(seen, want, data["lengths"])


@pytest.mark.parametrize("mode", MODES)
def test_reset_then_another_schedule(data, mode):
    """fl_reads_reset after a finalised run, then another schedule in the same context: a fresh context's result"""
    with new_ctx(data, mode) as ctx:
        run(ctx, data, schedule(data, mode, "alternating"))
        final(ctx)
        ctx.reset_reads()
        assert ctx.counts() == (0, 0, 0)
        seen = run(ctx, data, schedule(data, mode, "random_13"))
        got = final(ctx)
    want = baseline(data, mode)
    assert_same(got, want)
    check_observed(seen, want, data["lengths"])
