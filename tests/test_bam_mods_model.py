"""`--keep_mods` on the CPU: the model of tests/bam_mods_model.py against its own decoder (the worked example of SAMtags
1.7 MM / ML re-based to a child, random reads with random tags, one file per invalidity rule), and the host's children
(bam_child_record over fl_bam_mods.h, through the pass-2 writer without a context) against the model byte for byte."""
import os
import struct
import subprocess

import numpy as np
import pytest

from tests import bam_mods_model as mm
from tests import bam_util as bu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "filtlong_b200")
HOST_LIB = os.path.join(PKG, "libfiltlong_host.a")

EX_SEQ = b"ACGTCCGACGTC"
EX_AUX = bu.aux_z(b"RG", b"rg1") + bu.aux_z(b"MM", b"C+m?,1,0,1;C+h?,4;G-m.,0,1;") + bu.aux_b(b"ML", b"C", [200, 50, 180, 90, 30, 220]) + \
    bu.aux_i(b"MN", 12)


def shifted(calls, s, e):
    return sorted((p - s, st, c, q) for p, st, c, q in calls if s <= p < e)


def test_worked_example():
    extra, status = mm.rebase(EX_SEQ, EX_AUX, 3, 10)
    assert status == mm.KEPT
    assert extra == bu.aux_z(b"MM", b"C+m?,0,0;C+h?;G-m.,1;") + bu.aux_b(b"ML", b"C", [200, 50, 220]) + b"MNI" + struct.pack("<I", 7)
    raw = bu.bam_of([(b"r", EX_SEQ, bytes(range(1, 13)), EX_AUX)])
    r = bu.records(raw)[0]
    rec, _ = mm.child_record(raw, r, 3, 10, True)
    child = bu.records(bu.header() + rec)[0]
    assert child["name"] == b"r_4-10" and child["seq"] == b"TCCGACG"
    assert mm.decode(child["seq"], child["aux"]) == shifted(mm.decode(EX_SEQ, EX_AUX), 3, 10)
    assert [p for p, _, _, _ in mm.decode(child["seq"], child["aux"])] == [1, 2, 6]


def random_mm(rng, seq):
    """MM / ML over seq: several groups, both strands, every flag, multi-code and ChEBI codes, N and U, empty groups"""
    groups, ml = [], []
    for _ in range(int(rng.integers(1, 6))):
        base = "ACGTUN"[int(rng.integers(0, 6))]
        codes = ["m", "h", "mh", "a", "27551", "o", "mhf"][int(rng.integers(0, 7))]
        head = base + "+-"[int(rng.integers(0, 2))] + codes + ["", ".", "?"][int(rng.integers(0, 3))]
        where = mm.base_positions(seq, base)
        k = int(rng.integers(0, len(where) + 1)) if where and rng.random() < 0.8 else 0
        chosen = sorted(rng.choice(len(where), size=k, replace=False)) if k else []
        deltas, prev = [], -1
        for c in chosen:
            deltas.append(str(int(c) - prev - 1))
            prev = int(c)
        groups.append(head + "".join("," + d for d in deltas) + ";")
        ml += [int(x) for x in rng.integers(0, 256, size=len(deltas) * mm.n_codes(codes))]
    return "".join(groups).encode(), ml


def random_read(rng, i, lo=1, hi=400):
    L = int(rng.integers(lo, hi + 1))
    seq = np.frombuffer(b"ACGTACGTACGTN", np.uint8)[rng.integers(0, 13, size=L)].tobytes()
    mmv, ml = random_mm(rng, seq)
    aux = bu.aux_f(b"qs", 3.0)
    parts = [bu.aux_z(b"MM", mmv), bu.aux_b(b"ML", b"C", ml)]
    if rng.random() < 0.3:
        parts.reverse()
    if rng.random() < 0.15:
        parts = parts[:1] if parts[0][:2] == b"MM" else parts[1:]           # MM without ML
    aux += (bu.aux_z(b"RG", b"rg%d" % (i % 3)) if i % 4 else b"") + b"".join(parts)
    if rng.random() < 0.5:
        aux += bu.aux_i(b"MN", L)
    qual = None if i % 7 == 3 else bytes(rng.integers(1, 60, size=L).astype(np.uint8))
    return (b"read%d" % i, seq, qual, aux)


def children(rng, seq, calls):
    """child ranges that start and end on and next to called bases, and random ones"""
    L = len(seq)
    near = sorted({min(max(p + d, 0), L) for p, _, _, _ in calls for d in (-1, 0, 1)} | {0, L})
    out = []
    for _ in range(6):
        a, b = sorted(int(x) for x in rng.choice(near, size=2))
        if a < b:
            out.append((a, b))
        a, b = sorted(int(x) for x in rng.integers(0, L + 1, size=2))
        if a < b:
            out.append((a, b))
    return out


@pytest.mark.parametrize("seed", range(4))
def test_decode_of_every_child_is_the_parents_calls_inside_it(seed):
    rng = np.random.default_rng(seed)
    for i in range(150):
        name, seq, qual, aux = random_read(rng, i)
        assert mm.valid_tags(seq, aux) is not None
        calls = mm.decode(seq, aux)
        raw = bu.bam_of([(name, seq, qual, aux)])
        r = bu.records(raw)[0]
        for s, e in children(rng, seq, calls):
            rec, status = mm.child_record(raw, r, s, e, True)
            assert status == mm.KEPT
            c = bu.records(bu.header() + rec)[0]
            assert c["seq"] == seq[s:e]
            assert mm.decode(c["seq"], c["aux"]) == shifted(calls, s, e), (seq, aux, s, e)
            assert mm.valid_tags(c["seq"], c["aux"]) is not None


# one parent per rule: its children get RG only
INVALID = {
    "delta_past_last_base": (bu.aux_z(b"MM", b"C+m,5;") + bu.aux_b(b"ML", b"C", [1])),
    "ml_too_short": (bu.aux_z(b"MM", b"C+m,0,0;") + bu.aux_b(b"ML", b"C", [1])),
    "ml_too_long": (bu.aux_z(b"MM", b"C+m,0;") + bu.aux_b(b"ML", b"C", [1, 2])),
    "ml_not_bc": (bu.aux_z(b"MM", b"C+m,0;") + bu.aux_b(b"ML", b"S", [1])),
    "mn_not_l_seq": (bu.aux_z(b"MM", b"C+m,0;") + bu.aux_b(b"ML", b"C", [1]) + bu.aux_i(b"MN", 11)),
    "no_final_semicolon": (bu.aux_z(b"MM", b"C+m,0") + bu.aux_b(b"ML", b"C", [1])),
    "bad_base_letter": (bu.aux_z(b"MM", b"X+m,0;") + bu.aux_b(b"ML", b"C", [1])),
    "signed_delta": (bu.aux_z(b"MM", b"C+m,-0;") + bu.aux_b(b"ML", b"C", [1])),
    "delta_of_33_bits": (bu.aux_z(b"MM", b"C+m,4294967296;") + bu.aux_b(b"ML", b"C", [1])),
    "mm_not_z": (bu.aux_i(b"MM", 0)),
    "two_mm": (bu.aux_z(b"MM", b"C+m,0;") + bu.aux_z(b"MM", b"C+m,0;")),
}


@pytest.mark.parametrize("rule", sorted(INVALID))
def test_each_invalidity_rule_gives_an_rg_only_child(rule):
    aux = bu.aux_z(b"RG", b"rg1") + INVALID[rule]
    raw = bu.bam_of([(b"p", b"ACGTCCGACGTC", None, aux)])
    r = bu.records(raw)[0]
    assert mm.valid_tags(r["seq"], r["aux"]) is None
    rec, status = mm.child_record(raw, r, 2, 9, True)
    assert status == mm.INVALID
    assert rec == bu.child_record(raw, r, 2, 9)


def test_delta_of_32_bits_is_valid_and_u_and_n_count_their_bases():
    seq = b"T" * 5 + b"ACGU"[:3]
    assert mm.valid_tags(seq, bu.aux_z(b"MM", b"C+m,4294967295;")) is None        # valid number, past the last C
    assert mm.valid_tags(seq, bu.aux_z(b"MM", b"U+m,4;N-o,7;")) is not None
    assert mm.valid_tags(seq, bu.aux_z(b"MM", b"U+m,5;")) is None


# ---- the host's children, byte for byte ----
@pytest.fixture(scope="module")
def dumper(tmp_path_factory):
    if not os.path.exists(HOST_LIB):
        pytest.skip("host library not built")
    out = str(tmp_path_factory.mktemp("mods") / "bam_mods_dump")
    cmd = ["g++", "-std=c++17", "-O2", os.path.join(ROOT, "tests", "bam_mods_dump.cpp"), HOST_LIB, "-L" + PKG, "-lfiltlong_b200",
           "-lz", "-lpthread", "-Wl,-rpath," + PKG, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def results_for(rng, reads, max_children=6):
    """random results: whole reads kept or not, and children (sorted, some overlapping none) kept or not"""
    res = []
    for _, seq, _, _ in reads:
        L = len(seq)
        if rng.random() < 0.3:
            res.append((0, [(0, L, int(rng.random() < 0.7))]))
            continue
        cuts = sorted(set(int(x) for x in rng.integers(0, L + 1, size=2 * int(rng.integers(1, max_children + 1)))))
        rows = [(cuts[k], cuts[k + 1], int(rng.random() < 0.8)) for k in range(0, len(cuts) - 1, 2)] or [(0, L, 1)]
        res.append((len(rows), rows))
    return res


def spec_text(res):
    return "".join("%d %s\n" % (n, " ".join("%d %d %d" % row for row in rows)) for n, rows in res)


def test_host_children_equal_the_model(dumper, tmp_path):
    rng = np.random.default_rng(21)
    reads = [random_read(rng, i, hi=3000) for i in range(300)]
    reads += [(b"bad_%s" % k.encode(), b"ACGTCCGACGTC", b"\x10" * 12, bu.aux_z(b"RG", b"rg1") + v) for k, v in sorted(INVALID.items())]
    reads += [(b"nomods", b"ACGTACGTAC", None, bu.aux_z(b"RG", b"rg2"))]
    raw = bu.bam_of(reads)
    res = results_for(rng, reads)
    (tmp_path / "in.bam").write_bytes(bu.bgzf(raw))
    (tmp_path / "spec").write_text(spec_text(res))
    p = subprocess.run([dumper, str(tmp_path / "in.bam"), str(tmp_path / "spec")], capture_output=True)
    assert p.returncode == 0, p.stderr
    want, counts = mm.expected_output(raw, res, True)
    assert p.stdout == want
    assert [int(x) for x in p.stderr.split()] == counts
    assert counts[0] > 100 and counts[1] > 0
    # a kept whole read is its record byte for byte
    recs = bu.records(raw)
    for r, (n, rows) in zip(recs, res):
        if n == 0 and rows[0][2]:
            assert raw[r["start"]:r["start"] + r["size"]] in p.stdout
