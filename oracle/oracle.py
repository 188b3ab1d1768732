"""oracle/oracle.py -- TEST INFRASTRUCTURE, not product code.

ctypes front-end for (a) oracle/liboracle.so, our plain-C restatement of the reference path, and
(b) oracle/_ref/refdump + oracle/_ref/filtlong_ref, the UNMODIFIED reference compiled by
oracle/Makefile from a Filtlong v0.3.1 source tree (REF=<dir>). Only tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / --impl reference legs import this module; filtlong_b200/ never does.

Runs of (b) made by the tests are recorded in tests/golden/reference_runs.json.xz, keyed by the
command line and the CONTENT of its input files, and replayed from there: the comparisons with the
reference need neither its sources nor its binaries. FL_REFERENCE_RECORD=<file> runs the binaries
instead (they must exist) and appends every run to <file>; `python -m oracle.oracle merge <file>...`
then adds those runs to the golden store (a run recorded again replaces the stored one).
"""
import ctypes as C
import hashlib
import json
import lzma
import os
import subprocess
import zlib
from dataclasses import dataclass, field

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "liboracle.so")
REFDUMP = os.path.join(HERE, "_ref", "refdump")
REFCLI = os.path.join(HERE, "_ref", "filtlong_ref")


def build(quiet=True):
    """make liboracle.so (always) and _ref/ (only where the reference sources are found, oracle/Makefile)."""
    out = subprocess.run(["make", "-C", HERE, "all"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("oracle build failed:\n" + out.stdout + out.stderr)
    if not quiet:
        print(out.stdout)


class Params(C.Structure):
    _fields_ = [
        ("window_size", C.c_int),
        ("trim", C.c_int), ("split_set", C.c_int), ("split", C.c_int),
        ("min_length_set", C.c_int), ("min_length", C.c_int),
        ("max_length_set", C.c_int), ("max_length", C.c_int),
        ("min_mean_q_set", C.c_int), ("min_window_q_set", C.c_int),
        ("min_mean_q", C.c_double), ("min_window_q", C.c_double),
        ("length_weight", C.c_double), ("mean_q_weight", C.c_double), ("window_q_weight", C.c_double),
        ("target_bases_set", C.c_int), ("keep_percent_set", C.c_int),
        ("target_bases", C.c_longlong),
        ("keep_percent", C.c_double),
    ]


def make_params(window_size=250, trim=False, split=None, min_length=None, max_length=None,
                min_mean_q=None, min_window_q=None, length_weight=1.0, mean_q_weight=1.0,
                window_q_weight=1.0, target_bases=None, keep_percent=None):
    p = Params()
    p.window_size = window_size
    p.trim = int(bool(trim))
    p.split_set = int(split is not None)
    p.split = split or 0
    p.min_length_set = int(min_length is not None)
    p.min_length = min_length or 0
    p.max_length_set = int(max_length is not None)
    p.max_length = max_length or 0
    p.min_mean_q_set = int(min_mean_q is not None)
    p.min_mean_q = min_mean_q or 0.0
    p.min_window_q_set = int(min_window_q is not None)
    p.min_window_q = min_window_q or 0.0
    p.length_weight, p.mean_q_weight, p.window_q_weight = length_weight, mean_q_weight, window_q_weight
    p.target_bases_set = int(target_bases is not None)
    p.target_bases = target_bases or 0
    p.keep_percent_set = int(keep_percent is not None)
    p.keep_percent = keep_percent or 0.0
    return p


def params_to_cli(p):
    """The reference command-line flags equivalent to a Params block."""
    a = []
    if p.target_bases_set: a += ["--target_bases", str(p.target_bases)]
    if p.keep_percent_set: a += ["--keep_percent", repr(p.keep_percent)]
    if p.min_length_set: a += ["--min_length", str(p.min_length)]
    if p.max_length_set: a += ["--max_length", str(p.max_length)]
    if p.min_mean_q_set: a += ["--min_mean_q", repr(p.min_mean_q)]
    if p.min_window_q_set: a += ["--min_window_q", repr(p.min_window_q)]
    if p.trim: a += ["--trim"]
    if p.split_set: a += ["--split", str(p.split)]
    a += ["--length_weight", repr(p.length_weight), "--mean_q_weight", repr(p.mean_q_weight),
          "--window_q_weight", repr(p.window_q_weight), "--window_size", str(p.window_size)]
    return a


class Row(C.Structure):
    _fields_ = [
        ("parent", C.c_int), ("start", C.c_int), ("end", C.c_int), ("length", C.c_int),
        ("mean_q", C.c_double), ("window_q", C.c_double), ("length_score", C.c_double),
        ("passed", C.c_int), ("first", C.c_int), ("last", C.c_int),
        ("n_bad", C.c_int), ("n_child", C.c_int),
        ("norm_mean", C.c_double), ("norm_window", C.c_double), ("final_score", C.c_double),
        ("passed_final", C.c_int),
    ]


class Summary(C.Structure):
    _fields_ = [
        ("min_q", C.c_double), ("max_q", C.c_double), ("mean_q", C.c_double), ("stdev_q", C.c_double),
        ("min_z", C.c_double), ("max_z", C.c_double),
        ("status", C.c_int),
        ("target", C.c_longlong), ("passed_bases", C.c_longlong), ("keeping", C.c_longlong),
    ]


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        L = C.CDLL(LIB_PATH)
        L.orc_kmers_new.restype = C.c_void_p
        L.orc_kmers_free.argtypes = [C.c_void_p]
        L.orc_kmers_add_sequence.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int]
        L.orc_kmers_insert.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.orc_kmers_contains.argtypes = [C.c_void_p, C.c_uint32]
        L.orc_kmers_contains.restype = C.c_int
        L.orc_kmers_size.argtypes = [C.c_void_p]
        L.orc_kmers_size.restype = C.c_uint64
        L.orc_kmers_dump.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.orc_kmers_dump.restype = C.c_size_t
        L.orc_bloom_hash.argtypes = [C.c_uint32, C.c_int]
        L.orc_bloom_hash.restype = C.c_uint32
        L.orc_bloom_table_bits.restype = C.c_uint64
        for f in (L.orc_base_fwd, L.orc_base_rev):
            f.argtypes = [C.c_char]
            f.restype = C.c_uint32
        L.orc_qscore_to_quality.argtypes = [C.c_char]
        L.orc_qscore_to_quality.restype = C.c_double
        L.orc_length_score.argtypes = [C.c_int]
        L.orc_length_score.restype = C.c_double
        L.orc_score_read.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_int, C.POINTER(Params),
                                     C.c_int, C.POINTER(Row), C.POINTER(C.c_int), C.c_int,
                                     C.POINTER(Row), C.c_int]
        L.orc_score_read.restype = C.c_int
        L.orc_finalize.argtypes = [C.POINTER(Row), C.c_size_t, C.c_longlong, C.POINTER(Params),
                                   C.POINTER(Summary)]
        _lib = L
    return _lib


class Kmers:
    """Mirror of the reference's Kmers (kmers.h:28-55) over the C restatement."""

    def __init__(self):
        self._h = lib().orc_kmers_new()

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_kmers_free(self._h)
            self._h = None

    def add_sequence(self, seq: bytes, multiple_copies: bool):
        lib().orc_kmers_add_sequence(self._h, seq, len(seq), int(multiple_copies))

    def add_assembly(self, seqs):
        for s in seqs:
            self.add_sequence(s, False)

    def add_short_reads(self, seqs):
        for s in seqs:
            self.add_sequence(s, True)

    def insert(self, kmers):
        """Load an explicit list of 16-mers (numpy uint32)."""
        import numpy as np
        a = np.ascontiguousarray(kmers, dtype=np.uint32)
        lib().orc_kmers_insert(self._h, a.ctypes.data, a.size)

    def __contains__(self, kmer):
        return bool(lib().orc_kmers_contains(self._h, kmer))

    def __len__(self):
        return int(lib().orc_kmers_size(self._h))

    def dump(self):
        import numpy as np
        n = len(self)
        out = np.zeros(max(n, 1), dtype=np.uint32)
        lib().orc_kmers_dump(self._h, out.ctypes.data, n)
        return out[:n]


@dataclass
class Scored:
    parents: list            # Row per input read
    bad: list                # list of [(s, e), ...] per input read
    children: list           # list of [Row, ...] per input read
    rows: list = field(default_factory=list)      # reads2 table (file order) after finalize
    summary: Summary = None
    total_bases: int = 0


def score(reads, params, kmers=None, cap=4096):
    """reads: iterable of (seq: bytes, qual: bytes | None). Returns Scored (not yet finalized)."""
    L = lib()
    parents, bads, kids = [], [], []
    total = 0
    kh = kmers._h if kmers is not None else None
    for i, (seq, qual) in enumerate(reads):
        row = Row()
        bad = (C.c_int * (2 * cap))()
        ch = (Row * cap)()
        n = L.orc_score_read(kh, seq, qual, len(seq), C.byref(params), i, C.byref(row), bad, cap, ch, cap)
        if n < 0:
            raise RuntimeError("oracle capacity exceeded (or a child produced bad ranges)")
        parents.append(row)
        bads.append([(bad[2 * j], bad[2 * j + 1]) for j in range(row.n_bad)])
        kids.append([_copy_row(ch[j]) for j in range(n)])
        total += len(seq)
    return Scored(parents, bads, kids, total_bases=total)


def _copy_row(r):
    c = Row()
    C.memmove(C.byref(c), C.byref(r), C.sizeof(Row))
    return c


def finalize(sc: Scored, params):
    """main.cpp:138-261 on the scored reads; fills sc.rows / sc.summary."""
    flat = []
    for p, ch in zip(sc.parents, sc.children):
        flat.extend(ch if ch else [p])
    arr = (Row * max(len(flat), 1))()
    for i, r in enumerate(flat):
        C.memmove(C.byref(arr[i]), C.byref(r), C.sizeof(Row))
    s = Summary()
    lib().orc_finalize(arr, len(flat), sc.total_bases, C.byref(params), C.byref(s))
    sc.rows = [_copy_row(arr[i]) for i in range(len(flat))]
    sc.summary = s
    return sc


# ---------------------------------------------------------------------------------------------
# The real reference (oracle/_ref), when present
# ---------------------------------------------------------------------------------------------
def have_ref():
    return os.path.exists(REFDUMP) and os.path.exists(REFCLI)


GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden", "reference_runs.json.xz")
STDOUT_INLINE = 4096          # larger stdout is kept as its SHA-256 (and, for FASTQ, the record names)
_store = None


def _content_digest(path):
    """SHA-256 of what the reference reads from `path`: a gzip file by its inflated bytes (so that the
    header's time stamp does not matter; a truncated stream by what inflates before the cut)."""
    with open(path, "rb") as f:
        data = f.read()
    if data[:2] != b"\x1f\x8b":
        return "raw:" + hashlib.sha256(data).hexdigest()
    h, rest, ok = hashlib.sha256(), data, True
    while rest[:2] == b"\x1f\x8b":
        d = zlib.decompressobj(16 + zlib.MAX_WBITS)
        try:
            h.update(d.decompress(rest))
        except zlib.error:
            ok = False
            break
        if not d.eof:
            ok = False
            break
        rest = d.unused_data
    return ("gz:" if ok else "gz-truncated:") + h.hexdigest()


def _file_args(args):
    return [i for i, a in enumerate(args) if os.path.isfile(a)]


def _key(tool, args, mode):
    parts = [tool, mode] + [("file:" + _content_digest(a)) if os.path.isfile(a) else a for a in args]
    return hashlib.sha256(json.dumps(parts).encode()).hexdigest()[:32]


def _mask(text, args, files):
    for i in sorted(files, key=lambda i: -len(args[i])):
        text = text.replace(args[i], "{ARG%d}" % i)
    return text


def _unmask(text, args, files):
    for i in files:
        text = text.replace("{ARG%d}" % i, args[i])
    return text


def _load_store():
    global _store
    if _store is None:
        _store = {}
        if os.path.exists(GOLDEN):
            with lzma.open(GOLDEN, "rt") as f:
                _store = json.load(f)
    return _store


class RecordedStdout:
    """The stdout of a recorded reference run too large to keep: equal to the bytes with its SHA-256."""

    def __init__(self, sha256, size, fastq_names):
        self.sha256, self.size, self.fastq_names = sha256, size, fastq_names

    def __eq__(self, other):
        if isinstance(other, RecordedStdout):
            return (self.sha256, self.size) == (other.sha256, other.size)
        if isinstance(other, (bytes, bytearray)):
            return len(other) == self.size and hashlib.sha256(other).hexdigest() == self.sha256
        return NotImplemented

    def __len__(self):
        return self.size

    def __repr__(self):
        return "<reference stdout: %d bytes, sha256 %s>" % (self.size, self.sha256[:16])


def fastq_names(out):
    """Record names of FASTQ output (bytes or RecordedStdout), None if it is not 4-line FASTQ."""
    if isinstance(out, RecordedStdout):
        return out.fastq_names
    lines = out.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    if not lines or len(lines) % 4 or not all(l.startswith(b"@") for l in lines[0::4]):
        return None
    return [l[1:].split()[0].decode() for l in lines[0::4]]


def run_reference(tool, args, env_extra=None, cwd=None, timeout=3600, kmers_out=False):
    """One run of a reference binary ("refdump" or "filtlong_ref"): (returncode, stdout bytes, stderr str,
    SHA-256 of the k-mer dump or None). Replayed from the golden store; FL_REFERENCE_RECORD runs and records it.
    kmers_out: True for the dump's SHA-256, or a path to keep the dump itself (a live run only)."""
    args = [str(a) for a in args]
    env_extra = dict(env_extra or {})
    mode = env_extra.get("REFDUMP_MODE", "dump") + ("+kmers" if kmers_out else "") + ("+quiet" if "REFDUMP_QUIET" in env_extra else "")
    cwd_args = [os.path.join(cwd, a) if cwd and not os.path.isabs(a) and os.path.isfile(os.path.join(cwd, a)) else a for a in args]
    files = _file_args(cwd_args)
    key = _key(tool, cwd_args, mode)
    record_to = os.environ.get("FL_REFERENCE_RECORD")
    if not record_to:
        if isinstance(kmers_out, str):
            raise RuntimeError("writing the reference's k-mer dump needs a live run (FL_REFERENCE_RECORD=<file>)")
        rec = _load_store().get(key)
        if rec is None:
            raise RuntimeError("no recorded reference run for %s %s (key %s): record it with FL_REFERENCE_RECORD=<file> where "
                               "oracle/_ref is built, and merge the file into %s" % (tool, " ".join(args), key, GOLDEN))
        out = rec["stdout"].encode("latin-1") if "stdout" in rec else RecordedStdout(rec["stdout_sha256"], rec["stdout_size"],
                                                                                    rec.get("fastq_names"))
        if isinstance(out, bytes):
            out = _unmask(out.decode("latin-1"), args, files).encode("latin-1")
        return rec["rc"], out, _unmask(rec["stderr"], args, files), rec.get("kmers_sha256")
    kpath = None
    if kmers_out:
        import tempfile
        if isinstance(kmers_out, str):
            kpath = kmers_out
        else:
            fd, kpath = tempfile.mkstemp(prefix="refdump_kmers_")
            os.close(fd)
        env_extra["REFDUMP_KMERS_OUT"] = kpath
    binary = {"refdump": REFDUMP, "filtlong_ref": REFCLI}[tool]
    p = subprocess.run([binary] + args, capture_output=True, env=_env(env_extra), cwd=cwd, timeout=timeout)
    err = p.stderr.decode(errors="replace")
    rec = {"rc": p.returncode, "stderr": _mask(err, args, files)}
    if len(p.stdout) <= STDOUT_INLINE or tool == "refdump":
        rec["stdout"] = _mask(p.stdout.decode("latin-1"), args, files)
    else:
        rec.update(stdout_sha256=hashlib.sha256(p.stdout).hexdigest(), stdout_size=len(p.stdout), fastq_names=fastq_names(p.stdout))
    ksha = None
    if kpath:
        with open(kpath, "rb") as f:
            ksha = rec["kmers_sha256"] = hashlib.sha256(f.read()).hexdigest()
        if kpath is not kmers_out:
            os.unlink(kpath)
    with open(record_to, "a") as f:
        f.write(json.dumps({key: rec}) + "\n")
    return p.returncode, p.stdout, err, ksha


def _env(extra=None):
    e = dict(os.environ)
    e.pop("LANG", None)
    e.pop("LC_ALL", None)       # the reference aborts on an uninstalled locale (misc.cpp:37)
    e["LC_ALL"] = "C"
    if extra:
        e.update(extra)
    return e


def fromhex(s):
    return float.fromhex(s) if s not in ("nan", "-nan", "inf", "-inf") else float(s)


def run_refdump(cli_args, kmers_out=False, quiet=False, timeout=3600):
    """Run the link-harness over the reference objects; returns a dict of parsed records (with kmers_out, also
    "kmers_sha256": the SHA-256 of the sorted reference 16-mer set as raw little-endian uint32)."""
    extra = {"REFDUMP_QUIET": "1"} if quiet else {}
    rc, stdout, stderr, ksha = run_reference("refdump", cli_args, extra, timeout=timeout, kmers_out=kmers_out)
    if rc != 0:
        raise RuntimeError("refdump failed (%d): %s" % (rc, stderr[-2000:]))
    res = {"reads": [], "rows": [], "n_kmers": None, "global": None, "tail": None, "kmers_sha256": ksha}
    for line in stdout.decode("latin-1").splitlines():
        f = line.split(" ")
        if f[0] == "K":
            res["n_kmers"] = int(f[1])
        elif f[0] == "R":
            res["reads"].append(dict(idx=int(f[1]), name=f[2], length=int(f[3]), mean_q=fromhex(f[4]),
                                     window_q=fromhex(f[5]), length_score=fromhex(f[6]), passed=int(f[7]),
                                     first=int(f[8]), last=int(f[9]), n_bad=int(f[10]), n_child=int(f[11]),
                                     bad=[], children=[]))
        elif f[0] == "B":
            res["reads"][int(f[1])]["bad"].append((int(f[2]), int(f[3])))
        elif f[0] == "C":
            res["reads"][int(f[1])]["children"].append(dict(
                name=f[3], start=int(f[4]), end=int(f[5]), mean_q=fromhex(f[6]), window_q=fromhex(f[7]),
                length_score=fromhex(f[8]), passed=int(f[9]), n_bad=int(f[10]), n_child=int(f[11])))
        elif f[0] == "G":
            res["global"] = dict(n=int(f[1]), min_q=fromhex(f[2]), max_q=fromhex(f[3]), mean_q=fromhex(f[4]),
                                 stdev_q=fromhex(f[5]), min_z=fromhex(f[6]), max_z=fromhex(f[7]))
        elif f[0] == "F":
            res["rows"].append(dict(row=int(f[1]), name=f[2], length=int(f[3]), norm_mean=fromhex(f[4]),
                                    norm_window=fromhex(f[5]), final_score=fromhex(f[6]), passed_final=int(f[7])))
        elif f[0] == "T":
            res["tail"] = dict(status=int(f[1]), target=int(f[2]), total_bases=int(f[3]),
                               passed_bases=int(f[4]), keeping=int(f[5]))
    return res


def run_refdump_time(cli_args, timeout=3600):
    import json
    out = subprocess.run([REFDUMP] + list(cli_args), capture_output=True, text=True,
                         env=_env({"REFDUMP_MODE": "time"}), timeout=timeout)
    if out.returncode != 0:
        raise RuntimeError("refdump failed (%d): %s" % (out.returncode, out.stderr[-2000:]))
    return json.loads(out.stdout.strip().splitlines()[-1])


def run_refdump_bloom(keys):
    _, stdout, _, _ = run_reference("refdump", ["%08X" % k for k in keys], {"REFDUMP_MODE": "bloom"})
    res = {"salts": [], "hashes": {}}
    for line in stdout.decode("latin-1").splitlines():
        f = line.split()
        if f[0] == "BLOOM":
            res["k"], res["bits"] = int(f[1]), int(f[2])
        elif f[0] == "SALT":
            res["salts"].append(int(f[2], 16))
        elif f[0] == "H":
            res["hashes"][(int(f[1], 16), int(f[2]))] = (int(f[3], 16), int(f[4]))
    return res


def run_refcli(cli_args, cwd=None, timeout=3600):
    """Run the unmodified reference CLI; returns (returncode, stdout bytes or RecordedStdout, stderr str)."""
    rc, out, err, _ = run_reference("filtlong_ref", cli_args, cwd=cwd, timeout=timeout)
    return rc, out, err


def merge_recorded(paths, store=GOLDEN):
    """Adds the runs recorded under FL_REFERENCE_RECORD (JSON lines) to the golden store; returns its size."""
    runs = {}
    if os.path.exists(store):
        with lzma.open(store, "rt") as f:
            runs = json.load(f)
    for path in paths:
        with open(path) as f:
            for line in f:
                runs.update(json.loads(line))
    with lzma.open(store, "wt", preset=9 | lzma.PRESET_EXTREME) as f:
        json.dump(runs, f, sort_keys=True, separators=(",", ":"))
    return len(runs)


if __name__ == "__main__":
    import sys
    if len(sys.argv) < 3 or sys.argv[1] != "merge":
        raise SystemExit("usage: python -m oracle.oracle merge <recorded runs>...")
    print("%d reference runs in %s" % (merge_recorded(sys.argv[2:]), GOLDEN))
