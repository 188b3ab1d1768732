"""Seeded gzip inputs for the parallel inflater's tests (test_inflate_model.py on the CPU, test_gpu_gunzip.py on the
device), and the CPU model of it (tests/inflate_dump.cpp) built on demand."""
import gzip
import os
import random
import struct
import subprocess
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "filtlong_b200", "csrc")


def build_model(out_dir, sanitize=False):
    exe = os.path.join(out_dir, "inflate_dump_asan" if sanitize else "inflate_dump")
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-I", CSRC, os.path.join(ROOT, "tests", "inflate_dump.cpp"), "-o", exe]
    cmd += ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"] if sanitize else ["-O2"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def run_model(exe, path, chunk_bytes, max_dev, cap, out_path):
    r = subprocess.run([exe, "run", path, out_path, str(chunk_bytes), str(max_dev), str(cap)], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    rc, members, chunks, redecoded, rounds, n_out = (int(x) for x in r.stdout.split())
    data = open(out_path, "rb").read() if rc == 1 else None
    return rc, (members, chunks, redecoded, rounds), data


def fastq(rnd, n_bytes, lo=2000, hi=30000):
    out, n, i = [], 0, 0
    while n < n_bytes:
        L = rnd.randint(lo, hi)
        seq = "".join(rnd.choices("ACGT", k=L))
        qual = "".join(chr(33 + min(50, max(1, int(rnd.gauss(18, 6))))) for _ in range(L))
        r = "@%032x runid=abc read=%d ch=%d\n%s\n+\n%s\n" % (rnd.getrandbits(128), i, rnd.randint(1, 512), seq, qual)
        out.append(r)
        n += len(r)
        i += 1
    return "".join(out).encode()[:n_bytes]


def fasta(rnd, n_bytes):
    out, n, i = [], 0, 0
    while n < n_bytes:
        L = rnd.randint(500, 20000)
        seq = "".join(rnd.choices("ACGT", k=L))
        r = ">contig_%d\n%s\n" % (i, "\n".join(seq[j:j + 80] for j in range(0, L, 80)))
        out.append(r)
        n += len(r)
        i += 1
    return "".join(out).encode()[:n_bytes]


def deflate_gzip(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, flush_every=0, flush=zlib.Z_SYNC_FLUSH):
    c = zlib.compressobj(level, zlib.DEFLATED, 31, 8, strategy)
    if not flush_every:
        return c.compress(data) + c.flush()
    parts = []
    for i in range(0, len(data), flush_every):
        parts.append(c.compress(data[i:i + flush_every]))
        parts.append(c.flush(flush))
    parts.append(c.flush())
    return b"".join(parts)


def member_with_header(data, fname=None, comment=None, extra=None, hcrc=False, level=6):
    """One gzip member with the optional header fields of RFC 1952 2.3."""
    flg = (4 if extra is not None else 0) | (8 if fname else 0) | (16 if comment else 0) | (2 if hcrc else 0)
    h = bytearray(b"\x1f\x8b\x08" + bytes([flg]) + b"\0\0\0\0\0\xff")
    if extra is not None:
        h += struct.pack("<H", len(extra)) + extra
    if fname:
        h += fname + b"\0"
    if comment:
        h += comment + b"\0"
    if hcrc:
        h += struct.pack("<H", zlib.crc32(bytes(h)) & 0xFFFF)
    c = zlib.compressobj(level, zlib.DEFLATED, -15)
    body = c.compress(data) + c.flush()
    return bytes(h) + body + struct.pack("<II", zlib.crc32(data) & 0xFFFFFFFF, len(data) & 0xFFFFFFFF)


def gzread(blob):
    """What gzread (and the host path of inflate_gzip_memory) gives: members back to back, trailing bytes that do not
    start a gzip header ignored."""
    out, pos = [], 0
    while True:
        d = zlib.decompressobj(31)
        out.append(d.decompress(blob[pos:]))
        assert d.eof
        pos = len(blob) - len(d.unused_data)
        if len(blob) - pos < 2 or blob[pos:pos + 2] != b"\x1f\x8b":
            return b"".join(out)


def corpus(seed=11, size=1 << 20):
    """(name, gzip bytes) pairs: every container shape and zlib strategy the inflater has to take."""
    rnd = random.Random(seed)
    long_fq = fastq(rnd, size)
    short_fq = fastq(rnd, size, 100, 150)
    fa = fasta(rnd, size)
    noise = bytes(rnd.getrandbits(8) for _ in range(size // 2))
    cases = [
        ("ont_l1", deflate_gzip(long_fq, 1)),
        ("ont_l6", deflate_gzip(long_fq, 6)),
        ("ont_l9", deflate_gzip(long_fq, 9)),
        ("short_l6", deflate_gzip(short_fq, 6)),
        ("fasta_l6", deflate_gzip(fa, 6)),
        ("random_stored", deflate_gzip(noise, 6)),
        ("filtered", deflate_gzip(long_fq, 6, zlib.Z_FILTERED)),
        ("huffman_only", deflate_gzip(long_fq, 6, zlib.Z_HUFFMAN_ONLY)),
        ("rle", deflate_gzip(long_fq, 6, zlib.Z_RLE)),
        ("fixed", deflate_gzip(long_fq[:size // 8], 6, zlib.Z_FIXED)),
        ("sync_flush", deflate_gzip(short_fq, 6, flush_every=128 << 10)),
        ("full_flush", deflate_gzip(long_fq, 6, flush_every=128 << 10, flush=zlib.Z_FULL_FLUSH)),
        ("members", member_with_header(long_fq[:size // 3], fname=b"a.fastq") + gzip.compress(b"", mtime=0)
         + member_with_header(long_fq[size // 3:2 * size // 3], comment=b"chunk two", hcrc=True, level=1)
         + member_with_header(long_fq[2 * size // 3:], extra=b"XY\x02\x00ab", fname=b"c", level=9)),
        ("trailing_bytes", deflate_gzip(short_fq, 6) + b"not gzip at all\n" * 100),
    ]
    return cases
