"""Helpers of the BGZF tests: synthetic FASTQ / FASTA corpora, zlib's BGZF of the same blocks, member walking, and the
host build of the kernel's Huffman / CRC arithmetic (tests/bgzf_codes_dump.cpp over fl_bgzf.h)."""
import os
import struct
import subprocess
import zlib

import numpy as np

BLOCK = 0xff00
EOF_MEMBER = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "filtlong_b200", "csrc")


def build_codes_dumper(out_dir):
    """Compiles tests/bgzf_codes_dump.cpp (fl_bgzf.h for the host) into out_dir; returns the executable's path."""
    out = os.path.join(str(out_dir), "bgzf_codes_dump")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-I", CSRC, os.path.join(ROOT, "tests", "bgzf_codes_dump.cpp"), "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def huff_codes(dumper, freqs, maxbits):
    """fl_huff_lengths_sorted over the used symbols in ascending (frequency, symbol) order, then fl_huff_canonical:
    (lengths, bit-reversed codes), one entry per symbol of freqs."""
    r = subprocess.run([dumper, "huff", str(maxbits), str(len(freqs))] + [str(int(f)) for f in freqs],
                       capture_output=True, text=True, check=True)
    lines = r.stdout.split("\n")
    return [int(x) for x in lines[0].split()], [int(x) for x in lines[1].split()]


def ont_header(rng, i):
    u = rng.integers(0, 16, size=32)
    h = "".join("0123456789abcdef"[x] for x in u)
    uuid = "%s-%s-%s-%s-%s" % (h[:8], h[8:12], h[12:16], h[16:20], h[20:])
    return ("%s runid=8e3c7f42a5b1d9e06f2c4d8a1b3e5f7092c4d6e8 sampleid=sample_01 read=%d ch=%d "
            "start_time=2019-03-1%dT%02d:%02d:%02dZ" % (uuid, i, int(rng.integers(1, 513)), int(rng.integers(0, 10)),
                                                       int(rng.integers(0, 24)), int(rng.integers(0, 60)), int(rng.integers(0, 60))))


def fastq_corpus(rng, n_bytes, mean_len=None, lo=None, hi=None, fasta=False):
    """ONT-style reads: lognormal lengths around mean_len, or uniform in [lo, hi]; qualities around Q12 +- 4."""
    acgt = np.frombuffer(b"ACGT", np.uint8)
    out, size, i = [], 0, 0
    while size < n_bytes:
        if mean_len:
            L = int(np.clip(rng.lognormal(np.log(mean_len) - 0.32, 0.8), 200, 200000))
        else:
            L = int(rng.integers(lo, hi + 1))
        seq = acgt[rng.integers(0, 4, size=L)].tobytes()
        if fasta:
            rec = b">" + ont_header(rng, i).encode() + b"\n" + seq + b"\n"
        else:
            q = (np.clip(np.rint(rng.normal(12, 4, size=L)), 1, 50).astype(np.uint8) + 33).tobytes()
            rec = b"@" + ont_header(rng, i).encode() + b"\n" + seq + b"\n+\n" + q + b"\n"
        out.append(rec)
        size += len(rec)
        i += 1
    return b"".join(out)


def zlib_bgzf(data, level=1):
    """BGZF of data with zlib at `level` on the same 0xff00 cut, without the EOF member."""
    out = []
    for lo in range(0, len(data), BLOCK):
        chunk = data[lo:lo + BLOCK]
        co = zlib.compressobj(level, zlib.DEFLATED, -15)
        body = co.compress(chunk) + co.flush()
        bsize = 18 + len(body) + 8 - 1
        out.append(b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", bsize) + body
                   + struct.pack("<II", zlib.crc32(chunk) & 0xffffffff, len(chunk)))
    return b"".join(out)


def members(buf):
    """(offset, size, isize) of every member, checking the fixed header fields on the way."""
    res, pos = [], 0
    while pos < len(buf):
        h = buf[pos:pos + 18]
        assert h[:4] == b"\x1f\x8b\x08\x04" and h[4:8] == b"\0\0\0\0" and h[8] == 0 and h[9] == 0xff, h
        assert h[10:16] == b"\x06\0BC\x02\0", h
        size = struct.unpack("<H", h[16:18])[0] + 1
        isize = struct.unpack("<I", buf[pos + size - 4:pos + size])[0]
        res.append((pos, size, isize))
        pos += size
    assert pos == len(buf)
    return res
