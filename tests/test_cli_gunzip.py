"""The CLI on ordinary gzip input large enough for the GPU inflater (fl_gzip_inflate, at least
Kmers::kDeviceGunzipMinBytes compressed): every run must give the exit code, stdout and stderr log of the same command on
the plain files, and its FL_CLI_TIMING lines must show that the GPU inflater ran. A gzip file whose CRC is wrong must
give what the host z_stream gives (FL_GUNZIP_HOST=1 keeps every file there, as before the GPU inflater existed)."""
import os
import subprocess
import zlib

import numpy as np
import pytest

from tests.test_cli import CLI, final_lines, need_cli
from tests.test_cli_stdin import env_of, gpu_count, run_stream

pytestmark = [need_cli, pytest.mark.gpu]
TIMEOUT = 600
MIN_BYTES = 64 << 20          # Kmers::kDeviceGunzipMinBytes


def fastq(seed, n_bytes, lo, hi):
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    out, total, i = [], 0, 0
    while total < n_bytes:
        L = int(rng.integers(lo, hi))
        seq = acgt[rng.integers(0, 4, size=L)].tobytes()
        qual = (np.clip(rng.normal(18, 6, size=L), 1, 50).astype(np.uint8) + 33).tobytes()
        r = b"@read_%d ch=%d\n%s\n+\n%s\n" % (i, i % 512, seq, qual)
        out.append(r)
        total += len(r)
        i += 1
    return b"".join(out)


def gz(data, level=1):
    c = zlib.compressobj(level, zlib.DEFLATED, 31)
    return c.compress(data) + c.flush()


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("cli_gunzip")
    f = {}

    def put(name, data):
        f[name] = str(d / name)
        open(f[name], "wb").write(data)

    reads = fastq(41, 128 << 20, 3000, 30000)
    put("reads.fastq", reads)
    put("reads.fastq.gz", gz(reads))
    parts = [reads[:reads.index(b"\n@read_400 ") + 1], None]
    parts[1] = reads[len(parts[0]):]
    put("cat.fastq.gz", gz(parts[0], 1) + gz(parts[1][:len(parts[1]) // 2], 6) + gz(parts[1][len(parts[1]) // 2:], 1))
    short = fastq(42, 140 << 20, 100, 151)
    put("short.fastq", short)
    put("short.fastq.gz", gz(short))
    rng = np.random.default_rng(43)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    contigs = []
    for k in range(8):
        s = acgt[rng.integers(0, 4, size=32 << 20)].tobytes()
        contigs.append(b">contig_%d\n" % k + b"\n".join(s[i:i + 80] for i in range(0, len(s), 80)) + b"\n")
    asm = b"".join(contigs)
    put("asm.fasta", asm)
    put("asm.fasta.gz", gz(asm))
    put("few.fastq", fastq(44, 6 << 20, 2000, 20000))
    bad = bytearray(open(f["reads.fastq.gz"], "rb").read())
    bad[-6] ^= 0x10                                                # the CRC-32 of the (only) member
    put("bad_crc.fastq.gz", bytes(bad))
    for k in ("reads.fastq.gz", "cat.fastq.gz", "short.fastq.gz", "asm.fasta.gz"):
        assert os.path.getsize(f[k]) >= MIN_BYTES, (k, os.path.getsize(f[k]))
    return f


def run(args, env_extra=None):
    env = env_of(dict(env_extra or {}, FL_CLI_TIMING="1"))
    p = subprocess.run([CLI] + list(args), capture_output=True, env=env, timeout=TIMEOUT)
    return p.returncode, p.stdout, p.stderr.decode(errors="replace")


def log(err):
    """The stderr log without the FL_CLI_TIMING lines, and with `x.gz` file names read as `x` (the -a log names the file)."""
    return [x.replace(".gz", "") for x in final_lines(err) if not x.startswith("[timing]")]


def same(a, b, what):
    assert a[0] == b[0], (what, a[2][-2000:])
    assert a[1] == b[1], what
    assert log(a[2]) == log(b[2]), what


def gpu_inflated(err, n=1):
    lines = [x for x in err.split("\n") if "gzip input inflated into memory" in x and "GPU inflater:" in x]
    assert len(lines) >= n, err[-3000:]


def test_one_member(files):
    plain = run(["-p", "90", files["reads.fastq"]])
    gpu = run(["-p", "90", files["reads.fastq.gz"]])
    host = run(["-p", "90", files["reads.fastq.gz"]], {"FL_GUNZIP_HOST": "1"})
    assert plain[0] == 0 and len(plain[1]) > 0
    same(gpu, plain, "gzip on the GPU")
    same(host, plain, "gzip on the host")
    gpu_inflated(gpu[2])
    assert "GPU inflater:" not in host[2]


def test_one_member_from_a_pipe(files):
    plain = run(["-p", "90", files["reads.fastq"]])
    rc, out, err = run_stream(["-p", "90"], open(files["reads.fastq.gz"], "rb").read(), {"FL_CLI_TIMING": "1"})
    same((rc, out, err), plain, "cat reads.fastq.gz | filtlong -p 90 -")
    gpu_inflated(err)


def test_concatenated_members(files):
    plain = run(["-p", "90", files["reads.fastq"]])
    gpu = run(["-p", "90", files["cat.fastq.gz"]])
    same(gpu, plain, "cat of three .fastq.gz")
    gpu_inflated(gpu[2])


def test_short_read_references(files):
    plain = run(["-1", files["short.fastq"], "-2", files["short.fastq"], "-p", "90", files["few.fastq"]])
    gpu = run(["-1", files["short.fastq.gz"], "-2", files["short.fastq.gz"], "-p", "90", files["few.fastq"]])
    assert plain[0] == 0
    same(gpu, plain, "-1/-2 gzip")
    lines = [x for x in gpu[2].split("\n") if x.startswith("[timing] reference") and "GPU inflater:" in x]
    assert len(lines) == 2, gpu[2][-3000:]


def test_assembly_reference(files):
    plain = run(["-a", files["asm.fasta"], "-p", "90", "--trim", "--split", "500", files["few.fastq"]])
    gpu = run(["-a", files["asm.fasta.gz"], "-p", "90", "--trim", "--split", "500", files["few.fastq"]])
    assert plain[0] == 0
    same(gpu, plain, "-a gzip")
    assert any(x.startswith("[timing] reference") and "GPU inflater:" in x for x in gpu[2].split("\n")), gpu[2][-3000:]


@pytest.mark.skipif(gpu_count() < 2, reason="needs two GPUs")
def test_two_gpus(files):
    plain = run(["-p", "90", "--gpus", "2", files["reads.fastq"]])
    gpu = run(["-p", "90", "--gpus", "2", files["reads.fastq.gz"]])
    same(gpu, plain, "--gpus 2")
    gpu_inflated(gpu[2])


def test_bad_crc_behaves_as_the_host_path(files):
    gpu = run(["-p", "90", files["bad_crc.fastq.gz"]])
    host = run(["-p", "90", files["bad_crc.fastq.gz"]], {"FL_GUNZIP_HOST": "1"})
    same(gpu, host, "bad CRC")
    assert "GPU inflater:" not in gpu[2]
