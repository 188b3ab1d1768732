"""CPU pins of the BGZF kernel's arithmetic (filtlong_b200/csrc/fl_bgzf.h, compiled for the host): length-limited Huffman
code lengths and canonical codes on random and adversarial histograms, and the CRC-32 of a block assembled from its
threads' slices."""
import heapq
import subprocess
import zlib

import numpy as np
import pytest

from tests import bgzf_util as bu


@pytest.fixture(scope="module")
def dumper(tmp_path_factory):
    return bu.build_codes_dumper(tmp_path_factory.mktemp("bgzf"))


def codes(dumper, freqs, maxbits):
    return bu.huff_codes(dumper, freqs, maxbits)


def huffman_cost(freqs):
    """Cost of an unrestricted Huffman code, and its longest length."""
    h = [(f, i, 0) for i, f in enumerate(freqs) if f]
    if len(h) < 2:
        return sum(freqs), (1 if h else 0)
    depth = {}
    heap = [(f, i, (i,)) for f, i, _ in h]
    heapq.heapify(heap)
    k = len(freqs)
    while len(heap) > 1:
        a, b = heapq.heappop(heap), heapq.heappop(heap)
        for s in a[2] + b[2]:
            depth[s] = depth.get(s, 0) + 1
        heapq.heappush(heap, (a[0] + b[0], k, a[2] + b[2]))
        k += 1
    return sum(freqs[s] * d for s, d in depth.items()), max(depth.values())


def check(dumper, freqs, maxbits):
    lens, cds = codes(dumper, freqs, maxbits)
    used = [i for i, f in enumerate(freqs) if f]
    assert all((lens[i] > 0) == (freqs[i] > 0) for i in range(len(freqs)))
    assert max(lens, default=0) <= maxbits
    kraft = sum(2.0 ** -l for l in lens if l)
    assert kraft <= 1.0
    if len(used) >= 2:
        assert kraft == 1.0
    # prefix-free: the codes, read MSB first, are distinct and none is a prefix of another
    words = sorted(format(int(format(cds[i], "0%db" % lens[i])[::-1], 2), "0%db" % lens[i]) for i in used)
    for a, b in zip(words, words[1:]):
        assert not b.startswith(a), (a, b)
    cost = sum(freqs[i] * lens[i] for i in used)
    best, longest = huffman_cost(freqs)
    if longest <= maxbits and len(used) >= 2:
        assert cost <= 1.01 * best, (cost, best)
    return lens


def test_degenerate_histograms(dumper):
    assert check(dumper, [0] * 286, 15) == [0] * 286
    one = [0] * 286
    one[256] = 1
    assert check(dumper, one, 15)[256] == 1
    two = [0] * 30
    two[3], two[17] = 5, 1
    lens = check(dumper, two, 15)
    assert lens[3] == lens[17] == 1
    check(dumper, [1] * 286, 15)                                     # all 286 symbols
    check(dumper, [7] * 19, 7)


def test_fibonacci_counts_hit_the_length_limit(dumper):
    fib = [1, 1]
    while len(fib) < 30:
        fib.append(fib[-1] + fib[-2])
    assert huffman_cost(fib)[1] > 15
    lens = check(dumper, fib, 15)
    assert max(lens) == 15
    assert huffman_cost(fib[:19])[1] > 7
    assert max(check(dumper, fib[:19], 7)) == 7
    big = fib + [0] * 200 + fib[:30] + [1] * 26
    check(dumper, big, 15)


def test_random_histograms(dumper):
    rng = np.random.default_rng(5)
    for t in range(60):
        n = [286, 30, 19][t % 3]
        maxbits = 7 if n == 19 else 15
        f = rng.integers(0, 3, size=n) * rng.geometric(0.01 if t % 2 else 0.3, size=n)
        if t % 5 == 0:
            f = (rng.pareto(0.7, size=n) * 10).astype(np.int64) * (rng.random(n) < 0.7)
        check(dumper, [int(x) for x in f], maxbits)


@pytest.mark.parametrize("pieces", [1, 3, 512])
def test_crc_from_slices_matches_zlib(dumper, tmp_path, pieces):
    rng = np.random.default_rng(pieces)
    for size in (0, 1, 127, 65280):
        data = rng.integers(0, 256, size=size, dtype=np.uint8).tobytes()
        p = tmp_path / "d.bin"
        p.write_bytes(data)
        r = subprocess.run([dumper, "crc", str(pieces), str(p)], capture_output=True, text=True, check=True)
        assert int(r.stdout) == zlib.crc32(data) & 0xffffffff, (pieces, size)
