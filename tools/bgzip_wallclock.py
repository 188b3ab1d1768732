"""Wall-clock of `filtlong --bgzip > out.gz` against `filtlong | gzip -1 > out.gz` and the plain run writing an uncompressed
file, on a FASTQ file made by bgzf_bench.py's generator (bench.py's C2 read lengths and qualities, ONT-style headers).

    python tools/bgzip_wallclock.py --gbases 10 --dir /tmp/bgz [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CLI = os.path.join(ROOT, "filtlong_b200", "bin", "filtlong")


def timed(cmd, **kw):
    t0 = time.perf_counter()
    r = subprocess.run(cmd, shell=True, **kw)
    return time.perf_counter() - t0, r.returncode


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbases", type=float, default=10.0)
    ap.add_argument("--dir", required=True)
    ap.add_argument("--out")
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bgzf_bench
    os.makedirs(a.dir, exist_ok=True)
    fq = os.path.join(a.dir, "reads.fastq")
    with open(fq, "wb") as f:                                   # 2 Gbases per piece, each from its own seed
        left, seed = a.gbases * 1e9, 11
        while left > 0:
            t = bgzf_bench.fastq_text(min(left, 2e9) * 2.02, seed=seed)
            f.write(memoryview(t))
            left -= 2e9
            seed += 1
            del t
            print("written", f.tell(), flush=True)
    size = os.path.getsize(fq)
    args = "-p 90 " + fq
    res = {"input_bytes": size, "command": "filtlong " + args}
    d = a.dir
    res["plain_s"], rc1 = timed("%s %s > %s/plain.fastq" % (CLI, args, d), stderr=subprocess.DEVNULL)
    res["plain_bytes"] = os.path.getsize(d + "/plain.fastq")
    os.remove(d + "/plain.fastq")
    print("plain", res["plain_s"], flush=True)
    res["bgzip_s"], rc2 = timed("%s --bgzip %s > %s/bgzip.fastq.gz" % (CLI, args, d), stderr=subprocess.DEVNULL)
    res["bgzip_bytes"] = os.path.getsize(d + "/bgzip.fastq.gz")
    os.remove(d + "/bgzip.fastq.gz")
    print("bgzip", res["bgzip_s"], flush=True)
    res["pipe_gzip1_s"], rc3 = timed("set -o pipefail; %s %s | gzip -1 > %s/pipe.fastq.gz" % (CLI, args, d),
                                     stderr=subprocess.DEVNULL, executable="/bin/bash")
    res["pipe_gzip1_bytes"] = os.path.getsize(d + "/pipe.fastq.gz")
    os.remove(d + "/pipe.fastq.gz")
    os.remove(fq)
    res["exit_codes"] = [rc1, rc2, rc3]
    line = json.dumps(res)
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
