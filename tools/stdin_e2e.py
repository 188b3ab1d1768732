"""Input reads from a pipe against the same reads as a file, through the `filtlong` command line: C2-like reads (bench.py's
lengths and qualities, made by fl_synth with bgzf_bench.py's seeds) written once as FASTQ and once as BGZF (compressed on
the GPU with api.bgzf_compress), then `-p 90` on
    the file:                         filtlong -p 90 reads.fastq > out
    the file through a pipe:          cat reads.fastq | filtlong -p 90 - > out
    the compressed file, inflated:    gzip -dc reads.fastq.gz | filtlong -p 90 - > out
with FL_CLI_TIMING=1, beside the producers on their own (`cat reads.fastq | cat > /dev/null`, `gzip -dc reads.fastq.gz >
/dev/null`). Reports wall-clock seconds, the CLI's phases (the stream line included), whether the three outputs are
identical, and the card's name and power limit, as one JSON line.

    python tools/stdin_e2e.py --gbases 10 --dir /tmp/stdin [--out result.json]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
CLI = os.path.join(ROOT, "filtlong_b200", "bin", "filtlong")
EOF_MEMBER = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def pipeline(producer, consumer, out_path, env=None):
    """producer | consumer > out_path; (seconds, consumer's rc, consumer's stderr)"""
    t0 = time.perf_counter()
    with open(out_path, "wb") as out:
        p1 = subprocess.Popen(producer, stdout=subprocess.PIPE) if producer else None
        try:
            p2 = subprocess.Popen(consumer, stdin=p1.stdout if p1 else subprocess.DEVNULL, stdout=out, stderr=subprocess.PIPE, env=env)
            if p1:
                p1.stdout.close()
            _, err = p2.communicate()
        finally:
            if p1:
                if p1.poll() is None:
                    p1.kill()
                p1.wait()
    return time.perf_counter() - t0, p2.returncode, err.decode(errors="replace")


def phases(err):
    res = {m.group(1).strip(): float(m.group(2)) for m in re.finditer(r"^\[timing\] (.+?) +([0-9.]+) s$", err, re.M)}
    m = re.search(r"^\[timing\] (stream: .*)$", err, re.M)
    if m:
        res["stream"] = m.group(1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbases", type=float, default=10.0)
    ap.add_argument("--dir", required=True)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    import bgzf_bench
    from filtlong_b200 import api
    os.makedirs(a.dir, exist_ok=True)
    fq, gz = os.path.join(a.dir, "reads.fastq"), os.path.join(a.dir, "reads.fastq.gz")
    t0 = time.time()
    with open(fq, "wb") as ff, open(gz, "wb") as fz, api.Context() as ctx:
        left, seed = a.gbases, 11
        while left > 0:                                     # 2 Gbases per piece, each from its own seed
            text = bgzf_bench.fastq_text(min(left, 2.0) * 1e9 * 2.02, seed=seed).tobytes()
            ff.write(text)
            fz.write(ctx.bgzf_compress(text, append_eof=False))
            del text
            left -= 2.0
            seed += 1
            print("written", ff.tell(), flush=True)
        fz.write(EOF_MEMBER)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    res = dict(gbases=a.gbases, write_seconds=round(time.time() - t0, 1), fastq_bytes=os.path.getsize(fq), gz_bytes=os.path.getsize(gz),
               gpu=gpu.strip().splitlines()[0] if gpu.strip() else "unknown", host_cpus=os.cpu_count())
    env = dict(os.environ, LC_ALL="C", FL_CLI_TIMING="1")
    runs = [("file", None, [CLI, "-p", "90", fq]),
            ("cat_pipe", ["cat", fq], [CLI, "-p", "90", "-"]),
            ("gzip_dc_pipe", ["gzip", "-dc", gz], [CLI, "-p", "90", "-"]),
            ("cat_alone", ["cat", fq], ["cat"]),
            ("gzip_dc_alone", None, ["gzip", "-dc", gz])]
    first = os.path.join(a.dir, "out_file")
    for rep in range(a.repeats):                          # alternated, so that the page cache and the host's load treat them alike
        for tag, prod, cons in runs:
            out = first if tag == "file" else os.path.join(a.dir, "out")
            if tag.endswith("alone"):
                out = os.devnull
            dt, rc, err = pipeline(prod, cons, out, env)
            r = dict(seconds=round(dt, 3), rc=rc)
            if cons[0] == CLI:
                r["phases"] = phases(err)
                r["output_bytes"] = os.path.getsize(out)
                if tag != "file":
                    r["same_output_as_file"] = subprocess.run(["cmp", "-s", first, out]).returncode == 0
                    os.remove(out)
            res.setdefault(tag, []).append(r)
            print(tag, rep, r, flush=True)
    for p in (fq, gz, first):
        os.remove(p)
    line = json.dumps(res)
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
