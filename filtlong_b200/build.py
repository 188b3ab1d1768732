"""Builds libfiltlong_b200.so (hand-written sm_90a CUDA behind a C ABI) in-tree with nvcc.

The shared object is a build product, kept out of git. No CPU fallback exists:
if the library is missing or cannot be loaded, importing filtlong_b200.capi raises.
"""
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
BUILD = os.path.join(PKG, "build")
LIB = os.path.join(PKG, "libfiltlong_b200.so")
SOURCES = ["fl_api.cu", "fl_scan.cu", "fl_kmers.cu", "fl_score.cu", "fl_phred.cu", "fl_qtrim.cu", "fl_select.cu", "fl_comm.cu", "fl_text.cu", "fl_synth.cu",
           "fl_contam_k.cu", "fl_bgzf.cu", "fl_bam.cu", "fl_inflate.cu", "fl_synth_host.cpp"]
HEADERS = ["fl_internal.cuh", "fl_device.cuh", "fl_synth.h", "fl_bgzf.h", "fl_bam_mods.h", "fl_inflate.h", "fl_name_hash.h", os.path.join("..", "..", "include", "filtlong_b200.h")]
# host-only synthetic generators on their own (no CUDA inside): what bench.py's CPU legs load
SYNTH_LIB = os.path.join(PKG, "libflsynth_host.so")
CXX = os.environ.get("CXX", "g++")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# --fmad=false: the per-read scores must follow the reference's unfused double arithmetic
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "--fmad=false", "-std=c++17",
         "-Xcompiler", "-fPIC,-O2,-ffp-contract=off", "-Xptxas", "-v"]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    objs = []
    procs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(BUILD, src.replace(".cu", ".o").replace(".cpp", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + hdrs):
            cmd = [NVCC] + FLAGS + ["-c", s, "-o", o]
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        with open(os.path.join(BUILD, src + ".ptxas.log"), "w") as f:
            f.write(out)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s" % src)
    if force or procs or _stale(LIB, objs):
        cmd = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs + ["-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    sh = os.path.join(CSRC, "fl_synth_host.cpp")
    if force or _stale(SYNTH_LIB, [sh] + hdrs):
        r = subprocess.run([CXX, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", SYNTH_LIB, sh], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("libflsynth_host.so build failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose=True))
