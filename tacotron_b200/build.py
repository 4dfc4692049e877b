"""Build libtaco_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m tacotron_b200.build [--verbose]
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libtaco_b200.so")
SOURCES = ["api.cu", "gemm_simt.cu", "gemm_tc.cu", "gru.cu", "decoder.cu", "train.cu", "gru_bwd.cu", "decoder_bwd.cu", "audio.cu", "data.cu", "features.cu",
           "resample.cu", "summary.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _newest_src():
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "taco_b200.h")]
    return max(os.path.getmtime(p) for p in deps)


def build(force=False, verbose=False):
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _newest_src():
        return LIB
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc failed on {src} ---\n{out}\n")
        elif verbose or out.strip():
            sys.stderr.write(f"--- {src} ---\n{out}\n")
    if failed:
        raise RuntimeError("nvcc compilation failed")
    cmd = [NVCC, *FLAGS[:2], "-shared", "-o", LIB, *objs, "-lcudart_static", "-lrt", "-lpthread", "-ldl"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose="--verbose" in sys.argv))
