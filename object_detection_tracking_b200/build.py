"""Builds libb200det.so in-tree with nvcc for sm_90a (H100; no JIT cache: the .so sits next to this file)."""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libb200det.so")
SOURCES = ["engine_core.cu", "detplan.cu", "engine.cu", "ops.cu", "gemm_ws.cu", "conv_tc.cu", "conv_simt.cu", "stem.cu", "rpn.cu",
           "roialign.cu", "head.cu", "cosine.cu", "reid.cu", "reid_engine.cu", "effdet.cu", "effnet.cu", "effdet_engine.cu",
           "tracker.cpp", "tmot.cpp", "pairmatch.cu", "groupnorm.cu", "relation.cu", "deform.cu",
           "att_head.cu", "reid_ingest.cu", "small_objects.cu", "mask_head.cu",
           "mask_rle.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-Xcompiler", "-O2",
              "-Xcompiler", "-Wno-attributes"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.sep not in cand or os.path.exists(cand)):
            return cand
    return "nvcc"


def _digest() -> str:
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for name in sorted(os.listdir(root)):
            if name.endswith((".cu", ".cuh", ".h", ".cpp")):
                with open(os.path.join(root, name), "rb") as f:
                    h.update(name.encode())
                    h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    stamp = OUT + ".sha"
    dig = _digest()
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return OUT
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    objs = []
    for src in SOURCES:
        obj = os.path.join(objdir, os.path.splitext(src)[0] + ".o")
        objs.append(obj)
        cmd = [_nvcc(), *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write("nvcc failed for %s:\n%s\n" % (src, out))
        elif verbose and out:
            sys.stderr.write(out)
    if failed:
        raise RuntimeError("libb200det build failed")
    link = [_nvcc(), "-shared", "-o", OUT, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout)
    with open(stamp, "w") as f:
        f.write(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
