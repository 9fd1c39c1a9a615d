"""Build libmgproto_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m mgproto_b200.build [--force]

The .so and the objects under build/ are build products (git-ignored).
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmgproto_b200.so")
STAMP = LIB + ".stamp"
SOURCES = ["abi.cu", "normalize.cu", "logprob_simt.cu", "logprob_tc.cu", "logprob_tcz.cu", "log_density.cu", "head.cu", "bank.cu", "em.cu", "em_tc.cu", "em_api.cu", "push.cu", "aux_loss.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--use_fast_math=false",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-DMGP_WITH_TC"]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def _digest() -> str:
    h = hashlib.sha256()
    files = sorted(os.listdir(CSRC)) + ["../../include/mgproto_b200.h"]
    for f in files:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(f.encode())
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == dig:
        return LIB
    flags = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"]
    objs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    # per-object stamps: an object is recompiled when its source, any header or the flags changed
    hdr = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)) + ["../../include/mgproto_b200.h"]:
        if f.endswith((".cuh", ".h")):
            hdr.update(open(os.path.join(CSRC, f), "rb").read())
    hdr.update(" ".join(NVCC_FLAGS).encode())
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        objs.append(obj)
        h = hdr.copy()
        h.update(open(os.path.join(CSRC, src), "rb").read())
        odig = h.hexdigest()
        if os.path.exists(obj) and os.path.exists(obj + ".stamp") and open(obj + ".stamp").read().strip() == odig:
            continue
        cmd = [_nvcc(), *flags, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, obj, odig, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, obj, odig, p in procs:
        out, _ = p.communicate()
        log.append("== %s\n%s" % (src, out))
        if p.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, out))
        with open(obj + ".stamp", "w") as fh:
            fh.write(odig)
        with open(os.path.join(HERE, "build", src.replace(".cu", ".ptxas.log")), "w") as fh:
            fh.write(out)
    if verbose:
        print("\n".join(log))
    cmd = [_nvcc(), "-shared", "-o", LIB, *objs, "-lcudart", "-lcuda"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout)
    with open(STAMP, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
