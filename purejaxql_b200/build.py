"""Builds libpqn_b200.so in-tree with nvcc for sm_90a.

    python -m purejaxql_b200.build [--force]

Explicit nvcc (no torch cpp_extension): the library has a plain C ABI and does
not link libtorch.  pqn_env.cu is compiled with -fmad=false (fp32 physics round
as written); the network/optimizer units use default FMA contraction.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libpqn_b200.so")
BUILD = os.path.join(HERE, "csrc", "_build")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
UNITS = [
    ("pqn_api.cu", []),
    ("pqn_env.cu", ["-fmad=false"]),
    ("pqn_net.cu", []),
    ("pqn_optim.cu", []),
    ("pqn_perm.cu", []),
    ("pqn_pbt.cu", []),
    ("pqn_tc.cu", []),
]


def _deps():
    out = []
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for f in os.listdir(root):
            if f.endswith((".cu", ".cuh", ".h")):
                out.append(os.path.join(root, f))
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    deps = _deps()
    newest = max(os.path.getmtime(d) for d in deps)
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= newest:
        return OUT
    nvcc = os.environ.get("NVCC", "nvcc")
    objs = []
    procs = []
    for src, extra in UNITS:
        path = os.path.join(CSRC, src)
        if not os.path.exists(path):
            continue
        obj = os.path.join(BUILD, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc] + ARCH + COMMON + extra + ["-c", path, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, pr in procs:
        out, _ = pr.communicate()
        log.append(f"==== {src}\n{out}")
        if pr.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {src}")
    with open(os.path.join(BUILD, "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    subprocess.check_call([nvcc] + ARCH + ["-shared", "-o", OUT] + objs)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
