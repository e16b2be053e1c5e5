"""In-tree build of libsod_b200.so (nvcc, sm_90a only).  `python -m distributed_sod_project_b200.build`."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsod_b200.so")
OBJDIR = os.path.join(HERE, "build")
STAMP = os.path.join(OBJDIR, "arch.txt")   # the target LIB was built for: a library for another target is rebuilt
SOURCES = ("api.cu", "loss.cu", "sgd.cu", "syncbn.cu", "resample.cu", "nearest.cu", "maxpool.cu", "pipeline.cu", "resize.cu", "augment.cu", "joint.cu", "wfm.cu", "wsgn.cu", "gconv.cu")
ARCH = ("-gencode", "arch=compute_90a,code=sm_90a")
NVCC_FLAGS = (
    *ARCH, "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O2", "-I" + os.path.join(ROOT, "include"),
)


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (needed to build libsod_b200.so)")


def _stamp_text() -> str:
    return " ".join(ARCH) + "\n"


def needs_build() -> bool:
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        if f.read() != _stamp_text():
            return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "sod_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every .cu for sm_90a into one shared library next to this file. Returns its path."""
    if not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    os.makedirs(OBJDIR, exist_ok=True)
    procs = []
    for src in SOURCES:
        obj = os.path.join(OBJDIR, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    objs = []
    for src, obj, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
        if verbose and out:
            print(out)
        objs.append(obj)
    cmd = [nvcc, "-shared", "-o", LIB, *objs, *ARCH]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if out.returncode != 0:
        raise RuntimeError(f"link failed:\n{out.stdout}")
    with open(STAMP, "w") as f:
        f.write(_stamp_text())
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
