"""Build libbin_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libbin_b200.so")
SOURCES = ["conv_igemm.cu", "rdb_tail.cu", "aux_kernels.cu", "wgrad.cu", "metrics.cu", "png.cu", "api.cu"]
HEADERS = ["common.cuh", "wgmma.cuh", "xstack.cuh", "internal.h", os.path.join("..", "..", "include", "bin_b200.h")]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [*ARCH, "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _digest() -> str:
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def up_to_date(lib: str = LIB) -> bool:
    stamp = lib + ".sha256"
    return os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read().strip() == _digest()


def build(force: bool = False, verbose: bool = False) -> str:
    stamp = LIB + ".sha256"
    dig = _digest()
    if not force and up_to_date():
        return LIB
    objs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [_nvcc(), *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"== {src}\n{out}")
        if p.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed on {src}")
    # link to a temporary name and rename: a process that loads the library meanwhile never sees half a file
    fd, tmp = tempfile.mkstemp(prefix=".libbin_b200.", suffix=".so", dir=HERE)
    os.close(fd)
    cmd = [_nvcc(), "-shared", "-o", tmp, *objs, *ARCH]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    log.append(r.stdout)
    if r.returncode != 0:
        os.unlink(tmp)
        sys.stderr.write("\n".join(log))
        raise RuntimeError("link failed")
    os.chmod(tmp, 0o755)
    os.replace(tmp, LIB)
    with open(os.path.join(HERE, "build", "nvcc.log"), "w") as fh:
        fh.write("\n".join(log))
    with open(stamp, "w") as fh:
        fh.write(dig)
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
