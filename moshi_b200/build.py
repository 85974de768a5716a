"""Builds ``moshi_b200/_C/libmoshi_b200.so`` in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
OUT_DIR = HERE / "_C"
LIB = OUT_DIR / "libmoshi_b200.so"
SOURCES = ["common.cu", "mimi.cu", "lm.cu", "ops.cu", "gemm_sk.cu", "gemm_ns.cu", "dep_fused.cu", "frame.cu", "mimi_tc.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found; cannot build the sm_90a extension")


def _digest(files: list[Path]) -> str:
    h = hashlib.sha256()
    for f in sorted(files):
        h.update(f.name.encode())
        h.update(f.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    OUT_DIR.mkdir(exist_ok=True)
    srcs = [CSRC / s for s in SOURCES if (CSRC / s).exists()]
    deps = srcs + sorted(CSRC.glob("*.cuh")) + [HERE.parent / "include" / "moshi_b200.h"]
    stamp = OUT_DIR / "build.sha256"
    digest = _digest(deps)
    if LIB.exists() and stamp.exists() and stamp.read_text() == digest and not force:
        return LIB
    nvcc = _nvcc()
    objs, logs, procs = [], [], []
    for s in srcs:
        obj = OUT_DIR / (s.stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(s), "-o", str(obj)]
        procs.append((s, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = None
    for s, obj, p in procs:
        out, _ = p.communicate()
        logs.append(f"### {s.name}\n{out}")
        if p.returncode != 0:
            sys.stderr.write(out)
            failed = failed or s.name
        objs.append(str(obj))
    if failed:
        raise RuntimeError(f"nvcc failed on {failed}")
    cmd = [nvcc, "-shared", "-o", str(LIB), *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    (OUT_DIR / "ptxas.log").write_text("\n".join(logs))
    stamp.write_text(digest)
    if verbose:
        print("\n".join(logs))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
