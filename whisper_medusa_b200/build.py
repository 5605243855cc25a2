"""In-tree build of the CUDA engine: nvcc -> whisper_medusa_b200/_lib/libwm_b200.so (sm_90a only).

``python -m whisper_medusa_b200.build`` or ``__graft_entry__.build()``.  Objects are rebuilt only
when a source or header is newer.  nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess
import sys
from typing import List

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "_lib")
OBJ_DIR = os.path.join(OUT_DIR, "obj")
LIB_PATH = os.path.join(OUT_DIR, "libwm_b200.so")
ROOT = os.path.dirname(HERE)

SOURCES = ["engine.cu", "decode.cu", "mel.cu", "enc_gemm.cu", "enc_attn.cu", "enc_gemm_tc.cu", "enc_attn_tc.cu",
           "resample.cu", "scores.cu", "no_speech.cu", "timestamps.cu", "logits_proc.cu"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xptxas", "-v",
    # the stage-sequence templates are __host__ __device__ and are instantiated with host lambdas on
    # the host side only; nvcc warns about the (never taken) device instantiation
    "-diag-suppress=20013,20015",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _newer(src_paths: List[str], target: str) -> bool:
    if not os.path.isfile(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(p) > t for p in src_paths)


def build(verbose: bool = False, force: bool = False, extra_flags: List[str] = (), lib_path: str = LIB_PATH,
          obj_dir: str = OBJ_DIR) -> str:
    """``extra_flags`` / ``lib_path`` / ``obj_dir``: alternative builds for A/B timing (tests/gpu_ab.py), e.g.
    ``build(extra_flags=["-DWM_EPI_PIPELINE=1"], lib_path="ab_libs/v1.so", obj_dir="ab_libs/obj_v1")``."""
    os.makedirs(obj_dir, exist_ok=True)
    os.makedirs(os.path.dirname(os.path.abspath(lib_path)), exist_ok=True)
    nvcc = _nvcc()
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers.append(os.path.join(ROOT, "include", "whisper_medusa_b200.h"))
    srcs = [s for s in SOURCES if os.path.isfile(os.path.join(CSRC, s))]

    def compile_one(src: str):
        sp = os.path.join(CSRC, src)
        obj = os.path.join(obj_dir, src.replace(".cu", ".o"))
        if not force and not _newer([sp] + headers, obj):
            return obj, ""
        cmd = [nvcc] + NVCC_FLAGS + list(extra_flags) + ["-I", os.path.join(ROOT, "include"), "-c", sp, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return obj, r.stderr

    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(compile_one, srcs))
    objs = [o for o, _ in results]
    log = "\n".join(l for _, l in results if l)
    if log:
        # register / spill report of this build (a full rebuild starts the file afresh; alternative builds keep their own)
        log_path = os.path.join(OUT_DIR, "ptxas.log") if obj_dir == OBJ_DIR else os.path.join(obj_dir, "ptxas.log")
        with open(log_path, "w" if all(l for _, l in results) else "a") as f:
            f.write(log + "\n")
        if verbose:
            print(log)
    if force or _newer(objs, lib_path):
        cmd = [nvcc, "-shared", "-o", lib_path] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return lib_path


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
