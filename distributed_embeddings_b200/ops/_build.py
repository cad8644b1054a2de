"""In-tree build of the native extension (``distributed_embeddings_b200/_C.so``).

Kernels are compiled with nvcc for sm_90a only (``-gencode arch=compute_90a,code=sm_90a``);
the torch bindings are compiled with the host compiler so the CUDA files never include torch
headers (seconds per file).  The resulting shared object is loaded with
``torch.ops.load_library`` - there is no JIT step at import time, the .so travels with the tree.

Reference counterpart: ``Makefile`` (nvcc + g++ against TF flags, Makefile:22-55).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from typing import List

PKG_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(PKG_DIR, "ops", "csrc")
BUILD_DIR = os.path.join(PKG_DIR, "ops", "_build")
SO_PATH = os.path.join(PKG_DIR, "_C.so")

CU_SOURCES = ["lookup_kernels.cu", "sparse_update_kernels.cu", "misc_kernels.cu", "comm_kernels.cu",
              "dense_kernels.cu", "gemm_wgmma.cu", "radix_sort.cu",
              "offload_cache.cu", "eval_auc.cu"]
CPP_SOURCES = ["bindings.cpp"]

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc() -> str:
  cand = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
  if not os.path.exists(cand):
    raise RuntimeError("nvcc not found; set NVCC or add CUDA to PATH")
  return cand


def _cuda_home() -> str:
  return os.path.dirname(os.path.dirname(os.path.realpath(_nvcc())))


def _torch_paths():
  import torch
  from torch.utils import cpp_extension
  inc = cpp_extension.include_paths()
  lib = cpp_extension.library_paths()
  abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
  return inc, lib, abi


def _digest(paths: List[str], extra: str) -> str:
  h = hashlib.sha256(extra.encode())
  for p in sorted(paths):
    with open(p, "rb") as f:
      h.update(f.read())
  return h.hexdigest()


def _run(cmd: List[str]):
  res = subprocess.run(cmd, capture_output=True, text=True)
  if res.returncode != 0:
    raise RuntimeError("build command failed:\n" + " ".join(cmd) + "\n" + res.stdout + res.stderr)
  return res.stdout + res.stderr


def build(force: bool = False, verbose: bool = False) -> str:
  """Compile every CUDA/C++ source for sm_90a and link ``_C.so``.  Returns the .so path."""
  os.makedirs(BUILD_DIR, exist_ok=True)
  cu = [os.path.join(CSRC, s) for s in CU_SOURCES if os.path.exists(os.path.join(CSRC, s))]
  cpp = [os.path.join(CSRC, s) for s in CPP_SOURCES]
  headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
  inc, lib, abi = _torch_paths()
  stamp = os.path.join(BUILD_DIR, "stamp.txt")
  import torch
  digest = _digest(cu + cpp + headers, torch.__version__ + sys.version)
  if (not force and os.path.exists(SO_PATH) and os.path.exists(stamp) and
      open(stamp).read().strip() == digest):
    return SO_PATH

  nvcc = _nvcc()
  cuda_inc = os.path.join(_cuda_home(), "include")
  common_cu = [
      nvcc, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
      "-Xptxas", "-v" if verbose else "-warn-spills", "-diag-suppress", "550,177",
      "-Wno-deprecated-declarations"
  ] + ARCH_FLAGS + ["-I", CSRC]
  objs = []
  jobs = []
  for src in cu:
    obj = os.path.join(BUILD_DIR, os.path.basename(src) + ".o")
    objs.append(obj)
    jobs.append(common_cu + ["-c", src, "-o", obj])
  cxx = os.environ.get("CXX", "g++")
  for src in cpp:
    obj = os.path.join(BUILD_DIR, os.path.basename(src) + ".o")
    objs.append(obj)
    cmd = [cxx, "-O2", "-std=c++17", "-fPIC", "-Wno-deprecated-declarations",
           f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-DTORCH_API_INCLUDE_EXTENSION_H", "-I", CSRC, "-I",
           cuda_inc, "-I", sysconfig.get_paths()["include"]]
    for i in inc:
      cmd += ["-isystem", i]
    cmd += ["-c", src, "-o", obj]
    jobs.append(cmd)
  with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as pool:
    outs = list(pool.map(_run, jobs))
  if verbose:
    for o in outs:
      print(o)
  link = [cxx, "-shared", "-o", SO_PATH] + objs
  for l in lib:
    link += ["-L", l, f"-Wl,-rpath,{l}"]
  # static CUDA runtime of the toolkit that compiled the kernels (torch ships its own cudart)
  link += ["-lc10", "-ltorch_cpu", "-ltorch", "-lc10_cuda", "-ltorch_cuda", "-L",
           os.path.join(_cuda_home(), "lib64"), "-lcudart_static", "-lrt", "-ldl", "-lpthread"]
  _run(link)
  with open(stamp, "w") as f:
    f.write(digest)
  return SO_PATH


if __name__ == "__main__":
  path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
  print("built", path)
