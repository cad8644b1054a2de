#!/usr/bin/env python
"""First-party wgmma GEMM (+bias+ReLU epilogue) vs cuBLASLt (_addmm_activation) on the DLRM layer shapes."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from distributed_embeddings_b200.ops import _native

ops = _native.require()


def timeit(fn, iters=20, warmup=5):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(iters):
    fn()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / iters * 1e3  # us


rows = []
batch = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
for (n, k) in [(512, 16), (256, 512), (128, 256), (1024, 480), (1024, 1024), (512, 1024),
               (256, 512)]:
  x = torch.randn(batch, k, device="cuda").bfloat16()
  w = torch.randn(n, k, device="cuda").bfloat16()
  bias = torch.randn(n, device="cuda").bfloat16()
  out = torch.empty(batch, n, device="cuda", dtype=torch.bfloat16)
  flops = 2.0 * batch * n * k
  t_lib = timeit(lambda: torch._addmm_activation(bias, x, w.t(), out=out))
  res = {"M": batch, "N": n, "K": k, "cublaslt_us": round(t_lib, 1),
         "cublaslt_tflops": round(flops / t_lib / 1e6, 1)}
  for bn in (256, 128):
    if n < bn:
      continue
    t = timeit(lambda: ops.gemm_tn_bias_act(x, w, bias, out, True, bn))
    res[f"wgmma_bn{bn}_us"] = round(t, 1)
    res[f"wgmma_bn{bn}_tflops"] = round(flops / t / 1e6, 1)
  if n >= 256:
    # 2-CTA cluster kernel (B tile multicast), see gemm_tn_pair_kernel
    t = timeit(lambda: ops.gemm_tn_bias_act(x, w, bias, out, True, 512))
    res["wgmma_pair_us"] = round(t, 1)
    res["wgmma_pair_tflops"] = round(flops / t / 1e6, 1)
  rows.append(res)
  print(json.dumps(res))
os.makedirs("gpurun_out", exist_ok=True)
json.dump(rows, open("gpurun_out/bench_gemm.json", "w"), indent=1)
