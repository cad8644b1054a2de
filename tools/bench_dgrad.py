#!/usr/bin/env python
"""MLP data gradients of the DLRM step below a ReLU: cuBLAS + ``relu_bwd_bias`` against the fused
wgmma kernel (``gemm_dgrad_relu_bias``), on the five layer shapes the step runs.

  python tools/bench_dgrad.py [--batch 65536] [--launches 200] [--repeats 5] [--out-dir bench_out]

For each shape (TN form: ``dy`` [M, K] x ``W^T`` [N, K] -> ``dx`` [M, N], masked by ``act > 0``,
column sums into the bias gradient) it times, with CUDA events over ``--launches`` launches after
a warm-up:

* ``pair``: ``torch.mm`` (cuBLAS) + ``ops.relu_bwd_bias``, what the step ran before;
* ``fused_bn{0,128,256}``: ``ops.gemm_dgrad_relu_bias`` at each ``block_n`` (0 = the kernel's own
  choice);

once alone and once next to the layer's weight-gradient GEMM (``dy^T x``, fp32 out, cuBLAS) on a
second stream, the way the step overlaps them: each launch pairs one data-gradient variant with
one weight-gradient GEMM, and the time is that of the pair.  Bytes are computed from the shapes
(pair: 2MK + 2NK + 2MN for the GEMM and 6MN for the mask pass; fused: 2MK + 2NK + 4MN) and set
against the H100 SXM data-sheet 3.35 TB/s; TFLOP/s against its 989 dense bf16.

Prints one JSON line per shape and writes them all to ``<out-dir>/bench_dgrad.json``, with the
card's name and power limit read in the same run.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
BF16_FLOPS = 989e12
# (N, K) of the dgrad GEMMs that feed a ReLU in the DLRM step: top MLP 1024-1024-512-256 and
# bottom MLP 512-256-128
SHAPES = [("top[2]", 512, 256), ("top[1]", 1024, 512), ("top[0]", 1024, 1024),
          ("bottom[1]", 256, 128), ("bottom[0]", 512, 256)]
BLOCK_NS = (0, 128, 256)


def gpu_info():
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
  name, power, clock = [x.strip() for x in out.stdout.splitlines()[0].split(",")]
  return {"name": name, "power_limit": power, "max_sm_clock": clock}


def _median(xs):
  xs = sorted(xs)
  return xs[len(xs) // 2]


def _time(fn, launches, repeats):
  ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  for _ in range(10):
    fn()
  torch.cuda.synchronize()
  times = []
  for _ in range(repeats):
    ev[0].record()
    for _ in range(launches):
      fn()
    ev[1].record()
    torch.cuda.synchronize()
    times.append(ev[0].elapsed_time(ev[1]) * 1e3 / launches)
  return _median(times), [min(times), max(times)]


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
  ap.add_argument("--batch", type=int, default=65536)
  ap.add_argument("--launches", type=int, default=200)
  ap.add_argument("--repeats", type=int, default=5)
  ap.add_argument("--out-dir", default="bench_out")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_dgrad.py needs a CUDA GPU")
  from distributed_embeddings_b200.ops import _native
  ops = _native.require()
  torch.cuda.set_device(0)
  gpu = gpu_info()
  print(json.dumps({"gpu": gpu}), flush=True)
  dev = torch.device("cuda", 0)
  side = torch.cuda.Stream(device=dev)
  M = args.batch
  rows = []
  for name, N, K in SHAPES:
    g = torch.Generator(device=dev).manual_seed(N * 7 + K)
    dy = (torch.randn(M, K, device=dev, generator=g) * 0.1).bfloat16()
    w = (torch.randn(K, N, device=dev, generator=g) * 0.05).bfloat16()  # the layer's [out, in]
    wT = w.t().contiguous()  # [N, K], K-major: the fused kernel's B operand
    act = torch.randn(M, N, device=dev, generator=g).bfloat16()  # the ReLU output below
    dx = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
    gb = torch.zeros(N, dtype=torch.float32, device=dev)
    gw = torch.empty(K, N, dtype=torch.float32, device=dev)

    def pair():
      torch.mm(dy, w, out=dx)
      ops.relu_bwd_bias(dx, act, gb)

    variants = {"pair": pair}
    for bn in BLOCK_NS:
      if bn > N:
        continue
      variants[f"fused_bn{bn}"] = (lambda bn=bn: ops.gemm_dgrad_relu_bias(dy, wT, act, dx, gb, bn))

    def with_wgrad(fn):
      def run():
        main = torch.cuda.current_stream()
        side.wait_stream(main)
        with torch.cuda.stream(side):
          torch.mm(dy.t(), act, out_dtype=torch.float32, out=gw)
        fn()
        main.wait_stream(side)
      return run

    flops = 2.0 * M * N * K
    nbytes = {"pair": 2 * M * K + 2 * N * K + 8 * M * N,
              "fused": 2 * M * K + 2 * N * K + 4 * M * N}
    res = {"layer": name, "M": M, "N": N, "K": K, "flops": flops, "bytes": nbytes, "gpu": gpu}
    wgrad_us, _ = _time(lambda: torch.mm(dy.t(), act, out_dtype=torch.float32, out=gw),
                        args.launches, args.repeats)
    res["wgrad_alone_us"] = wgrad_us
    for vname, fn in variants.items():
      us, spread = _time(fn, args.launches, args.repeats)
      b = nbytes["pair" if vname == "pair" else "fused"]
      res[vname] = {"us": us, "spread_us": spread, "TFLOPs": flops / (us * 1e-6) / 1e12,
                    "share_of_989": flops / (us * 1e-6) / BF16_FLOPS,
                    "TBps": b / (us * 1e-6) / 1e12,
                    "share_of_3.35TBps": b / (us * 1e-6) / HBM_BYTES_PER_S}
      us, spread = _time(with_wgrad(fn), args.launches, args.repeats)
      res[vname]["with_wgrad_us"] = us
      res[vname]["with_wgrad_spread_us"] = spread
    res["pair_parts_us"] = {
        "mm": _time(lambda: torch.mm(dy, w, out=dx), args.launches, args.repeats)[0],
        "relu_bwd_bias": _time(lambda: ops.relu_bwd_bias(dx, act, gb), args.launches,
                               args.repeats)[0]}
    rows.append(res)
    print(json.dumps(res), flush=True)
    del dy, w, wT, act, dx, gb, gw
    torch.cuda.empty_cache()
  os.makedirs(args.out_dir, exist_ok=True)
  with open(os.path.join(args.out_dir, "bench_dgrad.json"), "w") as f:
    json.dump({"gpu": gpu, "shapes": rows}, f, indent=1)


if __name__ == "__main__":
  main()
