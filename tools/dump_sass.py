#!/usr/bin/env python
"""Full SASS listings of the hot kernels of ``_C.so`` (one file per kernel under
``sass/`` of the output directory, default the current one; cuobjdump runs without a GPU):

    python tools/dump_sass.py            # the curated list below
    python tools/dump_sass.py --all      # every kernel (large)

The listings are the evidence for what the kernels are built from: peer-memory ``STG`` /
``LDG`` and the system-scope flag protocol (``ST.E.STRONG.SYS`` / ``LD.E.STRONG.SYS``) inside the
data kernels, ``REDG.E.ADD.F32x4`` table updates, ``LDGSTS`` + ``LDSM`` + ``HMMA`` interaction,
``UTMALDG`` / ``HGMMA`` GEMMs, ``LDGMC`` multimem all-reduce."""
import argparse
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "distributed_embeddings_b200", "_C.so")
OUT = os.path.join(os.getcwd(), "sass")

# (file stem, regex on the demangled name): the instantiations the DLRM / synthetic steps run
HOT = [
    ("lookup_fwd_i32_bf16_v4", r"lookup_fwd_kernel<int, __nv_bfloat16, 4, float>"),
    ("lookup_fwd_i32_f32_v4", r"lookup_fwd_kernel<int, float, 4, float>"),
    ("scatter_add_bwd_i32_bf16_v4", r"scatter_add_bwd_kernel<int, __nv_bfloat16, 4>"),
    ("push_segments_i32", r"push_segments_kernel<int>"),
    ("push_grad_bf16_bf16", r"push_grad_kernel<__nv_bfloat16, __nv_bfloat16>"),
    ("sync_only", r"sync_only_kernel"),
    ("rowslice_reduce_bf16", r"rowslice_reduce_kernel<__nv_bfloat16>"),
    ("interact_fwd_128", r"interact_fwd_kernel<128>"),
    ("interact_bwd_v2_128", r"interact_bwd_v2_kernel<128>"),
    ("interact_bwd_apply_128", r"interact_bwd_apply_kernel<128>"),
    ("allreduce_p2p_f32", r"allreduce_p2p_kernel<(false|0)>"),
    ("allreduce_multimem_f32", r"allreduce_multimem_kernel<(false|0)>"),
    ("segment_update_bf16_v4", r"segment_update_kernel<__nv_bfloat16, 4, float, float, 0>"),
    ("balanced_update_bf16", r"balanced_update_kernel<__nv_bfloat16, float, float, 0>"),
    ("scatter_add_staged_i32_bf16", r"scatter_add_staged_kernel<int, __nv_bfloat16>"),
    ("stream_push", r"stream_push_kernel"),
    ("build_keys_i32_u32", r"build_keys_kernel<int, unsigned int>"),
    ("digit_hist_u32", r"digit_hist_kernel<unsigned int>"),
    ("digit_scatter_u32_u32", r"digit_scatter_kernel<unsigned int, unsigned int>"),
    ("head_compact", r"head_compact_kernel"),
    ("avgpool_fwd", r"avgpool_fwd_kernel"),
    ("gemm_tn_fused", r"gemm_tn_fused_kernel"),
    ("gemm_tn_pair", r"gemm_tn_pair_kernel"),
    ("integer_lookup", r"integer_lookup_kernel"),
    ("relu_bwd_bias", r"relu_bwd_bias_kernel"),
    ("cross_fwd", r"cross_fwd_kernel"),
    ("cross_bwd", r"cross_bwd_kernel"),
    ("cross_dx0", r"cross_dx0_kernel"),
    ("head_loss_8", r"head_loss_kernel<8>"),
    ("head_eval_8", r"head_eval_kernel<8>"),
    ("sgd_update", r"sgd_update_kernel"),
    ("dense_opt_adagrad", r"dense_opt_kernel<1>"),
    ("dense_opt_adam", r"dense_opt_kernel<3>"),
    ("cache_spill_writeback", r"cache_spill_writeback_kernel"),
    ("cache_probe", r"cache_probe_kernel"),
    ("cache_assign", r"cache_assign_kernel"),
    ("cache_fill", r"cache_fill_kernel"),
    ("cache_remap_i32", r"cache_remap_kernel<int>"),
    ("cache_flush", r"cache_flush_kernel"),
]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--all", action="store_true")
  args = ap.parse_args()
  sass = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True,
                        check=True).stdout
  blocks = [b for b in re.split(r"(?=\n\s*Function : )", sass) if "Function : " in b]
  names = [re.search(r"Function : (\S+)", b).group(1) for b in blocks]
  dem = subprocess.run(["cu++filt"] + names, capture_output=True, text=True,
                       check=False).stdout.splitlines()
  os.makedirs(OUT, exist_ok=True)
  written = []
  for body, mangled, name in zip(blocks, names, dem):
    name = re.sub(r"\(anonymous namespace\)::|<unnamed>::", "", name)
    name = re.sub(r"\((?:int|bool)\)", "", name)  # cu++filt prints template ints as (int)4
    stems = [s for s, rx in HOT if re.search(rx, name)]
    if args.all and not stems:
      stems = [re.sub(r"[^A-Za-z0-9]+", "_", name)[:80]]
    for stem in stems[:1]:
      # some templates are instantiated several times (e.g. tile shapes): number them
      path = os.path.join(OUT, stem + ".sass")
      k = 1
      while path in written:
        k += 1
        path = os.path.join(OUT, f"{stem}_{k}.sass")
      # drop the hex encodings (second line of every instruction + trailing comment): the
      # mnemonics and operands are the evidence, the listing stays half the size
      lines = []
      for line in body.strip().splitlines():
        if re.match(r"\s+/\* 0x[0-9a-f]{16} \*/\s*$", line):
          continue
        lines.append(re.sub(r"\s*/\* 0x[0-9a-f]{16} \*/\s*$", "", line))
      with open(path, "w") as f:
        f.write(f"// {name}\n// {mangled}\n" + "\n".join(lines) + "\n")
      written.append(path)
  for p in written:
    n = sum(1 for line in open(p) if re.match(r"\s+/\*[0-9a-f]{4}\*/", line))
    print(f"{os.path.relpath(p, ROOT)}: {n} instructions")


if __name__ == "__main__":
  sys.exit(main())
