"""``gemm_dgrad_relu_bias`` on the layer shapes of the DLRM step, against float64 references.

The op computes an MLP layer's data gradient with the ReLU backward of the layer below and that
layer's bias gradient in the GEMM epilogue: ``dx = (dy @ W) * (act > 0)``,
``colsum[:N] += sum_rows(dx)``.  The DLRM step runs it on every layer whose input is a ReLU output,
so these cases use the step's shapes (N x K = 512 x 256, 1024 x 512, 1024 x 1024 in the top MLP;
256 x 128 and 512 x 256 in the bottom MLP) at its batch of 65536 rows and at a ragged one.  The
bounds are those of ``test_dense_conformance.py``.

The kernel hands out tiles from a device counter that every launch resets, so it is also checked
next to a cuBLAS GEMM running on a second stream (CTAs become resident late and take fewer tiles)
and replayed from a CUDA graph (a counter left over from an earlier launch would skip tiles).
"""
import pytest
import torch

from test_dense_conformance import (  # pylint: disable=wrong-import-order
    _masked_colsum_bound, _ops, _randn, check_bits, check_close, check_zero, dot_bound, linear_ref)

# (N, K) of the step's dgrad GEMMs below a ReLU; 512 x 256 occurs in both MLPs
SHAPES = [(512, 256), (1024, 512), (1024, 1024), (256, 128)]
BATCH = 65536


def _inputs(m, n, k, seed):
  dy = _randn(m, k, scale=0.5, seed=seed)
  wt = _randn(n, k, scale=0.1, seed=seed + 1)
  act = _randn(m, n, seed=seed + 2)
  act.view(-1)[::5] = 0.0
  act.view(-1)[1::7] = -0.0
  dx_full = torch.full((m, n + 16), 3.0, dtype=torch.bfloat16, device="cuda")
  c0 = _randn(n + 8, seed=seed + 3, dtype=torch.float32)
  return dy, wt, act, dx_full, c0


def _check(case, dy, wt, act, dx_full, c0, colsum):
  n, k = wt.shape
  dx = dx_full[:, 8:8 + n]
  ref, mag = linear_ref(dy, wt)
  mask = act > 0
  eb = dot_bound(ref, mag, k)
  try:
    check_close("dgrad_epilogue/dx", dx, torch.where(mask, ref, torch.zeros_like(ref)), eb)
    check_zero("dgrad_epilogue/masked dx", torch.where(mask, torch.zeros_like(dx), dx))
    check_close("dgrad_epilogue/colsum", colsum[:n], c0[:n].double() + (ref * mask).sum(0),
                _masked_colsum_bound(ref, eb, mask, c0[:n].double()))
    check_bits("dgrad_epilogue/colsum beyond N", colsum[n:], c0[n:])
    check_bits("dgrad_epilogue/outside dx", dx_full[:, :8], torch.full_like(dx_full[:, :8], 3))
    check_bits("dgrad_epilogue/outside dx", dx_full[:, 8 + n:],
               torch.full_like(dx_full[:, 8 + n:], 3))
  except AssertionError as e:
    raise AssertionError(f"{case}: {e}") from None


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [0, 128, 256])
@pytest.mark.parametrize("n,k", SHAPES)
@pytest.mark.parametrize("m", [BATCH, BATCH - 37])
def test_dlrm_shapes(m, n, k, block_n):
  ops = _ops()
  dy, wt, act, dx_full, c0 = _inputs(m, n, k, seed=m + n + k + block_n)
  colsum = c0.clone()
  ops.gemm_dgrad_relu_bias(dy, wt, act, dx_full[:, 8:8 + n], colsum, block_n)
  torch.cuda.synchronize()
  _check(f"M={m} N={n} K={k} block_n={block_n}", dy, wt, act, dx_full, c0, colsum)


@pytest.mark.gpu
@pytest.mark.parametrize("n,k", [(1024, 1024), (256, 128)])
def test_next_to_a_concurrent_gemm(n, k):
  """The step runs the weight-gradient GEMMs on a second stream while the dgrad runs."""
  ops = _ops()
  m = BATCH - 37
  dy, wt, act, dx_full, c0 = _inputs(m, n, k, seed=5 * n + k)
  colsum = c0.clone()
  a = _randn(4096, 8192, seed=1)
  b = _randn(8192, 4096, seed=2)
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    for _ in range(4):
      c = a @ b
  ops.gemm_dgrad_relu_bias(dy, wt, act, dx_full[:, 8:8 + n], colsum, 0)
  torch.cuda.current_stream().wait_stream(side)
  torch.cuda.synchronize()
  _check(f"concurrent M={m} N={n} K={k}", dy, wt, act, dx_full, c0, colsum)
  del c


@pytest.mark.gpu
def test_graph_replays_match_eager_calls():
  """Three replays of a captured launch against three eager launches on the same inputs."""
  ops = _ops()
  m, n, k = BATCH - 37, 512, 256
  dy, wt, act, dx_full, c0 = _inputs(m, n, k, seed=11)
  colsum = c0.clone()
  dx = dx_full[:, 8:8 + n]
  ops.gemm_dgrad_relu_bias(dy, wt, act, dx, colsum, 0)  # module load outside the capture
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    ops.gemm_dgrad_relu_bias(dy, wt, act, dx, colsum, 0)
  for r in range(3):
    s_dy, s_wt, s_act, _, s_c0 = _inputs(m, n, k, seed=100 + r)
    dy.copy_(s_dy)
    wt.copy_(s_wt)
    act.copy_(s_act)
    dx_full.fill_(3.0)
    colsum.copy_(s_c0)
    g.replay()
    eager_full = torch.full_like(dx_full, 3.0)
    eager_colsum = s_c0.clone()
    ops.gemm_dgrad_relu_bias(s_dy, s_wt, s_act, eager_full[:, 8:8 + n], eager_colsum, 0)
    torch.cuda.synchronize()
    check_bits("dgrad_epilogue/graph replay vs eager dx", dx_full, eager_full)
    _check(f"graph replay {r}", dy, wt, act, dx_full, s_c0, colsum)
