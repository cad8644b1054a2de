"""Hand-written wgmma/TMA GEMM with fused bias+ReLU epilogue vs a PyTorch fp32 reference."""
import pytest
import torch

from distributed_embeddings_b200.ops import _native

pytestmark = pytest.mark.gpu

SHAPES = [
    (128, 256, 64), (128, 128, 64), (256, 256, 128), (1000, 512, 16), (4096, 1024, 480),
    (777, 256, 512), (8192, 1024, 1024), (300, 128, 256), (128, 8, 64), (5000, 1024, 200),
]


@pytest.mark.parametrize("m,n,k", SHAPES)
@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("block_n", [0, 128])
def test_gemm_matches_reference(m, n, k, relu, block_n):
  ops = _native.require()
  torch.manual_seed(m + n + k)
  a = (torch.randn(m, k, device="cuda") * 0.5).bfloat16()
  b = (torch.randn(n, k, device="cuda") * 0.5).bfloat16()
  bias = torch.randn(n, device="cuda").bfloat16()
  out = torch.full((m, n), 3.0, device="cuda", dtype=torch.bfloat16)
  ops.gemm_tn_bias_act(a, b, bias, out, relu, block_n)
  ref = a.float() @ b.float().t() + bias.float()
  if relu:
    ref = torch.relu(ref)
  torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=2e-2 * (k**0.5) * 0.25 + 1e-2)


def test_gemm_strided_views_and_no_bias():
  ops = _native.require()
  torch.manual_seed(0)
  big_a = (torch.randn(512, 96, device="cuda")).bfloat16()
  a = big_a[:, :64]                      # row stride 96, K = 64
  b = (torch.randn(256, 64, device="cuda")).bfloat16()
  big_out = torch.zeros(512, 320, device="cuda", dtype=torch.bfloat16)
  out = big_out[:, 32:288]               # column offset view, ldc = 320
  ops.gemm_tn_bias_act(a, b, None, out, False, 0)
  ref = a.float() @ b.float().t()
  torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=0.1)
  assert torch.count_nonzero(big_out[:, :32]) == 0 and torch.count_nonzero(big_out[:, 288:]) == 0


@pytest.mark.parametrize("m,n,k", [(4096, 512, 256), (777, 256, 1024), (8192, 1024, 1024),
                                   (1000, 128, 256)])
def test_fused_dgrad_relu_bias(m, n, k):
  """dx = (dy @ W) * (x > 0) and db = colsum(dx) in one wgmma kernel (W^T given K-major)."""
  ops = _native.require()
  torch.manual_seed(m + n)
  dy = (torch.randn(m, k, device="cuda") * 0.5).bfloat16()
  w = (torch.randn(k, n, device="cuda") * 0.1).bfloat16()      # layer weight [out=k, in=n]
  x = torch.relu(torch.randn(m, n, device="cuda")).bfloat16()   # activation of the layer below
  dx = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
  colsum = torch.zeros(n, device="cuda")
  ops.gemm_dgrad_relu_bias(dy, w.t().contiguous(), x, dx, colsum, 0)
  ref = (dy.float() @ w.float()) * (x > 0)
  torch.testing.assert_close(dx.float(), ref, rtol=2e-2, atol=5e-2)
  torch.testing.assert_close(colsum, ref.sum(0), rtol=2e-2, atol=0.5)


@pytest.mark.parametrize("m,n,k", [(256, 256, 64), (512, 256, 128), (4096, 1024, 480),
                                   (8192, 1024, 1024), (777, 512, 512), (300, 256, 256)])
@pytest.mark.parametrize("relu", [True, False])
def test_gemm_cta_pair_matches_reference(m, n, k, relu):
  """block_n=512 selects the 2-CTA cluster kernel (256x256 tile, B tile multicast to both CTAs)."""
  ops = _native.require()
  torch.manual_seed(m + n + k)
  a = (torch.randn(m, k, device="cuda") * 0.5).bfloat16()
  b = (torch.randn(n, k, device="cuda") * 0.5).bfloat16()
  bias = torch.randn(n, device="cuda").bfloat16()
  out = torch.full((m, n), 3.0, device="cuda", dtype=torch.bfloat16)
  ops.gemm_tn_bias_act(a, b, bias, out, relu, 512)
  torch.cuda.synchronize()
  ref = a.float() @ b.float().t() + bias.float()
  if relu:
    ref = torch.relu(ref)
  torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=2e-2 * (k**0.5) * 0.25 + 1e-2)
