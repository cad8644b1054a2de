"""Dense kernels of the DLRM step against float64 references, with bounds derived from each op.

Every reference runs in float64 on the same bf16 / fp32 operands the kernel reads, and every
tolerance follows from the operation (see the helpers below), so a kernel that rounds the wrong
way, drops a block of terms, adds its bias after rounding or writes one tail element off fails
here with the kernel, the case and the element named.  The second half checks every stage of the
single-GPU ``DLRMTrainStep`` on that stage's own inputs, taken from the step's retained buffers,
so errors do not compound and the same bounds apply unchanged.

Bounds (u16 = 2^-8 is the unit roundoff of bf16, u32 = 2^-24 that of fp32):

* bf16 output of an fp32-accumulated dot of K terms (a bias counts as one more term):
  ``|out - ref| <= u16 * (|ref| + E) + E + tiny`` with ``E = 2 * K * u32 * sum|a_i * b_i|``.
  ``K * u32 * sum|a_i b_i|`` is the classic first-order bound of any fp32 summation order.  The
  factor 2 is an assumption about the tensor cores: their accumulation may truncate instead of
  rounding to nearest, which doubles the per-add error.  ReLU is 1-Lipschitz, so the bound of the
  pre-activation value also holds after it.
* Pure data movement and casts are bit exact (``cast_pad``, the bottom copy and zero pad of the
  interaction output, masked gradients, ``p16 = bf16_rne(p32)``), and so is ``dense_sgd`` with a
  power-of-two ``lr`` and ``grad_scale = 1``: ``lr * g`` is exact, so the kernel's ``fmaf`` rounds
  once, like ``p - lr * g`` in fp32.  Other ``lr`` / ``grad_scale`` allow one fp32 ulp.
* fp32 reductions of n terms (bias gradients, column sums, weight gradients, the loss):
  ``|err| <= 2 * n * u32 * sum|terms|``, plus the error each term carries in.
* ``head_loss`` uses ``__expf``, documented with an error of ``2 + floor(1.17 * |x|)`` ulps; the
  loss and dlogit bounds below carry it through ``log1p`` and the sigmoid.

Each comparison records the worst ``|err| / bound`` per kernel / stage; the table is printed at
the end of the module (``-s`` shows it).  A CPU self-check applies typical kernel defects to exact
references and requires every one of them to fail its bound.
"""
import math
import os
import random
import subprocess
import sys

import pytest
import torch

U16 = 2.0 ** -8
U32 = 2.0 ** -24
TINY = 2.0 ** -126  # absorbs flush-to-zero of results below the smallest normal fp32

WORST = {}  # kernel or stage -> (worst |err| / bound, where)


# ------------------------------------------------------------------ bounds and comparisons
def dot_bound(ref, abs_sum, k):
  """Bound of a bf16 result of an fp32-accumulated dot of ``k`` terms (bias counted as a term).
  ``ref`` is the exact float64 value, ``abs_sum`` the float64 sum of the terms' magnitudes."""
  e = 2.0 * k * U32 * abs_sum
  return U16 * (ref.abs() + e) + e + TINY


def acc_bound(n, abs_sum):
  """Bound of an fp32 sum of ``n`` terms (any order, atomics included)."""
  return 2.0 * n * U32 * abs_sum + TINY


def _where(t, flat_idx):
  if t.dim() <= 1:
    return f"index {flat_idx}"
  idx = []
  for s in reversed(t.shape):
    idx.append(flat_idx % s)
    flat_idx //= s
  idx = tuple(reversed(idx))
  return f"row {idx[0]}, index {idx}"


def _record(name, worst, where):
  prev = WORST.get(name)
  if prev is None or worst > prev[0]:
    WORST[name] = (worst, where)


def check_close(name, out, ref, bound):
  """``|out - ref| <= bound`` element-wise; reports the worst ratio, its index and row."""
  out = out.double()
  ref = ref.double()
  bound = torch.as_tensor(bound, dtype=torch.float64, device=out.device).expand_as(ref)
  err = (out - ref).abs()
  ratio = torch.nan_to_num(err / bound, nan=math.inf)  # a NaN output fails
  if ratio.numel() == 0:
    return 0.0
  i = int(ratio.reshape(-1).argmax())
  worst = float(ratio.reshape(-1)[i])
  where = _where(ratio, i)
  _record(name, worst, where)
  if worst > 1.0:
    n_bad = int((ratio > 1.0).sum())
    raise AssertionError(
        f"{name}: {n_bad} of {ratio.numel()} elements exceed the bound; worst |err|/bound = "
        f"{worst:.3g} at {where}: out={float(out.reshape(-1)[i])!r} "
        f"ref={float(ref.reshape(-1)[i])!r} bound={float(bound.reshape(-1)[i]):.3g}")
  return worst


def _bits(t):
  return t.contiguous().view({2: torch.int16, 4: torch.int32}[t.element_size()])


def check_bits(name, out, ref):
  """Bit-for-bit equality (``ref`` is cast to ``out``'s dtype first)."""
  ref = ref.to(out.dtype)
  assert out.shape == ref.shape, (name, tuple(out.shape), tuple(ref.shape))
  diff = _bits(out) != _bits(ref)
  _record(name, 0.0 if not bool(diff.any()) else math.inf, "bit exact")
  if bool(diff.any()):
    i = int(diff.reshape(-1).nonzero()[0])
    raise AssertionError(
        f"{name}: {int(diff.sum())} of {diff.numel()} elements differ bitwise; first at "
        f"{_where(diff, i)}: out={float(out.reshape(-1)[i])!r} ref={float(ref.reshape(-1)[i])!r}")


def check_zero(name, t):
  """Exactly +0.0 everywhere (pad columns, cleared buffers, masked gradients)."""
  check_bits(name, t, torch.zeros_like(t))


# ------------------------------------------------------------------ float64 references
def linear_ref(x, w, bias=None):
  """x @ w^T (+ bias) in float64 and the matching sum of |terms|."""
  xd, wd = x.double(), w.double()
  ref = xd @ wd.t()
  mag = xd.abs() @ wd.abs().t()
  if bias is not None:
    ref = ref + bias.double()
    mag = mag + bias.double().abs()
  return ref, mag


def _features(bottom, emb, n_emb):
  b, d = bottom.shape
  return torch.cat([bottom.double()[:, None, :],
                    emb.double()[:, :n_emb * d].reshape(b, n_emb, d)], 1)


def interact_ref(bottom, emb, n_emb):
  """Strict lower triangle of F F^T (row-major), F = [bottom ; emb_0 ; ...]."""
  f = _features(bottom, emb, n_emb)
  ii, jj = torch.tril_indices(n_emb + 1, n_emb + 1, -1, device=bottom.device)
  g = f @ f.transpose(1, 2)
  ga = f.abs() @ f.abs().transpose(1, 2)
  return g[:, ii, jj], ga[:, ii, jj]


def interact_bwd_ref(bottom, emb, dz, n_emb, scale=1.0):
  """dF = G F with G the symmetric matrix of dz's triangle; returns (dbottom, |.|, demb, |.|),
  demb as [b, n_emb, dim] and already multiplied by ``scale``."""
  f = _features(bottom, emb, n_emb)
  b, nf, d = f.shape
  n_inter = nf * (nf - 1) // 2
  ii, jj = torch.tril_indices(nf, nf, -1, device=bottom.device)
  dzd = dz.double()
  g = torch.zeros(b, nf, nf, dtype=torch.float64, device=bottom.device)
  g[:, ii, jj] = dzd[:, :n_inter]
  g[:, jj, ii] = dzd[:, :n_inter]
  df = g @ f
  dfa = g.abs() @ f.abs()
  direct = dzd[:, n_inter:n_inter + d]
  return (df[:, 0] + direct, dfa[:, 0] + direct.abs(), df[:, 1:] * scale, dfa[:, 1:] * abs(scale))


# interaction kernels: the forward sums D products per output, the backward multiplies the
# 32 x 32 (zero padded) G by F on the tensor cores and then adds the direct term or the scale
def interact_fwd_bound(ref, mag, dim):
  return dot_bound(ref, mag, dim)


def interact_bwd_bound(ref, mag):
  return dot_bound(ref, mag, 32 + 1)


def head_ref(x, w, bias, labels, inv_b):
  """Final layer + BCE-with-logits + backward in float64, with the bounds of every output."""
  xd, wd = x.double(), w.double().reshape(-1)
  b0 = float(bias.double().reshape(-1)[0])
  y = labels.double()
  k = xd.shape[1]
  n = xd.shape[0]
  logit = xd @ wd + b0
  e_logit = 2.0 * (k + 1) * U32 * (xd.abs() @ wd.abs() + abs(b0))
  al = logit.abs()
  loss = logit.clamp_min(0) - logit * y + torch.log1p(torch.exp(-al))
  sig = torch.sigmoid(logit)
  rho = (2.0 + torch.floor(1.17 * al)) * 2.0 ** -23  # __expf: ulps -> relative error
  # loss: d loss / d logit = sig - y (|.| <= 1 for labels in [0, 1]); exp(-|l|) carries rho into
  # log1p with weight <= exp(-|l|); log1pf and the four fp32 operations each round once
  e_loss = e_logit + torch.exp(-al) * rho + 8 * U32 * (al * (1 + y.abs()) + 1)
  # sigmoid = 1 / (1 + exp(-l)): relative error rho of exp(-l) moves it by sig (1 - sig) rho,
  # the logit error by at most e_logit / 4, the add and the divide round once each
  e_sig = e_logit / 4 + sig * (1 - sig) * rho + 3 * U32 * sig
  dl = (sig - y) * inv_b
  e_dl = inv_b * (e_sig * (1 + 2 * U32) + 2 * U32 * (sig - y).abs())
  mask = xd > 0
  dx = torch.where(mask, dl[:, None] * wd[None, :], torch.zeros_like(xd))
  e_dx = torch.where(mask, e_dl[:, None] * wd.abs()[None, :] + U32 * dx.abs(), torch.zeros_like(xd))
  return {
      "logit": logit, "e_logit": e_logit + U32 * al,
      "loss_terms": loss * inv_b, "e_loss_terms": e_loss * inv_b,
      "dl": dl, "e_dl": e_dl,
      "dx": dx, "dx_bound": U16 * (dx.abs() + e_dx) + e_dx + TINY,
      "dw": dl @ xd, "dw_mag": dl.abs() @ xd.abs(), "dw_carried": e_dl @ xd.abs(),
      "dbp": dx.sum(0), "dbp_mag": dx.abs().sum(0), "dbp_carried": e_dx.sum(0),
      "db": dl.sum(), "db_mag": dl.abs().sum(), "db_carried": e_dl.sum(), "n": n,
  }


def check_head(name, h, out):
  """Compare head_loss outputs (``out`` values after the call, ``*0`` values before it)."""
  n = h["n"]
  check_close(f"{name}/dx", out["dx"], h["dx"], h["dx_bound"])
  dw0, dbp0, db0, ls0 = (out[k].double() for k in ("dw0", "dbp0", "db0", "ls0"))
  check_close(f"{name}/dw", out["dw"], dw0 + h["dw"],
              h["dw_carried"] + acc_bound(n + 1, dw0.abs() + h["dw_mag"]))
  check_close(f"{name}/dbias_prev", out["dbp"], dbp0 + h["dbp"],
              h["dbp_carried"] + acc_bound(n + 1, dbp0.abs() + h["dbp_mag"]))
  check_close(f"{name}/db", out["db"], db0 + h["db"],
              h["db_carried"] + acc_bound(n + 1, db0.abs() + h["db_mag"]))
  lt = h["loss_terms"]
  check_close(f"{name}/loss", out["ls"], ls0 + lt.sum(),
              h["e_loss_terms"].sum() + acc_bound(n + 2, ls0.abs() + lt.abs().sum()))
  if out.get("logits") is not None:
    check_close(f"{name}/logits", out["logits"], h["logit"], h["e_logit"] + TINY)


def bf16_trunc(x):
  """Round toward zero to bf16 (drop the low 16 bits of the fp32 pattern)."""
  bits = x.float().contiguous().view(torch.int32) & -65536
  return bits.view(torch.float32).bfloat16()


@pytest.fixture(scope="module", autouse=True)
def _report_worst_ratios():
  yield
  if WORST:
    print("\nworst |err| / bound per kernel / stage:")
    for name in sorted(WORST):
      r, where = WORST[name]
      print(f"  {name:60s} {r:9.4f}  ({where})")


# ------------------------------------------------------------------ CPU self-check of the bounds
def _gemm_case(seed=0, m=64, n=48, k=200):
  g = torch.Generator().manual_seed(seed)
  a = (torch.randn(m, k, generator=g) * 0.5).bfloat16()
  b = (torch.randn(n, k, generator=g) * 0.5).bfloat16()
  acc = a.double() @ b.double().t()
  # bias that nearly cancels row 0 (the case where rounding before the add shows), random elsewhere
  bias = (torch.randn(n, generator=g)).bfloat16()
  bias[:] = (-acc[0] * (1 + 2.0 ** -6)).bfloat16()
  return a, b, bias, acc


def test_bounds_accept_rounded_reference_and_reject_defects():
  a, b, bias, acc = _gemm_case()
  k = a.shape[1]
  ref, mag = linear_ref(a, b, bias)
  bound = dot_bound(ref, mag, k + 1)
  check_close("selfcheck/exact", ref.bfloat16(), ref, bound)
  check_close("selfcheck/exact_relu", ref.clamp_min(0).bfloat16(), ref.clamp_min(0), bound)
  defects = {
      "output rounded toward zero": bf16_trunc(ref),
      "accumulator rounded to bf16 before the bias add":
          (acc.bfloat16().double() + bias.double()).bfloat16(),
      "last K block dropped":
          (a[:, :192].double() @ b[:, :192].double().t() + bias.double()).bfloat16(),
  }
  tail = ref.bfloat16().clone()
  tail[-1, :-1] = tail[-1, 1:].clone()
  defects["one tail row off by one element"] = tail
  for what, out in defects.items():
    with pytest.raises(AssertionError, match="exceed the bound"):
      check_close(f"selfcheck/{what}", out, ref, bound)
  # an fp32 bias (the step's master copy) rounded to bf16 before it is added
  g = torch.Generator().manual_seed(1)
  bias32 = (-acc[0] * (1 + 2.0 ** -6)).float() + torch.rand(acc.shape[1], generator=g) * 1e-3
  ref32 = acc + bias32.double()
  bound32 = dot_bound(ref32, a.double().abs() @ b.double().abs().t() + bias32.double().abs(), k + 1)
  check_close("selfcheck/exact_fp32_bias", ref32.bfloat16(), ref32, bound32)
  with pytest.raises(AssertionError, match="exceed the bound"):
    check_close("selfcheck/bias rounded to bf16 before the add",
                (acc + bias32.bfloat16().double()).bfloat16(), ref32, bound32)


def test_bounds_reject_mask_defects_on_signed_zeros():
  g = torch.Generator().manual_seed(2)
  y = torch.randn(300, 24, generator=g).bfloat16()
  y.view(-1)[::5] = 0.0
  y.view(-1)[1::7] = -0.0
  dy = (torch.randn(300, 24, generator=g) + 0.01).bfloat16()
  want = torch.where(y > 0, dy, torch.zeros_like(dy))
  check_bits("selfcheck/mask_exact", want.clone(), want)
  wrong = torch.where(y >= 0, dy, torch.zeros_like(dy))
  with pytest.raises(AssertionError, match="differ bitwise"):
    check_bits("selfcheck/mask >= 0", wrong, want)
  # the bias gradient of the wrong mask fails the fp32 reduction bound as well
  ref_db = want.double().sum(0)
  bound = acc_bound(300, want.double().abs().sum(0))
  check_close("selfcheck/db_exact", want.float().sum(0), ref_db, bound)
  with pytest.raises(AssertionError, match="exceed the bound"):
    check_close("selfcheck/db of mask >= 0", wrong.float().sum(0), ref_db, bound)


def test_interaction_bounds_reject_defects():
  g = torch.Generator().manual_seed(3)
  n_emb, dim, b = 26, 128, 16
  bottom = (torch.randn(b, dim, generator=g) * 0.5).bfloat16()
  emb = (torch.randn(b, n_emb * dim, generator=g) * 0.5).bfloat16()
  ref, mag = interact_ref(bottom, emb, n_emb)
  bound = interact_fwd_bound(ref, mag, dim)
  check_close("selfcheck/interact_exact", ref.bfloat16(), ref, bound)
  with pytest.raises(AssertionError, match="exceed the bound"):
    check_close("selfcheck/interact truncated", bf16_trunc(ref), ref, bound)
  f = _features(bottom, emb, n_emb)[:, :, :dim - 16]  # last 16-wide K step dropped
  ii, jj = torch.tril_indices(n_emb + 1, n_emb + 1, -1)
  short = (f @ f.transpose(1, 2))[:, ii, jj]
  with pytest.raises(AssertionError, match="exceed the bound"):
    check_close("selfcheck/interact last K step dropped", short.bfloat16(), ref, bound)
  dz = (torch.randn(b, 480, generator=g) * 0.1).bfloat16()
  db_ref, db_mag, de_ref, de_mag = interact_bwd_ref(bottom, emb, dz, n_emb, 0.375)
  check_close("selfcheck/interact_bwd_exact", de_ref.bfloat16(), de_ref,
              interact_bwd_bound(de_ref, de_mag))
  with pytest.raises(AssertionError, match="exceed the bound"):  # scale applied to row 0 too
    check_close("selfcheck/interact_bwd scaled bottom", (db_ref * 0.375).bfloat16(), db_ref,
                interact_bwd_bound(db_ref, db_mag))


def test_head_bounds_reject_defects():
  g = torch.Generator().manual_seed(4)
  n, k = 200, 64
  x = torch.relu(torch.randn(n, k, generator=g)).bfloat16()
  w = (torch.randn(k, generator=g) * 12 / math.sqrt(k / 2)).bfloat16()
  bias = torch.tensor([0.3]).bfloat16()
  labels = torch.rand(n, generator=g)
  inv_b = float(torch.tensor(1.0 / n, dtype=torch.float32))
  h = head_ref(x, w, bias, labels, inv_b)
  zero = torch.zeros(k, dtype=torch.float64)
  exact = {"dx": h["dx"].bfloat16(), "dw": h["dw"], "dbp": h["dbp"], "db": h["db"],
           "ls": h["loss_terms"].sum(), "dw0": zero, "dbp0": zero, "db0": zero[0], "ls0": zero[0],
           "logits": h["logit"]}
  check_head("selfcheck/head_exact", h, exact)
  wrong = dict(exact, dx=bf16_trunc(h["dx"]))
  with pytest.raises(AssertionError, match="exceed the bound"):
    check_head("selfcheck/head dx truncated", h, wrong)
  wrong = dict(exact, db=h["db"] - h["dl"][-1])  # last sample's dlogit missing
  with pytest.raises(AssertionError, match="exceed the bound"):
    check_head("selfcheck/head db missing a sample", h, wrong)


# ------------------------------------------------------------------ GPU: kernels
def _ops():
  from distributed_embeddings_b200.ops import _native
  return _native.require()


def _sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def _randn(*shape, scale=1.0, seed=None, dtype=torch.bfloat16):
  g = torch.Generator(device="cuda")
  g.manual_seed(seed if seed is not None else 0)
  return (torch.randn(*shape, generator=g, device="cuda") * scale).to(dtype)


def _run_interact_fwd(dim, n_emb, batch, seed):
  ops = _ops()
  n_inter = (n_emb + 1) * n_emb // 2
  n_out = n_inter + dim
  zw = (n_out + 7) // 8 * 8 + 8
  # strided views: rows wider than the data, 16-byte aligned column offsets
  bottom_full = _randn(batch, dim + 24, scale=0.5, seed=seed)
  bottom = bottom_full[:, 8:8 + dim]
  emb_full = _randn(batch, n_emb * dim + 40, scale=0.5, seed=seed + 1)
  emb = emb_full[:, 16:16 + n_emb * dim]
  z_full = torch.full((batch, zw + 16), 7.0, dtype=torch.bfloat16, device="cuda")
  z = z_full[:, 8:8 + zw]
  ops.interact_fwd(bottom, emb, n_emb, z, [])
  ref, mag = interact_ref(bottom, emb, n_emb)
  check_close("interact_fwd", z[:, :n_inter], ref, interact_fwd_bound(ref, mag, dim))
  check_bits("interact_fwd/bottom copy", z[:, n_inter:n_out], bottom)
  check_zero("interact_fwd/zero pad", z[:, n_out:])
  check_bits("interact_fwd/columns outside z", z_full[:, :8], torch.full_like(z_full[:, :8], 7))
  check_bits("interact_fwd/columns outside z", z_full[:, 8 + zw:],
             torch.full_like(z_full[:, 8 + zw:], 7))


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [16, 32, 64, 128])
@pytest.mark.parametrize("n_emb", [1, 2, 15, 16, 26, 31])
def test_interact_fwd(dim, n_emb):
  for batch in (1, 3, 5, 777):
    try:
      _run_interact_fwd(dim, n_emb, batch, seed=dim * 100 + n_emb + batch)
    except AssertionError as e:
      raise AssertionError(f"dim={dim} n_emb={n_emb} batch={batch}: {e}") from None


@pytest.mark.gpu
@pytest.mark.parametrize("dim,n_emb", [(128, 26), (16, 31)])
def test_interact_fwd_grid_loops(dim, n_emb):
  """More samples than 8 blocks per SM x 4 warps: every warp handles several samples."""
  _run_interact_fwd(dim, n_emb, 8 * _sms() * 4 * 2 + 3, seed=5)


@pytest.mark.gpu
def test_interact_fwd_rejects_unsupported_shapes():
  ops = _ops()
  b = 4
  bottom = _randn(b, 128)
  z = torch.zeros(b, 1024, dtype=torch.bfloat16, device="cuda")
  with pytest.raises(RuntimeError, match="unsupported interaction shape"):
    ops.interact_fwd(bottom, _randn(b, 32 * 128), 32, z, [])
  with pytest.raises(RuntimeError, match="unsupported interaction shape"):
    ops.interact_fwd(_randn(b, 48), _randn(b, 4 * 48), 4, z, [])
  with pytest.raises(RuntimeError, match="n_emb"):
    ops.interact_fwd(bottom, _randn(b, 4 * 128 + 8), 4, z, [])
  with pytest.raises(RuntimeError, match="16-byte"):
    ops.interact_fwd(_randn(b, 140)[:, 4:132], _randn(b, 4 * 128), 4, z, [])


def _bwd_buffers(dim, n_emb, batch, seed, dz_aligned=True, dbottom_pad=8):
  n_inter = (n_emb + 1) * n_emb // 2
  n_out = n_inter + dim
  bottom_full = _randn(batch, dim + 16, scale=0.5, seed=seed)
  bottom = bottom_full[:, 8:8 + dim]
  emb_full = _randn(batch, n_emb * dim + 24, scale=0.5, seed=seed + 1)
  emb = emb_full[:, 8:8 + n_emb * dim]
  # an aligned dz row (multiple of 8 elements) allows the double-buffered kernel; an odd stride
  # selects the single-buffered one
  dzw = (n_out + 7) // 8 * 8 + 8 if dz_aligned else n_out + 3
  dz = _randn(batch, dzw, scale=0.1, seed=seed + 2)
  dbottom_full = torch.full((batch, dim + 2 * dbottom_pad), 5.0, dtype=torch.bfloat16,
                            device="cuda")
  dbottom = dbottom_full[:, dbottom_pad:dbottom_pad + dim]
  demb_full = torch.full((batch, n_emb * dim + 16), 5.0, dtype=torch.bfloat16, device="cuda")
  return bottom, emb, dz, dbottom_full, dbottom, demb_full


def _check_bwd(name, bottom, emb, dz, n_emb, scale, dbottom, demb):
  """demb: [batch, n_emb * dim] view of the embedding-gradient destination."""
  b, dim = bottom.shape
  db_ref, db_mag, de_ref, de_mag = interact_bwd_ref(bottom, emb, dz, n_emb, scale)
  check_close(f"{name}/dbottom", dbottom, db_ref, interact_bwd_bound(db_ref, db_mag))
  check_close(f"{name}/demb", demb.reshape(b, n_emb, dim), de_ref,
              interact_bwd_bound(de_ref, de_mag))


BWD_CASES = [  # (dim, n_emb, batch, dz_aligned): the double-buffered kernel needs dim 64 / 128,
    # aligned rows and n_inter + dim <= 512; everything else takes the single-buffered kernel
    (64, 1, 777, True), (64, 15, 5003, True), (64, 28, 777, True), (64, 31, 777, True),
    (128, 2, 3, True), (128, 16, 777, True), (128, 26, 5003, True), (128, 26, 1, True),
    (128, 28, 777, True), (128, 31, 5003, True), (32, 31, 777, True), (32, 7, 5, True),
    (128, 26, 777, False), (64, 7, 3001, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("dim,n_emb,batch,dz_aligned", BWD_CASES)
def test_interact_bwd_cases(dim, n_emb, batch, dz_aligned):
  ops = _ops()
  for scale in (1.0, 0.375):
    bottom, emb, dz, dbottom_full, dbottom, demb_full = _bwd_buffers(
        dim, n_emb, batch, seed=dim + n_emb + batch, dz_aligned=dz_aligned,
        dbottom_pad=8 if dz_aligned else 2)
    demb = demb_full[:, 8:8 + n_emb * dim]
    ops.interact_bwd(bottom, emb, n_emb, dz, dbottom, demb.data_ptr(), demb.stride(0), scale,
                     None, 0, [], None, 0)
    case = f"interact_bwd(dim={dim},n_emb={n_emb},batch={batch},scale={scale})"
    try:
      _check_bwd("interact_bwd", bottom, emb, dz, n_emb, scale, dbottom, demb)
      pad = dbottom.stride(0) - dim  # columns of the padded rows around the views stay untouched
      check_bits("interact_bwd/outside dbottom", dbottom_full[:, :pad // 2],
                 torch.full_like(dbottom_full[:, :pad // 2], 5))
      check_bits("interact_bwd/outside demb", demb_full[:, :8], torch.full_like(demb_full[:, :8], 5))
      check_bits("interact_bwd/outside demb", demb_full[:, 8 + n_emb * dim:],
                 torch.full_like(demb_full[:, 8 + n_emb * dim:], 5))
    except AssertionError as e:
      raise AssertionError(f"{case}: {e}") from None


@pytest.mark.gpu
def test_interact_bwd_forced_single_buffered():
  """DE_B200_INTERACT_V1=1 runs every unrouted launch on the single-buffered kernel.  The switch
  is read once per process, hence the subprocess."""
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  env = dict(os.environ, DE_B200_INTERACT_V1="1")
  out = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q",
                        "-p", "no:cacheprovider", "-k", "test_interact_bwd_cases"],
                       env=env, cwd=root, capture_output=True, text=True, timeout=900, check=False)
  assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
  assert " passed" in out.stdout


@pytest.mark.gpu
def test_interact_bwd_routes():
  """Gradient pieces routed to separate buffers: column slices, permuted features, a destination
  stride unlike the source; the scale applies to the embedding rows only."""
  import numpy as np
  from distributed_embeddings_b200.ops._native import GRAD_ROUTE, upload_struct_array
  ops = _ops()
  n_emb, dim, b = 5, 128, 3001
  bottom, emb, dz, _, dbottom, _ = _bwd_buffers(dim, n_emb, b, seed=7)
  a = torch.full((b, 2 * 128 + 64 + 8), 5.0, device="cuda", dtype=torch.bfloat16)
  bb = torch.full((b, 2 * 128 + 64), 5.0, device="cuda", dtype=torch.bfloat16)
  pieces = [(4 * 128, 128, a, 0), (0, 128, a, 128), (2 * 128 + 64, 64, a, 256),
            (1 * 128, 128, bb, 64), (2 * 128, 64, bb, 0), (3 * 128, 128, bb, 192)]
  routes = np.zeros(len(pieces), dtype=GRAD_ROUTE)
  for i, (sc, w, dst, dc) in enumerate(sorted(pieces, key=lambda p: p[0])):
    routes[i]["dst"], routes[i]["dst_stride"] = dst.data_ptr(), dst.stride(0)
    routes[i]["src_col"], routes[i]["width"], routes[i]["dst_col"] = sc, w, dc
  ops.interact_bwd(bottom, emb, n_emb, dz, dbottom, 0, 0, 0.375,
                   upload_struct_array(routes, "cuda"), len(pieces), [], None, 0)
  db_ref, db_mag, de_ref, de_mag = interact_bwd_ref(bottom, emb, dz, n_emb, 0.375)
  check_close("interact_bwd routed/dbottom", dbottom, db_ref, interact_bwd_bound(db_ref, db_mag))
  de_ref, de_bound = de_ref.reshape(b, -1), interact_bwd_bound(de_ref, de_mag).reshape(b, -1)
  for sc, w, dst, dc in pieces:
    check_close("interact_bwd routed/demb", dst[:, dc:dc + w], de_ref[:, sc:sc + w],
                de_bound[:, sc:sc + w])
  check_bits("interact_bwd routed/outside", a[:, 320:], torch.full_like(a[:, 320:], 5))


@pytest.mark.gpu
def test_interact_bwd_done_counters():
  """Progress counters of the streamed push: counter k counts the samples of chunk k, and the
  outputs equal those of the same launch without counters."""
  ops = _ops()
  n_emb, dim, b, chunk = 26, 128, 777, 100
  bottom, emb, dz, _, dbottom, demb_full = _bwd_buffers(dim, n_emb, b, seed=11)
  demb = demb_full[:, :n_emb * dim]
  ops.interact_bwd(bottom, emb, n_emb, dz, dbottom, demb.data_ptr(), demb.stride(0), 1.0, None, 0,
                   [], None, 0)
  want_db, want_de = dbottom.clone(), demb.clone()
  dbottom.fill_(3.0)
  demb.fill_(3.0)
  n_chunks = -(-b // chunk)
  counters = torch.zeros(n_chunks + 2, dtype=torch.int32, device="cuda")
  ops.interact_bwd(bottom, emb, n_emb, dz, dbottom, demb.data_ptr(), demb.stride(0), 1.0, None, 0,
                   [], counters, chunk)
  check_bits("interact_bwd counters/dbottom", dbottom, want_db)
  check_bits("interact_bwd counters/demb", demb, want_de)
  want = [min(chunk, b - k * chunk) for k in range(n_chunks)] + [0, 0]
  assert counters.tolist() == want
  _check_bwd("interact_bwd counters", bottom, emb, dz, n_emb, 1.0, dbottom, demb)


@pytest.mark.gpu
def test_interact_bwd_rejects_bad_arguments():
  ops = _ops()
  n_emb, dim, b = 4, 128, 8
  bottom, emb, dz, _, dbottom, demb_full = _bwd_buffers(dim, n_emb, b, seed=1)
  p, s = demb_full.data_ptr(), demb_full.stride(0)

  def call(**kw):
    args = dict(bottom=bottom, emb=emb, dz=dz, dbottom=dbottom, demb=p, stride=s, counters=None,
                chunk=0)
    args.update(kw)
    ops.interact_bwd(args["bottom"], args["emb"], n_emb, args["dz"], args["dbottom"],
                     args["demb"], args["stride"], 1.0, None, 0, [], args["counters"],
                     args["chunk"])

  with pytest.raises(RuntimeError, match="n_emb"):
    call(emb=_randn(b, (n_emb + 1) * dim))
  with pytest.raises(RuntimeError, match="dz is too narrow"):
    call(dz=_randn(b, 136))
  with pytest.raises(RuntimeError, match="dbottom"):
    call(dbottom=torch.empty(b, 64, dtype=torch.bfloat16, device="cuda"))
  with pytest.raises(RuntimeError, match="gradient buffer or routes"):
    call(demb=0, stride=0)
  with pytest.raises(RuntimeError, match="16-byte"):
    call(bottom=_randn(b, dim + 12)[:, 4:4 + dim])  # row stride of 280 bytes
  counters = torch.zeros(4, dtype=torch.int32, device="cuda")
  with pytest.raises(RuntimeError, match="chunk_rows"):
    call(counters=counters, chunk=0)
  with pytest.raises(RuntimeError, match="chunk_rows"):
    call(counters=counters, chunk=-3)
  with pytest.raises(RuntimeError, match="one counter per chunk"):
    call(counters=counters, chunk=1)
  torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("cols", [8, 24, 128, 480, 1000, 1024, 2048])
def test_relu_bwd_bias(cols):
  ops = _ops()
  rows_par = 256 // (cols // 8)
  rows_per_block = rows_par * 16  # 4 passes of 4 rows in flight per thread
  for rows in (1, 3, 3000, 3 * rows_per_block + 5):
    y = _randn(rows, cols, seed=rows + cols)
    y.view(-1)[::5] = 0.0
    y.view(-1)[1::7] = -0.0
    dy0 = _randn(rows, cols, seed=rows + cols + 1)
    dy = dy0.clone()
    db0 = _randn(cols + 8, seed=cols, dtype=torch.float32)
    db = db0.clone()
    ops.relu_bwd_bias(dy, y, db)
    want = torch.where(y > 0, dy0, torch.zeros_like(dy0))
    case = f"rows={rows} cols={cols}"
    try:
      check_bits("relu_bwd_bias/dy", dy, want)
      check_close("relu_bwd_bias/db", db[:cols], db0[:cols].double() + want.double().sum(0),
                  acc_bound(rows + 1, db0[:cols].double().abs() + want.double().abs().sum(0)))
      check_bits("relu_bwd_bias/db beyond cols", db[cols:], db0[cols:])
    except AssertionError as e:
      raise AssertionError(f"{case}: {e}") from None


@pytest.mark.gpu
def test_relu_bwd_bias_rejects_bad_arguments():
  ops = _ops()
  db = torch.zeros(4096, device="cuda")
  with pytest.raises(RuntimeError, match="8..2048 columns"):
    ops.relu_bwd_bias(_randn(4, 2056), _randn(4, 2056), db)
  with pytest.raises(RuntimeError, match="shape of dy"):
    ops.relu_bwd_bias(_randn(4, 128), _randn(3, 128), db)
  with pytest.raises(RuntimeError, match="shape of dy"):
    ops.relu_bwd_bias(_randn(4, 128), _randn(4, 64), db)
  torch.cuda.synchronize()


def _head_inputs(b, k, seed, frac_labels):
  x = torch.relu(_randn(b, k, seed=seed, dtype=torch.float32)).bfloat16()
  # logits spread to about +-30 and beyond: std 12
  w = _randn(k, scale=12 / math.sqrt(k / 2), seed=seed + 1)
  bias = torch.tensor([0.3], device="cuda").bfloat16()
  g = torch.Generator(device="cuda").manual_seed(seed + 2)
  if frac_labels:
    labels = torch.rand(b, generator=g, device="cuda")
  else:
    labels = torch.randint(0, 2, (b,), generator=g, device="cuda").float()
  return x, w, bias, labels


def _run_head(ops, x, w, bias, labels, with_logits, seed):
  b, k = x.shape
  inv_b = float(torch.tensor(1.0 / b, dtype=torch.float32))
  out = {"dx": torch.full_like(x, 9.0)}
  for key, n in (("dw", k), ("dbp", k), ("db", 8), ("ls", 1)):
    out[key + "0"] = _randn(n, seed=seed + n, dtype=torch.float32)
    out[key] = out[key + "0"].clone()
  out["logits"] = torch.full((b,), 9.0, device="cuda") if with_logits else None
  ops.head_loss(x, w, bias, labels, inv_b, out["dx"], out["dw"], out["db"], out["dbp"], out["ls"],
                out["logits"])
  check_bits("head_loss/db beyond [0]", out["db"][1:], out["db0"][1:])
  out["db"], out["db0"], out["ls"], out["ls0"] = out["db"][0], out["db0"][0], out["ls"][0], \
      out["ls0"][0]
  return head_ref(x, w, bias, labels, inv_b), out


@pytest.mark.gpu
@pytest.mark.parametrize("k", [64, 128, 256, 512, 1024])
def test_head_loss(k):
  ops = _ops()
  big = 4 * _sms() * 8 + 9
  for b, frac, with_logits in ((1, False, True), (7, True, True), (1000, False, False),
                               (big, True, True)):
    x, w, bias, labels = _head_inputs(b, k, seed=k + b, frac_labels=frac)
    h, out = _run_head(ops, x, w, bias, labels, with_logits, seed=k + b)
    try:
      check_head("head_loss", h, out)
    except AssertionError as e:
      raise AssertionError(f"K={k} batch={b} fractional labels={frac}: {e}") from None


@pytest.mark.gpu
def test_head_loss_rejects_bad_arguments():
  ops = _ops()
  b, k = 16, 256
  x, w, bias, labels = _head_inputs(b, k, seed=1, frac_labels=False)
  f = lambda n: torch.zeros(n, device="cuda")  # noqa: E731
  dx = torch.empty_like(x)

  def call(**kw):
    a = dict(w=w, dx=dx, dw=f(k), db=f(1), dbp=f(k), ls=f(1), labels=labels)
    a.update(kw)
    ops.head_loss(x, a["w"], bias, a["labels"], 1.0 / b, a["dx"], a["dw"], a["db"], a["dbp"],
                  a["ls"], None)

  with pytest.raises(RuntimeError, match="w must hold K"):
    call(w=_randn(k // 2))
  with pytest.raises(RuntimeError, match="dx must be"):
    call(dx=torch.empty(b, k // 2, dtype=torch.bfloat16, device="cuda"))
  with pytest.raises(RuntimeError, match="dw must be"):
    call(dw=f(k - 8))
  with pytest.raises(RuntimeError, match="dbias_prev must be"):
    call(dbp=f(k // 2))
  with pytest.raises(RuntimeError, match="db must be"):
    call(db=f(0))
  with pytest.raises(RuntimeError, match="labels"):
    call(labels=labels[:b // 2])
  torch.cuda.synchronize()


def _ulp32(x):
  a = x.float().abs()
  return (torch.nextafter(a, torch.full_like(a, math.inf)) - a).double()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4, 12, 4100, 3 << 20])
def test_dense_sgd(n):
  ops = _ops()
  p0 = _randn(n, scale=4.0, seed=n, dtype=torch.float32)
  g0 = _randn(n, seed=n + 1, dtype=torch.float32)
  g0[::9] = 0.0
  for lr, gs in ((0.5, 1.0), (2.0 ** -7, 1.0), (0.3, 0.7)):
    p32, g32 = p0.clone(), g0.clone()
    p16 = torch.full((n,), 9.0, dtype=torch.bfloat16, device="cuda")
    lr_t = torch.tensor([lr], dtype=torch.float32, device="cuda")
    ops.dense_sgd(p32, p16, g32, lr_t, gs)
    if gs == 1.0:  # power-of-two lr: lr * g is exact, the fma rounds once like p - lr * g
      check_bits("dense_sgd/p32 (power-of-two lr)", p32, p0 - lr_t * g0)
    else:  # the kernel forms -(lr * grad_scale) in fp32 and rounds p + step * g once
      step = (-(lr_t * torch.tensor(gs, dtype=torch.float32))).double()
      want = p0.double() + step * g0.double()
      check_close("dense_sgd/p32", p32, want, _ulp32(want) + TINY)
    check_bits("dense_sgd/p16", p16, p32.bfloat16())
    check_zero("dense_sgd/g32", g32)


@pytest.mark.gpu
@pytest.mark.parametrize("src_cols,dst_cols", [(13, 16), (16, 16)])
@pytest.mark.parametrize("rows", [1, 3, 40000])
def test_cast_pad(src_cols, dst_cols, rows):
  ops = _ops()
  src = _randn(rows, src_cols, scale=100.0, seed=rows, dtype=torch.float32)
  bits = src.view(torch.int32)
  bits.view(-1)[::3] = (bits.view(-1)[::3] & -65536) | 0x8000  # exact ties: round to even
  bits.view(-1)[1::5] = (bits.view(-1)[1::5] & -65536) | 0x18000
  src.view(-1)[2::11] = 1e-40  # subnormal
  dst = torch.full((rows, dst_cols), 5.0, dtype=torch.bfloat16, device="cuda")
  ops.cast_pad(src, dst)
  check_bits("cast_pad", dst[:, :src_cols], src.bfloat16())
  check_zero("cast_pad/pad", dst[:, src_cols:])


def _avgpool_ref(x, n, stride):
  """Keras AveragePooling1D(stride, stride, padding="same"): a partial window divides by the
  number of its real elements."""
  out_len = -(-n // stride)
  pad = max(0, (out_len - 1) * stride + stride - n)
  left = pad // 2
  j = torch.arange(out_len, device=x.device)
  lo = (j * stride - left).clamp(0, n)
  hi = ((j + 1) * stride - left).clamp(0, n)
  xd = x.double()
  z = torch.zeros(x.shape[0], 1, dtype=torch.float64, device=x.device)
  cs = torch.cat([z, xd.cumsum(1)], 1)
  ca = torch.cat([z, xd.abs().cumsum(1)], 1)
  cnt = (hi - lo).double()
  return (cs[:, hi] - cs[:, lo]) / cnt, (ca[:, hi] - ca[:, lo]) / cnt, lo, hi, left


@pytest.mark.gpu
@pytest.mark.parametrize("stride", [1, 2, 3, 7])
@pytest.mark.parametrize("n", [2, 10, 11, 26, 3329])
def test_avgpool(stride, n):
  ops = _ops()
  rows = 37
  out_len = -(-n // stride)
  x_full = _randn(rows, n + 24, seed=n * stride)
  x = x_full[:, 3:3 + n]
  out_full = torch.full((rows, out_len + 16), 3.0, dtype=torch.bfloat16, device="cuda")
  out = out_full[:, 5:5 + out_len]
  ops.avgpool_fwd(x, n, out, stride)
  ref, mag, lo, hi, left = _avgpool_ref(x, n, stride)
  case = f"n={n} stride={stride} left pad={left}"
  try:
    check_close("avgpool_fwd", out, ref, dot_bound(ref, mag, stride + 1))
    check_bits("avgpool_fwd/outside out", out_full[:, :5], torch.full_like(out_full[:, :5], 3))
    check_bits("avgpool_fwd/outside out", out_full[:, 5 + out_len:],
               torch.full_like(out_full[:, 5 + out_len:], 3))
    dout_full = _randn(rows, out_len + 16, seed=n + stride)
    dout = dout_full[:, 2:2 + out_len]
    dx_full = torch.full((rows, n + 16), 3.0, dtype=torch.bfloat16, device="cuda")
    dx = dx_full[:, 7:7 + n]
    ops.avgpool_bwd(dout, dx, n, stride)
    c = torch.arange(n, device="cuda")
    j = (c + left) // stride
    want = dout.double()[:, j] / (hi - lo).double()[j]
    check_close("avgpool_bwd", dx, want, dot_bound(want, want.abs(), 1))
    check_bits("avgpool_bwd/outside dx", dx_full[:, :7], torch.full_like(dx_full[:, :7], 3))
    check_bits("avgpool_bwd/outside dx", dx_full[:, 7 + n:], torch.full_like(dx_full[:, 7 + n:], 3))
  except AssertionError as e:
    raise AssertionError(f"{case}: {e}") from None


_NS = [8, 24, 136, 264, 392, 1000, 2048]
_MS = [1, 64, 129, 777, 8192]
_KS = [8, 24, 72, 200, 1024]


def _gemm_shapes(n_cases, block_ns, seed):
  """A fixed, seeded list that visits every N, M and K at least once (not the full product)."""
  rng = random.Random(seed)
  out = []
  for i in range(n_cases):
    n = _NS[i % len(_NS)] if i < len(_NS) else rng.choice(_NS)
    m = _MS[i % len(_MS)] if i < len(_MS) else rng.choice(_MS)
    k = _KS[(3 * i + 1) % len(_KS)] if i < len(_KS) + 2 else rng.choice(_KS)
    if m * n * k > 8192 * 1024 * 1024:
      m = 777
    out.append((m, n, k, block_ns[i % len(block_ns)]))
  return out


FWD_GEMM = _gemm_shapes(16, [0, 128, 256, 512], seed=90)
DGRAD_GEMM = _gemm_shapes(12, [0, 128, 256], seed=91)


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,k,block_n", FWD_GEMM)
def test_gemm_tn_bias_act(m, n, k, block_n):
  ops = _ops()
  seed = m + n + k + block_n
  a_full = _randn(m, k + 8, scale=0.5, seed=seed)
  a = a_full[:, :k]  # row stride wider than K
  b = _randn(n, k, scale=0.5, seed=seed + 1)
  for relu, with_bias in ((True, True), (False, seed % 2 == 0)):
    bias = _randn(n, seed=seed + 2) if with_bias else None
    out_full = torch.full((m, n + 16), 3.0, dtype=torch.bfloat16, device="cuda")
    out = out_full[:, 8:8 + n]
    ops.gemm_tn_bias_act(a, b, bias, out, relu, block_n)
    ref, mag = linear_ref(a, b, bias)
    case = f"M={m} N={n} K={k} block_n={block_n} relu={relu} bias={with_bias}"
    try:
      check_close("gemm_tn_bias_act", out, ref.clamp_min(0) if relu else ref,
                  dot_bound(ref, mag, k + (1 if with_bias else 0)))
      check_bits("gemm_tn_bias_act/outside out", out_full[:, :8], torch.full_like(out_full[:, :8], 3))
      check_bits("gemm_tn_bias_act/outside out", out_full[:, 8 + n:],
                 torch.full_like(out_full[:, 8 + n:], 3))
    except AssertionError as e:
      raise AssertionError(f"{case}: {e}") from None


def _masked_colsum_bound(ref, elem_bound, mask, c0):
  """Column sums of masked dot results: each term carries its element bound, plus the fp32
  accumulation of M terms onto the initial value."""
  m = ref.shape[0]
  carried = (elem_bound * mask).sum(0)
  return carried + acc_bound(m + 1, c0.abs() + ((ref.abs() + elem_bound) * mask).sum(0))


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,k,block_n", DGRAD_GEMM)
def test_gemm_dgrad_relu_bias(m, n, k, block_n):
  ops = _ops()
  seed = m + n + k + block_n + 1
  dy = _randn(m, k, scale=0.5, seed=seed)
  wt = _randn(n, k, scale=0.1, seed=seed + 1)
  act = _randn(m, n, seed=seed + 2)
  act.view(-1)[::5] = 0.0
  act.view(-1)[1::7] = -0.0
  dx_full = torch.full((m, n + 16), 3.0, dtype=torch.bfloat16, device="cuda")
  dx = dx_full[:, 8:8 + n]
  c0 = _randn(n + 8, seed=seed + 3, dtype=torch.float32)
  colsum = c0.clone()
  ops.gemm_dgrad_relu_bias(dy, wt, act, dx, colsum, block_n)
  ref, mag = linear_ref(dy, wt)
  mask = act > 0
  eb = dot_bound(ref, mag, k)
  case = f"M={m} N={n} K={k} block_n={block_n}"
  try:
    check_close("gemm_dgrad_relu_bias/dx", dx, torch.where(mask, ref, torch.zeros_like(ref)), eb)
    check_zero("gemm_dgrad_relu_bias/masked dx", torch.where(mask, torch.zeros_like(dx), dx))
    check_close("gemm_dgrad_relu_bias/colsum", colsum[:n],
                c0[:n].double() + (ref * mask).sum(0),
                _masked_colsum_bound(ref, eb, mask, c0[:n].double()))
    check_bits("gemm_dgrad_relu_bias/colsum beyond N", colsum[n:], c0[n:])
    check_bits("gemm_dgrad_relu_bias/outside dx", dx_full[:, :8], torch.full_like(dx_full[:, :8], 3))
  except AssertionError as e:
    raise AssertionError(f"{case}: {e}") from None


@pytest.mark.gpu
def test_gemm_dgrad_rejects_wide_n():
  ops = _ops()
  m, n, k = 64, 2056, 64
  with pytest.raises(RuntimeError, match="unsupported"):
    ops.gemm_dgrad_relu_bias(_randn(m, k), _randn(n, k), _randn(m, n),
                             torch.empty(m, n, dtype=torch.bfloat16, device="cuda"),
                             torch.zeros(n, device="cuda"), 0)
  torch.cuda.synchronize()


# ------------------------------------------------------------------ GPU: the DLRM step, stage by stage
SIZES = [300 + 11 * i for i in range(26)]
LR = 0.5  # power of two: the SGD update is exact to compare bit for bit


class _SnapshotOps:
  """Forwards every custom op of the step; snapshots p32 / p16 / g32 right before dense_sgd."""

  def __init__(self, ops):
    self._ops = ops
    self.before_sgd = []

  def __getattr__(self, name):
    fn = getattr(self._ops, name)
    if name != "dense_sgd":
      return fn

    def dense_sgd(p32, p16, g32, lr, grad_scale):
      self.before_sgd.append((p32.clone(), p16.clone(), g32.clone(), float(lr.item()),
                              float(grad_scale)))
      return fn(p32, p16, g32, lr, grad_scale)

    return dense_sgd


def _batch(b, seed):
  g = torch.Generator().manual_seed(seed)
  num = torch.randn(b, 13, generator=g).cuda()
  cat = torch.stack([torch.randint(0, s, (b,), generator=g, dtype=torch.int32)
                     for s in SIZES]).cuda()
  lab = torch.randint(0, 2, (b,), generator=g).float().cuda()
  return num, cat, lab


def _make_step(gemm, use_graph, seed=0, like=None):
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  torch.manual_seed(seed)
  model = DLRM(SIZES, device=torch.device("cuda", 0), compute_dtype=torch.bfloat16,
               backend="fused")
  if like is not None:  # identical initial weights (before the step takes the parameters over)
    model.load_state_dict(like.state_dict())
    model.embedding.set_weights(like.embedding.get_weights())
  step = DLRMTrainStep(model, lr=LR, embedding_optimizer="sgd", use_cuda_graph=use_graph,
                       gemm=gemm)
  return model, step


def _tables(model):
  """The unsharded tables in feature order (the engine may fuse them into one local table)."""
  return [torch.from_numpy(w).cuda() for w in model.embedding.get_weights()]


def _old(step, p16_old, L):
  w = p16_old[L.w_off:L.w_off + L.w_numel].view(L.out_f, L.in_pad)
  return w, p16_old[L.b_off:L.b_off + L.out_f]


def _flat(t, L, which):
  if which == "w":
    return t[L.w_off:L.w_off + L.w_numel].view(L.out_f, L.in_pad)
  return t[L.b_off:L.b_off + L.b_numel]


def _check_step(gemm, b):
  model, step = _make_step(gemm, use_graph=False)
  proxy = _SnapshotOps(step.ops)
  step.ops = proxy
  num, cat, lab = _batch(b, seed=b)
  p16_old = step.p16.clone()
  tables_old = _tables(model)
  step.step(num, cat, lab)
  torch.cuda.synchronize()
  assert len(proxy.before_sgd) == 1
  p32_0, p16_0, g32, lr, grad_scale = proxy.before_sgd[0]
  assert lr == LR and grad_scale == 1.0
  check_bits("step/p16 unchanged before the update", p16_0, p16_old)
  eng = step.engine
  n_emb, dim = step.n_emb, step.dim
  S = f"step[{gemm}]"

  # forward: every stage from the previous stage's buffer and the old bf16 weights
  check_bits(f"{S}/x0", step.x0[:, :13], num.bfloat16())
  check_zero(f"{S}/x0 pad", step.x0[:, 13:])
  inputs = {}
  x = step.x0
  for i, L in enumerate(step.bottom):
    inputs[id(L)] = x
    w, bias = _old(step, p16_old, L)
    ref, mag = linear_ref(x, w, bias)
    check_close(f"{S}/bottom[{i}].y", L.y, ref.clamp_min(0), dot_bound(ref, mag, L.in_pad + 1))
    x = L.y
  hb = step.bottom[-1]
  n_inter = (n_emb + 1) * n_emb // 2
  ref, mag = interact_ref(hb.y, eng.out, n_emb)
  check_close(f"{S}/z", step.z[:, :n_inter], ref, interact_fwd_bound(ref, mag, dim))
  check_bits(f"{S}/z bottom copy", step.z[:, n_inter:n_inter + dim], hb.y)
  check_zero(f"{S}/z pad", step.z[:, n_inter + dim:])
  x = step.z
  for i, L in enumerate(step.top):
    inputs[id(L)] = x
    w, bias = _old(step, p16_old, L)
    ref, mag = linear_ref(x, w, bias)
    check_close(f"{S}/top[{i}].y", L.y, ref.clamp_min(0), dot_bound(ref, mag, L.in_pad + 1))
    x = L.y

  # head: loss, the masked dx of the last top layer and the head / last-layer gradients
  H, last = step.head, step.top[-1]
  inputs[id(H)] = last.y
  w, bias = _old(step, p16_old, H)
  inv_b = float(torch.tensor(1.0 / b, dtype=torch.float32))
  h = head_ref(last.y, w.reshape(-1), bias, lab, inv_b)
  zk = torch.zeros(H.in_pad, dtype=torch.float64, device="cuda")
  check_head(f"{S}/head", h, {
      "dx": last.dy, "dw": _flat(g32, H, "w").reshape(-1), "dbp": _flat(g32, last, "b")[:last.out_f],
      "db": _flat(g32, H, "b")[0], "ls": step.loss[0], "dw0": zk, "dbp0": zk, "db0": zk[0],
      "ls0": zk[0]})

  def dgrad(name, L, below_y, below_dy, below_gb):
    w, _ = _old(step, p16_old, L)
    ref, mag = linear_ref(L.dy, w.t())
    eb = dot_bound(ref, mag, L.out_f)
    mask = below_y > 0
    check_close(f"{S}/{name}.dy", below_dy, torch.where(mask, ref, torch.zeros_like(ref)), eb)
    check_zero(f"{S}/{name}.dy masked", torch.where(mask, torch.zeros_like(below_dy), below_dy))
    check_close(f"{S}/{name}.gb", below_gb[:ref.shape[1]], (ref * mask).sum(0),
                _masked_colsum_bound(ref, eb, mask, torch.zeros_like(ref[0])))

  for i in range(len(step.top) - 1, 0, -1):
    below = step.top[i - 1]
    dgrad(f"top[{i - 1}]", step.top[i], below.y, below.dy, _flat(g32, below, "b"))
  # dz = dy @ W of the first top layer (no activation below: the interaction)
  w, _ = _old(step, p16_old, step.top[0])
  ref, mag = linear_ref(step.top[0].dy, w.t())
  check_close(f"{S}/dz", step.dz, ref, dot_bound(ref, mag, step.top[0].out_f))
  # interaction backward followed by relu_bwd_bias: the masked gradient of the bottom output
  db_ref, db_mag, de_ref, de_mag = interact_bwd_ref(hb.y, eng.out, step.dz, n_emb, 1.0)
  mask = hb.y > 0
  check_close(f"{S}/bottom[-1].dy", hb.dy, torch.where(mask, db_ref, torch.zeros_like(db_ref)),
              interact_bwd_bound(db_ref, db_mag))
  check_zero(f"{S}/bottom[-1].dy masked", torch.where(mask, torch.zeros_like(hb.dy), hb.dy))
  hdy = hb.dy.double()
  check_close(f"{S}/bottom[-1].gb", _flat(g32, hb, "b")[:hb.out_f], hdy.sum(0),
              acc_bound(b, hdy.abs().sum(0)))
  for i in range(len(step.bottom) - 1, 0, -1):
    below = step.bottom[i - 1]
    dgrad(f"bottom[{i - 1}]", step.bottom[i], below.y, below.dy, _flat(g32, below, "b"))

  # weight gradients dy^T x (fp32 outputs; K = batch products of bf16 values)
  layers = [(f"bottom[{i}]", L) for i, L in enumerate(step.bottom)] + \
      [(f"top[{i}]", L) for i, L in enumerate(step.top)]
  for name, L in layers:
    xin = inputs[id(L)]
    ref, mag = linear_ref(L.dy.t(), xin.t())
    check_close(f"{S}/{name}.gw", _flat(g32, L, "w"), ref, acc_bound(b, mag))

  # update: bit exact with a power-of-two lr; bf16 shadow; cleared gradients; transposes
  lr_t = torch.tensor(LR, dtype=torch.float32, device="cuda")
  check_bits(f"{S}/p32 update", step.p32, p32_0 - lr_t * g32)
  check_bits(f"{S}/p16 = bf16(p32)", step.p16, step.p32.bfloat16())
  check_zero(f"{S}/g32 cleared", step.g32)
  if gemm != "cublas":
    for L in step.bottom[1:] + step.top[1:]:
      check_bits(f"{S}/w16T", L.w16T, L.w16.t())
  for name, L in layers + [("head", H)]:
    for buf, what in ((step.p32, "p32"), (step.p16, "p16"), (g32, "g32")):
      check_zero(f"{S}/{name} {what} weight pad", _flat(buf, L, "w")[:, L.in_f:])
      check_zero(f"{S}/{name} {what} bias pad", _flat(buf, L, "b")[L.out_f:])

  # tables: touched rows move by -lr x the sum of their samples' embedding gradients
  tables_new = _tables(model)
  de_bound = interact_bwd_bound(de_ref, de_mag)
  for t in range(n_emb):
    assert tables_old[t].shape == (SIZES[t], dim)
    ids = cat[t].long()
    old, new = tables_old[t].double(), tables_new[t].double()
    rows = old.shape[0]
    gsum = torch.zeros(rows, dim, dtype=torch.float64, device="cuda")
    gsum.index_add_(0, ids, de_ref[:, t])
    carried = torch.zeros_like(gsum).index_add_(0, ids, de_bound[:, t])
    gabs = torch.zeros_like(gsum).index_add_(0, ids, de_ref[:, t].abs() + de_bound[:, t])
    occ = torch.bincount(ids, minlength=rows).double()[:, None]
    touched = occ[:, 0] > 0
    check_close(f"{S}/table {t} update", new[touched], (old - LR * gsum)[touched],
                (LR * carried + acc_bound(occ + 1, old.abs() + LR * gabs))[touched])
    check_bits(f"{S}/table {t} untouched rows", tables_new[t][~touched], tables_old[t][~touched])


@pytest.mark.gpu
@pytest.mark.parametrize("gemm", ["cublas", "fused_dgrad", "tcgen05", "tcgen05_pair"])
@pytest.mark.parametrize("b", [512, 777])
def test_step_stages(gemm, b):
  _check_step(gemm, b)


@pytest.mark.gpu
def test_step_stages_wgrad_stream(monkeypatch):
  """The weight-gradient GEMMs on their own stream (read when the step is built)."""
  monkeypatch.setenv("DE_B200_WGRAD_STREAM", "1")
  _check_step("tcgen05", 777)


@pytest.mark.gpu
def test_graph_replay_matches_eager():
  """Three graph replays against three eager steps of an identical model.

  The two runs execute the same kernels on the same data; they differ only in the order of fp32
  atomic additions (bias gradients, column sums, loss head, table updates).  In the first step
  that moves each gradient by at most 2 n u32 sum|terms|; afterwards a bf16 value that sits on a
  rounding boundary may flip by one bf16 ulp and move the gradients that depend on it by about
  u16 of their size.  Each step is therefore allowed lr * 2 u16 (|g| + mean |g| of the layer)
  per element, with |g| the eager step's gradient, plus two fp32 ulps of the weight."""
  model_e, eager = _make_step("tcgen05", use_graph=False, seed=4)
  _, graph = _make_step("tcgen05", use_graph=True, seed=4, like=model_e)
  proxy = _SnapshotOps(eager.ops)
  eager.ops = proxy
  batches = [_batch(640, seed=40 + i) for i in range(3)]
  for num, cat, lab in batches:
    eager.step(num, cat, lab)
    graph.step(num, cat, lab)
  torch.cuda.synchronize()
  layers = eager.bottom + eager.top + [eager.head]
  tol = 2 * _ulp32(eager.p32)
  for _, _, g32, _, _ in proxy.before_sgd:
    ga = g32.double().abs()
    for L in layers:
      for which in ("w", "b"):
        _flat(tol, L, which).add_(LR * 2 * U16 * (_flat(ga, L, which) + _flat(ga, L, which).mean()))
  check_close("graph replay vs eager/p32", graph.p32, eager.p32, tol + TINY)
  for L, Lg in zip(layers, graph.bottom + graph.top + [graph.head]):
    for buf in (graph.p32, graph.p16):
      check_zero("graph replay/weight pad", _flat(buf, Lg, "w")[:, Lg.in_f:])
      check_zero("graph replay/bias pad", _flat(buf, Lg, "b")[Lg.out_f:])
  check_zero("graph replay/z pad", graph.z[:, (eager.n_emb + 1) * eager.n_emb // 2 + eager.dim:])
