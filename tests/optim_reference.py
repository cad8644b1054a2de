"""float64 models of the optimizers with error bounds from operation counts, shared by the dense
(``test_dense_optimizers.py``) and the embedding (``test_fused_optimizers.py``) optimizer tests.

``reference`` is one element-wise Adagrad / Adam update on fp32 inputs, with the rounding bounds
of the kernels' fp32 operations.  ``table_step`` is one lazy step of an embedding optimizer on a
whole table: it sums the gradient of every row from its id occurrences, adds the weight decay,
applies SGD / Adagrad / row-wise Adagrad / Adam to the rows at least one id touched, and bounds
the result by the rounding of those operations plus the error of an fp32 gradient sum in any
order.  Untouched rows get a bound of zero: they must not change at all.
"""
import numpy as np
import torch

U = 2.0**-24  # fp32 unit roundoff
TINY = 1e-37


def _ulp32(x):
  """ulp of fp32 numbers of magnitude |x| (float64 tensor), subnormal floor included."""
  e = torch.floor(torch.log2(x.abs().clamp_min(2.0**-126)))
  return torch.pow(2.0, e - 23)


def f32(v):
  """The fp32 value of a scalar the kernels take as an fp32 argument."""
  return float(np.float32(v))


def reference(kind, p, g, s0, s1, lr, t, cfg, defect=None):
  """float64 result of one update on fp32 inputs, with its error bounds.  ``defect`` models a
  wrong kernel: 'bias_t_minus_1', 'eps_in_sqrt', 'no_state_writeback', 'no_grad_zero'."""
  f = lambda x: x.double()
  p, g, s0 = f(p), f(g), f(s0)
  lr, eps = f32(lr), f32(cfg["eps"])
  out, bound = {}, {}
  if kind == "adagrad":
    a = s0 + g * g
    den = (a + eps).sqrt() if defect == "eps_in_sqrt" else a.sqrt() + eps
    d = lr * g / den
    out["s0"] = s0 if defect == "no_state_writeback" else a
    bound["s0"] = _ulp32(a) + TINY  # one fma: exactly rounded
    e_d = 6 * U * d.abs()
  else:
    s1 = f(s1)
    b1, b2 = f32(cfg["beta1"]), f32(cfg["beta2"])
    c1, c2 = 1.0 - b1, 1.0 - b2  # exact in fp32 (Sterbenz)
    tt = t - 1 if defect == "bias_t_minus_1" else t
    m = b1 * s0 + c1 * g
    v = b2 * s1 + c2 * g * g
    pw1, pw2 = b1**tt, b2**tt
    bias1, bias2 = 1.0 - pw1, 1.0 - pw2
    mh, vh = m / bias1, v / bias2
    sq = (vh + eps).sqrt() if defect == "eps_in_sqrt" else vh.sqrt()
    den = sq if defect == "eps_in_sqrt" else sq + eps
    d = lr * mh / den
    out["s0"] = s0 if defect == "no_state_writeback" else m
    out["s1"] = s1 if defect == "no_state_writeback" else v
    # moments: two or three roundings of the terms (fma contraction only removes some)
    e_m = 2.5 * U * ((b1 * s0).abs() + (c1 * g).abs())
    e_v = 3.5 * U * ((b2 * s1).abs() + c2 * g * g)
    bound["s0"], bound["s1"] = e_m + TINY, e_v + TINY
    # bias corrections: powf within 4 ulps, then one rounding of 1 - x
    rb1 = 4 * float(_ulp32(torch.tensor(pw1))) / bias1 + U
    rb2 = 4 * float(_ulp32(torch.tensor(pw2))) / bias2 + U
    e_mh = e_m / bias1 + mh.abs() * (rb1 + U)
    rv = torch.where(v > 0, e_v / v.clamp_min(1e-300), torch.zeros_like(v)) + rb2 + U
    e_sq = sq * (rv / 2 + U)
    e_den = e_sq + U * den
    e_d = (lr * e_mh + U * lr * mh.abs()) / den + d.abs() * (e_den / den + U)
  out["p"] = p - d
  bound["p"] = 1.05 * e_d + U * out["p"].abs() + TINY
  out["g"] = g if defect == "no_grad_zero" else torch.zeros_like(g)
  return out, bound


# ------------------------------------------------------------------ embedding optimizers
# Defects ``table_step`` can model (each must fail the bounds while the exact result passes):
TABLE_DEFECTS = ("decay_dropped", "decay_twice", "rowwise_acc_without_decay", "bias_t_minus_1",
                 "eps_in_sqrt", "mean_weight_dropped", "duplicate_applied_twice",
                 "untouched_decayed")


def row_update(kind, w, gp, e_gp, s0, s1, lr, t, cfg, defect=None):
  """One update of the touched rows from their decayed gradient ``gp`` ([R, W] float64, known to
  within ``e_gp`` of what the kernel computes).  Returns (out, bound) for 'p', 's0', 's1'.

  SGD, Adagrad and Adam are element-wise: the rounding of their own operations comes from
  :func:`reference` (SGD: one fma), the error of the input from the envelope of the same float64
  update evaluated at ``gp -/+ e_gp`` (twice the larger deviation: the update is smooth at that
  scale, and Adam is not monotone in g when m != 0).  Row-wise Adagrad bounds its accumulator
  first (a sum of W squares in any order, then / W and + a), then the shared denominator."""
  lr = f32(lr)
  out, bound = {}, {}
  if kind == "sgd":
    out["p"] = w - lr * gp
    bound["p"] = 1.05 * lr * e_gp + U * out["p"].abs() + TINY
    return out, bound
  if kind == "rowwise_adagrad":
    eps = f32(cfg["eps"])
    width = gp.shape[1]
    sq = (gp * gp).sum(1)
    acc = s0 + sq / width
    e_acc = (((2 * gp.abs() * e_gp + e_gp * e_gp).sum(1) + (width + 3) * U * sq) / width +
             U * acc.abs() + TINY)
    out["s0"], bound["s0"] = acc, 1.05 * e_acc
    root = acc.clamp_min(0).sqrt()
    den = ((acc + eps).sqrt() if defect == "eps_in_sqrt" else root + eps).unsqueeze(1)
    e_den = ((root - (acc - e_acc).clamp_min(0).sqrt()) + U * root + U * (root + eps)).unsqueeze(1)
    d = lr * gp / den
    e_d = lr * e_gp / den + d.abs() * (e_den / (den - e_den).clamp_min(TINY) + 3 * U)
    out["p"] = w - d
    bound["p"] = 1.05 * e_d + U * out["p"].abs() + TINY
    return out, bound
  fwd = lambda g: reference(kind, w.flatten(), g.flatten(), s0.flatten(),
                            None if s1 is None else s1.flatten(), lr, t, cfg,
                            defect=defect if defect in ("bias_t_minus_1", "eps_in_sqrt") else None)
  o, b = fwd(gp)
  lo, _ = fwd(gp - e_gp)
  hi, _ = fwd(gp + e_gp)
  for k in ("p", "s0", "s1"):
    if k in o:
      env = torch.maximum((lo[k] - o[k]).abs(), (hi[k] - o[k]).abs())
      out[k] = o[k].reshape(w.shape)
      bound[k] = (b[k] + 2 * env).reshape(w.shape)
  return out, bound


def table_step(kind, weights, state, occ_rows, occ_vals, scale, lr, t, cfg, defect=None,
               atomic=False):
  """float64 result of one lazy step of an embedding optimizer on one table, with bounds.

  weights [rows, W]: the table's values before the step (fp32, or 16-bit values widened);
  state: list of the state slots before the step ([rows, W], row-wise Adagrad [rows]);
  occ_rows [N]: the table row of every id occurrence of the step (ids outside the table left
  out); occ_vals [N, W]: c_k * g_k of each occurrence, the pooling weight (1, or the fp32 value of
  1/n for the mean of n ids) times the gradient row as the kernel reads it (after rounding to the
  compute dtype): the product is exact in float64.  ``scale``: the gradient scale (1 / world);
  ``cfg``: eps, beta1, beta2, weight_decay; ``t``: Adam's step after this one.

  The fp32 sum of n terms, then the scale, is within (n + 2) u |s| sum_k |c_k g_k| of the exact
  value whatever the order (chunked, RED atomics, fma contraction); the decay adds one fma.
  ``atomic``: SGD without decay as an atomic scatter, which adds each occurrence's scaled
  -lr c_k g_k into the weight on its own: n roundings of values up to |w| + lr |s| sum |c_k g_k|,
  plus the roundings of each product.
  Returns (out, bound, touched): dicts with 'p' and the state slots 's0' / 's1' over the whole
  table, bound 0 on rows no id touched (those must be bit-identical), and the touched mask."""
  w = torch.as_tensor(np.asarray(weights, dtype=np.float64))
  rows = w.shape[0]
  occ_rows = np.asarray(occ_rows, dtype=np.int64)
  vals = torch.as_tensor(np.asarray(occ_vals, dtype=np.float64))
  if defect == "mean_weight_dropped":
    raise ValueError("mean_weight_dropped is modelled by the caller (occurrence values)")
  s = f32(scale)
  wd = f32(cfg.get("weight_decay", 0.0))
  st = [torch.as_tensor(np.asarray(x, dtype=np.float64)) for x in state]
  touched = np.zeros(rows, dtype=bool)
  touched[occ_rows] = True
  if defect == "untouched_decayed":
    touched[:] = True
  idx = torch.as_tensor(np.nonzero(touched)[0])
  gsum = torch.zeros_like(w).index_add_(0, torch.as_tensor(occ_rows), vals)
  gabs = torch.zeros_like(w).index_add_(0, torch.as_tensor(occ_rows), vals.abs())
  n_occ = torch.zeros(rows, dtype=torch.float64).index_add_(
      0, torch.as_tensor(occ_rows), torch.ones(len(occ_rows), dtype=torch.float64))
  out = {"p": w.clone()}
  bound = {"p": torch.zeros_like(w)}
  for k, x in zip(("s0", "s1"), st):
    out[k], bound[k] = x.clone(), torch.zeros_like(x)
  if defect == "duplicate_applied_twice":
    # every occurrence applied as its own step (an unsorted scatter of a stateful update)
    cur_w, cur_s = w.clone(), [x.clone() for x in st]
    for r, v in zip(occ_rows, vals):
      o, _ = _one(kind, cur_w[r:r + 1], s * v[None], torch.zeros_like(v[None]), wd,
                  [x[r:r + 1] for x in cur_s], lr, t, cfg, None)
      cur_w[r] = o["p"][0]
      for j, k in enumerate(("s0", "s1")[:len(cur_s)]):
        cur_s[j][r] = o[k][0]
    out["p"] = cur_w
    for j, k in enumerate(("s0", "s1")[:len(cur_s)]):
      out[k] = cur_s[j]
    _, b = _one(kind, w[idx], s * gsum[idx], _e_sum(s, n_occ[idx], gabs[idx]), wd,
                [x[idx] for x in st], lr, t, cfg, None)
    for k in b:
      bound[k][idx] = b[k]
    return out, bound, touched
  o, b = _one(kind, w[idx], s * gsum[idx], _e_sum(s, n_occ[idx], gabs[idx]), wd,
              [x[idx] for x in st], lr, t, cfg, defect)
  if atomic and kind == "sgd":
    n, ga = n_occ[idx].unsqueeze(1), f32(lr) * abs(s) * gabs[idx]
    b["p"] = 1.05 * ((n + 3) * U * ga + n * U * (w[idx].abs() + ga)) + U * o["p"].abs() + TINY
  for k in o:
    out[k][idx] = o[k]
    bound[k][idx] = b[k]
  return out, bound, touched


def _e_sum(s, n, gabs):
  return (n.unsqueeze(1) + 2) * U * abs(s) * gabs


def _one(kind, w, g, e_g, wd, st, lr, t, cfg, defect):
  """Decay (one fma) then :func:`row_update` on the selected rows."""
  gp = g
  if defect == "decay_twice":
    gp = g + 2 * wd * w
  elif defect not in ("decay_dropped",):
    gp = g + wd * w
  e_gp = e_g + U * gp.abs() + TINY
  s0 = st[0] if st else None
  s1 = st[1] if len(st) > 1 else None
  if defect == "rowwise_acc_without_decay" and kind == "rowwise_adagrad":
    o_acc, _ = row_update(kind, w, g, e_gp, s0, s1, lr, t, cfg)
    o, b = row_update(kind, w, gp, e_gp, s0, s1, lr, t, cfg)
    acc = o_acc["s0"]
    den = (acc.sqrt() + f32(cfg["eps"])).unsqueeze(1)
    o["s0"], o["p"] = acc, w - f32(lr) * gp / den
    return o, b
  return row_update(kind, w, gp, e_gp, s0, s1, lr, t, cfg, defect)


def worst_table_ratio(out, bound, got):
  """max |got - ref| / bound over the weights and state of a table; a nonzero difference where
  the bound is zero (an untouched row) or a non-finite value gives inf."""
  worst = 0.0
  for k in out:
    g = torch.as_tensor(np.asarray(got[k], dtype=np.float64))
    err = (g - out[k]).abs()
    if not torch.isfinite(g).all() or bool((err[bound[k] == 0] != 0).any()):
      return float("inf")
    nz = bound[k] > 0
    if nz.any():
      worst = max(worst, float((err[nz] / bound[k][nz]).max()))
  return worst


def half_within(got16, ref, bound, dtype, step, keys, stream=0, mask=False):
  """16-bit result check: the kernel rounds its fp32 value x, known to lie in
  [ref - bound, ref + bound], stochastically with the bits of ``ops/stochastic_rounding.py``.  That
  rule is monotone in x for fixed bits, so the result must lie between the rounding of the two
  ends (rounded outward to fp32): exactly the reference's rounding wherever the interval holds no
  16-bit value.  Returns the number of elements outside (``mask``: whether each one is inside)."""
  from distributed_embeddings_b200.ops.stochastic_rounding import stochastic_round
  lo = (ref - bound).numpy()
  hi = (ref + bound).numpy()
  lo32 = lo.astype(np.float32)
  lo32 = np.where(lo32.astype(np.float64) > lo, np.nextafter(lo32, np.float32(-np.inf)), lo32)
  hi32 = hi.astype(np.float32)
  hi32 = np.where(hi32.astype(np.float64) < hi, np.nextafter(hi32, np.float32(np.inf)), hi32)
  keys = np.asarray(keys, dtype=np.int64)
  r_lo = stochastic_round(torch.from_numpy(lo32), dtype, step, keys, stream=stream).float()
  r_hi = stochastic_round(torch.from_numpy(hi32), dtype, step, keys, stream=stream).float()
  g = torch.as_tensor(got16).float()
  outside = (g < r_lo) | (g > r_hi)
  return ~outside.numpy() if mask else int(outside.sum())
