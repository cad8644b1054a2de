"""The single-table lookup ops against a float64 model, on every kernel path they take.

``embedding_lookup_fwd``, ``embedding_lookup_grad`` (the sorted "emit" route) and
``embedding_scatter_add`` are the GPU path of ``embedding_lookup``, ``de.Embedding`` and the
torch back end of ``DistributedEmbedding``, which several GPU tests use as their reference.  They
launch the same lookup, key-building, radix-sort and segment kernels as the fused engine, so a
defect there would cancel out of a fused-versus-torch comparison.  Here every op is checked
directly against a numpy float64 model computed from the kernel's own stored operands (16-bit
tables and gradients upcast exactly).

Semantics the model implements:

* pooling runs in fp32 and is stored once, in the table's dtype or in bf16 with ``out_bf16``;
* ids outside ``[0, rows)`` contribute zero, but ``mean`` still counts them; an empty row is zero;
* ``combiner=None`` (and any one-id pooling) is a copy;
* the sparse gradient holds the sorted unique in-range ids, out-of-range ids are dropped;
* the dense gradient is ``dst[id] += scale * w * g`` with ``w = 1 / n`` for ``mean``.

Bounds follow from the operation counts (u = 2^-24, gamma(n) = n u / (1 - n u)):

* an fp32 sum of k terms in any order: ``gamma(k - 1) * sum|x|``;
* ``mean``: the rounded reciprocal and the multiply add ``gamma(2)`` of the result;
* gradient terms scaled before the sum (mean weights, ``scale``) add one rounding per factor;
* a 16-bit result adds half an ulp: ``u16 * (|ref| + e)`` plus half the smallest subnormal;
* copies are bit exact, entries that must be zero are exactly zero, and guard rows and elements
  around the outputs keep their bits.

A CPU self-check requires every modelled defect to fail these bounds on the cases' data, and the
CPU implementation (the suite's other oracle) is run against the model on every CPU-sized case.
"""
import math

import numpy as np
import pytest
import torch

from distributed_embeddings_b200.ops import embedding_lookup_ops as elo
from distributed_embeddings_b200.ops.ragged import RaggedIds, SparseIds
from optim_reference import TINY, U  # pylint: disable=wrong-import-order

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]
TABLE_DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
U_OUT = {torch.float32: 0.0, torch.bfloat16: 2.0**-8, torch.float16: 2.0**-11}
# half the smallest subnormal of the output type (absolute rounding error near zero)
TINY_OUT = {torch.float32: TINY, torch.bfloat16: 2.0**-134, torch.float16: 2.0**-25}
COMBINER = {"sum": 0, "mean": 1}
# 4-wide and 8-wide classes, scalar widths, several column passes (4-wide, 8-wide, scalar)
WIDTHS = [4, 8, 6, 10, 1000, 1001, 2048]
LAYOUTS = ["hot1", "hot3", "hot64", "ragged", "coo"]
INT32_MAX = 2**31 - 1


def gamma(n):
  n = np.maximum(np.asarray(n, dtype=np.float64), 0.0)
  return n * U / (1.0 - n * U)


# ------------------------------------------------------------------ float64 model
def seg_sum(x, seg, nseg):
  """Row sums of ``x`` per segment (``seg`` non-decreasing in [0, nseg)), accumulated in float64."""
  out = np.zeros((nseg, x.shape[1]), dtype=np.float64)
  if len(seg) == 0:
    return out
  starts = np.flatnonzero(np.r_[True, seg[1:] != seg[:-1]])
  out[seg[starts]] = np.add.reduceat(x, starts, axis=0, dtype=np.float64)
  return out


def sample_of(counts):
  return np.repeat(np.arange(len(counts)), counts)


def fwd_model(tab, vals, counts, combiner, out_dtype, valid_rows=None, hot_unroll=None,
              mean_of_valid=False):
  """Pooled rows (float64) and their bounds.  ``valid_rows``, ``hot_unroll`` and
  ``mean_of_valid`` model defects for the self-check (ids up to ``valid_rows`` read, tails after
  the unroll dropped, the mean taken over the in-range ids only)."""
  rows = tab.shape[0] if valid_rows is None else valid_rows
  batch = len(counts)
  sample = sample_of(counts)
  ok = (vals >= 0) & (vals < rows)
  if hot_unroll is not None:
    pos = np.arange(len(vals)) - np.repeat(np.cumsum(counts) - counts, counts)
    ok &= pos < np.repeat(counts // hot_unroll * hot_unroll, counts)
  x = tab[vals[ok]]
  s = seg_sum(x, sample[ok], batch)
  a = seg_sum(np.abs(x), sample[ok], batch)
  k = np.bincount(sample[ok], minlength=batch)[:, None]
  e = gamma(k - 1) * a
  ref = s
  if combiner == "mean":
    n = np.maximum(k[:, 0] if mean_of_valid else counts, 1)[:, None].astype(np.float64)
    ref = s / n
    e = (e + gamma(2) * (np.abs(s) + e)) / n
  e = e + U_OUT[out_dtype] * (np.abs(ref) + e) + TINY_OUT[out_dtype]
  return {"ref": ref, "bound": e, "zero": np.broadcast_to(k == 0, ref.shape)}


def grad_model(vals, counts, g, combiner, num_rows, dup_twice=False, mean_of_valid=False):
  """Sparse gradient: sorted unique in-range ids, their summed rows (float64) and bounds.
  ``g`` is the gradient as stored, upcast exactly (fp32 or float64 array, any strides).
  ``dup_twice`` and ``mean_of_valid`` model defects for the self-check."""
  sample = sample_of(counts)
  ok = (vals >= 0) & (vals < num_rows)
  ids = vals[ok]
  order = np.argsort(ids, kind="stable")
  ids_s = ids[order]
  smp = sample[ok][order]
  uniq, starts = np.unique(ids_s, return_index=True)
  k = np.diff(np.r_[starts, len(ids_s)])[:, None]
  if combiner == "mean":
    n = np.bincount(sample[ok], minlength=len(counts)) if mean_of_valid else counts
    w = 1.0 / np.maximum(n, 1).astype(np.float64)
    terms = g[smp].astype(np.float64) * w[smp][:, None]
  else:
    terms = g[smp]
  if len(ids_s) == 0:
    rows = np.zeros((0, g.shape[1]))
    a = rows
  else:
    rows = np.add.reduceat(terms, starts, axis=0, dtype=np.float64)
    a = np.add.reduceat(np.abs(terms), starts, axis=0, dtype=np.float64)
    if dup_twice:  # the first occurrence of every repeated id counted twice
      rows = rows + np.where(k > 1, terms[starts].astype(np.float64), 0.0)
  ops = k + 1 if combiner == "mean" else k - 1  # the mean weight adds two roundings per term
  return {"ids": uniq, "rows": rows, "abs": a, "k": k,
          "bound": gamma(ops) * a + TINY}


def scatter_model(d0, gm, combiner, scale):
  """``dst0 + scale * sum w g`` on the touched rows; untouched rows keep their bits."""
  ref = d0.astype(np.float64).copy()
  bound = np.zeros_like(ref)
  ids = gm["ids"]
  ref[ids] += scale * gm["rows"]
  ops = gm["k"] + (2 if combiner == "mean" else 1)  # w * g rounds, and every add into dst
  bound[ids] = gamma(ops) * (np.abs(d0[ids]) + abs(scale) * gm["abs"]) + TINY
  return ref, bound


# ------------------------------------------------------------------ comparisons
def _np(t):
  return t.detach().to(torch.float64).cpu().numpy()


def check_close(name, out, ref, bound, zero=None):
  """``|out - ref| <= bound`` element-wise, and exactly zero where ``zero`` says so."""
  o = _np(out) if isinstance(out, torch.Tensor) else np.asarray(out, dtype=np.float64)
  assert o.shape == ref.shape, (name, o.shape, ref.shape)
  err = np.abs(o - ref)
  with np.errstate(invalid="ignore", divide="ignore"):
    # a NaN output fails; a zero bound admits only an exact result
    ratio = np.where(err == 0, 0.0, np.nan_to_num(err / bound, nan=math.inf))
  if ratio.size and ratio.max() > 1.0:
    i = np.unravel_index(int(ratio.argmax()), ratio.shape)
    raise AssertionError(
        f"{name}: {int((ratio > 1).sum())} of {ratio.size} elements exceed the bound; worst "
        f"|err|/bound = {ratio[i]:.3g} at {i}: out={o[i]!r} ref={ref[i]!r} bound={bound[i]:.3g}")
  if zero is not None and np.any(o[zero] != 0):
    i = tuple(np.argwhere(zero & (o != 0))[0])
    raise AssertionError(f"{name}: element {i} must be exactly zero, is {o[i]!r}")


def _bits(t):
  t = t.detach().cpu().contiguous()
  return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def check_bits(name, out, ref):
  assert out.dtype == ref.dtype and out.shape == ref.shape, (name, out.dtype, ref.dtype)
  diff = _bits(out) != _bits(ref)
  if bool(diff.any()):
    i = int(diff.reshape(-1).nonzero()[0])
    raise AssertionError(f"{name}: {int(diff.sum())} of {diff.numel()} elements differ bitwise; "
                         f"first at flat index {i}: out={float(out.reshape(-1)[i])!r} "
                         f"ref={float(ref.reshape(-1)[i].cpu())!r}")


# ------------------------------------------------------------------ cases
def _values(gen, n, rows, specials=True):
  """Ids in range with ~12 % of them outside: ``rows``, negative, and the int32 extremes."""
  v = gen.integers(0, rows, n)
  if specials and n:
    bad = gen.random(n) < 0.12
    v[bad] = gen.choice([rows, -1, -7, INT32_MAX, -2**31], int(bad.sum()))
  return v.astype(np.int64)


def make_layout(layout, width, rows, seed):
  """(values, counts, hotness or None) of one id layout; ``hotness=None`` means CSR / COO."""
  gen = np.random.default_rng(seed)
  if layout.startswith("hot"):
    hot = int(layout[3:])
    batch = max(4, min(256, 1_500_000 // (hot * width)))
    counts = np.full(batch, hot)
    return _values(gen, batch * hot, rows), counts, hot
  # ragged: empty rows, rows of one id, rows of many (tails after every unroll width) and one
  # very long row among rows of one id (it spreads over many warps of the tile heuristic)
  long_row = 50_000 if width <= 16 else 2_000
  counts = gen.choice([0, 0, 1, 1, 2, 3, 5, 7, 9, 13, 31, 64, 127, 300], 48)
  if layout == "coo":
    counts[-1] = 0  # trailing empty rows only exist in the dense shape of a COO input
    counts = np.r_[counts, [1] * 6, long_row // 5, [1] * 6, 0, 0]
  else:
    counts = np.r_[counts, [1] * 16, long_row, [1] * 16]
  return _values(gen, int(counts.sum()), rows), counts, None


def _table(rows, width, dtype, seed):
  g = torch.Generator().manual_seed(seed)
  # non-dyadic normal values of mixed signs and magnitudes
  t = torch.randn(rows, width, generator=g)
  t = (t.sign() * (t.abs() + 0.05)) * torch.exp2(torch.randint(-3, 3, (rows, 1), generator=g).float())
  return t.to(dtype)


def _id_dtypes(device):
  """The CPU implementation widens every id to int64 first: one id dtype is enough there."""
  return (torch.int32, torch.int64) if device == "cuda" else (torch.int64,)


def _ids(vals, id_dtype, device):
  return torch.from_numpy(vals).to(id_dtype).to(device)


def _splits(counts, device):
  return torch.from_numpy(np.r_[0, np.cumsum(counts)].astype(np.int64)).to(device)


def _coo(vals, counts, id_dtype, device):
  rows = np.repeat(np.arange(len(counts)), counts)
  cols = np.arange(len(vals)) - np.repeat(np.cumsum(counts) - counts, counts)
  idx = torch.from_numpy(np.stack([rows, cols], 1).astype(np.int64)).to(device)
  return SparseIds(idx, _ids(vals, id_dtype, device), (len(counts), int(counts.max()) + 1))


def _offsets(layout, counts, device):
  """CSR offsets as the public wrappers build them (``row_to_split`` for COO)."""
  if layout == "coo":
    rows = np.repeat(np.arange(len(counts)), counts)
    idx = torch.from_numpy(np.stack([rows, np.zeros_like(rows)], 1).astype(np.int64)).to(device)
    got = elo.row_to_split(idx, len(counts))
    assert torch.equal(got.cpu(), _splits(counts, "cpu")), "row_to_split"
    return got
  return _splits(counts, device)


# ------------------------------------------------------------------ forward
def _fwd_public(param, vals, counts, hot, layout, id_dtype, combiner):
  dev = param.device
  if hot is not None:
    return elo.embedding_lookup(param, _ids(vals, id_dtype, dev).reshape(len(counts), hot),
                                combiner)
  if layout == "coo":
    return elo.embedding_lookup(param, _coo(vals, counts, id_dtype, dev), combiner)
  return elo.embedding_lookup(param, RaggedIds(_ids(vals, id_dtype, dev), _splits(counts, dev)),
                              combiner)


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("width", WIDTHS)
@pytest.mark.parametrize("tdt", sorted(TABLE_DTYPES))
def test_forward(device, tdt, width, layout):
  dtype = TABLE_DTYPES[tdt]
  rows = 97
  param = _table(rows, width, dtype, seed=width).to(device)
  vals, counts, hot = make_layout(layout, width, rows, seed=width + len(layout))
  tab = _np(param)
  for combiner in ("sum", "mean"):
    for id_dtype in _id_dtypes(device):
      name = f"fwd/{tdt}/w{width}/{layout}/{combiner}/{id_dtype}"
      # the public op stores in the table's dtype
      m = fwd_model(tab, vals, counts, combiner, dtype)
      out = _fwd_public(param, vals, counts, hot, layout, id_dtype, combiner)
      assert out.dtype == dtype
      check_close(name, out, m["ref"], m["bound"], m["zero"])
      # out_bf16: pooled in fp32, rounded once to bf16
      m16 = fwd_model(tab, vals, counts, combiner, torch.bfloat16)
      out16 = elo.lookup_forward(param, _ids(vals, id_dtype, device),
                                 None if hot else _offsets(layout, counts, device), hot or 0,
                                 len(counts), COMBINER[combiner], True)
      assert out16.dtype == torch.bfloat16
      check_close(name + "/out_bf16", out16, m16["ref"], m16["bound"], m16["zero"])
      if hot == 1:  # one id per sample: a copy, bit exact
        want = torch.where(torch.from_numpy((vals >= 0) & (vals < rows))[:, None],
                           param.cpu()[torch.from_numpy(vals).clamp(0, rows - 1)].float(), 0.0)
        check_bits(name + "/copy", out.cpu(), want.to(dtype))
        check_bits(name + "/copy_bf16", out16.cpu(), want.to(torch.bfloat16))


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("width", [4, 8, 6, 1001])
@pytest.mark.parametrize("tdt", sorted(TABLE_DTYPES))
def test_forward_unpooled_copy(device, tdt, width):
  """``combiner=None``: every id is its own output row, a bit-exact copy (zero outside)."""
  dtype = TABLE_DTYPES[tdt]
  rows = 61
  param = _table(rows, width, dtype, seed=7 + width).to(device)
  vals = _values(np.random.default_rng(width), 150 * 5, rows)
  ok = torch.from_numpy((vals >= 0) & (vals < rows))[:, None]
  want = torch.where(ok, param.cpu()[torch.from_numpy(vals).clamp(0, rows - 1)].float(), 0.0)
  for id_dtype in _id_dtypes(device):
    ids = _ids(vals, id_dtype, device).reshape(150, 5)
    out = elo.embedding_lookup(param, ids, None)
    assert out.shape == (150, 5, width)
    check_bits(f"none/{tdt}/w{width}/{id_dtype}", out.cpu().reshape(-1, width), want.to(dtype))
    out16 = elo.lookup_forward(param, ids.reshape(-1), None, 1, 750, 0, True)
    check_bits(f"none/{tdt}/w{width}/{id_dtype}/bf16", out16.cpu(), want.to(torch.bfloat16))


# ------------------------------------------------------------------ backward
GRAD_DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}


def _grad(batch, width, dtype, kind, seed, device):
  """(tensor handed to the op, its values as stored, upcast to fp32 as a numpy array)."""
  g = torch.Generator().manual_seed(seed)
  if kind == "broadcast":  # stride 0 over the batch
    t = torch.randn(width, generator=g).to(dtype).to(device)[None, :].expand(batch, width)
  elif kind == "strided":  # row stride not a multiple of 4, base off the 16-byte grid
    pad = 2 if (width + 2) % 4 else 3
    t = torch.randn(batch, width + pad, generator=g).to(dtype).to(device)[:, 1:width + 1]
    assert t.stride(0) % 4 != 0
  else:
    t = torch.randn(batch, width, generator=g).to(dtype).to(device)
  return t, t.float().cpu().numpy()


def _grad_offsets(layout, counts, hot, device):
  return None if hot is not None else _offsets(layout, counts, device)


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("width", WIDTHS)
@pytest.mark.parametrize("gdt", sorted(GRAD_DTYPES))
def test_grad_sparse(device, gdt, width, layout):
  rows = 97
  vals, counts, hot = make_layout(layout, width, rows, seed=3 * width + len(layout))
  batch = len(counts)
  offsets = _grad_offsets(layout, counts, hot, device)
  for kind in ("contiguous", "strided", "broadcast"):
    grad, g = _grad(batch, width, GRAD_DTYPES[gdt], kind, seed=width, device=device)
    for combiner in ("sum", "mean"):
      m = grad_model(vals, counts, g, combiner, rows)
      for id_dtype in _id_dtypes(device):
        name = f"grad/{gdt}/w{width}/{layout}/{kind}/{combiner}/{id_dtype}"
        ids, out = elo.lookup_grad_sparse(_ids(vals, id_dtype, device), offsets, hot or 0, batch,
                                          COMBINER[combiner], grad, rows)
        assert ids.dtype == torch.int64 and out.dtype == torch.float32
        assert np.array_equal(ids.cpu().numpy(), m["ids"]), name + ": ids"
        check_close(name, out, m["rows"], m["bound"])


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("width", WIDTHS)
@pytest.mark.parametrize("gdt", sorted(GRAD_DTYPES))
def test_scatter_add(device, gdt, width, layout):
  """Dense backward into a pre-filled ``dst`` with ``scale != 1``; guard rows keep their bits."""
  rows = 97
  vals, counts, hot = make_layout(layout, width, rows, seed=5 * width + len(layout))
  batch = len(counts)
  offsets = _grad_offsets(layout, counts, hot, device)
  scale = 0.37
  gen = torch.Generator().manual_seed(width)
  for kind in ("contiguous", "strided", "broadcast"):
    grad, g = _grad(batch, width, GRAD_DTYPES[gdt], kind, seed=width + 1, device=device)
    for combiner in ("sum", "mean"):
      gm = grad_model(vals, counts, g, combiner, rows)
      for id_dtype in _id_dtypes(device):
        name = f"scatter/{gdt}/w{width}/{layout}/{kind}/{combiner}/{id_dtype}"
        buf = torch.randn(rows + 2, width, generator=gen).to(device)
        before = buf.clone()
        dst = buf[1:rows + 1]
        d0 = _np(dst)
        ref, bound = scatter_model(d0, gm, combiner, float(np.float32(scale)))
        out = elo.scatter_add_rows(dst, _ids(vals, id_dtype, device), offsets, hot or 0, batch,
                                   COMBINER[combiner], grad, scale)
        assert out.data_ptr() == dst.data_ptr()
        check_close(name, dst, ref, bound)
        untouched = torch.from_numpy(bound[:, 0] == 0)
        check_bits(name + "/untouched", dst.cpu()[untouched], before.cpu()[1:rows + 1][untouched])
        check_bits(name + "/guard", buf.cpu()[[0, rows + 1]], before.cpu()[[0, rows + 1]])


AUTOGRAD_FORMS = ["fixed/sum", "fixed/mean", "none", "ragged/mean", "ragged/sum", "coo/mean"]


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("sparse_grad", [True, False])
@pytest.mark.parametrize("form", AUTOGRAD_FORMS)
def test_autograd(device, form, sparse_grad):
  """``embedding_lookup`` end to end: forward, then the sparse or dense parameter gradient."""
  rows, width = 53, 12
  gen = np.random.default_rng(len(form))
  kind, _, combiner = form.partition("/")
  if kind in ("fixed", "none"):
    hot = 4
    counts = np.full(90, hot)
    vals = _values(gen, counts.sum(), rows)
  else:
    vals, counts, _ = make_layout(kind, width, rows, seed=11)
  param = _table(rows, width, torch.float32, seed=12).to(device).requires_grad_(True)
  ids = _ids(vals, torch.int64, device)
  if kind == "fixed":
    out = elo.embedding_lookup(param, ids.reshape(-1, hot), combiner, sparse_grad)
  elif kind == "none":
    out = elo.embedding_lookup(param, ids.reshape(-1, hot), None, sparse_grad).reshape(-1, width)
    counts, combiner = np.ones(len(vals), dtype=np.int64), "sum"
  elif kind == "ragged":
    out = elo.embedding_lookup(param, RaggedIds(ids, _splits(counts, device)), combiner,
                               sparse_grad)
  else:
    out = elo.embedding_lookup(param, _coo(vals, counts, torch.int64, device), combiner,
                               sparse_grad)
  tab = _np(param)
  m = fwd_model(tab, vals, counts, combiner, torch.float32)
  if kind == "none":
    check_bits(f"autograd/{form}/fwd", out.detach().cpu(), torch.from_numpy(m["ref"]).float())
  else:
    check_close(f"autograd/{form}/fwd", out, m["ref"], m["bound"], m["zero"])
  up = torch.randn(out.shape, generator=torch.Generator().manual_seed(3)).to(device)
  (out * up).sum().backward()
  gm = grad_model(vals, counts, up.cpu().numpy(), combiner, rows)
  if sparse_grad:
    assert param.grad.is_sparse
    grad = param.grad.coalesce()
    assert np.array_equal(grad.indices()[0].cpu().numpy(), gm["ids"]), form
    check_close(f"autograd/{form}/sparse", grad.values(), gm["rows"], gm["bound"])
  else:
    assert not param.grad.is_sparse
    ref, bound = scatter_model(np.zeros((rows, width)), gm, combiner, 1.0)
    check_close(f"autograd/{form}/dense", param.grad, ref, bound)


# ------------------------------------------------------------------ views off the vector grid
@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("width", [4, 8, 1000])
@pytest.mark.parametrize("tdt", sorted(TABLE_DTYPES))
def test_views_at_odd_element_offsets(device, tdt, width):
  """A contiguous table or ``dst`` view one element into its buffer is a legal input: the ops
  take their scalar path for it and compute the same values; elements around ``dst`` keep
  their bits."""
  dtype = TABLE_DTYPES[tdt]
  rows = 41
  buf = _table(rows * width + 1, 1, dtype, seed=width).reshape(-1).to(device)
  param = buf[1:].view(rows, width)
  assert param.is_contiguous() and param.storage_offset() == 1
  tab = _np(param)
  for layout in ("hot1", "hot3", "ragged"):
    vals, counts, hot = make_layout(layout, width, rows, seed=width)
    offsets = None if hot else _splits(counts, device)
    for combiner in ("sum", "mean"):
      name = f"odd/{tdt}/w{width}/{layout}/{combiner}"
      for out_bf16 in (False, True):
        m = fwd_model(tab, vals, counts, combiner, torch.bfloat16 if out_bf16 else dtype)
        out = elo.lookup_forward(param, _ids(vals, torch.int64, device), offsets, hot or 0,
                                 len(counts), COMBINER[combiner], out_bf16)
        check_close(f"{name}/fwd/bf16={out_bf16}", out, m["ref"], m["bound"], m["zero"])
      g = torch.randn(len(counts), width, generator=torch.Generator().manual_seed(1))
      gm = grad_model(vals, counts, g.numpy(), combiner, rows)
      dbuf = torch.randn(rows * width + 2, generator=torch.Generator().manual_seed(2)).to(device)
      before = dbuf.clone()
      dst = dbuf[1:1 + rows * width].view(rows, width)
      ref, bound = scatter_model(_np(dst), gm, combiner, float(np.float32(0.37)))
      elo.scatter_add_rows(dst, _ids(vals, torch.int32, device), offsets, hot or 0, len(counts),
                           COMBINER[combiner], g.to(device), 0.37)
      check_close(f"{name}/scatter", dst, ref, bound)
      check_bits(f"{name}/guard", dbuf.cpu()[[0, -1]], before.cpu()[[0, -1]])


# ------------------------------------------------------------------ key space and sort size
@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("id_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("num_rows", [2**32 - 2, 2**32 - 1, 2**33 + 7])
def test_grad_sparse_key_space(device, num_rows, id_dtype):
  """Row keys near and above 2^32: below 2^32 - 1 rows the keys sort as uint32 with the
  out-of-range sentinel (= rows) at the top of the key space, from 2^32 - 1 rows on as int64."""
  gen = np.random.default_rng(num_rows % 1000)
  top = INT32_MAX if id_dtype == torch.int32 else num_rows
  specials = [0, 1, num_rows - 1, num_rows, num_rows + 1, 2**32 - 3, 2**32 - 2, 2**32 - 1, 2**32,
              2**32 + 5, 2**33 + 6, -1, -2**31, 2**62, INT32_MAX, INT32_MAX - 1]
  if id_dtype == torch.int32:
    specials = [s for s in specials if -2**31 <= s <= INT32_MAX]
  pool = np.r_[gen.integers(0, top, 300), specials].astype(np.int64)
  counts = gen.choice([0, 1, 2, 5, 9, 33], 400)
  vals = gen.choice(pool, int(counts.sum()))
  offsets = _splits(counts, device)
  for width, gdt in ((8, torch.float32), (6, torch.bfloat16)):
    grad, g = _grad(len(counts), width, gdt, "contiguous", seed=width, device=device)
    for combiner in ("sum", "mean"):
      m = grad_model(vals, counts, g, combiner, num_rows)
      name = f"keys/{num_rows}/{id_dtype}/w{width}/{combiner}"
      ids, out = elo.lookup_grad_sparse(_ids(vals, id_dtype, device), offsets, 0, len(counts),
                                        COMBINER[combiner], grad, num_rows)
      assert np.array_equal(ids.cpu().numpy(), m["ids"]), name + ": ids"
      check_close(name, out, m["rows"], m["bound"])


@pytest.mark.gpu
def test_grad_sparse_beyond_one_scan_chunk():
  """32768 x 160 = 5.2 M int32 ids: more than 1024 sort tiles of 4096 pairs, so the digit and
  head scans carry their running totals across chunks."""
  batch, hot, width, rows = 32768, 160, 8, 200_003
  gen = np.random.default_rng(0)
  vals = (gen.random(batch * hot) ** 3 * rows).astype(np.int64)  # power-law: long segments
  vals[gen.random(vals.size) < 0.01] = rows
  counts = np.full(batch, hot)
  grad, g = _grad(batch, width, torch.float32, "contiguous", seed=0, device="cuda")
  m = grad_model(vals, counts, g, "sum", rows)
  ids, out = elo.lookup_grad_sparse(_ids(vals, torch.int32, "cuda"), None, hot, batch, 0, grad,
                                    rows)
  assert np.array_equal(ids.cpu().numpy(), m["ids"])
  check_close("keys/scan_carry", out, m["rows"], m["bound"])


# ------------------------------------------------------------------ the sort itself
SORT_SIZES = [4_194_305, 2**23 + 1]  # 1024 tiles + 1 pair, 2048 tiles + 1 pair


def _sort_keys(n, end_bit, pattern):
  gen = torch.Generator(device="cuda").manual_seed(n + end_bit)
  lo = torch.randint(0, 2**31, (n,), generator=gen, device="cuda", dtype=torch.int64)
  hi = torch.randint(0, 2**32, (n,), generator=gen, device="cuda", dtype=torch.int64)
  keys = ((hi << 31) | lo) & ((1 << end_bit) - 1)
  if pattern == "equal":
    keys = torch.full_like(keys, (1 << end_bit) - 1)
  elif pattern == "sorted":
    keys = torch.sort(keys).values
  elif pattern == "reverse":
    keys = torch.sort(keys, descending=True).values
  return keys


def _check_sort(ks, it, keys):
  ref_k, ref_i = torch.sort(keys, stable=True)
  assert torch.equal(ks, ref_k)
  assert torch.equal(it.long(), ref_i)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", ["random", "equal", "sorted", "reverse"])
@pytest.mark.parametrize("end_bit", [9, 16, 17, 24, 32])
@pytest.mark.parametrize("n", SORT_SIZES)
def test_radix_sort_pairs32_multi_chunk(n, end_bit, pattern):
  from distributed_embeddings_b200.ops import _native
  keys = _sort_keys(n, end_bit, pattern)
  k32 = torch.where(keys >= 2**31, keys - 2**32, keys).to(torch.int32)  # same bits, signed
  items = torch.arange(n, device="cuda", dtype=torch.int32)
  ks, it = _native.require().radix_sort_pairs32(k32, items, end_bit)
  assert ks.dtype == torch.int64
  _check_sort(ks, it, keys)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", ["random", "equal", "sorted", "reverse"])
@pytest.mark.parametrize("end_bit", [33, 48, 63])
@pytest.mark.parametrize("n", SORT_SIZES)
def test_radix_sort_pairs_multi_chunk(n, end_bit, pattern):
  from distributed_embeddings_b200.ops import _native
  keys = _sort_keys(n, end_bit, pattern)
  items = torch.arange(n, device="cuda", dtype=torch.int32)
  ks, it = _native.require().radix_sort_pairs(keys, items, end_bit)
  _check_sort(ks, it, keys)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", ["random", "equal", "distinct", "few"])
@pytest.mark.parametrize("n", SORT_SIZES)
def test_head_segments_multi_chunk(n, pattern):
  from distributed_embeddings_b200.ops import _native
  keys = torch.sort(_sort_keys(n, 40, "random")).values
  if pattern == "equal":
    keys = torch.full_like(keys, 12345)
  elif pattern == "distinct":
    keys = torch.arange(n, device="cuda", dtype=torch.int64) * 3
  elif pattern == "few":
    keys = keys >> 36  # 16 runs
  seg, nu = _native.require().head_segments(keys)
  uniq, counts = torch.unique_consecutive(keys, return_counts=True)
  u = int(nu.item())
  assert u == uniq.numel()
  assert torch.equal(seg[:u], torch.cumsum(counts, 0) - counts)
  assert int(seg[u].item()) == n


# ------------------------------------------------------------------ CPU self-check of the bounds
def _rounded(ref, dtype):
  """The exactly rounded result: float64 -> fp32 -> the output dtype."""
  return torch.from_numpy(ref).float().to(dtype)


def _truncated(ref, dtype):
  """The fp32 result rounded toward zero to ``dtype`` (a store that truncates)."""
  x = ref.astype(np.float32)
  if dtype == torch.bfloat16:
    return (torch.from_numpy(x).view(torch.int32) & -65536).view(torch.float32).bfloat16()
  r = x.astype(np.float16)
  over = np.abs(r.astype(np.float32)) > np.abs(x)
  r[over] = np.nextafter(r[over], np.float16(0))
  return torch.from_numpy(r)


def _bf16_pooled(tab, vals, counts):
  """Fixed hotness pooled with a bf16 accumulator (vectorised over the batch)."""
  hot = int(counts[0])
  x = torch.from_numpy(tab[np.clip(vals, 0, tab.shape[0] - 1)].reshape(len(counts), hot, -1))
  x = x * torch.from_numpy((vals >= 0) & (vals < tab.shape[0])).reshape(len(counts), hot, 1)
  acc = torch.zeros(x.shape[0], x.shape[2], dtype=torch.bfloat16)
  for h in range(hot):
    acc = (acc.float() + x[:, h].float()).bfloat16()
  return acc.double().numpy()


def _expect_fail(name, out, ref, bound, zero=None):
  with pytest.raises(AssertionError, match="exceed the bound|exactly zero"):
    check_close(f"selfcheck/{name}", out, ref, bound, zero)


def test_bounds_reject_forward_defects():
  rows = 97
  cases = {}
  for layout, width, tdt in (("hot64", 8, "fp32"), ("ragged", 6, "fp32"), ("ragged", 8, "bf16"),
                             ("hot3", 1001, "fp32"), ("hot3", 10, "bf16"), ("hot3", 10, "fp16")):
    tab = _np(_table(rows, width, TABLE_DTYPES[tdt], seed=width))
    vals, counts, _ = make_layout(layout, width, rows, seed=width + len(layout))
    cases[(layout, width, tdt)] = (tab, vals, counts)
    for combiner in ("sum", "mean"):
      for out_dtype in (torch.float32, torch.bfloat16, TABLE_DTYPES[tdt]):
        m = fwd_model(tab, vals, counts, combiner, out_dtype)
        check_close("selfcheck/rounded", _rounded(m["ref"], out_dtype), m["ref"], m["bound"],
                    m["zero"])
  tab, vals, counts = cases[("hot64", 8, "fp32")]
  m = fwd_model(tab, vals, counts, "sum", torch.float32)
  _expect_fail("pooled in bf16", _bf16_pooled(tab, vals, counts), m["ref"], m["bound"])
  tab, vals, counts = cases[("ragged", 6, "fp32")]
  m = fwd_model(tab, vals, counts, "mean", torch.float32)
  _expect_fail("mean over valid ids",
               fwd_model(tab, vals, counts, "mean", torch.float32, mean_of_valid=True)["ref"],
               m["ref"], m["bound"], m["zero"])
  for key, unroll in ((("ragged", 6, "fp32"), 8), (("ragged", 8, "bf16"), 4)):
    tab, vals, counts = cases[key]
    m = fwd_model(tab, vals, counts, "sum", torch.float32)
    _expect_fail(f"tail after the {unroll}-wide unroll dropped",
                 fwd_model(tab, vals, counts, "sum", torch.float32, hot_unroll=unroll)["ref"],
                 m["ref"], m["bound"], m["zero"])
  tab, vals, counts = cases[("hot3", 1001, "fp32")]
  m = fwd_model(tab, vals, counts, "sum", torch.float32)
  short = m["ref"].copy()
  short[:, -1] = 0.0  # the last column pass stops one column early
  _expect_fail("last column pass one short", short, m["ref"], m["bound"], m["zero"])
  guard = np.vstack([tab, np.full((1, tab.shape[1]), 0.3)])  # the row behind the table
  _expect_fail("id == rows read", fwd_model(guard, vals, counts, "sum", torch.float32,
                                            valid_rows=rows + 1)["ref"],
               m["ref"], m["bound"], m["zero"])
  for tdt in ("bf16", "fp16"):
    tab, vals, counts = cases[("hot3", 10, tdt)]
    for combiner in ("sum", "mean"):
      m = fwd_model(tab, vals, counts, combiner, TABLE_DTYPES[tdt])
      _expect_fail(f"{tdt} store truncated", _truncated(m["ref"], TABLE_DTYPES[tdt]), m["ref"],
                   m["bound"], m["zero"])


def test_bounds_reject_backward_defects():
  rows, width = 97, 8
  for layout in ("hot3", "ragged"):
    vals, counts, _ = make_layout(layout, width, rows, seed=4)
    g = torch.randn(len(counts), width, generator=torch.Generator().manual_seed(5)).numpy()
    for combiner in ("sum", "mean"):
      m = grad_model(vals, counts, g, combiner, rows)
      check_close("selfcheck/grad_rounded", m["rows"].astype(np.float32), m["rows"], m["bound"])
      _expect_fail(f"{layout}/{combiner}: duplicate id summed twice",
                   grad_model(vals, counts, g, combiner, rows, dup_twice=True)["rows"], m["rows"],
                   m["bound"])
      d0 = torch.randn(rows, width, generator=torch.Generator().manual_seed(6)).numpy()
      ref, bound = scatter_model(d0, m, combiner, 0.37)
      check_close("selfcheck/scatter_rounded", ref.astype(np.float32), ref, bound)
    m = grad_model(vals, counts, g, "mean", rows)
    bad = grad_model(vals, counts, g, "mean", rows, mean_of_valid=True)
    _expect_fail(f"{layout}: sparse mean over valid ids", bad["rows"], m["rows"], m["bound"])
    ref, bound = scatter_model(d0, m, "mean", 0.37)
    _expect_fail(f"{layout}: dense mean over valid ids", scatter_model(d0, bad, "mean", 0.37)[0],
                 ref, bound)
