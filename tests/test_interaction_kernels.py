"""The DLRM dot-interaction kernels beyond the float64 bounds of ``test_dense_conformance.py``.

GPU:
  * the double-buffered backward (v2) is bit identical to the single-buffered one (v1) on the same
    inputs: both run the same MMAs in the same order on the same operands;
  * NaN in the memory next to the rows the kernels stage (past each feature row, past the dz
    row's used columns, past the batch) reaches neither ``z`` nor the gradients;
  * the table update applied by the backward equals the scatter of its gradient rows within fp32
    rounding when the samples of a block hit the same few rows many times;
  * ``z`` written through a view whose rows are not 16-byte aligned equals ``z`` written through
    an aligned one, and the columns around the view are left untouched.
"""
import numpy as np
import pytest
import torch

U32 = 2.0 ** -24


def _ops():
  from distributed_embeddings_b200.ops import _native
  return _native.require()


def _randn(g, *shape, scale=1.0):
  return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _z_width(n_emb, dim):
  return (n_emb * (n_emb + 1) // 2 + dim + 7) // 8 * 8


def _max_v2_emb(dim):
  """Largest n_emb whose staged dz row (triangle + bottom gradient) fits v2's 512 elements."""
  n = 1
  while (n + 2) * (n + 1) // 2 + dim <= 512:
    n += 1
  return n


def _inputs(dim, n_emb, batch, seed):
  g = torch.Generator(device="cuda").manual_seed(seed)
  zw = _z_width(n_emb, dim)
  return (_randn(g, batch, dim), _randn(g, batch, n_emb * dim), _randn(g, batch, zw, scale=0.1))


def _bwd(bottom, emb, n_emb, dz, dbottom, demb, apply=()):
  _ops().interact_bwd(bottom, emb, n_emb, dz, dbottom, demb.data_ptr(), demb.stride(0), 0.75,
                      None, 0, [], None, 0, *apply)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [64, 128])
@pytest.mark.parametrize("n_emb", [1, 26, "max"])
def test_bwd_v2_bit_identical_to_v1(dim, n_emb):
  n_emb = _max_v2_emb(dim) if n_emb == "max" else n_emb
  batch = 3 * 132 * 4 * 2 + 5  # several samples per warp, a ragged tail
  bottom, emb, dz = _inputs(dim, n_emb, batch, seed=dim + n_emb)
  demb2 = torch.empty(batch, n_emb * dim, dtype=torch.bfloat16, device="cuda")
  db2 = torch.empty(batch, dim, dtype=torch.bfloat16, device="cuda")
  _bwd(bottom, emb, n_emb, dz, db2, demb2)
  # a dbottom row stride that is not a multiple of 8 elements leaves only v1 eligible
  demb1 = torch.empty_like(demb2)
  db1 = torch.empty(batch, dim + 2, dtype=torch.bfloat16, device="cuda")[:, :dim]
  _bwd(bottom, emb, n_emb, dz, db1, demb1)
  torch.cuda.synchronize()
  assert torch.equal(db1, db2), f"dbottom differs (dim {dim}, n_emb {n_emb})"
  assert torch.equal(demb1, demb2), f"embedding gradient differs (dim {dim}, n_emb {n_emb})"


def _nan_padded(t, extra_cols, extra_rows=3):
  """A view equal to t inside a buffer whose other columns and rows hold NaN."""
  buf = torch.full((t.shape[0] + extra_rows, t.shape[1] + extra_cols), float("nan"),
                   dtype=t.dtype, device=t.device)
  v = buf[:t.shape[0], :t.shape[1]]
  v.copy_(t)
  return v


@pytest.mark.gpu
@pytest.mark.parametrize("dim,n_emb", [(128, 26), (128, 5), (64, 29)])
def test_nan_next_to_staged_rows_does_not_leak(dim, n_emb):
  batch = 1000
  bottom, emb, dz = _inputs(dim, n_emb, batch, seed=11 * n_emb)
  n_used = n_emb * (n_emb + 1) // 2 + dim
  dz[:, n_used:] = 0  # columns of z that are zero pad
  ops = _ops()
  zw = dz.shape[1]
  z_ref = torch.empty(batch, zw, dtype=torch.bfloat16, device="cuda")
  ops.interact_fwd(bottom, emb, n_emb, z_ref, [])
  db_ref = torch.empty(batch, dim, dtype=torch.bfloat16, device="cuda")
  de_ref = torch.empty(batch, n_emb * dim, dtype=torch.bfloat16, device="cuda")
  _bwd(bottom, emb, n_emb, dz, db_ref, de_ref)

  nb, ne = _nan_padded(bottom, 8), _nan_padded(emb, 8)
  ndz = _nan_padded(dz, 8)
  ndz[:, n_used:] = float("nan")  # staged with the row's last chunk, never an operand
  z = torch.empty_like(z_ref)
  ops.interact_fwd(nb, ne, n_emb, z, [])
  db = torch.empty_like(db_ref)
  de = torch.empty_like(de_ref)
  _bwd(nb, ne, n_emb, ndz, db, de)
  torch.cuda.synchronize()
  assert not bool(z.isnan().any()) and torch.equal(z, z_ref)
  assert not bool(db.isnan().any()) and torch.equal(db, db_ref)
  assert not bool(de.isnan().any()) and torch.equal(de, de_ref)


@pytest.mark.gpu
@pytest.mark.parametrize("ids64", [False, True])
def test_applied_update_with_duplicate_ids(ids64):
  from distributed_embeddings_b200.ops._native import INPUT_DESC
  dim, n_emb, batch, rows = 128, 8, 4096, 1000
  bottom, emb, dz = _inputs(dim, n_emb, batch, seed=3)
  g = torch.Generator(device="cuda").manual_seed(4)
  applied = [0, 2, 3, 7]  # the others stay routed
  # every sample of feature f hits one of a few rows (fewer for the later features)
  ids = [torch.randint(0, 1 + 7 * (f % 3), (batch,), generator=g, device="cuda",
                       dtype=torch.int64 if ids64 else torch.int32) for f in range(n_emb)]
  tables = [torch.randn(rows, dim, generator=g, device="cuda") for _ in applied]
  old = [t.clone() for t in tables]
  descs = np.zeros(n_emb, dtype=INPUT_DESC)
  for k, f in enumerate(applied):
    descs[f]["table"] = tables[k].data_ptr()
    descs[f]["ids"] = ids[f].data_ptr()
    descs[f]["sub_rows"] = rows
    descs[f]["width"] = dim
    descs[f]["hotness"] = 1
  scale = -0.5
  demb_ref = torch.empty(batch, n_emb * dim, dtype=torch.bfloat16, device="cuda")
  db_ref = torch.empty(batch, dim, dtype=torch.bfloat16, device="cuda")
  _bwd(bottom, emb, n_emb, dz, db_ref, demb_ref)
  demb = torch.full_like(demb_ref, 7.0)
  db = torch.empty_like(db_ref)
  _bwd(bottom, emb, n_emb, dz, db, demb,
       (torch.from_numpy(descs.view(np.uint8).copy()), scale, 0, ids64))
  torch.cuda.synchronize()
  assert torch.equal(db, db_ref)
  for f in range(n_emb):
    cols = slice(f * dim, (f + 1) * dim)
    if f in applied:
      assert bool((demb[:, cols] == 7.0).all()), f"applied feature {f} was also stored"
    else:
      assert torch.equal(demb[:, cols], demb_ref[:, cols]), f"routed feature {f}"
  for k, f in enumerate(applied):
    grad = demb_ref[:, f * dim:(f + 1) * dim].double() * scale
    idx = ids[f].long()
    gsum = torch.zeros(rows, dim, dtype=torch.float64, device="cuda").index_add_(0, idx, grad)
    gabs = torch.zeros_like(gsum).index_add_(0, idx, grad.abs())
    occ = torch.zeros(rows, dtype=torch.float64, device="cuda").index_add_(
        0, idx, torch.ones(batch, dtype=torch.float64, device="cuda"))
    ref = old[k].double() + gsum
    bound = 2 * (occ[:, None] + 1) * U32 * (old[k].double().abs() + gabs) + 1e-30
    err = (tables[k].double() - ref).abs()
    assert bool((err <= bound).all()), \
        f"feature {f}: max excess {float((err - bound).max()):.3e}"
    assert float(occ.max()) > 100  # many duplicates of one row
    touched = occ > 0
    assert torch.equal(tables[k][~touched], old[k][~touched])


@pytest.mark.gpu
@pytest.mark.parametrize("dim,n_emb", [(128, 26), (64, 3), (16, 1)])
def test_fwd_unaligned_z(dim, n_emb):
  batch = 777
  bottom, emb, _ = _inputs(dim, n_emb, batch, seed=5 + dim)
  ops = _ops()
  zw = _z_width(n_emb, dim)
  z_ref = torch.empty(batch, zw, dtype=torch.bfloat16, device="cuda")
  ops.interact_fwd(bottom, emb, n_emb, z_ref, [])
  for lead, stride in ((1, zw + 3), (3, zw + 8), (8, zw + 9)):
    buf = torch.full((batch, stride), -3.0, dtype=torch.bfloat16, device="cuda")
    z = buf[:, lead:lead + zw]
    ops.interact_fwd(bottom, emb, n_emb, z, [])
    torch.cuda.synchronize()
    assert torch.equal(z, z_ref), f"lead {lead}, stride {stride}"
    assert bool((buf[:, :lead] == -3.0).all()) and bool((buf[:, lead + zw:] == -3.0).all()), \
        f"lead {lead}, stride {stride}: neighbours written"
