"""bf16 / fp16 storage of model-parallel tables (``DistributedEmbedding(table_dtype=...)``):
the stochastic-rounding rule, the plan interpreter at world sizes 1-8, checkpoints, the plan
report and - on an H100 - the fused kernels against the Python rule and the torch back end."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from distributed_embeddings_b200.ops import stochastic_rounding as sr
from distributed_embeddings_b200.parallel import dry_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HALF = [torch.bfloat16, torch.float16]


def _bits(t):
  return t.view(torch.int16).numpy().view(np.uint16)


# ----------------------------------------------------------------------------- rounding rule
@pytest.mark.parametrize("dtype", HALF)
def test_representable_values_are_unchanged(dtype):
  x = torch.randn(4096).to(dtype)
  x = torch.cat([x, torch.tensor([0.0, -0.0, float("inf"), -float("inf")], dtype=dtype)])
  out = sr.stochastic_round(x.float().view(1, -1), dtype, 7, [3])
  assert np.array_equal(_bits(out.view(-1)), _bits(x))
  assert torch.isnan(sr.stochastic_round(torch.tensor([[float("nan")]]), dtype, 1, [0])).all()


@pytest.mark.parametrize("dtype", HALF)
def test_result_is_a_neighbour_and_deterministic(dtype):
  torch.manual_seed(0)
  x = torch.randn(64, 32) * 3
  a = sr.stochastic_round(x, dtype, 5, torch.arange(64))
  b = sr.stochastic_round(x, dtype, 5, torch.arange(64))
  assert torch.equal(a.view(torch.int16), b.view(torch.int16))
  rn = x.to(dtype).float()
  af = a.float()
  # either the nearest value or the neighbour on the other side of x, never further away
  assert bool(((af == rn) | ((af - x) * (rn - x) < 0)).all())
  ulp = torch.maximum(af.abs(), rn.abs()) * (2.0**-7 if dtype == torch.bfloat16 else 2.0**-10)
  ulp = ulp.clamp(min=torch.finfo(dtype).smallest_normal * 2.0**-10)  # subnormal spacing
  assert bool(((af - x).abs() <= ulp).all())
  c = sr.stochastic_round(x, dtype, 6, torch.arange(64))
  assert not torch.equal(a.view(torch.int16), c.view(torch.int16)), "a new step draws new bits"


@pytest.mark.parametrize("dtype", HALF)
def test_mean_is_unbiased_where_round_to_nearest_is_not(dtype):
  base = torch.tensor(1.0, dtype=dtype).float()
  ulp = float(torch.nextafter(torch.tensor(1.0, dtype=dtype),
                              torch.tensor(2.0, dtype=dtype)).float() - 1.0) if dtype == \
      torch.float16 else 2.0**-7
  x = base + 0.1 * ulp  # a sub-half-ulp offset: round-to-nearest returns 1.0 every time
  n = 20000
  vals = sr.stochastic_round(torch.full((n, 1), float(x)), dtype, 3, torch.arange(n)).float()
  mean, se = float(vals.mean()), ulp * np.sqrt(0.1 * 0.9 / n)
  assert abs(mean - float(x)) < 5 * se, (mean, float(x), se)
  assert abs(float(torch.full((n,), float(x)).to(dtype).float().mean()) - float(x)) > 20 * se


def test_random_bits_match_the_documented_hash():
  # the fused kernels compute the same words (ops/csrc/common.cuh, sr_row_seed / sr_bits)
  def mix(h):
    h ^= h >> 16
    h = (h * 0x7FEB352D) & 0xFFFFFFFF
    h ^= h >> 15
    h = (h * 0x846CA68B) & 0xFFFFFFFF
    return h ^ (h >> 16)
  step, key, col = 12, (5 << 32) + 77, 9
  h = mix((step + 0x9E3779B9) & 0xFFFFFFFF)
  h = mix(h ^ (key & 0xFFFFFFFF))
  h = mix(h ^ (key >> 32))
  assert int(sr.random_bits(step, [key], [col])[0]) == mix(h ^ col)


# ----------------------------------------------------------------------------- plan interpreter
def run_half_plan(seed, world, kind, table_dtype, ragged=False):
  """One step of a random plan with half-precision tables against an fp32 unsharded model."""
  rng = random.Random(seed)
  nrng = np.random.default_rng(seed)
  n_tables = rng.randint(max(1, world // 2), 2 * world + 2)
  if kind == "rowwise_adagrad":
    n_tables = max(n_tables, world)
  sizes = [(rng.randint(3, 50), rng.choice([4, 8, 12, 16])) for _ in range(n_tables)]
  combiners = [rng.choice(["sum", "mean"]) for _ in sizes]
  imap = list(range(n_tables))
  hots = {t: rng.choice([1, 1, 2, 3]) for t in range(n_tables)}
  kw = {"strategy": rng.choice(["basic", "memory_balanced", "memory_optimized"]),
        "input_table_map": imap, "dp_input": True, "table_dtype": table_dtype}
  if rng.random() < 0.5 and kind != "rowwise_adagrad":
    kw["column_slice_threshold"] = rng.choice([40, 100, 250])
  plain = ragged or kind == "rowwise_adagrad"
  if world > 1 and rng.random() < 0.5 and not plain:
    kw["data_parallel_threshold"] = rng.choice([30, 80])
  if world > 1 and rng.random() < 0.5 and not plain:
    kw["row_slice_threshold"] = rng.choice([300, 500])
  embs = [{"input_dim": r, "output_dim": w, "combiner": c} for (r, w), c in zip(sizes, combiners)]
  try:
    sim, des = dry_run.build_engines(embs, world, **kw)
  except ValueError as e:
    if "Not enough table" in str(e):
      return "infeasible"
    raise
  # start from values every dtype stores exactly
  tables = [torch.from_numpy(nrng.standard_normal(s).astype(np.float32)).to(table_dtype).float()
            .numpy() for s in sizes]
  for de in des:
    de.set_weights(tables)
    if kind != "none":
      de.set_optimizer(kind, lr=0.5)
  lb = rng.choice([2, 3, 5])
  B = lb * world
  glob = [nrng.integers(0, sizes[t][0], size=(B, hots[t])) for t in imap]
  rag = [ragged and rng.random() < 0.6 for _ in imap]
  for i, t in enumerate(imap):
    if rag[i]:
      glob[i] = [list(nrng.integers(0, sizes[t][0], size=rng.randint(0, 4))) for _ in range(B)]
  if ragged:
    for de in des:
      de.ragged_capacity = 4

  def as_input(i, lo, hi):
    from distributed_embeddings_b200.ops.ragged import RaggedIds
    if rag[i]:
      rows = glob[i][lo:hi]
      return RaggedIds.from_row_lengths(
          torch.tensor([v for row in rows for v in row], dtype=torch.int64),
          torch.tensor([len(row) for row in rows], dtype=torch.int64))
    return torch.from_numpy(glob[i][lo:hi])

  widths = [sizes[t][1] for t in imap]
  grads = [nrng.standard_normal((B, w)).astype(np.float32) * 0.1 for w in widths]
  st = des[0].strategy
  dp_tables = set(st.table_groups[0])
  for de in des:
    for layer in de.dp_layers:
      assert layer.embeddings.dtype == torch.float32, "replicated tables stay fp32"
    for w in de.weights[len(de.dp_layers):]:
      assert w.dtype == table_dtype

  def rank_fn(r):
    de = des[r]
    out = de([as_input(i, r * lb, (r + 1) * lb) for i in range(len(imap))], concat=True)
    assert de._engine.ops.calls.get("lookup_fwd", 0) > 0
    gout = torch.from_numpy(np.concatenate([g[r * lb:(r + 1) * lb] for g in grads], 1))
    out.backward(gout)
    if kind == "none":
      from distributed_embeddings_b200.parallel.hybrid import SparseRowOptimizer
      mp = [p for p in de.mp_parameters() if p.grad is not None]
      for p in mp:
        assert p.grad.dtype == table_dtype
      SparseRowOptimizer(mp, "sgd", lr=0.5).step()
    return out.detach().float().numpy()

  outs = dry_run.run_ranks(sim, rank_fn)
  from test_dry_run import reference_step  # noqa: E402  pylint: disable=import-outside-toplevel
  ref = [t.copy() for t in tables]
  ref_outs = reference_step(ref, imap, glob, combiners, grads, 0.5, world,
                            "sgd" if kind == "none" else kind, {})
  for r, out in enumerate(outs):
    exp = np.concatenate([o[r * lb:(r + 1) * lb] for o in ref_outs], 1)
    np.testing.assert_allclose(out, exp, rtol=1e-5, atol=1e-5, err_msg=f"forward, rank {r}")
  got = des[0].get_weights() if world == 1 else dry_run.run_ranks(
      sim, lambda r: des[r].get_weights(all_ranks=True))[0]
  for t in range(n_tables):
    assert got[t].dtype == np.float32
    if t in dp_tables:
      np.testing.assert_array_equal(got[t], tables[t])  # replicated: untouched by the engine
      continue
    # one stochastic rounding per element: within one ulp of the fp32 result
    ulp = 2.0**-7 if table_dtype == torch.bfloat16 else 2.0**-10
    np.testing.assert_allclose(got[t], ref[t], rtol=2 * ulp, atol=1e-3,
                               err_msg=f"table {t} after the {kind} step")
  return "ok"


@pytest.fixture(autouse=True)
def _tests_on_path():
  sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
  yield
  sys.path.remove(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("kind", ["sgd", "adagrad", "rowwise_adagrad", "adam", "none"])
def test_random_plans_half_tables(world, kind, dtype):
  n = 3 if world < 8 else 2
  outcomes = [run_half_plan(11000 * world + 17 * s + len(kind), world, kind, dtype)
              for s in range(n)]
  assert outcomes.count("ok") >= 1, outcomes


@pytest.mark.parametrize("world", [1, 2, 4])
def test_random_plans_half_tables_ragged(world):
  outcomes = [run_half_plan(13000 * world + s, world, "adagrad", torch.bfloat16, ragged=True)
              for s in range(3)]
  assert outcomes.count("ok") >= 1, outcomes


def test_interpreter_catches_out_of_bounds_at_the_half_element_size():
  sim, des = dry_run.build_engines([{"input_dim": 10, "output_dim": 8, "combiner": "sum"}], 1,
                                   table_dtype=torch.bfloat16)
  de = des[0]
  de.set_optimizer("sgd", lr=0.1)
  ids = torch.tensor([[9]])
  de([ids], concat=True)
  eng = de._engine
  d = eng.fwd_main_np.copy()
  d[0]["sub_rows"] = 11  # one row past the table: 16 bytes in bf16
  blob = torch.from_numpy(np.frombuffer(d.tobytes(), dtype=np.uint8).copy())
  eng.ids_mp = None
  with pytest.raises(RuntimeError, match="outside any buffer"):
    eng.ops.lookup_fwd(blob, 1, 1, 1, 1, 8, [], [eng.out.data_ptr()], 0, True, 0, True, [], 32,
                       1, True)


@pytest.mark.parametrize("kind", ["sgd", "adagrad", "rowwise_adagrad", "adam"])
def test_dry_updates_leave_half_tables_bit_identical(kind):
  sim, des = dry_run.build_engines([{"input_dim": 30, "output_dim": 8, "combiner": "sum"},
                                    {"input_dim": 20, "output_dim": 16, "combiner": "mean"}], 1,
                                   table_dtype=torch.bfloat16)
  de = des[0]
  de.set_optimizer(kind, lr=0.5)
  ids = [torch.randint(0, 30, (6, 2)), torch.randint(0, 20, (6, 3))]
  de(ids, concat=True).sum().backward()  # one real step: state exists and is non-trivial
  before = [w.detach().clone() for w in de.weights]
  state = {m: [s.clone() for s in v] for m, v in de._engine.opt_state.items()}
  step = de._engine.step_count()
  de._engine.dry_updates(True)
  for _ in range(2):
    de(ids, concat=True).sum().backward()
  de._engine.dry_updates(False)
  for a, b in zip(before, de.weights):
    assert torch.equal(a.view(torch.int16), b.detach().view(torch.int16))
  for m, v in state.items():
    for a, b in zip(v, de._engine.opt_state[m]):
      assert torch.equal(a, b)
  assert de._engine.step_count() == step


def test_invalid_table_dtype_is_rejected():
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  with pytest.raises(ValueError, match="table_dtype"):
    DistributedEmbedding([{"input_dim": 4, "output_dim": 4}], device="cpu",
                         table_dtype=torch.float64)


# ----------------------------------------------------------------------------- checkpoints
def test_checkpoint_crosses_table_dtype_and_world_size(tmp_path):
  embs = [{"input_dim": 40, "output_dim": 8, "combiner": "sum"},
          {"input_dim": 25, "output_dim": 16, "combiner": "sum"},
          {"input_dim": 33, "output_dim": 4, "combiner": "sum"}]
  nrng = np.random.default_rng(0)
  w32 = [nrng.standard_normal((e["input_dim"], e["output_dim"])).astype(np.float32) for e in embs]
  # fp32 values load into bf16 tables as round-to-nearest
  sim2, des2 = dry_run.build_engines(embs, 2, table_dtype=torch.bfloat16,
                                     column_slice_threshold=200)
  dry_run.run_ranks(sim2, lambda r: des2[r].set_weights(w32, chunk=24))
  got = dry_run.run_ranks(sim2, lambda r: des2[r].get_weights(all_ranks=True))[0]
  for g, w in zip(got, w32):
    assert g.dtype == np.float32
    np.testing.assert_array_equal(g, torch.from_numpy(w).to(torch.bfloat16).float().numpy())
  # bf16 tables saved at W=2 (small chunks) load into fp32 tables at W=3 exactly
  dry_run.run_ranks(sim2, lambda r: des2[r].save_weights(str(tmp_path), chunk=24))
  sim3, des3 = dry_run.build_engines(embs, 3)
  dry_run.run_ranks(sim3, lambda r: des3[r].load_weights(str(tmp_path), chunk=24))
  got3 = dry_run.run_ranks(sim3, lambda r: des3[r].get_weights(all_ranks=True))[0]
  for a, b in zip(got, got3):
    np.testing.assert_array_equal(a, b)


class _Fp32Sizes(torch.overrides.TorchFunctionMode):
  """Records the size of every fp32 tensor a torch call produces."""

  def __init__(self):
    super().__init__()
    self.sizes = []

  def __torch_function__(self, func, types, args=(), kwargs=None):
    out = func(*args, **(kwargs or {}))
    for t in out if isinstance(out, (tuple, list)) else (out,):
      if isinstance(t, torch.Tensor) and t.dtype == torch.float32:
        self.sizes.append(t.numel())
    return out


def test_checkpoint_chunks_bound_every_fp32_staging_buffer(tmp_path):
  """set / get / save / load of bf16 tables go through fp32 chunks of at most ``chunk``
  elements: no fp32 copy of a whole table is ever made."""
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  embs = [{"input_dim": 400, "output_dim": 16, "combiner": "sum"},
          {"input_dim": 300, "output_dim": 8, "combiner": "sum"}]
  de = DistributedEmbedding(embs, device="cpu", backend="torch", table_dtype=torch.bfloat16)
  w32 = [np.random.default_rng(i).standard_normal((e["input_dim"], e["output_dim"]))
         .astype(np.float32) for i, e in enumerate(embs)]
  chunk = 256  # 16 rows of the first table, 1/25 of it
  with _Fp32Sizes() as mode:
    de.set_weights(w32, chunk=chunk)
    got = de.get_weights(chunk=chunk)
    de.save_weights(str(tmp_path), chunk=chunk)
    de.load_weights(str(tmp_path), chunk=chunk)
  assert mode.sizes, "no fp32 staging observed"
  assert max(mode.sizes) <= chunk, max(mode.sizes)
  for g, w in zip(got, w32):
    np.testing.assert_array_equal(g, torch.from_numpy(w).to(torch.bfloat16).float().numpy())


def test_offloaded_half_table_pools_in_fp32_in_the_torch_back_end():
  from distributed_embeddings_b200.layers.embedding import _embedding_lookup_native
  from distributed_embeddings_b200.ops.ragged import RaggedIds
  torch.manual_seed(3)
  w = (torch.randn(60, 8) * 100).to(torch.bfloat16)
  ids = torch.randint(0, 60, (5, 40))
  for comb in ("sum", "mean"):
    ref = w.float()[ids].sum(1) / (40 if comb == "mean" else 1)
    out = _embedding_lookup_native(w, ids, comb)
    assert out.dtype == torch.bfloat16
    assert torch.equal(out, ref.to(torch.bfloat16))  # one rounding of the fp32 pool
  rag = RaggedIds.from_row_lengths(ids.reshape(-1)[:30], torch.tensor([10, 0, 20]))
  ref = torch.stack([w.float()[ids.reshape(-1)[:10]].sum(0), torch.zeros(8),
                     w.float()[ids.reshape(-1)[10:30]].sum(0)])
  assert torch.equal(_embedding_lookup_native(w, rag, "sum"), ref.to(torch.bfloat16))


# ----------------------------------------------------------------------------- single layer (CPU)
@pytest.mark.parametrize("dtype", HALF)
def test_single_layer_cpu_pools_in_fp32(dtype):
  from distributed_embeddings_b200.layers.embedding import Embedding
  layer = Embedding(50, 12, combiner="sum", dtype=dtype)
  ids = torch.randint(0, 50, (7, 30))
  out = layer(ids).detach()
  assert out.dtype == dtype
  ref = layer.embeddings.detach().float()[ids].sum(1)
  ulp = 2.0**-7 if dtype == torch.bfloat16 else 2.0**-10
  np.testing.assert_allclose(out.float().numpy(), ref.numpy(), rtol=ulp, atol=1e-6)


# ----------------------------------------------------------------------------- tools / examples
def test_plan_report_table_dtype_fits_mlperf_on_one_gpu():
  def run(extra):
    return subprocess.run([sys.executable, "tools/plan_report.py", "--model", "dlrm-mlperf",
                           "--world", "1"] + extra, cwd=ROOT, capture_output=True, text=True,
                          check=True).stdout
  assert "GiB!" not in run(["--table-dtype", "bf16"])
  assert "GiB!" in run([])


def test_dlrm_example_learns_with_bf16_tables(tmp_path):
  data = str(tmp_path / "criteo")
  env = dict(os.environ, PYTHONPATH=ROOT, CUDA_VISIBLE_DEVICES="")
  subprocess.run([sys.executable, "tools/make_synthetic_criteo.py", data, "--train", "16384",
                  "--test", "4096", "--table_sizes", "5,300,7000,40,900,60,15,2000"], cwd=ROOT,
                 env=env, check=True, capture_output=True)
  out = subprocess.run([sys.executable, "examples/dlrm/main.py", "--dataset_path", data,
                        "--batch_size", "256", "--embedding_dim", "16", "--bottom_mlp_dims",
                        "32,16", "--top_mlp_dims", "64,32,1", "--learning_rate", "2.0",
                        "--warmup_steps", "20", "--decay_start_step", "100000", "--epochs", "3",
                        "--save_path", str(tmp_path / "w"), "--table_dtype", "bf16"],
                       cwd=ROOT, env=env, check=True, capture_output=True, text=True, timeout=900)
  auc = float(out.stdout.split("AUC:")[1].split(",")[0])
  assert auc > 0.7, out.stdout[-500:]


# ----------------------------------------------------------------------------- GPU (one H100)
def _cuda():
  return torch.device("cuda", 0)


def _de(embs, dtype, **kw):
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  return DistributedEmbedding(embs, device=_cuda(), backend="fused", table_dtype=dtype, **kw)


# width classes of the fused forward: every width / column a multiple of 8 (16-bit rows read 8
# columns per lane, 16-byte loads), of 4 but not all of 8 (8-byte loads), and not all of 4 (one
# column per lane).  The engine picks one path per launch, so each class gets its own layer.
WIDTH_CLASSES = {"vec8": [128, 64, 16], "vec4": [12, 20, 36], "scalar": [6, 10, 8]}


def _assert_path(de, cls):
  eng = de._engine
  assert eng.vec4 == (cls != "scalar"), (cls, eng.vec4)
  assert eng.fwd_vec8 == (cls == "vec8"), (cls, eng.fwd_vec8)


@pytest.mark.gpu
@pytest.mark.parametrize("cls", sorted(WIDTH_CLASSES))
@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("ids64", [False, True])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_gpu_one_hot_lookup_returns_stored_rows(cls, dtype, ids64, out_dtype):
  torch.manual_seed(0)
  widths = WIDTH_CLASSES[cls]
  de = _de([{"input_dim": 1000, "output_dim": w, "combiner": None} for w in widths], dtype,
           compute_dtype=out_dtype)
  idt = torch.int64 if ids64 else torch.int32
  ids = [torch.randint(0, 1000, (512,), device=_cuda(), dtype=idt) for _ in widths]
  outs = de(ids)
  _assert_path(de, cls)
  for w, i, o in zip(de.get_weights(), ids, outs):  # global tables, upcast exactly to fp32
    assert o.dtype == out_dtype
    # the stored value, converted to the output dtype once (exact unless fp16 -> bf16)
    exp = torch.from_numpy(w).to(_cuda())[i.long()].to(out_dtype)
    assert torch.equal(o, exp)


@pytest.mark.gpu
@pytest.mark.parametrize("cls", sorted(WIDTH_CLASSES))
@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("ids64", [False, True])
def test_gpu_multi_hot_pooling_matches_fp32_reference(cls, dtype, ids64):
  torch.manual_seed(1)
  widths = WIDTH_CLASSES[cls]
  embs = [{"input_dim": 700, "output_dim": w, "combiner": c}
          for w, c in zip(widths, ["sum", "mean", "sum"])]
  embs.append({"input_dim": 5000, "output_dim": widths[0], "combiner": "mean"})  # offloaded
  de = _de(embs, dtype, compute_dtype=torch.float32,
           gpu_embedding_size=700 * sum(widths) + 1)
  assert any(getattr(l, "cpu_offloaded", False) for l in de.local_embedding_layers)
  idt = torch.int64 if ids64 else torch.int32
  ids = [torch.randint(0, e["input_dim"], (300, 7), device=_cuda(), dtype=idt) for e in embs]
  outs = de(ids)
  _assert_path(de, cls)
  for w, e, i, o in zip(de.get_weights(), embs, ids, outs):
    ref = torch.from_numpy(w).to(_cuda())[i.long()].sum(1)  # fp32 pooling of the stored rows
    if e["combiner"] == "mean":
      ref = ref / 7
    torch.testing.assert_close(o, ref, rtol=1e-5, atol=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("width", [128, 12, 6])  # 16-byte, 8-byte and 2-byte row loads
@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("ids64", [False, True])
def test_gpu_single_layer_op(width, dtype, ids64):
  from distributed_embeddings_b200.layers.embedding import Embedding
  torch.manual_seed(2)
  idt = torch.int64 if ids64 else torch.int32
  one = Embedding(900, width, combiner=None, dtype=dtype, device=_cuda())
  ids = torch.randint(0, 900, (333, 1), device=_cuda(), dtype=idt)
  out = one(ids).detach()
  assert out.dtype == dtype
  assert torch.equal(out.view(torch.int16), one.embeddings.detach()[ids.long()].view(torch.int16))
  pooled = Embedding(900, width, combiner="sum", dtype=dtype, device=_cuda())
  ids = torch.randint(0, 900, (333, 9), device=_cuda(), dtype=idt)
  out = pooled(ids).detach()
  assert out.dtype == dtype
  ref = pooled.embeddings.detach().float()[ids.long()].sum(1)  # fp32 pooling, one rounding
  ulp = 2.0**-7 if dtype == torch.bfloat16 else 2.0**-10
  torch.testing.assert_close(out.float(), ref, rtol=ulp, atol=1e-6)


def _sgd_bit_exact(dtype, width):
  rows, n = 4096, 1024
  de = _de([{"input_dim": rows, "output_dim": width, "combiner": None}], dtype,
           compute_dtype=torch.float32)
  de.set_optimizer("sgd", lr=0.5)
  g = torch.Generator().manual_seed(width)
  # weights on a coarse grid, gradients of few significant bits: w - lr * g is exact in fp32
  w0 = (torch.randint(-64, 64, (rows, width), generator=g).float() / 64).to(dtype)
  de.set_weights([w0.float().numpy()])
  ids = torch.randperm(rows, generator=g)[:n]
  grad = torch.randint(-512, 512, (n, width), generator=g).float() * 2.0**-17
  out = de([ids.to(_cuda())], concat=True)
  out.backward(grad.to(_cuda()))
  torch.cuda.synchronize()
  exact = w0.float().clone()
  exact[ids] = exact[ids] - 0.5 * grad
  expect = sr.stochastic_round(exact, dtype, 1, torch.arange(rows))
  got = de.weights[0].detach().cpu()
  assert torch.equal(got.view(torch.int16), expect.view(torch.int16))
  assert not torch.equal(got.view(torch.int16), w0.view(torch.int16))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("width", [64, 192])  # balanced kernel (<= 128) / per-row kernel
def test_gpu_fused_update_matches_python_rounding_bit_for_bit(dtype, width):
  _sgd_bit_exact(dtype, width)


@pytest.mark.gpu
def test_gpu_sub_ulp_updates_move_the_mean():
  rows, width, steps = 64, 128, 200
  de = _de([{"input_dim": rows, "output_dim": width, "combiner": None}], torch.bfloat16,
           compute_dtype=torch.float32)
  de.set_optimizer("sgd", lr=1.0)
  de.set_weights([np.ones((rows, width), dtype=np.float32)])
  ids = torch.arange(rows, device=_cuda())
  step = 0.1 * 2.0**-7  # 0.1 ulp of bf16 at 1.0 per step (fp32 oracle: exact linear drift)
  for _ in range(steps):
    de([ids], concat=True).backward(torch.full((rows, width), -step, device=_cuda()))
  torch.cuda.synchronize()
  w = de.weights[0].detach().float()
  expect = 1.0 + steps * step
  se = 2.0**-7 * np.sqrt(steps * 0.25) / np.sqrt(rows * width)
  assert abs(float(w.mean()) - expect) < 5 * se + 1e-6, (float(w.mean()), expect, se)
  assert float(w.mean()) > 1.0 + 0.5 * steps * step, "the table froze"


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sgd", "adagrad", "rowwise_adagrad", "adam"])
def test_gpu_optimizers_match_torch_backend(kind):
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  from distributed_embeddings_b200.parallel.hybrid import SparseRowOptimizer
  torch.manual_seed(4)
  embs = [{"input_dim": 500, "output_dim": 64, "combiner": "sum"},
          {"input_dim": 300, "output_dim": 16, "combiner": "mean"}]
  w0 = [(np.random.default_rng(i).standard_normal((e["input_dim"], e["output_dim"])) * 0.1)
        .astype(np.float32) for i, e in enumerate(embs)]
  fused = _de(embs, torch.bfloat16, compute_dtype=torch.float32)
  fused.set_weights(w0)
  fused.set_optimizer(kind, lr=0.05)
  ref = DistributedEmbedding(embs, device=_cuda(), backend="torch", table_dtype=torch.bfloat16,
                             compute_dtype=torch.float32)
  ref.set_weights(w0)
  opt = SparseRowOptimizer(ref.mp_parameters(), kind, lr=0.05)
  for _ in range(3):
    ids = [torch.randint(0, e["input_dim"], (256, 3), device=_cuda()) for e in embs]
    gout = torch.randn(256, 80, device=_cuda())
    fused(ids, concat=True).backward(gout)
    ref(ids, concat=True).backward(gout)
    opt.step()
  torch.cuda.synchronize()
  for a, b in zip(fused.get_weights(), ref.get_weights()):
    if kind != "adam":
      np.testing.assert_allclose(a, b, rtol=2 * 2.0**-7, atol=2e-3)
      continue
    # Adam divides by sqrt(v): where a gradient element is near zero, the torch back end's bf16
    # sparse gradient (autograd casts it to the table dtype) and the fused fp32 segment sum can
    # give that element a different sign, moving the weight by up to ~lr per step in opposite
    # directions.  Those elements are rare; all others agree at the same tolerance.
    bad = ~np.isclose(a, b, rtol=2 * 2.0**-7, atol=2e-3)
    assert bad.mean() < 2e-3, bad.mean()
    assert np.abs(a - b).max() <= 3 * 3 * 0.05


def _dlrm_pair(table_dtype):
  from distributed_embeddings_b200.models.dlrm import DLRM
  sizes = [200 + 13 * i for i in range(26)]
  torch.manual_seed(7)
  half = DLRM(sizes, device=_cuda(), compute_dtype=torch.bfloat16, backend="fused",
              table_dtype=table_dtype)
  torch.manual_seed(7)
  ref = DLRM(sizes, device=_cuda(), compute_dtype=torch.bfloat16, backend="fused")
  ref.load_state_dict({k: v for k, v in half.state_dict().items() if "embedding" not in k},
                      strict=False)
  ref.embedding.set_weights(half.embedding.get_weights())  # fp32 copy of the half tables
  return sizes, half, ref


def _dlrm_oracle(model, tables, batches, lr):
  """Plain PyTorch, fp32 throughout: SGD on the global batch with fp32 copies of the tables and
  dense weights (indexing, bmm interaction, F.linear, BCE with logits, autograd)."""
  F = torch.nn.functional
  lins = [m for m in list(model.bottom_mlp.net) + list(model.top_mlp.net)
          if isinstance(m, torch.nn.Linear)]
  n_bottom = sum(isinstance(m, torch.nn.Linear) for m in model.bottom_mlp.net)
  dense = [(l.weight.detach().float().clone().requires_grad_(True),
            l.bias.detach().float().clone().requires_grad_(True)) for l in lins]
  tabs = [torch.from_numpy(t).to(_cuda()).requires_grad_(True) for t in tables]
  params = tabs + [x for wb in dense for x in wb]
  n = len(tabs) + 1
  ii, jj = torch.tril_indices(n, n, offset=-1, device=_cuda())
  losses = []
  for num, cat, lab in batches:
    x = num
    for w, bias in dense[:n_bottom]:
      x = torch.relu(F.linear(x, w, bias))
    feats = torch.stack([x] + [tabs[t][cat[t].long()] for t in range(len(tabs))], dim=1)
    h = torch.cat([torch.bmm(feats, feats.transpose(1, 2))[:, ii, jj], x], dim=1)
    top = dense[n_bottom:]
    for i, (w, bias) in enumerate(top):
      h = F.linear(h, w, bias)
      if i < len(top) - 1:
        h = torch.relu(h)
    loss = F.binary_cross_entropy_with_logits(h.reshape(-1), lab)
    losses.append(float(loss.detach()))
    grads = torch.autograd.grad(loss, params)
    with torch.no_grad():
      for p_, g_ in zip(params, grads):
        p_ -= lr * g_
  return [t.detach().cpu().numpy() for t in tabs], losses


@pytest.mark.gpu
def test_gpu_dlrm_train_step_with_bf16_tables():
  """DLRMTrainStep (CUDA graph) on bf16 tables against the plain-PyTorch fp32 oracle run on an
  upcast copy of the same tables.  The trainer computes the dense side in bf16 and rounds the
  tables stochastically, so the check is the one bench.py's verify uses: the aggregate error of
  the table update relative to the update itself, and the per-step loss."""
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  sizes = [200 + 13 * i for i in range(26)]
  torch.manual_seed(7)
  model = DLRM(sizes, device=_cuda(), compute_dtype=torch.bfloat16, backend="fused",
               table_dtype=torch.bfloat16)
  # small initial values, so that one bf16 ulp of a table element (~1e-7 here) is far below the
  # per-step update (~1e-5): the stochastic rounding then adds a few percent of noise to the
  # update instead of hiding it, and a misrouted or mis-scaled update shows as an error of the
  # order of the update itself
  model.embedding.set_weights([w * 1e-3 for w in model.embedding.get_weights()])
  w0 = model.embedding.get_weights()  # the stored bf16 values, upcast exactly
  lr = 4.0
  g = torch.Generator().manual_seed(3)
  batches = []
  for _ in range(3):
    batches.append((torch.rand(512, 13, generator=g).to(_cuda()),
                    torch.stack([torch.randint(0, s, (512,), generator=g, dtype=torch.int32)
                                 for s in sizes]).to(_cuda()),
                    torch.randint(0, 2, (512,), generator=g).float().to(_cuda())))
  ref_tabs, ref_losses = _dlrm_oracle(model, w0, batches, lr)
  trainer = DLRMTrainStep(model, lr=lr, embedding_optimizer="sgd", use_cuda_graph=True)
  losses = [float(trainer.step(*b)) for b in batches]
  torch.cuda.synchronize()
  got = model.embedding.get_weights()
  for w in model.embedding.weights:
    assert w.dtype == torch.bfloat16
  sq_err = sum(float(((a.astype(np.float64) - b)**2).sum()) for a, b in zip(got, ref_tabs))
  sq_upd = sum(float(((b.astype(np.float64) - c)**2).sum()) for b, c in zip(ref_tabs, w0))
  rel = (sq_err / sq_upd)**0.5
  assert sq_upd > 0 and rel <= 0.3, (rel, sq_upd)
  assert max(abs(a - b) for a, b in zip(losses, ref_losses)) <= 3e-2, (losses, ref_losses)


@pytest.mark.gpu
def test_gpu_dlrm_graph_warmup_leaves_bf16_tables_untouched():
  """The passes DLRMTrainStep runs before capturing its graph (zero lr, dry updates)."""
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  sizes, half, _ = _dlrm_pair(torch.bfloat16)
  t = DLRMTrainStep(half, lr=0.5, embedding_optimizer="sgd", use_cuda_graph=True)
  before = [w.detach().clone() for w in half.embedding.weights]
  num = torch.rand(512, 13, device=_cuda())
  cat = torch.stack([torch.randint(0, s, (512,), device=_cuda(), dtype=torch.int32)
                     for s in sizes])
  lab = torch.randint(0, 2, (512,), device=_cuda()).float()
  t.load_batch(num, cat, lab)
  t.lr_t.zero_()
  t.engine.dry_updates(True)
  for _ in range(2):
    t._step_impl()
  t.engine.dry_updates(False)
  torch.cuda.synchronize()
  for a, w in zip(before, half.embedding.weights):
    assert torch.equal(a.view(torch.int16), w.detach().view(torch.int16))


@pytest.mark.gpu
def test_gpu_synthetic_train_step_bf16_tables_adagrad():
  from distributed_embeddings_b200.models.configs import expand, scaled, synthetic_models_v3
  from distributed_embeddings_b200.models.synthetic import SyntheticModel
  from distributed_embeddings_b200.models.synthetic_fast import SyntheticTrainStep
  cfg = scaled(synthetic_models_v3["tiny"], 2e-4)
  tables, imap, hots = expand(cfg)[:3]
  torch.manual_seed(5)
  m = SyntheticModel(cfg, dp_input=True, device=_cuda(), compute_dtype=torch.bfloat16,
                     backend="fused", table_dtype=torch.bfloat16)
  torch.manual_seed(5)
  r = SyntheticModel(cfg, dp_input=True, device=_cuda(), compute_dtype=torch.bfloat16,
                     backend="fused")
  r.load_state_dict({k: v for k, v in m.state_dict().items() if "embedding" not in k},
                    strict=False)
  r.embedding.set_weights(m.embedding.get_weights())
  tm = SyntheticTrainStep(m, lr=0.01, embedding_optimizer="adagrad", use_cuda_graph=True)
  tr = SyntheticTrainStep(r, lr=0.01, embedding_optimizer="adagrad", use_cuda_graph=False)
  g = torch.Generator().manual_seed(4)
  for _ in range(3):
    num = (torch.rand(128, cfg.num_numerical_features, generator=g) * 2).to(_cuda())
    ids = [torch.randint(0, tables[t][0], (128, h), generator=g).to(_cuda())
           for t, h in zip(imap, hots)]
    lab = torch.randint(0, 2, (128, 1), generator=g).float().to(_cuda())
    lm = tm.step(num, ids, lab).clone()
    lr_ = tr.step(num, ids, lab).clone()
    torch.testing.assert_close(lm, lr_, rtol=2e-2, atol=2e-3)
  for a, b in zip(m.embedding.get_weights(), r.embedding.get_weights()):
    np.testing.assert_allclose(a, b, rtol=4 * 2.0**-7, atol=2e-3)
