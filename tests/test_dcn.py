"""DLRM-DCNv2: the low-rank cross network and multi-hot features, from the module to the
hand-scheduled step.

CPU:
- The ``dcnv2`` module's forward (multi-hot, h = 1 and h > 1) equals a float64 formula on the
  same weights; with the default arguments the model is today's (same parameters, same keys).
- ``HybridTrainer`` on the ``dcnv2`` model at gloo world 2 equals one process on the global
  batch; the dense-optimizer checkpoint round trip covers the cross parameters.
- The DLRM example with ``--interaction dcnv2`` learns the generated dataset (AUC > 0.7).
- Self-check of the kernel bounds used on the GPU: the float64 model of each kernel, rounded the
  way the kernel rounds, passes; a model of each plausible defect (missing ``+ xl``, ``dy * s``
  in place of ``dy * x0``, a dropped layer term in ``dx0``, the bias sum over the wrong axis)
  fails.

GPU (one H100):
- ``cross_fwd`` / ``cross_bwd`` / ``cross_dx0`` against float64 at rounding-level bounds, D in
  {8, 136, 3456}, rows in {1, 3, 777, 65536}, L in {1, 3}; argument checks raise before launch.
- ``DLRMTrainStep`` on the ``dcnv2`` model against ``HybridTrainer`` on a copy (loss, relative
  error of the dense and table updates), eager and graph, embedding sgd / adagrad /
  rowwise_adagrad, dense sgd / adam, hotness mixes with 1 and 100, fp32 and bf16 tables.
- ``prefetch`` / ``run_prefetched`` equal ``step``; ``evaluate`` / ``predict`` equal the sigmoid
  of the module forward, with a padded last chunk.
- World 2 (skips on fewer GPUs): the step against ``HybridTrainer``.

The multi-rank cases run one spawned process per rank (launcher at the end of this file).
"""
import os
import socket
import subprocess
import sys
import traceback

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U16 = 2.0**-8   # bf16 unit roundoff
U32 = 2.0**-24  # fp32 unit roundoff
TINY = 1e-30


# ------------------------------------------------------------------ float64 models + bounds
def ratio(got, ref, bound):
  """max |got - ref| / bound (inf on non-finite output)."""
  got = got.double()
  if not torch.isfinite(got).all():
    return float("inf")
  return float(((got - ref).abs() / bound).max()) if ref.numel() else 0.0


def fwd_ratio(x0, s, xl, out):
  """out = bf16(x0 * s + xl) with one fp32 fma: one bf16 rounding plus one fp32 rounding."""
  x0, s, xl = x0.double(), s.double(), xl.double()
  ref = x0 * s + xl
  bound = U16 * ref.abs() + U32 * ((x0 * s).abs() + xl.abs()) + TINY
  return ratio(out, ref, bound)


def bwd_ratio(dy, x0, g, db):
  """g = bf16(dy * x0) (the product is exact in fp32); db = column sums in fp32, summed along
  chains of at most rows / 16 + 300 additions (per-thread runs, the block reduction, one atomic
  per block)."""
  p = dy.double() * x0.double()
  rows = p.shape[0]
  rg = ratio(g, p, U16 * p.abs() + TINY)
  ref = p.sum(0)
  depth = rows / 16 + 300
  rb = ratio(db, ref, depth * U32 * p.abs().sum(0) + TINY)
  return max(rg, rb)


def dx0_ratio(d_chain, dys, ss, dx0, d_bottom):
  """d_chain + sum_l dy_l * s_l: L fp32 fmas, one bf16 rounding; embedding columns in dx0, the
  bottom columns in d_bottom."""
  ref = d_chain.double()
  mag = ref.abs()
  for dy, s in zip(dys, ss):
    t = dy.double() * s.double()
    ref = ref + t
    mag = mag + t.abs()
  bound = U16 * ref.abs() + (len(dys) + 1) * U32 * mag + TINY
  e = ref.shape[1] - d_bottom.shape[1]
  got = torch.cat([dx0[:, :e].double(), d_bottom.double()], dim=1)
  return ratio(got, ref, bound)


def _rand(shape, gen, scale=1.0):
  return (torch.randn(*shape, generator=gen) * scale).bfloat16()


def _rounded_fwd(x0, s, xl):
  return torch.addcmul(xl.float(), x0.float(), s.float()).bfloat16()


def _rounded_bwd(dy, x0):
  p = dy.float() * x0.float()
  return p.bfloat16(), p.double().sum(0).float()


def _rounded_dx0(d_chain, dys, ss, nb):
  acc = d_chain.double()
  for dy, s in zip(dys, ss):
    acc = acc + dy.double() * s.double()
  out = acc.float().bfloat16()
  return out, out[:, out.shape[1] - nb:].contiguous()


@pytest.mark.parametrize("defect", ["missing_xl", "dy_times_s", "dropped_layer", "bias_axis"])
def test_bounds_catch_defects(defect):
  gen = torch.Generator().manual_seed(4)
  rows, D, nb = 777, 136, 128
  x0, s, xl, dy = (_rand((rows, D), gen) for _ in range(4))
  # the exactly rounded results pass every bound
  assert fwd_ratio(x0, s, xl, _rounded_fwd(x0, s, xl)) <= 1.0
  assert bwd_ratio(dy, x0, *_rounded_bwd(dy, x0)) <= 1.0
  dys = [_rand((rows, D), gen) for _ in range(3)]
  ss = [_rand((rows, D), gen) for _ in range(3)]
  assert dx0_ratio(xl, dys, ss, *_rounded_dx0(xl, dys, ss, nb)) <= 1.0
  if defect == "missing_xl":
    assert fwd_ratio(x0, s, xl, (x0.float() * s.float()).bfloat16()) > 1.0
  elif defect == "dy_times_s":
    assert bwd_ratio(dy, x0, *_rounded_bwd(dy, s)) > 1.0
  elif defect == "dropped_layer":
    out, bottom = _rounded_dx0(xl, dys[:-1], ss[:-1], nb)
    assert dx0_ratio(xl, dys, ss, out, bottom) > 1.0
  else:
    g, _ = _rounded_bwd(dy, x0)
    rowsum = (dy.double() * x0.double()).sum(1)[:D].float()
    assert bwd_ratio(dy, x0, g, rowsum) > 1.0


# ------------------------------------------------------------------ module (CPU)
def _small(seed, interaction="dcnv2", hots=None, device="cpu", dtype=torch.float32, **kw):
  from distributed_embeddings_b200.models.dlrm import DLRM
  torch.manual_seed(seed)
  sizes = kw.pop("sizes", [20 + 3 * i for i in range(4)])
  return DLRM(sizes, embedding_dim=8, bottom_mlp_dims=(16, 8), top_mlp_dims=(16, 1),
              compute_dtype=dtype, device=device, backend=kw.pop("backend", "torch"),
              interaction=interaction, dcn_num_layers=kw.pop("layers", 2),
              dcn_low_rank_dim=kw.pop("rank", 8), multi_hot_sizes=hots, **kw)


def _batch(sizes, hots, b, seed, device="cpu"):
  g = torch.Generator().manual_seed(seed)
  num = torch.rand(b, 13, generator=g).to(device)
  cat = [torch.randint(0, s, (b, h), generator=g).to(device) for s, h in zip(sizes, hots)]
  lab = torch.randint(0, 2, (b, 1), generator=g).float().to(device)
  return num, cat, lab


def test_module_forward_matches_float64_formula():
  sizes, hots = [20 + 3 * i for i in range(4)], [1, 3, 1, 5]
  m = _small(0, hots=hots)
  num, cat, _ = _batch(sizes, hots, 9, 1)
  got = m(num, cat).double()
  f64 = lambda t: t.detach().double()
  relu = torch.relu

  def mlp(x, net, last_relu):
    lins = [l for l in net if isinstance(l, torch.nn.Linear)]
    for i, l in enumerate(lins):
      x = x @ f64(l.weight).t() + f64(l.bias)
      if i < len(lins) - 1 or last_relu:
        x = relu(x)
    return x

  bottom = mlp(num.double(), m.bottom_mlp.net, True)
  tables = [torch.as_tensor(w).double() for w in m.embedding.get_weights()]
  emb = [t[c].sum(1) for t, c in zip(tables, cat)]  # sum over the h ids of each sample
  x0 = torch.cat(emb + [bottom], dim=1)
  assert x0.shape[1] == m.cross_dim == 5 * 8
  x = x0
  for layer in m.cross_layers:
    s = (x @ f64(layer.V.weight).t()) @ f64(layer.W.weight).t() + f64(layer.W.bias)
    x = x0 * s + x
  ref = mlp(x, m.top_mlp.net, False)
  torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-6)
  assert all(layer.V.bias is None for layer in m.cross_layers)
  assert all(torch.equal(layer.W.bias, torch.zeros_like(layer.W.bias)) for layer in m.cross_layers)
  # the dot model takes the same multi-hot inputs
  d = _small(0, interaction="dot", hots=hots)
  assert d(num, cat).shape == (9, 1)


def test_default_model_is_unchanged():
  from distributed_embeddings_b200.models.dlrm import DLRM
  torch.manual_seed(3)
  a = DLRM([30, 40, 50], embedding_dim=8, bottom_mlp_dims=(16, 8), top_mlp_dims=(16, 1),
           backend="torch")
  keys = list(a.state_dict().keys())
  mlp = lambda pre, n: [f"{pre}.net.{2 * i}.{k}" for i in range(n) for k in ("weight", "bias")]
  assert [k for k in keys if "embedding" not in k] == mlp("bottom_mlp", 2) + mlp("top_mlp", 2)
  assert not any("cross" in n for n, _ in a.named_parameters())
  assert a.top_mlp.net[0].in_features == 6 + 8 and hasattr(a, "tril")
  torch.manual_seed(3)
  b = DLRM([30, 40, 50], embedding_dim=8, bottom_mlp_dims=(16, 8), top_mlp_dims=(16, 1),
           backend="torch", interaction="dot", dcn_num_layers=5, dcn_low_rank_dim=7,
           multi_hot_sizes=None)
  for (n, p), (m, q) in zip(a.named_parameters(), b.named_parameters()):
    assert n == m and torch.equal(p, q)


def test_module_rejects_bad_arguments():
  with pytest.raises(ValueError, match="interaction"):
    _small(0, interaction="cat")
  with pytest.raises(ValueError, match="multi_hot_sizes"):
    _small(0, hots=[1, 2])


def test_hybrid_gloo_world2_matches_single_process():
  _launch("case_dcnv2_hybrid_world", world=2)


@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_hybrid_checkpoint_round_trip_covers_cross(kind):
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  sizes, hots = [20 + 3 * i for i in range(4)], [2, 1, 4, 1]
  batches = [_batch(sizes, hots, 32, 200 + i) for i in range(5)]
  a = _small(1, hots=hots)
  ta = HybridTrainer(a, lr=0.01, embedding_optimizer="sgd", dense_optimizer=kind)
  for bt in batches:
    ta.step(*bt)
  b = _small(1, hots=hots)
  tb = HybridTrainer(b, lr=0.01, embedding_optimizer="sgd", dense_optimizer=kind)
  for bt in batches[:3]:
    tb.step(*bt)
  saved = tb.dense_optimizer_state()
  assert {"cross_layers.0.V.weight", "cross_layers.1.W.weight",
          "cross_layers.1.W.bias"} <= set(saved["slots"])
  weights = {k: v.clone() for k, v in b.state_dict().items()}
  tables = b.embedding.get_weights()
  c = _small(2, hots=hots)
  c.load_state_dict(weights)
  c.embedding.set_weights(tables)
  tc = HybridTrainer(c, lr=0.01, embedding_optimizer="sgd", dense_optimizer=kind)
  tc.load_dense_optimizer_state(saved)
  for bt in batches[3:]:
    tc.step(*bt)
  for (n, p), q in zip(a.named_parameters(), c.parameters()):
    assert torch.equal(p, q), n


def test_dlrm_example_dcnv2_learns(tmp_path):
  env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
  data = str(tmp_path / "criteo")

  def run(args):
    out = subprocess.run([sys.executable] + args, cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=900, check=False)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    return out.stdout

  run(["tools/make_synthetic_criteo.py", data, "--train", "16384", "--test", "4096",
       "--table_sizes", "5,300,7000,40,900,60,15,2000"])
  out = run(["examples/dlrm/main.py", "--dataset_path", data, "--batch_size", "256",
             "--embedding_dim", "16", "--bottom_mlp_dims", "32,16", "--top_mlp_dims", "64,32,1",
             "--interaction", "dcnv2", "--dcn_num_layers", "2", "--dcn_low_rank_dim", "32",
             "--learning_rate", "2.0", "--warmup_steps", "20", "--decay_start_step", "100000",
             "--epochs", "3", "--save_path", str(tmp_path / "w")])
  auc = float(out.split("AUC:")[1].split(",")[0])
  assert auc > 0.7, out[-500:]


def test_dlrm_example_dcnv2_multi_hot_synthetic(tmp_path):
  env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
  out = subprocess.run([sys.executable, "examples/dlrm/main.py", "--batch_size", "32",
                        "--num_batches", "2", "--table_sizes", "50,60,70", "--embedding_dim", "8",
                        "--bottom_mlp_dims", "16,8", "--top_mlp_dims", "16,1", "--interaction",
                        "dcnv2", "--dcn_low_rank_dim", "16", "--multi_hot_sizes", "1,3,7",
                        "--save_path", str(tmp_path / "w")], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600, check=False)
  assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
  assert "Evaluation completed" in out.stdout


# ------------------------------------------------------------------ GPU: kernels
def _ops():
  from distributed_embeddings_b200.ops import _native
  return _native.require()


DS = [8, 136, 3456]
ROWS = [1, 3, 777, 65536]


@pytest.mark.gpu
@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("rows", ROWS)
def test_cross_fwd_kernel(D, rows):
  ops, dev = _ops(), torch.device("cuda", 0)
  gen = torch.Generator().manual_seed(D + rows)
  x0, s, xl = (_rand((rows, D), gen).to(dev) for _ in range(3))
  out = torch.full_like(x0, float("nan"))
  ops.cross_fwd(x0, s, xl, out)
  assert fwd_ratio(x0, s, xl, out) <= 1.0
  ops.cross_fwd(x0, s, xl, xl)  # in place on x_l
  assert torch.equal(xl, out)


@pytest.mark.gpu
@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("rows", ROWS)
def test_cross_bwd_kernel(D, rows):
  ops, dev = _ops(), torch.device("cuda", 0)
  gen = torch.Generator().manual_seed(7 * D + rows)
  dy, x0 = _rand((rows, D), gen, 1e-2).to(dev), _rand((rows, D), gen).to(dev)
  g = torch.full_like(x0, float("nan"))
  db = torch.zeros(D, device=dev)
  ops.cross_bwd(dy, x0, g, db)
  assert bwd_ratio(dy, x0, g, db) <= 1.0
  ops.cross_bwd(dy, x0, g, db)  # db accumulates (+=): twice the column sums
  assert bwd_ratio(dy, x0, g, db / 2) <= 1.01


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 3])
@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("rows", ROWS)
def test_cross_dx0_kernel(L, D, rows):
  ops, dev = _ops(), torch.device("cuda", 0)
  gen = torch.Generator().manual_seed(13 * D + rows + L)
  nb = 8 if D == 8 else 128
  d_chain = _rand((rows, D), gen).to(dev)
  dys = [_rand((rows, D), gen).to(dev) for _ in range(L)]
  ss = [_rand((rows, D), gen).to(dev) for _ in range(L)]
  dx0 = torch.full_like(d_chain, float("nan"))
  d_bottom = torch.full((rows, nb), float("nan"), dtype=torch.bfloat16, device=dev)
  ops.cross_dx0(d_chain, dys, ss, dx0, d_bottom)
  assert dx0_ratio(d_chain, dys, ss, dx0, d_bottom) <= 1.0
  assert torch.isnan(dx0[:, D - nb:].float()).all()  # the bottom columns go to d_bottom only


@pytest.mark.gpu
def test_cross_argument_checks():
  ops, dev = _ops(), torch.device("cuda", 0)
  bf = dict(dtype=torch.bfloat16, device=dev)
  a = torch.zeros(4, 16, **bf)
  b = torch.zeros(4, 16, **bf)
  db = torch.zeros(16, dtype=torch.float32, device=dev)
  mis = torch.zeros(4 * 16 + 1, **bf)[1:].view(4, 16)  # 2-byte offset
  bad = [
      lambda: ops.cross_fwd(a, b, a.float(), b),
      lambda: ops.cross_fwd(a, b, a, torch.zeros(4, 24, **bf)),
      lambda: ops.cross_fwd(a, b, a, torch.zeros(5, 16, **bf)),
      lambda: ops.cross_fwd(a, b, a.cpu(), b),
      lambda: ops.cross_fwd(torch.zeros(4, 12, **bf), torch.zeros(4, 12, **bf),
                            torch.zeros(4, 12, **bf), torch.zeros(4, 12, **bf)),
      lambda: ops.cross_fwd(a, b, mis, b),
      lambda: ops.cross_fwd(a, b, torch.zeros(16, 4, **bf).t(), b),
      lambda: ops.cross_bwd(a, b, a, db.double()),
      lambda: ops.cross_bwd(a, b, a, torch.zeros(8, dtype=torch.float32, device=dev)),
      lambda: ops.cross_dx0(a, [a, a], [b], a, torch.zeros(4, 8, **bf)),
      lambda: ops.cross_dx0(a, [], [], a, torch.zeros(4, 8, **bf)),
      lambda: ops.cross_dx0(a, [a] * 9, [b] * 9, a, torch.zeros(4, 8, **bf)),
      lambda: ops.cross_dx0(a, [a], [b], a, torch.zeros(4, 24, **bf)),
      lambda: ops.cross_dx0(a, [a], [b], a, torch.zeros(4, 4, **bf)),
      lambda: ops.cross_dx0(a, [a], [mis], a, torch.zeros(4, 8, **bf)),
  ]
  for i, f in enumerate(bad):
    with pytest.raises(RuntimeError):
      f()
    torch.cuda.synchronize()
  ops.cross_dx0(a, [a], [b], a.clone(), torch.zeros(4, 8, **bf))  # a valid call still runs


# ------------------------------------------------------------------ GPU: the step
MLPERF_LIKE = [3, 2, 1, 2, 6, 1, 100, 7]


def _gpu_model(seed, hots, table_dtype=torch.float32, n_tables=8, **kw):
  from distributed_embeddings_b200.models.dlrm import DLRM
  torch.manual_seed(seed)
  sizes = kw.pop("sizes", [300 + 11 * i for i in range(n_tables)])
  return DLRM(sizes, embedding_dim=32, bottom_mlp_dims=(64, 32), top_mlp_dims=(128, 64, 1),
              device=torch.device("cuda", 0), compute_dtype=torch.bfloat16,
              backend=kw.pop("backend", "fused"),
              table_dtype=table_dtype, interaction="dcnv2", dcn_num_layers=3,
              dcn_low_rank_dim=64, multi_hot_sizes=hots, **kw)


def _gpu_batch(sizes, hots, b, seed):
  dev = torch.device("cuda", 0)
  g = torch.Generator().manual_seed(seed)
  num = torch.rand(b, 13, generator=g).to(dev)
  cat = [torch.randint(0, s, (b, h), generator=g, dtype=torch.int32).to(dev)
         for s, h in zip(sizes, hots)]
  lab = torch.randint(0, 2, (b, 1), generator=g).float().to(dev)
  return num, cat, lab


def _rel(a, b):
  return float((a - b).norm() / (b.norm() + 1e-12))


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph,emb_opt,dense_opt,hots,table_dtype", [
    (False, "sgd", "sgd", MLPERF_LIKE, torch.float32),
    (True, "sgd", "sgd", MLPERF_LIKE, torch.float32),
    (True, "adagrad", "adam", MLPERF_LIKE, torch.float32),
    (False, "rowwise_adagrad", "sgd", MLPERF_LIKE, torch.bfloat16),
    (True, "sgd", "adam", [1] * 8, torch.bfloat16),
    (True, "rowwise_adagrad", "adam", [1, 1, 100, 1, 2, 1, 1, 4], torch.float32),
])
def test_dcn_step_matches_hybrid_trainer(use_graph, emb_opt, dense_opt, hots, table_dtype):
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  ref = _gpu_model(0, hots, table_dtype)
  fast = _gpu_model(0, hots, table_dtype)
  fast.load_state_dict(ref.state_dict())
  fast.embedding.set_weights(ref.embedding.get_weights())
  b, lr = 512, 0.05 if dense_opt == "adam" or emb_opt != "sgd" else 0.5
  num, cat, lab = _gpu_batch(ref.table_sizes, hots, b, 1)
  w0 = [p.detach().clone() for p in ref.dense_parameters()]
  e0 = [torch.as_tensor(w).float().clone() for w in ref.embedding.get_weights()]
  kw = dict(lr=lr, embedding_optimizer=emb_opt, dense_optimizer=dense_opt)
  t_ref = HybridTrainer(ref, **kw)
  loss_ref = t_ref.step(num, cat, lab)
  t_fast = DLRMTrainStep(fast, use_cuda_graph=use_graph, **kw)
  loss_fast = t_fast.step(num, cat, lab).clone()
  torch.cuda.synchronize()
  torch.testing.assert_close(loss_fast[0], loss_ref, rtol=2e-2, atol=2e-3)
  names = [n for n, p in ref.named_parameters() if not getattr(p, "de_local", False)]
  if dense_opt == "adam":
    # Adam's first update is about +-lr * sign(g): compare its first moment, (1 - beta1) * g
    m_ref = t_ref.dense_optimizer_state()["slots"]
    m_fast = t_fast.dense_optimizer_state()["slots"]
    for n in names:
      assert _rel(m_fast[n][0], m_ref[n][0]) < 0.08, (n, _rel(m_fast[n][0], m_ref[n][0]))
  else:
    for n, p_ref, p_fast, p0 in zip(names, ref.dense_parameters(), fast.dense_parameters(), w0):
      d_ref, d_fast = p_ref.detach() - p0, p_fast.detach() - p0
      assert _rel(d_fast, d_ref) < 0.08, (n, _rel(d_fast, d_ref))
  # bf16 tables: both sides round every updated element stochastically, so each element of the
  # update is off by up to one bf16 ulp of the weight on either side
  tol = 0.08 if table_dtype == torch.float32 else 0.3
  for w_ref, w_fast, w0_ in zip(ref.embedding.get_weights(), fast.embedding.get_weights(), e0):
    d_ref = torch.as_tensor(w_ref).float() - w0_
    d_fast = torch.as_tensor(w_fast).float() - w0_
    assert d_ref.abs().sum() > 0
    assert _rel(d_fast, d_ref) < tol, _rel(d_fast, d_ref)
  loss2 = t_fast.step(num, cat, lab)
  torch.cuda.synchronize()
  assert torch.isfinite(loss2).all() and float(loss2) != float(loss_fast)


@pytest.mark.gpu
def test_dcn_step_rejects_unsupported_configurations():
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  with pytest.raises(ValueError, match="cublas"):
    DLRMTrainStep(_gpu_model(0, None), gemm="fused_dgrad")
  torch.manual_seed(0)
  dot = DLRM([300] * 4, embedding_dim=32, bottom_mlp_dims=(64, 32), top_mlp_dims=(128, 64, 1),
             device=torch.device("cuda", 0), backend="fused", multi_hot_sizes=[1, 2, 1, 1])
  with pytest.raises(ValueError, match="multi-hot"):
    DLRMTrainStep(dot)


@pytest.mark.gpu
def test_dcn_prefetch_matches_step():
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  hots = MLPERF_LIKE
  a, b_ = _gpu_model(3, hots), _gpu_model(3, hots)
  b_.load_state_dict(a.state_dict())
  b_.embedding.set_weights(a.embedding.get_weights())
  bs = 256
  batches = []
  for i in range(4):
    num, cat, lab = _gpu_batch(a.table_sizes, hots, bs, 20 + i)
    flat = torch.cat([c.reshape(-1) for c in cat])
    batches.append((num, cat, lab, flat))
  ta = DLRMTrainStep(a, lr=0.3, use_cuda_graph=True)
  tb = DLRMTrainStep(b_, lr=0.3, use_cuda_graph=True)
  la = [float(ta.step(n, c, l)) for n, c, l, _ in batches]
  pin = lambda t: t.cpu().pin_memory()
  lb = []
  tb.prefetch(pin(batches[0][0]), pin(batches[0][3]), pin(batches[0][2]))
  for i in range(len(batches)):
    loss = tb.run_prefetched()
    if i + 1 < len(batches):
      n, _, l, f = batches[i + 1]
      tb.prefetch(pin(n), pin(f), pin(l))
    lb.append(float(loss))
  torch.cuda.synchronize()
  assert la == pytest.approx(lb, rel=1e-5)
  for p, q in zip(a.dense_parameters(), b_.dense_parameters()):
    torch.testing.assert_close(p, q, rtol=1e-4, atol=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True])
def test_dcn_evaluate_and_predict_match_module(use_graph):
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  hots = MLPERF_LIKE
  m = _gpu_model(5, hots)
  ref = _gpu_model(5, hots, backend="torch")
  ref.load_state_dict(m.state_dict())
  ref.embedding.set_weights(m.embedding.get_weights())
  t = DLRMTrainStep(m, lr=0.0, use_cuda_graph=use_graph)
  t.load_batch(*_gpu_batch(m.table_sizes, hots, 256, 1))  # sets the chunk size
  n = 2 * 256 + 37
  num, cat, lab = _gpu_batch(m.table_sizes, hots, n, 2)
  probs = t.predict(num, cat)
  with torch.no_grad():
    want = torch.sigmoid(ref(num, cat).float()).reshape(-1)
  torch.testing.assert_close(probs, want, rtol=0, atol=1e-2)
  t.evaluate(num, cat, lab)
  res = t.eval_metrics()
  assert res["samples"] == n
  bce = torch.nn.functional.binary_cross_entropy(probs.double().clamp(1e-7, 1 - 1e-7),
                                                 lab.reshape(-1).double())
  assert abs(res["log_loss"] - float(bce)) < 1e-4


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2,
                    reason="needs 2 GPUs (not run on a single H100)")
def test_dcn_step_world2():
  _launch("case_dcnv2_fast_step_world", world=2, device_type="cuda")


# ------------------------------------------------------------------ multi-rank cases + launcher
def _dcnv2_pair(device, backend, world, hots, sizes, **kw):
  """A single-process reference and this rank's model of the same DLRM-DCNv2 weights."""
  from distributed_embeddings_b200.models.dlrm import DLRM
  cfg = dict(embedding_dim=8, bottom_mlp_dims=(16, 8), top_mlp_dims=(64, 1), device=device,
             interaction="dcnv2", dcn_num_layers=2, dcn_low_rank_dim=16, multi_hot_sizes=hots,
             **kw)
  torch.manual_seed(11)
  ref = DLRM(sizes, world_size=1, rank=0, backend="torch", **cfg)
  test = DLRM(sizes, backend=backend, **cfg)
  test.load_state_dict({k: v for k, v in ref.state_dict().items() if "embedding" not in k},
                       strict=False)
  test.embedding.set_weights(ref.embedding.get_weights())
  return ref, test


def _dcnv2_batch(sizes, hots, b, seed, device):
  g = torch.Generator().manual_seed(seed)
  num = torch.rand(b, 13, generator=g).to(device)
  cat = [torch.randint(0, s, (b, h), generator=g).to(device) for s, h in zip(sizes, hots)]
  lab = torch.randint(0, 2, (b, 1), generator=g).float().to(device)
  return num, cat, lab


def case_dcnv2_hybrid_world(rank, world, device, backend):
  """HybridTrainer on the dcnv2 model (multi-hot, model-parallel tables) equals one process on
  the global batch."""
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  sizes, hots = [20 + 7 * i for i in range(5)], [1, 3, 2, 1, 4]
  ref, test = _dcnv2_pair(device, "torch" if backend == "auto" else backend, world, hots, sizes,
                          dp_input=True)
  kw = dict(lr=0.05, embedding_optimizer="sgd")
  t_ref, t_test = HybridTrainer(ref, **kw), HybridTrainer(test, **kw)
  gb, lb = 8 * world, 8
  for i in range(3):
    num, cat, lab = _dcnv2_batch(sizes, hots, gb, 40 + i, device)
    l_ref = t_ref.step(num, cat, lab)
    sl = slice(rank * lb, (rank + 1) * lb)
    l_test = t_test.step(num[sl], [c[sl] for c in cat], lab[sl]).clone()
    dist.all_reduce(l_test)
    torch.testing.assert_close(l_test / world, l_ref, rtol=1e-5, atol=1e-6)
  mine = dict(test.named_parameters())
  for n, p in ref.named_parameters():
    if "embedding" not in n:
      torch.testing.assert_close(mine[n], p, rtol=1e-5, atol=1e-6, msg=lambda m: f"{n}: {m}")
  for a, b in zip(ref.embedding.get_weights(), test.embedding.get_weights(all_ranks=True)):
    torch.testing.assert_close(torch.as_tensor(b), torch.as_tensor(a), rtol=1e-5, atol=1e-6)


def case_dcnv2_fast_step_world(rank, world, device, backend):
  """DLRMTrainStep on the dcnv2 model at world > 1 against HybridTrainer on the global batch."""
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  sizes, hots = [300 + 11 * i for i in range(6)], [1, 3, 2, 1, 100, 4]
  ref, test = _dcnv2_pair(device, "fused", world, hots, sizes, dp_input=True,
                          compute_dtype=torch.bfloat16)
  gb, lb = 64 * world, 64
  num, cat, lab = _dcnv2_batch(sizes, hots, gb, 5, device)
  w0 = [p.detach().clone() for p in ref.dense_parameters()]
  l_ref = HybridTrainer(ref, lr=0.5).step(num, cat, lab)
  sl = slice(rank * lb, (rank + 1) * lb)
  t = DLRMTrainStep(test, lr=0.5, use_cuda_graph=False)
  l_test = t.step(num[sl], [c[sl] for c in cat], lab[sl]).clone()
  dist.all_reduce(l_test)
  torch.testing.assert_close(l_test[0] / world, l_ref, rtol=2e-2, atol=2e-3)
  for p, q, p0 in zip(ref.dense_parameters(), test.dense_parameters(), w0):
    d_ref, d_test = p.detach() - p0, q.detach() - p0
    assert float((d_test - d_ref).norm() / (d_ref.norm() + 1e-12)) < 0.08


def _free_port():
  with socket.socket() as sk:
    sk.bind(("127.0.0.1", 0))
    return sk.getsockname()[1]


def _worker(rank, world, port, case, device_type, errq):
  try:
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world))
    torch.set_num_threads(1)
    sys.path.insert(0, ROOT)
    if device_type == "cuda":
      torch.cuda.set_device(rank)
      device = f"cuda:{rank}"
      dist.init_process_group("nccl", rank=rank, world_size=world,
                              device_id=torch.device(device))
    else:
      device = "cpu"
      dist.init_process_group("gloo", rank=rank, world_size=world)
    globals()[case](rank, world, device, "auto")
    if device_type == "cuda":
      torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()
  except Exception:  # pylint: disable=broad-except
    errq.put((rank, traceback.format_exc()))
    raise


def _launch(case, world=2, device_type="cpu", timeout=300):
  ctx = mp.get_context("spawn")
  errq = ctx.SimpleQueue()
  port = _free_port()
  procs = [ctx.Process(target=_worker, args=(r, world, port, case, device_type, errq))
           for r in range(world)]
  for p in procs:
    p.start()
  failed = False
  for p in procs:
    p.join(timeout)
    if p.is_alive():
      p.terminate()
      p.join()
      failed = True
    failed = failed or p.exitcode != 0
  msgs = []
  while not errq.empty():
    msgs.append(errq.get())
  assert not failed and not msgs, "\n".join(f"--- rank {r} ---\n{tb}" for r, tb in msgs) or \
      "timeout / crash"
