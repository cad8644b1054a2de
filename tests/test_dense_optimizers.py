"""Dense Adagrad and Adam (``dense_optimizer``) in ``DLRMTrainStep``, ``SyntheticTrainStep`` and
``HybridTrainer``, and the fused ``dense_adagrad`` / ``dense_adam`` kernels.

CPU (no GPU needed):
- ``HybridTrainer`` at world 1 (small fp32 ``DLRM``, ``backend="torch"``): over 4 steps of dense
  Adagrad / Adam its dense parameters match ``torch.optim.Adagrad`` / ``torch.optim.Adam`` to
  rounding level, with and without a ``LearningRateScheduler``; momentum with a non-SGD dense
  optimizer and unknown hyperparameters raise.
- gloo at world 2 with replicated tables and dense Adagrad: tables and dense parameters equal a
  single-process run on the global batch, and both ranks' dense parameters are bit-identical
  (own spawn launcher below).
- Checkpoint round trip on ``HybridTrainer``: 3 steps, save, load into a fresh trainer, 2 more
  steps == 5 continuous steps, bit for bit; a state of another kind raises.
- With ``sgd``, the flat-buffer optimizer launches ``dense_sgd`` and nothing else.
- The synthetic example runs end to end with ``--dense_optimizer adagrad``.
- Self-check of the kernel bounds used on the GPU: a float64 model of each defect (bias
  correction with ``t - 1``, ``eps`` inside the square root, accumulator not written back,
  gradient not zeroed) fails the bound while the exactly rounded result passes.

GPU:
- ``dense_adagrad`` / ``dense_adam`` against float64 references computed on the same fp32 inputs,
  sizes 4 to 12.6 M (odd multiples of 4), gradients up to +-1e3 with exact zeros, Adam t = 1, 2,
  1000.  ``p32`` and the state within bounds derived from the operation count (Adagrad's
  accumulator, one fma, within 1 ulp; Adam's moments within their 2-3 roundings);
  ``p16 == bf16(p32)`` and ``g32 == 0`` bit for bit; argument checks raise before any launch.
- ``DLRMTrainStep`` with dense and embedding Adagrad / Adam, eager and graph, cuBLAS and
  first-party GEMMs, against ``HybridTrainer`` (relative update error < 0.08, the tolerance of
  ``test_dlrm_fast.py``) of the update and the optimizer state, tables included; Adam's first
  step is about ``+-lr * sign(g)``, so there its moments are compared and the update must follow
  from them (``_check_update``); ``SyntheticTrainStep`` the same way.
- Graph warm-up leaks nothing: Adam's step word equals the number of graph steps, and Adagrad's
  accumulator after one graph step equals the eager one.
- Pad elements of ``p32`` / ``p16`` stay zero and their state at its initial value.
- With the default ``sgd`` an eager step launches ``dense_sgd`` once and no new op.
- Checkpoint round trip on ``DLRMTrainStep`` (eager, Adagrad embeddings): the continued run
  matches the continuous run as closely as a second continuous run does (bit for bit when the
  step is deterministic; the atomic fp32 sums of the step's gradient kernels make it differ in
  the last bits); a ``HybridTrainer`` state loads slot for slot.
- World 2 (skips on fewer GPUs): ``DLRMTrainStep`` with replicated tables and dense Adagrad
  matches the single-process step, ranks bit-identical.
"""
import json
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
U = 2.0**-24  # fp32 unit roundoff
TINY = 1e-37


# ------------------------------------------------------------------ float64 model + bounds
def _ulp32(x):
  """ulp of fp32 numbers of magnitude |x| (float64 tensor), subnormal floor included."""
  e = torch.floor(torch.log2(x.abs().clamp_min(2.0**-126)))
  return torch.pow(2.0, e - 23)


def reference(kind, p, g, s0, s1, lr, t, cfg, defect=None):
  """float64 result of one update on fp32 inputs, with its error bounds.  ``defect`` models a
  wrong kernel: 'bias_t_minus_1', 'eps_in_sqrt', 'no_state_writeback', 'no_grad_zero'."""
  f = lambda x: x.double()
  p, g, s0 = f(p), f(g), f(s0)
  f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))
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


def worst_ratio(kind, inputs, got, cfg, t=1):
  """max |got - ref| / bound over p32 and the state; inf when p16 / g32 are not exact."""
  ref, bound = reference(kind, *inputs, t, cfg)
  worst = 0.0
  for k in ("p", "s0", "s1"):
    if k not in ref:
      continue
    err = (got[k].double() - ref[k]).abs()
    r = err / bound[k]
    if not torch.isfinite(got[k]).all() or torch.isnan(r).any():
      return float("inf")
    worst = max(worst, float(r.max()))
  if not torch.equal(got["p16"], got["p"].float().bfloat16()) or bool((got["g"] != 0).any()):
    return float("inf")
  return worst


def make_inputs(kind, n, seed, device="cpu"):
  """fp32 parameters, gradients (up to +-1e3, 1 in 8 exactly zero) and plausible state."""
  gen = torch.Generator().manual_seed(seed)
  r = lambda: torch.randn(n, generator=gen, dtype=torch.float64)
  mag = lambda lo, hi: torch.pow(10.0, torch.rand(n, generator=gen, dtype=torch.float64) *
                                 (hi - lo) + lo)
  p = r()
  g = (r() * mag(-4, 3)).clamp(-1e3, 1e3)
  g[torch.rand(n, generator=gen) < 0.125] = 0.0
  if kind == "adagrad":
    s0, s1 = 0.1 + r().abs() * mag(-3, 3), None
  else:
    s0 = r() * mag(-4, 2)
    s1 = s0 * s0 * (1 + 9 * torch.rand(n, generator=gen, dtype=torch.float64))
  cast = lambda x: None if x is None else x.float().to(device)
  return cast(p), cast(g), cast(s0), cast(s1)


CFGS = {
    "adagrad": [{"eps": 1e-7, "initial_accumulator_value": 0.1},
                {"eps": 1e-2, "initial_accumulator_value": 0.0}],
    "adam": [{"beta1": 0.9, "beta2": 0.999, "eps": 1e-8},
             {"beta1": 0.8, "beta2": 0.99, "eps": 1e-3}],
}


def _rounded(kind, inputs, cfg, t, defect=None):
  out, _ = reference(kind, *inputs, t, cfg, defect=defect)
  got = {k: v.float() for k, v in out.items()}
  got["p16"] = got["p"].bfloat16()
  return got


@pytest.mark.parametrize("kind,defect", [("adam", "bias_t_minus_1"), ("adam", "eps_in_sqrt"),
                                         ("adagrad", "eps_in_sqrt"),
                                         ("adagrad", "no_state_writeback"),
                                         ("adam", "no_state_writeback"),
                                         ("adagrad", "no_grad_zero"), ("adam", "no_grad_zero")])
def test_bounds_catch_defects(kind, defect):
  """The exactly rounded result passes every bound; each modelled defect fails it."""
  for cfg in CFGS[kind]:
    inputs = make_inputs(kind, 4096, 11) + (0.01,)
    for t in ((2, 1000) if kind == "adam" else (1,)):
      assert worst_ratio(kind, inputs, _rounded(kind, inputs, cfg, t), cfg, t) <= 1.0
  # every defect is visible with the configuration that makes it matter (eps 1e-2 / 1e-3 for
  # eps_in_sqrt: at 1e-7 / 1e-8 it changes the update by less than a rounding)
  cfg = CFGS[kind][1] if defect == "eps_in_sqrt" else CFGS[kind][0]
  inputs = make_inputs(kind, 4096, 11) + (0.01,)
  for t in ((2, 1000) if kind == "adam" else (1,)):
    bad = _rounded(kind, inputs, cfg, t, defect)
    assert worst_ratio(kind, inputs, bad, cfg, t) > 1.0, (defect, t)


# ------------------------------------------------------------------ CPU: HybridTrainer
def _small_dlrm(seed, device="cpu", dtype=torch.float32, **kw):
  from distributed_embeddings_b200.models.dlrm import DLRM
  torch.manual_seed(seed)
  sizes = kw.pop("sizes", [20 + 3 * i for i in range(4)])
  return DLRM(sizes, embedding_dim=8, bottom_mlp_dims=(16, 8), top_mlp_dims=(16, 1),
              compute_dtype=dtype, device=device, backend=kw.pop("backend", "torch"), **kw)


def _batch(sizes, b, seed, device="cpu"):
  g = torch.Generator().manual_seed(seed)
  num = torch.rand(b, 13, generator=g).to(device)
  cat = [torch.randint(0, s, (b,), generator=g).to(device) for s in sizes]
  lab = torch.randint(0, 2, (b, 1), generator=g).float().to(device)
  return num, cat, lab


@pytest.mark.parametrize("kind", ["adagrad", "adam"])
@pytest.mark.parametrize("sched", [False, True])
def test_hybrid_matches_torch_optim(kind, sched):
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  from distributed_embeddings_b200.utils.lr_schedule import LearningRateScheduler
  model, ref = _small_dlrm(0), _small_dlrm(0)  # same seed: same weights, de_local tags kept
  lr = 0.01
  mk = lambda: LearningRateScheduler(lr, 2, 3, 4) if sched else None
  tr = HybridTrainer(model, lr=lr, embedding_optimizer="sgd", dense_optimizer=kind,
                     scheduler=mk())
  dense = [p for p in ref.parameters() if not getattr(p, "de_local", False)]
  tables = [p for p in ref.parameters() if getattr(p, "de_local", False)]
  opt = torch.optim.Adagrad(dense, lr=lr, initial_accumulator_value=0.1, eps=1e-7) \
      if kind == "adagrad" else torch.optim.Adam(dense, lr=lr, eps=1e-8)
  topt = torch.optim.SGD(tables, lr=lr)  # the model-parallel tables take the embedding SGD
  ref_sched = mk()
  sizes = model.table_sizes
  for i in range(4):
    num, cat, lab = _batch(sizes, 32, 100 + i)
    tr.step(num, cat, lab)
    if ref_sched is not None:
      cur = ref_sched.step()
      for o in (opt, topt):
        for grp in o.param_groups:
          grp["lr"] = cur
    ref.zero_grad()
    torch.nn.functional.binary_cross_entropy_with_logits(ref(num, cat).float(), lab).backward()
    opt.step()
    topt.step()
  for (n, a), b in zip([(n, p) for n, p in model.named_parameters()
                        if not getattr(p, "de_local", False)], dense):
    # Adam's m / sqrt(v) amplifies the gradients' last-bit differences (summation order) where
    # they are tiny: allowed 1e-4 of one step's size (lr)
    torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-4 * lr, msg=lambda m: f"{n}: {m}")
  st = tr.dense_optimizer_state()
  assert st["kind"] == kind and st["step"] == (4 if kind == "adam" else 0)


def test_hybrid_argument_errors():
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  with pytest.raises(ValueError, match="momentum"):
    HybridTrainer(_small_dlrm(0), lr=0.1, momentum=0.9, dense_optimizer="adam")
  with pytest.raises(ValueError, match="dense_optimizer"):
    HybridTrainer(_small_dlrm(0), lr=0.1, dense_optimizer="rmsprop")
  with pytest.raises(ValueError, match="takes no argument"):
    HybridTrainer(_small_dlrm(0), lr=0.1, dense_optimizer="adagrad",
                  dense_optimizer_kwargs={"beta1": 0.5})


@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_hybrid_checkpoint_round_trip(kind):
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  sizes = [20 + 3 * i for i in range(4)]
  batches = [_batch(sizes, 32, 200 + i) for i in range(5)]
  a = _small_dlrm(1)
  ta = HybridTrainer(a, lr=0.01, embedding_optimizer="sgd", dense_optimizer=kind)
  for bt in batches:
    ta.step(*bt)
  b = _small_dlrm(1)
  tb = HybridTrainer(b, lr=0.01, embedding_optimizer="sgd", dense_optimizer=kind)
  for bt in batches[:3]:
    tb.step(*bt)
  saved = tb.dense_optimizer_state()
  weights = {k: v.clone() for k, v in b.state_dict().items()}
  tables = b.embedding.get_weights()
  c = _small_dlrm(2)  # different initial weights: everything comes from the checkpoint
  c.load_state_dict(weights)
  c.embedding.set_weights(tables)
  tc = HybridTrainer(c, lr=0.01, embedding_optimizer="sgd", dense_optimizer=kind)
  tc.load_dense_optimizer_state(saved)
  for bt in batches[3:]:
    tc.step(*bt)
  for (n, p), q in zip(a.named_parameters(), c.parameters()):
    assert torch.equal(p, q), n
  other = "adam" if kind == "adagrad" else "adagrad"
  td = HybridTrainer(_small_dlrm(1), lr=0.01, dense_optimizer=other)
  with pytest.raises(ValueError, match="cannot be loaded"):
    td.load_dense_optimizer_state(saved)


def test_flat_sgd_launches_dense_sgd_only():
  """The default keeps today's schedule: one dense_sgd, no state, no step word."""
  from distributed_embeddings_b200.models.dense_optimizer import (FlatDenseOptimizer,
                                                                  dense_optimizer_config)
  calls = []

  class Rec:

    def __getattr__(self, name):
      return lambda *a, **k: calls.append(name)

  p32 = torch.zeros(16)
  opt = FlatDenseOptimizer(dense_optimizer_config("sgd"), p32)
  assert opt.state == [] and opt.step_t is None and opt.snapshot() == []
  opt.apply(Rec(), torch.zeros(16, dtype=torch.bfloat16), torch.zeros(16), torch.ones(1))
  assert calls == ["dense_sgd"]


def test_synthetic_example_dense_adagrad():
  env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
  out = subprocess.run([sys.executable, "examples/benchmarks/synthetic_models/main.py", "--model",
                        "tiny", "--row_scale", "0.001", "--batch_size", "16", "--num_steps", "3",
                        "--device", "cpu", "--optimizer", "adagrad", "--dense_optimizer",
                        "adagrad"], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600, check=False)
  assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
  rec = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])
  assert rec["dense_optimizer"] == "adagrad" and rec["optimizer"] == "adagrad"
  assert rec["samples_per_sec"] > 0


# ------------------------------------------------------------------ world-2 launcher
def _free_port():
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    return s.getsockname()[1]


def _worker(rank, world, port, fn_name, device_type, errq):
  try:
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world))
    torch.set_num_threads(1)
    sys.path.insert(0, ROOT)
    if device_type == "cuda":
      torch.cuda.set_device(rank)
      dist.init_process_group("nccl", rank=rank, world_size=world,
                              device_id=torch.device("cuda", rank))
      device = torch.device("cuda", rank)
    else:
      dist.init_process_group("gloo", rank=rank, world_size=world)
      device = torch.device("cpu")
    globals()[fn_name](rank, world, device)
    dist.barrier()
    dist.destroy_process_group()
  except Exception:  # pylint: disable=broad-except
    errq.put((rank, traceback.format_exc()))
    raise


def _launch(fn_name, world=2, device_type="cpu", timeout=300):
  ctx = mp.get_context("spawn")
  errq = ctx.SimpleQueue()
  port = _free_port()
  procs = [ctx.Process(target=_worker, args=(r, world, port, fn_name, device_type, errq))
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


def _assert_ranks_identical(tensors):
  for t in tensors:
    got = [torch.empty_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(got, t.contiguous())
    for x in got[1:]:
      assert torch.equal(x, got[0]), "dense parameters differ between ranks"


def _case_gloo_replicated_adagrad(rank, world, device):
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  sizes = [20 + 3 * i for i in range(4)] + [400, 500]
  ref = _small_dlrm(5, sizes=sizes, world_size=1, rank=0)
  test = _small_dlrm(5, sizes=sizes, data_parallel_threshold=40 * 8)
  assert len(test.embedding.dp_layers) > 0
  test.load_state_dict({k: v for k, v in ref.state_dict().items() if "embedding" not in k},
                       strict=False)
  test.embedding.set_weights(ref.embedding.get_weights())
  kw = dict(lr=0.02, embedding_optimizer="adagrad", dense_optimizer="adagrad")
  t_ref, t_test = HybridTrainer(ref, **kw), HybridTrainer(test, **kw)
  gb, lb = 16 * world, 16
  for i in range(3):
    num, cat, lab = _batch(sizes, gb, 300 + i)
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
  _assert_ranks_identical([p.detach() for p in test.dense_parameters()])


def test_gloo_world2_replicated_tables_dense_adagrad():
  _launch("_case_gloo_replicated_adagrad", world=2, device_type="cpu")


# ------------------------------------------------------------------ GPU: kernels
def _kernel_run(kind, n, seed, cfg, t=1):
  from distributed_embeddings_b200.ops import _native
  ops = _native.require()
  dev = torch.device("cuda", 0)
  p, g, s0, s1 = make_inputs(kind, n, seed, dev)
  inputs = [x.clone() if x is not None else None for x in (p, g, s0, s1)]
  lr = torch.full((1,), 0.01, dtype=torch.float32, device=dev)
  p16 = torch.empty(n, dtype=torch.bfloat16, device=dev)
  if kind == "adagrad":
    ops.dense_adagrad(p, p16, g, s0, lr, cfg["eps"])
  else:
    step = torch.full((1,), float(t), dtype=torch.float32, device=dev)
    ops.dense_adam(p, p16, g, s0, s1, lr, step, cfg["beta1"], cfg["beta2"], cfg["eps"])
  torch.cuda.synchronize()
  got = {"p": p, "p16": p16, "g": g, "s0": s0, "s1": s1}
  inputs = [inputs[0], inputs[1], inputs[2], inputs[3], 0.01]
  return inputs, got


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4, 12, 4 * 1001, 4 * (3 * 2**20 + 1)])
@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_kernel_against_float64(kind, n):
  worst = 0.0
  for ci, cfg in enumerate(CFGS[kind]):
    for t in ((1, 2, 1000) if kind == "adam" else (1,)):
      inputs, got = _kernel_run(kind, n, 7 + ci + t, cfg, t)
      if kind == "adagrad":
        got.pop("s1")
      r = worst_ratio(kind, inputs, got, cfg, t)
      assert r <= 1.0, (kind, n, cfg, t, r)
      worst = max(worst, r)
  print(f"dense_{kind} n={n}: worst |err| / bound {worst:.3f}")


@pytest.mark.gpu
def test_kernel_argument_checks():
  from distributed_embeddings_b200.ops import _native
  ops = _native.require()
  dev = torch.device("cuda", 0)
  f32 = lambda n=16: torch.zeros(n, dtype=torch.float32, device=dev)
  p, g, a, m, v = f32(), f32(), f32(), f32(), f32()
  p16 = torch.zeros(16, dtype=torch.bfloat16, device=dev)
  lr = torch.full((1,), 0.5, device=dev)
  step = torch.ones(1, device=dev)
  g.fill_(1.0)
  bad = [
      lambda: ops.dense_adagrad(p.double(), p16, g, a, lr, 1e-7),
      lambda: ops.dense_adagrad(p, p16.float(), g, a, lr, 1e-7),
      lambda: ops.dense_adagrad(p, p16, g, f32(20), lr, 1e-7),
      lambda: ops.dense_adagrad(p[:6], p16[:6], g[:6], a[:6], lr, 1e-7),
      lambda: ops.dense_adagrad(p[1:9], p16[1:9], g[1:9], a[1:9], lr, 1e-7),
      lambda: ops.dense_adagrad(f32(32)[::2], p16, g, a, lr, 1e-7),
      lambda: ops.dense_adagrad(p, p16, g, a, torch.full((2,), 0.5, device=dev), 1e-7),
      lambda: ops.dense_adagrad(p, p16, g, a, torch.full((1,), 0.5), 1e-7),
      lambda: ops.dense_adagrad(p, p16, g, a.cpu(), lr, 1e-7),
      lambda: ops.dense_adam(p, p16, g, m, v, lr, step.double(), 0.9, 0.999, 1e-8),
      lambda: ops.dense_adam(p, p16, g, m, v, lr, torch.ones(2, device=dev), 0.9, 0.999, 1e-8),
      lambda: ops.dense_adam(p, p16, g, m, f32(8), lr, step, 0.9, 0.999, 1e-8),
      lambda: ops.dense_adam(p, p16, g, m.half(), v, lr, step, 0.9, 0.999, 1e-8),
  ]
  for i, call in enumerate(bad):
    with pytest.raises(RuntimeError):
      call()
    torch.cuda.synchronize()
    assert bool((g == 1.0).all()) and bool((p == 0).all()), f"call {i} launched"


# ------------------------------------------------------------------ GPU: trainers
def _dlrm(seed, dev, **kw):
  from distributed_embeddings_b200.models.dlrm import DLRM
  torch.manual_seed(seed)
  sizes = kw.pop("sizes", [300 + 11 * i for i in range(26)])
  return DLRM(sizes, device=dev, compute_dtype=torch.bfloat16, backend="fused", **kw)


def _dense_named(model):
  from distributed_embeddings_b200.models.dense_optimizer import dense_named_parameters
  return dense_named_parameters(model)


def _rel(a, b):
  return float((a - b).norm() / (b.norm() + 1e-12))


LR = {"adagrad": 0.05, "adam": 0.002}


def _check_update(kind, d_fast, d_ref, state_fast, state_ref, what):
  """One step of the fast trainer against HybridTrainer, relative error below 0.08 (the tolerance
  of test_dlrm_fast.py).  Adagrad: the update and the accumulator.  Adam's first step is
  ``-lr * g / (|g| + eps)``, about ``+-lr`` wherever ``|g| >> eps = 1e-8``: comparing the updates
  would compare signs of gradients that are bf16 rounding noise between the two paths (near-zero
  sums).  So for Adam the moments are compared (m and sqrt(v), proportional to the gradients, at
  0.08), and the update must follow from the fast trainer's own moments to fp32 rounding."""
  init = 0.1 if kind == "adagrad" else 0.0
  for i, (a, b) in enumerate(zip(state_ref, state_fast)):
    a, b = a.double().cpu() - init, b.double().cpu() - init
    if kind == "adam" and i == 1:
      a, b = a.sqrt(), b.sqrt()
    assert _rel(b, a) < 0.08, (what, "state", i, _rel(b, a))
  if kind != "adam":
    assert _rel(d_fast, d_ref) < 0.08, (what, _rel(d_fast, d_ref))
    return
  m, v = (x.double().to(d_fast.device).view(d_fast.shape) for x in state_fast)
  lr = float(torch.tensor(LR["adam"], dtype=torch.float32))
  want = -lr * (m / 0.1) / ((v / (1 - 0.999)).sqrt() + 1e-8)
  torch.testing.assert_close(d_fast.double(), want, rtol=1e-3, atol=1e-3 * lr,
                             msg=lambda msg: f"{what}: {msg}")


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph,gemm", [(False, "cublas"), (True, "cublas"),
                                            (False, "tcgen05"), (True, "tcgen05")])
@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_dlrm_step_matches_hybrid(kind, use_graph, gemm):
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  dev = torch.device("cuda", 0)
  ref, fast = _dlrm(0, dev), _dlrm(0, dev)
  fast.load_state_dict(ref.state_dict())
  fast.embedding.set_weights(ref.embedding.get_weights())
  sizes = ref.table_sizes
  num, cat, lab = _batch(sizes, 512, 1, dev)
  cat = [c.int() for c in cat]
  w0 = [p.detach().clone() for p in ref.dense_parameters()]
  e0 = ref.embedding.get_weights()  # global tables, the layout of get_optimizer_state()
  kw = dict(lr=LR[kind], embedding_optimizer=kind, dense_optimizer=kind)
  t_ref = HybridTrainer(ref, **kw)
  loss_ref = t_ref.step(num, cat, lab)
  t_fast = DLRMTrainStep(fast, use_cuda_graph=use_graph, gemm=gemm, **kw)
  loss_fast = t_fast.step(num, torch.stack(cat), lab).clone()
  torch.cuda.synchronize()
  torch.testing.assert_close(loss_fast[0], loss_ref, rtol=2e-2, atol=2e-3)
  s_ref, s_fast = t_ref.dense_optimizer_state(), t_fast.dense_optimizer_state()
  assert s_ref["step"] == s_fast["step"] == (1 if kind == "adam" else 0)
  named = zip(_dense_named(ref), _dense_named(fast), w0)
  for (name, p_ref), (_, p_fast), p0 in named:
    d_ref, d_fast = p_ref.detach() - p0, p_fast.detach() - p0
    assert d_ref.abs().sum() > 0
    _check_update(kind, d_fast, d_ref, s_fast["slots"][name], s_ref["slots"][name], name)
  e_ref, e_fast = ref.embedding.get_optimizer_state(), fast.embedding.get_optimizer_state()
  # all tables as one vector, like test_dlrm_fast.py's comparison of the merged local tables
  flat = lambda arrays: torch.cat([torch.as_tensor(a).reshape(-1) for a in arrays])
  d_ref = flat(ref.embedding.get_weights()) - flat(e0)
  d_fast = flat(fast.embedding.get_weights()) - flat(e0)
  slots = len(e_ref["tables"][0])
  st = [flat([t[j] for t in e_fast["tables"]]) for j in range(slots)]
  sr = [flat([t[j] for t in e_ref["tables"]]) for j in range(slots)]
  _check_update(kind, d_fast, d_ref, st, sr, "tables")
  loss2 = t_fast.step(num, torch.stack(cat), lab)
  torch.cuda.synchronize()
  assert torch.isfinite(loss2).all() and float(loss2) != float(loss_fast)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_synthetic_step_matches_hybrid(kind):
  from distributed_embeddings_b200.models.configs import scaled, synthetic_models_v3
  from distributed_embeddings_b200.models.synthetic import InputGenerator, SyntheticModel
  from distributed_embeddings_b200.models.synthetic_fast import SyntheticTrainStep
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  dev = torch.device("cuda", 0)
  cfg = scaled(synthetic_models_v3["tiny"], 2e-4)
  mk = lambda: SyntheticModel(cfg, device=dev, compute_dtype=torch.bfloat16, backend="fused")
  torch.manual_seed(21)
  ref = mk()
  torch.manual_seed(21)
  fast = mk()
  fast.load_state_dict(ref.state_dict())
  fast.embedding.set_weights(ref.embedding.get_weights())
  (num, cat), lab = InputGenerator(cfg, 256, alpha=1.05, device=dev,
                                   mp_input_ids=ref.embedding.strategy.input_ids_list[0])[0]
  w0 = [p.detach().clone() for p in ref.dense_parameters()]
  kw = dict(lr=LR[kind], embedding_optimizer=kind, dense_optimizer=kind)
  t_ref = HybridTrainer(ref, **kw)
  t_ref.step(num, cat, lab)
  t_fast = SyntheticTrainStep(fast, use_cuda_graph=True, **kw)
  t_fast.step(num, cat, lab)
  torch.cuda.synchronize()
  s_ref, s_fast = t_ref.dense_optimizer_state(), t_fast.dense_optimizer_state()
  assert s_ref["step"] == s_fast["step"] == (1 if kind == "adam" else 0)
  for (name, p_ref), (_, p_fast), p0 in zip(_dense_named(ref), _dense_named(fast), w0):
    d_ref, d_fast = p_ref.detach() - p0, p_fast.detach() - p0
    assert d_ref.abs().sum() > 0
    _check_update(kind, d_fast, d_ref, s_fast["slots"][name], s_ref["slots"][name], name)


@pytest.mark.gpu
def test_graph_warmup_leaks_no_state():
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  dev = torch.device("cuda", 0)
  sizes = [100 + 7 * i for i in range(26)]
  num, cat, lab = _batch(sizes, 256, 5, dev)
  cat = torch.stack([c.int() for c in cat])
  m = _dlrm(3, dev, sizes=sizes)
  t = DLRMTrainStep(m, lr=0.002, embedding_optimizer="adam", dense_optimizer="adam")
  for k in range(1, 4):
    t.step(num, cat, lab)
    torch.cuda.synchronize()
    assert float(t.dense_opt.step_t) == k
  graph, eager = _dlrm(4, dev, sizes=sizes), _dlrm(4, dev, sizes=sizes)
  kw = dict(lr=0.05, embedding_optimizer="adagrad", dense_optimizer="adagrad")
  tg = DLRMTrainStep(graph, use_cuda_graph=True, **kw)
  te = DLRMTrainStep(eager, use_cuda_graph=False, **kw)
  tg.step(num, cat, lab)
  te.step(num, cat, lab)
  torch.cuda.synchronize()
  torch.testing.assert_close(tg.dense_opt.state[0], te.dense_opt.state[0], rtol=1e-6, atol=1e-7)
  torch.testing.assert_close(tg.p32, te.p32, rtol=1e-6, atol=1e-7)


def _pad_mask(t):
  """True at the elements of the flat buffers that belong to no parameter."""
  mask = torch.ones(t.n_flat, dtype=torch.bool, device=t.p32.device)
  for p in t.model.dense_parameters():
    mask.as_strided(p.shape, p.stride(), p.storage_offset()).fill_(False)
  return mask


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_pad_elements_stay_put(kind):
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  dev = torch.device("cuda", 0)
  sizes = [100 + 7 * i for i in range(26)]
  num, cat, lab = _batch(sizes, 256, 6, dev)
  t = DLRMTrainStep(_dlrm(5, dev, sizes=sizes), lr=LR[kind], embedding_optimizer=kind,
                    dense_optimizer=kind)
  for _ in range(3):
    t.step(num, torch.stack([c.int() for c in cat]), lab)
  torch.cuda.synchronize()
  pad = _pad_mask(t)
  assert int(pad.sum()) > 0
  assert bool((t.p32[pad] == 0).all()) and bool((t.p16[pad] == 0).all())
  init = 0.1 if kind == "adagrad" else 0.0
  for s in t.dense_opt.state:
    assert bool((s[pad] == init).all())


@pytest.mark.gpu
def test_default_sgd_launches_same_ops():
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from distributed_embeddings_b200.ops import _native
  dev = torch.device("cuda", 0)
  sizes = [100 + 7 * i for i in range(26)]
  num, cat, lab = _batch(sizes, 256, 7, dev)
  t = DLRMTrainStep(_dlrm(6, dev, sizes=sizes), lr=0.1, use_cuda_graph=False)
  names = []
  real = t.ops

  class Rec:

    def __getattr__(self, name):
      names.append(name)
      return getattr(real, name)

  t.ops = Rec()
  _native.reset_launch_count()
  t.step(num, torch.stack([c.int() for c in cat]), lab)
  torch.cuda.synchronize()
  assert names.count("dense_sgd") == 1
  assert "dense_adagrad" not in names and "dense_adam" not in names
  assert t.dense_opt.state == [] and t.dense_opt.step_t is None


@pytest.mark.gpu
def test_dlrm_checkpoint_round_trip():
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  dev = torch.device("cuda", 0)
  sizes = [100 + 7 * i for i in range(26)]
  batches = [_batch(sizes, 256, 400 + i, dev) for i in range(5)]
  batches = [(n, torch.stack([c.int() for c in cat]), l) for n, cat, l in batches]
  kw = dict(lr=0.05, embedding_optimizer="adagrad", dense_optimizer="adagrad",
            use_cuda_graph=False)
  a, a2 = _dlrm(8, dev, sizes=sizes), _dlrm(8, dev, sizes=sizes)
  ta, ta2 = DLRMTrainStep(a, **kw), DLRMTrainStep(a2, **kw)
  for bt in batches:
    ta.step(*bt)
    ta2.step(*bt)
  b = _dlrm(8, dev, sizes=sizes)
  tb = DLRMTrainStep(b, **kw)
  for bt in batches[:3]:
    tb.step(*bt)
  torch.cuda.synchronize()
  dense_state = tb.dense_optimizer_state()
  emb_state = b.embedding.get_optimizer_state()
  weights = {k: v.clone() for k, v in b.state_dict().items()}
  tables = b.embedding.get_weights()
  c = _dlrm(9, dev, sizes=sizes)
  c.load_state_dict(weights)
  tc = DLRMTrainStep(c, **kw)
  c.embedding.set_weights(tables)
  c.embedding.set_optimizer_state(emb_state)
  tc.load_dense_optimizer_state(dense_state)
  for bt in batches[3:]:
    tc.step(*bt)
  torch.cuda.synchronize()
  # a second continuous run is the control: the continued run must match the continuous one as
  # closely as two continuous runs match each other (bit for bit when the step is deterministic)
  def flat(m, t):
    dense = [p.detach().reshape(-1) for n, p in m.named_parameters() if "embedding" not in n]
    tabs = [torch.from_numpy(w).reshape(-1).to(dev) for w in m.embedding.get_weights()]
    st = [s[0].reshape(-1) for s in t.dense_optimizer_state()["slots"].values()]
    return torch.cat(dense + tabs + st)
  ref, ctl, got = flat(a, ta), flat(a2, ta2), flat(c, tc)
  noise = float((ctl - ref).abs().max())
  diff = float((got - ref).abs().max())
  print(f"checkpoint round trip: max |continued - continuous| {diff:.3g}, "
        f"control run {noise:.3g}")
  if noise == 0.0:
    assert torch.equal(got, ref)
  else:
    assert diff <= 4 * noise, (diff, noise)
  # a HybridTrainer state loads slot for slot
  h = _dlrm(10, dev, sizes=sizes)
  th = HybridTrainer(h, lr=0.05, embedding_optimizer="adagrad", dense_optimizer="adagrad")
  n0, c0, l0 = batches[0]
  th.step(n0, list(c0), l0.view(-1, 1))
  hs = th.dense_optimizer_state()
  d = _dlrm(10, dev, sizes=sizes)
  td = DLRMTrainStep(d, **kw)
  td.load_dense_optimizer_state(hs)
  back = td.dense_optimizer_state()
  assert set(back["slots"]) == set(hs["slots"])
  for name, slots in hs["slots"].items():
    assert torch.equal(back["slots"][name][0], slots[0]), name
  with pytest.raises(ValueError, match="cannot be loaded"):
    DLRMTrainStep(_dlrm(10, dev, sizes=sizes), lr=0.01, dense_optimizer="adam",
                  embedding_optimizer="adam").load_dense_optimizer_state(hs)


def _case_gpu_replicated_adagrad(rank, world, device):
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  sizes = [200 + 13 * i for i in range(26)]
  ref = _dlrm(7, device, sizes=sizes, world_size=1, rank=0)
  test = _dlrm(7, device, sizes=sizes, data_parallel_threshold=250 * 128)
  assert len(test.embedding.dp_layers) > 0
  test.load_state_dict({k: v for k, v in ref.state_dict().items() if "embedding" not in k},
                       strict=False)
  test.embedding.set_weights(ref.embedding.get_weights(all_ranks=True))
  with pytest.raises(ValueError, match="dense_optimizer"):  # replicated tables need one kind
    DLRMTrainStep(_dlrm(7, device, sizes=sizes, data_parallel_threshold=250 * 128), lr=0.05,
                  embedding_optimizer="adagrad", dense_optimizer="adam")
  kw = dict(lr=0.05, embedding_optimizer="adagrad", dense_optimizer="adagrad")
  t_ref = DLRMTrainStep(ref, use_cuda_graph=False, **kw)
  t_test = DLRMTrainStep(test, use_cuda_graph=True, **kw)
  gb, lb = 256 * world, 256
  for i in range(2):
    num, cat, lab = _batch(sizes, gb, 500 + i, device)
    cat = torch.stack([c.int() for c in cat])
    l_ref = t_ref.step(num, cat, lab.view(-1)).clone()
    sl = slice(rank * lb, (rank + 1) * lb)
    l_test = t_test.step(num[sl], cat[:, sl].contiguous(), lab.view(-1)[sl]).clone()
    dist.all_reduce(l_test)
    torch.testing.assert_close(l_test / world, l_ref, rtol=1e-2, atol=1e-3)
  t_test.ctx.check_errors()
  mine = dict(test.named_parameters())
  for n, p in ref.named_parameters():
    if "embedding" not in n:
      torch.testing.assert_close(mine[n], p, rtol=3e-2, atol=3e-3, msg=lambda m: f"{n}: {m}")
  for a, b in zip(ref.embedding.get_weights(all_ranks=True),
                  test.embedding.get_weights(all_ranks=True)):
    torch.testing.assert_close(torch.from_numpy(b), torch.from_numpy(a), rtol=3e-2, atol=3e-3)
  _assert_ranks_identical([t_test.p32])


@pytest.mark.gpu
@pytest.mark.multigpu
def test_gpu_world2_replicated_tables_dense_adagrad():
  _launch("_case_gpu_replicated_adagrad", world=2, device_type="cuda")
