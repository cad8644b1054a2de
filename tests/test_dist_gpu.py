"""GPU runs of the distributed cases: fused back end (sm_90a kernels + P2P) and the torch/NCCL
back end.  world=1 exercises the kernels on one GPU; world>=2 needs several GPUs (NVLink P2P)."""
import pytest
import torch

from dist_utils import launch

FUSED_CASES = [
    "case_basic", "case_memory_balanced", "case_memory_optimized", "case_shared_dp",
    "case_shared_mp", "case_mp_input", "case_column_slice_threshold",
    "case_fewer_tables_than_workers", "case_multihot_dp", "case_multihot_mp", "case_multihot_mean",
    "case_int32_ids", "case_errors", "case_hybrid_optimizer", "case_row_slice",
    "case_data_parallel", "case_all_modes", "case_checkpoint_resharding", "case_cpu_offload",
    "case_ragged_dp", "case_ragged_mean", "case_ragged_mp",
]
TORCH_CASES = ["case_basic", "case_ragged_dp", "case_custom_layer", "case_cpu_offload",
               "case_dp_to_mp_input", "case_broadcast"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", FUSED_CASES)
def test_fused_world1(case):
  launch(case, world=1, device_type="cuda", backend="fused")


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["case_basic", "case_ragged_dp", "case_custom_layer",
                                  "case_cpu_offload"])
def test_torch_backend_world1(case):
  launch(case, world=1, device_type="cuda", backend="torch" if case != "case_custom_layer"
         else "auto")


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("case", FUSED_CASES + ["case_column_slice_merge"][:0])
def test_fused_world2(case):
  launch(case, world=2, device_type="cuda", backend="fused")


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("case", TORCH_CASES)
def test_nccl_world2(case):
  launch(case, world=2, device_type="cuda", backend="auto" if case == "case_custom_layer"
         else "torch")


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("case", ["case_column_slice_merge", "case_column_slice_dup_worker",
                                  "case_all_modes", "case_row_slice"])
def test_fused_world4(case):
  if torch.cuda.device_count() < 4:
    pytest.skip("needs 4 GPUs")
  launch(case, world=4, device_type="cuda", backend="fused")


@pytest.mark.gpu
@pytest.mark.parametrize("optimizer", ["sgd", "adagrad"])
def test_dlrm_fast_world1(optimizer):
  launch("case_dlrm_fast_step", world=1, device_type="cuda", backend="fused", optimizer=optimizer)


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("optimizer", ["sgd", "adagrad", "rowwise_adagrad"])
def test_dlrm_fast_world2(optimizer):
  launch("case_dlrm_fast_step", world=2, device_type="cuda", backend="fused", optimizer=optimizer)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 4])
def test_fuzz_plans_fused(world):
  if torch.cuda.device_count() < world:
    pytest.skip(f"needs {world} GPUs")
  launch("case_fuzz", world=world, device_type="cuda", backend="fused", n_seeds=12,
         seed0=500 * world)


@pytest.mark.gpu
@pytest.mark.multigpu
def test_subgroups_fused():
  if torch.cuda.device_count() < 4:
    pytest.skip("needs 4 GPUs")
  launch("case_subgroups", world=4, device_type="cuda", backend="fused")


@pytest.mark.gpu
@pytest.mark.multigpu
def test_dlrm_fast_world2_replicated_tables():
  # tables have 200..525 rows x 128: replicate those up to 300 rows
  launch("case_dlrm_fast_step", world=2, device_type="cuda", backend="fused", optimizer="sgd",
         dp_threshold=300 * 128)




@pytest.mark.gpu
@pytest.mark.parametrize("optimizer,dp_input,stride", [("adagrad", False, None), ("sgd", True, None),
                                                        ("adagrad", True, 4), ("adam", False, None)])
def test_synthetic_fast_world1(optimizer, dp_input, stride):
  if optimizer == "adam":
    pytest.skip("the plain-PyTorch oracle of this case covers sgd / adagrad")
  launch("case_synthetic_fast_step", world=1, device_type="cuda", backend="fused",
         optimizer=optimizer, dp_input=dp_input, interact_stride=stride)


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("optimizer,dp_input,stride", [("adagrad", False, None), ("sgd", True, 4)])
def test_synthetic_fast_world2(optimizer, dp_input, stride):
  launch("case_synthetic_fast_step", world=2, device_type="cuda", backend="fused",
         optimizer=optimizer, dp_input=dp_input, interact_stride=stride)


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("case", ["case_all_modes", "case_multihot_dp", "case_fuzz"])
def test_fused_world8(case):
  """The exchange protocol at the full NVSwitch domain (8 ranks): every sharding mode at once,
  multi-hot inputs, and randomised plans, against the unsharded model."""
  if torch.cuda.device_count() < 8:
    pytest.skip("needs 8 GPUs")
  kw = {"n_seeds": 6, "seed0": 4000} if case == "case_fuzz" else {}
  launch(case, world=8, device_type="cuda", backend="fused", timeout=600, **kw)


@pytest.mark.gpu
@pytest.mark.multigpu
def test_dlrm_fast_world8():
  if torch.cuda.device_count() < 8:
    pytest.skip("needs 8 GPUs")
  launch("case_dlrm_fast_step", world=8, device_type="cuda", backend="fused", optimizer="sgd",
         dp_threshold=300 * 128, timeout=600)
