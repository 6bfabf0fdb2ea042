"""train_tiktok.py's data-parallel step (DDP + ZeroRedundancyOptimizer) on the CPU over gloo, at world sizes 2 and 3,
for stage 2 (cldm_v15_reference_only_pose.yaml) and stage 1 (cldm_v15_reference_only.yaml): the kernels are the
layout-checking PyTorch stand-ins of tests/fake_ops.py and tests/fake_train_ops.py, the networks are the yaml's with 128
model channels, the latent 16x16.  tests/ddp_train_cases.py lists the properties each rank checks over two steps."""
import pytest

from tests import ddp_train_cases as D

# fp32 sums in another order, and fp16 roundings of the activation gradients that move with the per-rank scale
GRAD_REL_L2 = 1e-2


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("stage", [2, 1])
def test_ddp_zero_training_step_gloo(stage, world):
    reports = D.run(world, "gloo", stage, small=True, latent=16, per_rank=2, steps=2, device="cpu")
    worst = max(r["b_worst_rel_l2"] for r in reports)
    name = max(reports, key=lambda r: r["b_worst_rel_l2"])["b_worst_param"]
    print(f"stage {stage}, world {world}: worst per-parameter gradient rel-L2 against the single-process batch "
          f"{worst:.3e} ({name}); gradients populated per step {reports[0]['grads']}")
    assert worst <= GRAD_REL_L2
    assert all(r["grads"] == reports[0]["grads"] for r in reports)
