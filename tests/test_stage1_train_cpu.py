"""Stage-1 training on the CPU: p_losses -> backward through the drop-in ControlLDMReferenceOnly with the autograd ops
replaced by the layout-checking, fp16-rounding stand-ins of tests/fake_train_ops.py, held to the gradients the
UNMODIFIED reference's stage-1 model produced (tests/golden/stage1_grad16.npz: use_checkpoint True, the stage-1 freeze).
Its own module, so that the inference tests' model is freed before these build theirs."""
import pytest
import torch

from tests.test_stage1_cpu import TOL, compare_grads, release_memory, stage1_model, train_step


@pytest.fixture(scope="module")
def train_runs():
    from magicdance_b200 import ops
    from tests import fake_train_ops
    with pytest.MonkeyPatch.context() as mp:
        for name in fake_train_ops.PATCHED:
            mp.setattr(ops, name, getattr(fake_train_ops, name))
        m = stage1_model()
        yield m, train_step(m, checkpointing=True), train_step(m, checkpointing=False)
    del m
    release_memory()


def test_training_gradients_match_the_reference(train_runs):
    _, (loss, ld, dx, grads), _ = train_runs
    assert set(ld) == {"train/loss_simple", "train/loss_vlb", "train/loss"}
    compare_grads(loss, dx, grads, TOL)


def test_checkpointing_changes_memory_not_values(train_runs):
    _, on, off = train_runs
    assert torch.equal(on[0], off[0]) and torch.equal(on[2], off[2])
    for k, g in on[3].items():
        assert (g is None) == (off[3][k] is None) and (g is None or torch.equal(g, off[3][k])), k


def test_stage1_freeze_policy(train_runs):
    """the UNet's blocks and `out` get no gradient; its time_embed does; so does every appearance-net parameter up to
    its last norm1 and none after it (hint block included)"""
    model, (_, _, _, grads), _ = train_runs
    dm = model.model.diffusion_model
    frozen = [p for blk in list(dm.input_blocks) + [dm.middle_block] + list(dm.output_blocks) + list(dm.out)
              for p in blk.parameters()]
    assert frozen and all(p.grad is None and not p.requires_grad for p in frozen)
    assert all(p.grad is not None for p in dm.time_embed.parameters())
    dead = [k for k, g in grads.items() if g is None]
    assert len(dead) == 36 and all(k.startswith("control_model.") for k in dead)
    assert all(p.grad is None for p in model.control_model.input_hint_block.parameters())
