"""TEST INFRASTRUCTURE — exact FLOP count of one TRAINING sample of the reference (SURVEY 8d: "measure with the same
counter ... and publish the exact figure"), by running the UNMODIFIED reference's `p_losses` -> `backward()` under
torch.utils.flop_counter.FlopCounterMode on the CPU, at the training shape (latent 64x64, B = 1), stage-2 freeze policy
(train_tiktok.py:798-822), once with `use_checkpoint: True` (the yaml: CheckpointFunction recomputes every ResBlock and
CrossAttention inside backward, util.py:118-187) and once without.

Run in the build container only (needs /root/reference):

    python oracle/count_training_flops.py      # writes profiles/r02_training_flops.md
"""
from __future__ import annotations

import importlib.util
import os
import sys
import time

import torch
from torch.utils.flop_counter import FlopCounterMode

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO in sys.path:
    sys.path.remove(REPO)
sys.path.append(REPO)


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    sys.modules[name] = m
    spec.loader.exec_module(m)
    return m


grad = _load("mdb_oracle_make_golden_grad", os.path.join(REPO, "oracle", "make_golden_grad.py"))
ref_shim, synth = grad.ref_shim, grad.synth  # ONE import of the reference per process


def count(use_checkpoint, weights, inp):
    model = grad.build(use_checkpoint, weights)
    cond = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]], "image_control": [inp["ref"]], "wonoise": True}
    g = torch.Generator().manual_seed(3)
    x0 = torch.randn(1, 4, 64, 64, generator=g)
    noise = torch.randn(1, 4, 64, 64, generator=g)
    t = torch.tensor([500], dtype=torch.long)
    out = {}
    with FlopCounterMode(display=False) as fwd:
        loss, _ = model.p_losses(x0, cond, t, noise=noise)
    out["forward"] = fwd.get_total_flops()
    t0 = time.time()
    with FlopCounterMode(display=False) as bwd:
        loss.backward()
    out["backward"] = bwd.get_total_flops()
    out["backward_by_op"] = {str(k): v for k, v in bwd.get_flop_counts().get("Global", {}).items()}
    out["seconds_backward"] = time.time() - t0
    return out


def main():
    torch.manual_seed(0)
    probe = ref_shim.build_reference_ldm()
    manifest = {k: list(v.shape) for k, v in probe.state_dict().items()}
    del probe
    weights = synth.synth_state_dict(manifest, seed=0)
    inp = synth.synth_inputs(1, 64, seed=0, shared_reference=True)
    rows = {}
    for flag in (True, False):
        rows[flag] = count(flag, weights, inp)
        print(flag, {k: v for k, v in rows[flag].items() if k != "backward_by_op"}, flush=True)
    ck, pl = rows[True], rows[False]
    path = os.path.join(REPO, "profiles", "r02_training_flops.md")
    with open(path, "w") as f:
        f.write("# FLOPs of one training sample of the REFERENCE (oracle/count_training_flops.py; CPU, FlopCounterMode, multiply-add = 2)\n\n")
        f.write("`LatentDiffusionReferenceOnly.p_losses` -> `backward()`, latent 64x64 (512x512 image), B = 1, stage-2 freeze policy\n"
                "(SD UNet frozen: dgrad only; appearance net + pose ControlNet trained: dgrad + wgrad).  The forward as the reference\n"
                "executes it in training: appearance pass + pose ControlNet + UNet read (no unconditional call).\n\n")
        f.write("| | forward | backward | total per sample |\n|---|---|---|---|\n")
        f.write("| `use_checkpoint: True` (the yaml; backward includes the recompute of every ResBlock / CrossAttention) | %.1f GF | %.1f GF | **%.1f GF** |\n"
                % (ck["forward"] / 1e9, ck["backward"] / 1e9, (ck["forward"] + ck["backward"]) / 1e9))
        f.write("| `use_checkpoint: False` | %.1f GF | %.1f GF | %.1f GF |\n"
                % (pl["forward"] / 1e9, pl["backward"] / 1e9, (pl["forward"] + pl["backward"]) / 1e9))
        f.write("\nRecompute share of the checkpointed backward: %.1f GF (= %.2f of one forward).\n"
                % ((ck["backward"] - pl["backward"]) / 1e9, (ck["backward"] - pl["backward"]) / pl["forward"]))
        f.write("\nBackward by operator (checkpointed run):\n\n| aten op | GF |\n|---|---|\n")
        for k, v in sorted(ck["backward_by_op"].items(), key=lambda kv: -kv[1]):
            f.write("| `%s` | %.1f |\n" % (k, v / 1e9))
    print("wrote", path)


if __name__ == "__main__":
    main()
