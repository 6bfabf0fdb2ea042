"""Inputs of tests/golden/anysize40x24.npz (oracle/make_golden_anysize.py: anysize_inputs, the same recipe), and the
check that they still are what the golden was made from (its input fingerprints)."""
import os

import numpy as np
import torch

H, W = 40, 24
KEYS = ("x", "ref", "pose", "context", "t", "x0", "noise", "t_train", "uc_context")


def anysize_inputs():
    """B = 2 at a 40x24 latent (320x192 pose maps): apply_model and p_losses inputs; uc_context for the chain"""
    g = torch.Generator().manual_seed(4024)
    b = 2
    x = torch.randn(b, 4, H, W, generator=g)
    ref = 0.8 * torch.randn(b, 4, H, W, generator=g)
    u = torch.rand(b, 3, 8 * H, 8 * W, generator=g)
    v = torch.rand(b, 3, 8 * H, 8 * W, generator=g)
    pose = torch.where(u > 0.97, v, torch.zeros_like(v))
    context = torch.randn(b, 77, 768, generator=g)
    x0 = 0.9 * torch.randn(b, 4, H, W, generator=g)
    noise = torch.randn(b, 4, H, W, generator=g)
    uc_context = torch.randn(1, 77, 768, generator=g)
    return {"x": x, "ref": ref, "pose": pose, "context": context, "t": torch.tensor([621, 135]), "x0": x0,
            "noise": noise, "t_train": torch.tensor([812, 97]), "uc_context": uc_context}


def fingerprints(inp):
    return np.array([float(inp[k].double().sum()) for k in KEYS])


def load():
    """(golden, inputs), the inputs checked against the fingerprints the golden stores"""
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "anysize40x24.npz"))
    inp = anysize_inputs()
    assert np.allclose(fingerprints(inp), gold["inputs/sums"], rtol=1e-9, atol=1e-6), "the inputs changed"
    return gold, inp


def _rel(a, b):
    a, b = a.detach().double().reshape(-1).cpu(), b.detach().double().reshape(-1).cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def compare_grads(gold, loss, dx, grads, tol):
    """worst errors of (loss, d_x_noisy, trained-parameter gradients) against the golden's grad16-layout record, each
    checked against tol[name] (the grad16 gates); returns them"""
    names = [str(n) for n in gold["names"]]
    assert sorted(names) == sorted(grads)
    worst = {"loss": abs(float(loss) - float(gold["loss"])) / float(gold["loss"]),
             "d_x_noisy": _rel(dx, torch.from_numpy(gold["d_x_noisy"])), "norm": 0.0, "sample": 0.0, "sum": 0.0,
             "full": 0.0}
    reached = {n for n in names if grads[n] is not None and float(grads[n].abs().max()) > 0}
    assert reached == {n for n, h, g in zip(names, gold["has_grad"], gold["gnorm"]) if h and float(g) > 0}
    for i, n in enumerate(names):
        if n not in reached:
            continue
        g = grads[n].double().cpu().flatten()
        norm = float(gold["gnorm"][i])
        worst["norm"] = max(worst["norm"], abs(float(g.norm()) - norm) / norm)
        pos = np.arange(g.numel()) if g.numel() <= 16 else (np.arange(16, dtype=np.int64) * (g.numel() - 1)) // 15
        err = float((g[torch.from_numpy(pos)] - torch.from_numpy(gold["gsample"][i, :len(pos)])).norm()) / (
            norm / np.sqrt(g.numel()) * np.sqrt(len(pos)))
        worst["sample"] = max(worst["sample"], err)
        worst["sum"] = max(worst["sum"], abs(float(g.sum()) - float(gold["gsum"][i])) / (norm * np.sqrt(g.numel())))
    for key in gold.files:
        if key.startswith("full/"):
            worst["full"] = max(worst["full"], _rel(grads[key[5:]], torch.from_numpy(gold[key])))
    print({k: f"{v:.3e}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v <= tol[k], (k, v, tol[k])
    return worst
