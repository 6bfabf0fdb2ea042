"""GPU parity of the VAE decoder and encoder in magicdance_b200/vae.py against the pinned CPU oracle and
the reference goldens.  Run on an H100:

    python tests/gpu_vae_parity_report.py            # latent 16 (B=2) and latent 64 (B=1)

Gates: rel-L2 <= 5e-3 against the reference golden image (fp16 storage / fp32 accumulate vs fp32), per stage
taps are printed to localise a failure.
"""
import json
import os
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from magicdance_b200 import ops, synth  # noqa: E402
from magicdance_b200.vae import PackedVaeDecoder, PackedVaeEncoder, VaeDecoder, VaeEncoder  # noqa: E402
from oracle import vae_restatement as V  # noqa: E402  (checker only)

TOL = 5e-3


def rel(a, b):
    a, b = a.double().reshape(-1).cpu(), b.double().reshape(-1).cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def main():
    torch.set_grad_enabled(False)
    with open(os.path.join(REPO, "magicdance_b200", "vae_manifest.json")) as f:
        manifest = json.load(f)
    sd = synth.synth_state_dict(manifest, seed=0)
    dec = VaeDecoder(PackedVaeDecoder(sd, "cuda"))
    bad = 0
    # unit check of the new softmax kernel
    x = torch.randn(300, 4096, device="cuda").half() * 4
    ref = torch.softmax(x.float() * 0.37, dim=1)
    got = ops.softmax_rows(x.clone(), 0.37).float()
    e = rel(got, ref)
    print(f"softmax_rows 300x4096: rel-L2 {e:.2e}")
    bad += e > 2e-3
    # GroupNorm with 4 channels per group (the VAE's 128-channel level)
    xg = torch.randn(2 * 1024, 128, device="cuda").half()
    g_, b_ = torch.randn(128, device="cuda") * 0.1 + 1, torch.randn(128, device="cuda") * 0.1
    yg = ops.groupnorm(xg, g_, b_, batch=2, hw=1024, eps=1e-6, silu=True).float()
    rg = torch.nn.functional.silu(torch.nn.functional.group_norm(
        xg.float().reshape(2, 1024, 128).permute(0, 2, 1), 32, g_, b_, eps=1e-6)).permute(0, 2, 1).reshape(2048, 128)
    e = rel(yg, rg)
    print(f"groupnorm c=128 (4 channels per group): rel-L2 {e:.2e}")
    bad += e > 2e-3
    for batch, latent, gname in ((2, 16, "vae16"), (1, 64, "vae64")):
        z, _, _ = V.vae_inputs(batch, latent)
        t0 = time.time()
        img = dec.decode(z.cuda())
        torch.cuda.synchronize()
        dt = time.time() - t0
        oracle = V.decode_first_stage(sd, z)
        e = rel(img, oracle)
        print(f"decode latent {latent} B={batch}: rel-L2 vs CPU oracle {e:.3e} (first call {dt * 1e3:.1f} ms, "
              f"finite={bool(torch.isfinite(img).all())})")
        bad += not (e <= TOL)
        g = np.load(os.path.join(REPO, "tests", "golden", gname + ".npz"))
        if gname + "/decoded" in g.files:
            e2 = rel(img, torch.from_numpy(g[gname + "/decoded"]))
            print(f"   vs reference golden: {e2:.3e}")
            bad += not (e2 <= TOL)
        if latent == 64:
            for _ in range(2):
                dec.decode(z.cuda())
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                dec.decode(z.cuda())
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 5
            print(f"   decode 64x64 -> 512x512: {ms:.2f} ms/frame = {2514.5 / ms:.1f} TFLOP/s (2514.5 GFLOP per frame)")
    # ---- encoder (encode_first_stage): the br-padded im2col, then the whole stack against the golden moments ----
    xi = torch.randn(2 * 16 * 16, 64, device="cuda").half()
    col = ops.im2col3x3(xi, batch=2, h=16, w=16, c=64, stride=2, pad="br").float()
    xp = torch.nn.functional.pad(xi.float().reshape(2, 16, 16, 64).permute(0, 3, 1, 2), (0, 1, 0, 1))
    rc = torch.nn.functional.unfold(xp, 3, padding=0, stride=2).reshape(2, 64, 9, 64).permute(0, 3, 2, 1).reshape(128, 576)
    e = rel(col, rc)
    print(f"im2col3x3 pad=br stride 2: rel-L2 {e:.2e}")
    bad += e > 1e-6
    enc = VaeEncoder(PackedVaeEncoder(sd, "cuda"))
    for batch, latent, gname in ((2, 16, "vae16"), (1, 64, None)):
        _, img_in, noise = V.vae_inputs(batch, latent)
        t0 = time.time()
        mom = enc.encode(img_in.cuda())
        torch.cuda.synchronize()
        dt = time.time() - t0
        oracle = V.vae_encode_moments(sd, img_in)
        e = rel(mom, oracle)
        print(f"encode {latent * 8}x{latent * 8} B={batch}: moments rel-L2 vs CPU oracle {e:.3e} (first call {dt * 1e3:.1f} ms, "
              f"finite={bool(torch.isfinite(mom).all())})")
        bad += not (e <= TOL)
        if gname:
            g = np.load(os.path.join(REPO, "tests", "golden", gname + ".npz"))
            e2 = rel(mom, torch.from_numpy(g[gname + "/moments"]))
            print(f"   vs reference golden moments: {e2:.3e}")
            bad += not (e2 <= TOL)
    print("FAILED" if bad else "OK")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
