"""Drop-in for the reference's first-stage VAE class (model_lib/ControlNet/ldm/models/autoencoder.py:13-91):
same constructor kwargs, the same 248 state-dict keys and shapes (`encoder.*`, `decoder.*`, `quant_conv.*`,
`post_quant_conv.*`, recorded from the unmodified reference in magicdance_b200/vae_manifest.json), the same
`encode(x) -> posterior` / `decode(z) -> image` / `forward(input, sample_posterior)` calls — running on the hot
path's kernels through magicdance_b200/vae.py.

Checked against the goldens of the unmodified reference AutoencoderKL (tests/test_vae_gpu.py: decode and encode
within rel-L2 5e-3 at fp16 storage) and re-exported under the reference's dotted path
`model_lib/ControlNet/ldm/models/autoencoder.py`, so the YAML's first_stage_config resolves to it.
Parameters stay fp32 in PyTorch-native layouts (checkpoint compatible); the fp16 kernel layouts are packed lazily on
the GPU and dropped by load_state_dict.  Inference only: no loss, no EMA, no training_step.
"""
from __future__ import annotations

import json
import os

import torch
import torch.nn as nn

from .. import ops, vae

_MANIFEST = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vae_manifest.json")
_SUPPORTED = dict(double_z=True, z_channels=4, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2, 4, 4], num_res_blocks=2,
                  attn_resolutions=[], dropout=0.0)  # yaml:98-112; `resolution` only sizes the (absent) attention maps


class DiagonalGaussianDistribution:
    """ldm/modules/distributions/distributions.py:24-60 over the [B, 8, h, w] moments the encoder returns."""

    def __init__(self, parameters: torch.Tensor, deterministic: bool = False):
        self.parameters = parameters
        self.mean, logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if deterministic:
            self.var = self.std = torch.zeros_like(self.mean)

    def sample(self):
        return self.mean + self.std * torch.randn(self.mean.shape, device=self.parameters.device)

    def mode(self):
        return self.mean

    def kl(self, other=None):
        if self.deterministic:
            return torch.zeros((), device=self.parameters.device)
        if other is None:
            return 0.5 * torch.sum(self.mean ** 2 + self.var - 1.0 - self.logvar, dim=[1, 2, 3])
        return 0.5 * torch.sum((self.mean - other.mean) ** 2 / other.var + self.var / other.var - 1.0 - self.logvar
                               + other.logvar, dim=[1, 2, 3])


def _register_tree(root: nn.Module, shapes: dict):
    """Registers one fp32 nn.Parameter per dotted name, creating plain nn.Module containers on the way, so that
    state_dict() yields exactly the reference's keys ('decoder.up.3.block.0.norm1.weight', ...)."""
    for name, shape in shapes.items():
        parts = name.split(".")
        mod = root
        for p in parts[:-1]:
            if p not in mod._modules:
                mod.add_module(p, nn.Module())
            mod = mod._modules[p]
        t = torch.empty(tuple(shape), dtype=torch.float32)
        if t.dim() > 1:
            nn.init.kaiming_uniform_(t, a=5 ** 0.5)  # Conv2d's default; a checkpoint overwrites it anyway
        elif parts[-1] == "weight" and "norm" in parts[-2]:
            nn.init.ones_(t)
        else:
            nn.init.zeros_(t)
        mod.register_parameter(parts[-1], nn.Parameter(t, requires_grad=False))


class AutoencoderKL(nn.Module):
    def __init__(self, ddconfig, lossconfig=None, embed_dim=4, ckpt_path=None, ignore_keys=(), image_key="image",
                 colorize_nlabels=None, monitor=None, ema_decay=None, learn_logvar=False):
        super().__init__()
        dd = {k: (list(v) if isinstance(v, (list, tuple)) or type(v).__name__ == "ListConfig" else v)
              for k, v in dict(ddconfig).items()}
        for k, want in _SUPPORTED.items():
            got = dd.get(k, want)
            if (list(got) if isinstance(want, list) else got) != want:
                raise NotImplementedError(f"magicdance_b200 AutoencoderKL supports the SD1.5 first stage only "
                                          f"(ddconfig.{k}={got!r}, expected {want!r})")
        assert embed_dim == 4 and ema_decay is None and colorize_nlabels is None and not learn_logvar
        self.embed_dim, self.image_key = embed_dim, image_key
        if monitor is not None:
            self.monitor = monitor
        with open(_MANIFEST) as f:
            manifest = json.load(f)
        _register_tree(self, {k[len(vae.PREFIX):]: v for k, v in manifest.items() if k.startswith(vae.PREFIX)})
        self._dec = self._enc = None
        self.register_load_state_dict_post_hook(lambda module, incompatible: module._drop_packed())
        if ckpt_path is not None:
            self.init_from_ckpt(ckpt_path, ignore_keys=ignore_keys)

    # ---- checkpoint plumbing (autoencoder.py:50-60) ---------------------------------------------------
    def init_from_ckpt(self, path, ignore_keys=()):
        sd = torch.load(path, map_location="cpu")["state_dict"]
        sd = {k: v for k, v in sd.items() if not any(k.startswith(ik) for ik in ignore_keys)}
        self.load_state_dict(sd, strict=False)
        print(f"Restored from {path}")

    def _drop_packed(self):
        self._dec = self._enc = None

    def _apply(self, fn, *a, **kw):  # .cuda() / .to(): the packed copies live on the old device
        self._drop_packed()
        return super()._apply(fn, *a, **kw)

    def _prefixed_state(self):
        return {vae.PREFIX + k: v for k, v in self.state_dict().items()}

    def _device(self):
        dev = next(self.parameters()).device
        ops.require_cuda(dev)
        return dev

    def decoder_engine(self) -> vae.VaeDecoder:
        if self._dec is None:
            self._dec = vae.VaeDecoder(vae.PackedVaeDecoder(self._prefixed_state(), self._device(), scale_factor=1.0))
        return self._dec

    def encoder_engine(self) -> vae.VaeEncoder:
        if self._enc is None:
            self._enc = vae.VaeEncoder(vae.PackedVaeEncoder(self._prefixed_state(), self._device()))
        return self._enc

    # ---- the reference's calls (autoencoder.py:82-102) -------------------------------------------------
    @torch.no_grad()
    def encode(self, x):
        return DiagonalGaussianDistribution(self.encoder_engine().encode(x))

    @torch.no_grad()
    def decode(self, z):
        """z is the UNSCALED latent here (the LDM divides by scale_factor before calling, ddpm.py:2107)."""
        return self.decoder_engine().decode(z)

    def forward(self, input, sample_posterior=True):
        posterior = self.encode(input)
        z = posterior.sample() if sample_posterior else posterior.mode()
        return self.decode(z), posterior

    def get_last_layer(self):
        return self.decoder.conv_out.weight


class IdentityFirstStage(nn.Module):
    """ldm/models/autoencoder.py:201-219: a first stage that returns its input (used by configs without a VAE)"""

    def __init__(self, *args, vq_interface=False, **kwargs):
        super().__init__()
        self.vq_interface = vq_interface

    def encode(self, x, *args, **kwargs):
        return x

    def decode(self, x, *args, **kwargs):
        return x

    def quantize(self, x, *args, **kwargs):
        return (x, None, [None, None, None]) if self.vq_interface else x

    def forward(self, x, *args, **kwargs):
        return x
