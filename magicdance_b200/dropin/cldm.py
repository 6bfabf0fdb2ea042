"""Drop-in for model_lib/ControlNet/cldm/cldm.py's hot-path classes:

  ControlledUnetModelAttnPose      cldm.py:59-112
  ControlNetReferenceOnly          cldm.py:164-497
  ControlNet                       cldm.py:500-757
  ControlLDMReferenceOnlyPose      cldm.py:1087-1121

Same constructor kwargs (models/cldm_v15_reference_only_pose.yaml), same forward / apply_model
signatures, same state-dict keys.  Tensors cross this boundary exactly as in the reference (NCHW fp32
latents, (B,77,768) context, lists of tensors for the bank and the pose residuals); inside, everything
runs on the sm_90a kernels in fp16 channels-last.
"""
from __future__ import annotations

import torch

from .. import ops, train
from ..engine import DenoiseEngine
from .ddpm import LatentDiffusionReferenceOnly
from .modules import UNetModel
from .util import _one, instantiate_from_config


def _tokens_to_nchw(data, b, h, w):
    return ops.nhwc_f16_to_nchw_f32(data, batch=b, c=data.shape[1], h=h, w=w)


class ControlledUnetModelAttnPose(UNetModel):
    _kind = "unet"

    def forward(self, x, timesteps=None, context=None, control=None, pose_control=None, only_mid_control=False,
                attention_mode=None, uc=False, **kwargs):
        """cldm.py:60-112.  control = attention bank as produced by ControlNetReferenceOnly.forward (a list
        of [tensor(B,N,C)] entries); pose_control = the 13 NCHW residuals of ControlNet.forward.  Both are
        consumed (the reference pops pose_control; so do we)."""
        assert not only_mid_control, "only_mid_control is not used by MagicPose (yaml: only_mid_control: False)"
        eng = DenoiseEngine.from_packed(self.packed(x.device), None, None)
        t = timesteps.to(device=x.device, dtype=torch.int64)
        if uc:
            return eng.unet_forward(x, t, context, uc=True)
        bank_kv = None
        if control:
            bank = [e[0].reshape(-1, e[0].shape[-1]).to(torch.float16).contiguous() for e in control]
            bank_kv = eng.project_bank(bank, control[0][0].shape[0])
        pose = None
        if pose_control is not None:
            pose = [ops.nchw_f32_to_nhwc_f16(p.float()) for p in pose_control]
            del pose_control[:]
        return eng.unet_forward(x, t, context, bank_kv=bank_kv, pose=pose, uc=False)


class ControlNetReferenceOnly(UNetModel):
    """Appearance Control Model: a UNet twin run in 'write' mode on the reference latent."""
    _kind = "appearance"

    def forward(self, x, hint, timesteps, context, attention_bank=None, attention_mode=None, uc=False, **kwargs):
        """cldm.py:469-497: fills attention_bank with one [norm1(x)] entry per transformer block
        (attention.py:287-298) and returns the (always empty) list of outputs."""
        assert attention_mode == "write" and attention_bank is not None
        eng = DenoiseEngine.from_packed(None, self.packed(x.device), None)
        t = timesteps.to(device=x.device, dtype=torch.int64)
        b = x.shape[0]
        for n1 in eng.appearance_write(x, t, context):
            attention_bank.append([n1.view(b, -1, n1.shape[-1])])
        return []


class ControlNet(UNetModel):
    """OpenPose ControlNet (encoder half + zero convs)."""
    _kind = "controlnet"

    def forward(self, x, hint, timesteps, context, **kwargs):
        """cldm.py:736-757 -> list of 13 NCHW fp32 residuals."""
        eng = DenoiseEngine.from_packed(None, None, self.packed(x.device))
        t = timesteps.to(device=x.device, dtype=torch.int64)
        outs = eng.controlnet(x, eng.hint_features(hint), t, context)
        b, _, h, w = x.shape
        res = []
        for o in outs:
            hw = o.shape[0] // b
            s = int(round((h * w / hw) ** 0.5))
            res.append(_tokens_to_nchw(o, b, h // s, w // s))
        return res


class ControlLDMReferenceOnlyPose(LatentDiffusionReferenceOnly):
    def __init__(self, control_key, only_mid_control, appearance_control_stage_config, pose_control_stage_config,
                 *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.control_key = control_key
        self.only_mid_control = only_mid_control
        self.control_enabled = True
        self.appearance_control_model = instantiate_from_config(appearance_control_stage_config)
        self.pose_control_model = instantiate_from_config(pose_control_stage_config)
        self._engine = None

    # ---- engine over the three sub-networks' (lazily) packed weights ----------------------------------
    def engine(self, device=None) -> DenoiseEngine:
        dev = torch.device(device) if device is not None else self.device
        nets = (self.model.diffusion_model, self.appearance_control_model, self.pose_control_model)
        packed = [n.packed(dev) for n in nets]
        if self._engine is None or any(a is not b for a, b in zip(self._engine_nets, packed)):
            self._engine = DenoiseEngine.from_packed(*packed)
            self._engine_nets = packed
        return self._engine

    def _nets(self):
        return self.model.diffusion_model, self.appearance_control_model, self.pose_control_model

    def wants_grad(self, x_noisy):
        """Does this call build a graph?  Grad mode on, and x_noisy or any parameter of the three nets requires grad."""
        if not torch.is_grad_enabled():
            return False
        return x_noisy.requires_grad or any(p.requires_grad for n in self._nets() for p in n.parameters())

    def apply_model(self, x_noisy, t, cond, reference_image_noisy, uc=False, *args, **kwargs):
        """cldm.py:1099-1117 — same arguments, returns eps (B,4,h,w) fp32.  Differentiable (magicdance_b200.train)
        when grad mode is on and something requires grad; the inference engine otherwise."""
        assert isinstance(cond, dict)
        assert not self.only_mid_control
        cond_txt = _one(cond["c_crossattn"])
        if self.control_enabled and cond.get("c_crossattn_void") is not None:
            raise NotImplementedError("c_crossattn_void is never passed by the MagicPose scripts")
        assert self.control_enabled and cond.get("c_concat") is not None, "the pose map (c_concat) is required"
        cond_hint = _one(cond["c_concat"])
        if not uc and self.wants_grad(x_noisy):
            nets = self._nets()
            eps = train.apply_model(*nets, x_noisy, t, cond_txt, cond_hint, reference_image_noisy)
            for n in nets:  # an optimizer step will change these weights, maybe without bumping version counters
                if any(p.requires_grad for p in n.parameters()):
                    n.invalidate()
            return eps
        eng = self.engine(x_noisy.device)
        return eng.apply_model(x_noisy, t, cond_txt, cond_hint, reference_image_noisy, uc=uc)

    @torch.no_grad()
    def get_unconditional_conditioning(self, N):
        return self.get_learned_conditioning([""] * N)
