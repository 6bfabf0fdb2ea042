"""Drop-in for model_lib/ControlNet/cldm/cldm.py's hot-path classes:

  ControlledUnetModelAttnPose      cldm.py:59-112
  ControlledUnetModelAttn          cldm.py:115-161
  ControlNetReferenceOnly          cldm.py:164-497
  ControlNet                       cldm.py:500-757
  ControlLDMReferenceOnly          cldm.py:1055-1081   (stage-1 appearance-control pre-training)
  ControlLDMReferenceOnlyPose      cldm.py:1087-1121

Same constructor kwargs (models/cldm_v15_reference_only_pose.yaml, models/cldm_v15_reference_only.yaml), same forward / apply_model
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


def _unet_forward(module, x, timesteps, context, control, pose_control, only_mid_control, uc):
    """the UNet in 'read' mode: control = attention bank as produced by ControlNetReferenceOnly.forward (a list of
    [tensor(B,N,C)] entries, or empty); pose_control = the 13 NCHW residuals of ControlNet.forward, or None"""
    assert not only_mid_control, "only_mid_control is not used by MagicPose (yaml: only_mid_control: False)"
    eng = DenoiseEngine.from_packed(module.packed(x.device), None, None)
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


class ControlledUnetModelAttnPose(UNetModel):
    _kind = "unet"

    def forward(self, x, timesteps=None, context=None, control=None, pose_control=None, only_mid_control=False,
                attention_mode=None, uc=False, **kwargs):
        """cldm.py:60-112.  The bank and the pose residuals are both consumed (the reference pops pose_control;
        so do we)."""
        return _unet_forward(self, x, timesteps, context, control, pose_control, only_mid_control, uc)


class ControlledUnetModelAttn(UNetModel):
    """The stage-1 UNet: ControlledUnetModelAttnPose without pose residuals."""
    _kind = "unet"

    def forward(self, x, timesteps=None, context=None, control=None, pose_control=None, only_mid_control=False,
                attention_mode=None, uc=False, **kwargs):
        """cldm.py:116-161: the same signature as ControlledUnetModelAttnPose.forward; pose_control is ignored (and
        left as it is).  In 'read' mode every input, middle and output block reads the bank; uc=True is the plain
        SD UNet."""
        return _unet_forward(self, x, timesteps, context, control, None, only_mid_control, uc)


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


class _ControlLDM(LatentDiffusionReferenceOnly):
    """What the stage-1 and stage-2 models share: the engine over their networks' packed weights and the choice
    between the training path and the inference engine."""

    def _nets(self):
        """(SD UNet, appearance net, pose ControlNet or None)"""
        raise NotImplementedError

    # ---- engine over the sub-networks' (lazily) packed weights ----------------------------------------
    def engine(self, device=None) -> DenoiseEngine:
        dev = torch.device(device) if device is not None else self.device
        packed = [None if n is None else n.packed(dev) for n in self._nets()]
        if self._engine is None or any(a is not b for a, b in zip(self._engine_nets, packed)):
            self._engine = DenoiseEngine.from_packed(*packed)
            self._engine_nets = packed
        return self._engine

    def wants_grad(self, x_noisy):
        """Does this call build a graph?  Grad mode on, and x_noisy or any parameter of the networks requires grad."""
        if not torch.is_grad_enabled():
            return False
        return x_noisy.requires_grad or any(p.requires_grad for n in self._nets() if n is not None
                                            for p in n.parameters())

    def _train_apply(self, x_noisy, t, cond_txt, cond_hint, reference_image_noisy):
        """the differentiable forward (magicdance_b200.train); the packing of every net it trains is dropped"""
        nets = self._nets()
        eps = train.apply_model(*nets, x_noisy, t, cond_txt, cond_hint, reference_image_noisy)
        for n in nets:  # an optimizer step will change these weights, maybe without bumping version counters
            if n is not None and any(p.requires_grad for p in n.parameters()):
                n.invalidate()
        return eps

    @torch.no_grad()
    def get_unconditional_conditioning(self, N):
        return self.get_learned_conditioning([""] * N)


class ControlLDMReferenceOnly(_ControlLDM):
    """Stage-1 appearance-control pre-training (models/cldm_v15_reference_only.yaml): the SD UNet reads the bank that
    the appearance net `control_model` writes; there is no pose ControlNet."""

    def __init__(self, control_key, only_mid_control, control_stage_config, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.control_key = control_key
        self.only_mid_control = only_mid_control
        self.control_enabled = True
        self.control_model = instantiate_from_config(control_stage_config)
        self._engine = None

    def _nets(self):
        return self.model.diffusion_model, self.control_model, None

    def apply_model(self, x_noisy, t, cond, reference_image_noisy, uc=False, *args, **kwargs):
        """cldm.py:1067-1077 — same arguments, returns eps (B,4,h,w) fp32.  cond['c_concat'] (a pose map, which the
        reference's training script passes anyway) is ignored; reference_image_noisy None means no bank.
        Differentiable (magicdance_b200.train) when grad mode is on and something requires grad; the inference
        engine otherwise."""
        assert isinstance(cond, dict)
        assert not self.only_mid_control
        cond_txt = _one(cond["c_crossattn"])
        if not uc and self.wants_grad(x_noisy):
            return self._train_apply(x_noisy, t, cond_txt, None, reference_image_noisy)
        eng = self.engine(x_noisy.device)
        return eng.apply_model(x_noisy, t, cond_txt, None, reference_image_noisy, uc=uc)


class ControlLDMReferenceOnlyPose(_ControlLDM):
    def __init__(self, control_key, only_mid_control, appearance_control_stage_config, pose_control_stage_config,
                 *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.control_key = control_key
        self.only_mid_control = only_mid_control
        self.control_enabled = True
        self.appearance_control_model = instantiate_from_config(appearance_control_stage_config)
        self.pose_control_model = instantiate_from_config(pose_control_stage_config)
        self._engine = None

    def _nets(self):
        return self.model.diffusion_model, self.appearance_control_model, self.pose_control_model

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
            return self._train_apply(x_noisy, t, cond_txt, cond_hint, reference_image_noisy)
        eng = self.engine(x_noisy.device)
        return eng.apply_model(x_noisy, t, cond_txt, cond_hint, reference_image_noisy, uc=uc)
