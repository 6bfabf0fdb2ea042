"""Drop-in for DDIMSampler_ReferenceOnly (model_lib/ControlNet/ldm/models/diffusion/ddim.py:346-730):
same constructor, make_schedule / sample / ddim_sampling / p_sample_ddim signatures and return values,
for the configuration the MagicPose scripts drive (test_tiktok.py:261-268, and the sample logging of
train_tiktok.py:437-444 for both training stages): eps-prediction, DDIM, classifier-free guidance through the
'controlnet is more important' branch (ddim.py:598-605).  A stage-1 model (ControlLDMReferenceOnly) has no pose
ControlNet: the same step runs without hint features and pose residuals.

Host code only: the step itself (pose ControlNet, paired conditional/unconditional UNet, fused
CFG + DDIM update) runs on the sm_90a kernels via magicdance_b200.pipeline.DenoisePipeline, which also
keeps the per-sequence caches (text K/V, per-timestep appearance bank, per-frame hint features) across
the frames of a video — the reference recomputes all of them for every frame and step.
"""
from __future__ import annotations


import numpy as np
import torch

from ..engine import tensor_key
from ..pipeline import DenoisePipeline, ddim_parameters, ddim_timesteps_uniform
from .util import _one


class DDIMSampler_ReferenceOnly(object):
    # ddim_sampling replays the captured step / bank-build CUDA graphs (pipeline.GraphedDenoiser — the code bench.py
    # times) whenever the call is the one the MagicPose scripts make; False forces the eager per-step loop.
    use_graphs = True

    def __init__(self, model, schedule="linear", **kwargs):
        super().__init__()
        self.model = model
        self.ddpm_num_timesteps = model.num_timesteps
        self.schedule = schedule

    def register_buffer(self, name, attr):
        setattr(self, name, attr)

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=True):
        """ddim.py:359-388 (uniform discretisation)."""
        assert ddim_discretize == "uniform"
        acp = self.model.alphas_cumprod.detach().cpu().numpy().astype(np.float32)
        self.ddim_timesteps = ddim_timesteps_uniform(ddim_num_steps, self.ddpm_num_timesteps)
        sig, a, a_prev = ddim_parameters(acp, self.ddim_timesteps, ddim_eta)
        self.ddim_sigmas, self.ddim_alphas, self.ddim_alphas_prev = sig, a, a_prev
        self.ddim_sqrt_one_minus_alphas = np.sqrt(1.0 - a)
        self.ddim_eta = ddim_eta
        self.alphas_cumprod = acp

    def _pipeline(self, scale) -> DenoisePipeline:
        """One pipeline (and its caches) per (steps, eta, scale), kept on the model so that successive
        sample_log() calls for the frames of one video share the appearance bank and the text K/V."""
        cache = self.model.__dict__.setdefault("_mdb_pipelines", {})
        key = (len(self.ddim_timesteps), float(self.ddim_eta), float(scale))
        eng = self.model.engine()
        pipe = cache.get(key)
        if pipe is None or pipe.engine is not eng:
            cache.clear()
            pipe = DenoisePipeline(eng, ddim_steps=key[0], scale=scale, eta=self.ddim_eta,
                                   alphas_cumprod=self.alphas_cumprod)
            cache[key] = pipe
        return pipe

    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, callback=None, normals_sequence=None, img_callback=None,
               quantize_x0=False, eta=0., mask=None, x0=None, temperature=1., noise_dropout=0., score_corrector=None,
               corrector_kwargs=None, verbose=True, x_T=None, log_every_t=100, unconditional_guidance_scale=1.,
               unconditional_conditioning=None, dynamic_threshold=None, ucg_schedule=None, inpaint=None, **kwargs):
        """ddim.py:390-458"""
        self.make_schedule(ddim_num_steps=S, ddim_eta=eta, verbose=verbose)
        C, H, W = shape
        return self.ddim_sampling(conditioning, (batch_size, C, H, W), callback=callback, img_callback=img_callback,
                                  quantize_denoised=quantize_x0, mask=mask, x0=x0, x_T=x_T, log_every_t=log_every_t,
                                  temperature=temperature, noise_dropout=noise_dropout, score_corrector=score_corrector,
                                  corrector_kwargs=corrector_kwargs,
                                  unconditional_guidance_scale=unconditional_guidance_scale,
                                  unconditional_conditioning=unconditional_conditioning,
                                  dynamic_threshold=dynamic_threshold, ucg_schedule=ucg_schedule, inpaint=inpaint)

    @torch.no_grad()
    def ddim_sampling(self, cond, shape, x_T=None, ddim_use_original_steps=False, callback=None, timesteps=None,
                      quantize_denoised=False, mask=None, x0=None, img_callback=None, log_every_t=100, temperature=1.,
                      noise_dropout=0., score_corrector=None, corrector_kwargs=None, unconditional_guidance_scale=1.,
                      unconditional_conditioning=None, dynamic_threshold=None, ucg_schedule=None, inpaint=None):
        """ddim.py:460-516"""
        if ddim_use_original_steps or timesteps is not None or mask is not None or ucg_schedule is not None:
            raise NotImplementedError("DDIMSampler_ReferenceOnly.ddim_sampling: ddim_use_original_steps / timesteps / mask / "
                                      "ucg_schedule are not used by the MagicPose scripts and are not implemented")
        device = self.model.betas.device
        b = shape[0]
        img = torch.randn(shape, device=device) if x_T is None else x_T.to(device)
        intermediates = {"x_inter": [img], "pred_x0": [img]}
        total = self.ddim_timesteps.shape[0]
        if (self.use_graphs and not quantize_denoised and temperature == 1.
                and noise_dropout == 0. and score_corrector is None and dynamic_threshold is None and inpaint is None):
            out = self._ddim_sampling_graphed(cond, img, unconditional_guidance_scale, unconditional_conditioning,
                                              callback, img_callback, log_every_t, intermediates)
            if out is not None:
                return out
        for i, step in enumerate(np.flip(self.ddim_timesteps)):
            index = total - i - 1
            ts = torch.full((b,), int(step), device=device, dtype=torch.long)
            img, pred_x0 = self.p_sample_ddim(img, cond, ts, index=index, quantize_denoised=quantize_denoised,
                                              temperature=temperature, noise_dropout=noise_dropout,
                                              score_corrector=score_corrector, corrector_kwargs=corrector_kwargs,
                                              unconditional_guidance_scale=unconditional_guidance_scale,
                                              unconditional_conditioning=unconditional_conditioning,
                                              dynamic_threshold=dynamic_threshold, inpaint=inpaint)
            if callback:
                callback(i)
            if img_callback:
                img_callback(pred_x0, i)
            if index % log_every_t == 0 or index == total - 1:
                intermediates["x_inter"].append(img)
                intermediates["pred_x0"].append(pred_x0)
        return img, intermediates

    @torch.no_grad()
    def _ddim_sampling_graphed(self, c, img, scale, uc, callback, img_callback, log_every_t, intermediates):
        """The same chain as the loop above, but every step is
        one replay of pipeline.GraphedDenoiser's captured step graph and the appearance bank of the reference is built
        by its timestep-batched bank graph — what bench.py times — instead of ~650 eager launches per step driven from
        Python.  Returns None (the caller falls back to the eager loop) for anything the graphs do not cover: eta != 0,
        a noised or per-sample reference, no classifier-free guidance, CPU tensors."""
        from .. import parallel
        from ..pipeline import GraphedDenoiser
        if not (isinstance(c, dict) and c.get("image_control") is not None and c.get("wonoise") and uc is not None
                and uc.get("image_control") is None and scale != 1.0 and not c.get("overlap_sampling")
                and not np.any(self.ddim_sigmas) and img.is_cuda):
            return None
        ref, ctx = _one(c["image_control"]), _one(c["c_crossattn"])
        if not (self._rows_identical(ref) and self._rows_identical(ctx)):
            return None  # one reference image and one prompt per batch only (the scripts repeat them per sample)
        pipe = self._pipeline(scale)
        b, _, h, w = img.shape
        total = int(self.ddim_timesteps.shape[0])
        # The captured graphs bake in the text keys/values of the context they were captured with, and the bank slots
        # belong to one reference image.  The scripts build NEW tensors with the SAME content for every frame
        # (get_learned_conditioning([""] * N), the encoded reference image), so both are recognised by content
        # (torch.equal against the copy kept with the graphs), not by identity.
        # Sequence-parallel bank (SURVEY §8e): when the caller has set model.bank_process_group (all ranks of that group
        # sample frames of the SAME reference image in lock-step, e.g. bench.py's config 4), the timesteps of the
        # appearance pass are dealt over the ranks and exchanged once per reference (parallel.build_and_gather_bank).
        group = getattr(self.model, "bank_process_group", None)
        world, rank = 1, 0
        if group is not None:
            import torch.distributed as dist
            world, rank = dist.get_world_size(group), dist.get_rank(group)
        graphs = self.model.__dict__.setdefault("_mdb_graphs", {})
        gkey = (id(pipe), b, h, w, tuple(ctx.shape), world)
        ctx_dev = ctx[:1].to(pipe.device)  # all rows are identical (checked above): one row, broadcast in-kernel
        ent = graphs.get(gkey)
        if ent is None or not torch.equal(ent["ctx"], ctx_dev):
            graphs.clear()  # one captured configuration at a time: each owns gigabytes of graph memory
            ctx_own = ctx_dev.clone()
            gd = GraphedDenoiser(pipe, b, (h, w), ctx_own, bank_chunk=parallel.bank_chunk_size(total, world))
            gd.capture()
            ent = {"gd": gd, "ctx": ctx_own, "ref": None,
                   "storage": parallel.bank_storage((total + world - 1) // world, gd.layout, pipe.device, world)}
            graphs[gkey] = ent
        gd = ent["gd"]
        ref_dev = ref[:1].to(device=pipe.device, dtype=torch.float32)
        if ent["ref"] is None or not torch.equal(ent["ref"], ref_dev):
            # a new reference image: one batched appearance pass per chunk of (this rank's) timesteps
            order = list(range(total - 1, -1, -1))
            ent["bank"] = parallel.build_and_gather_bank(
                order, gd.layout, lambda part, slots: gd.build_bank(part, ref_dev, slots), pipe.device, world, rank,
                group=group, chunk=gd.bank_chunk, storage=ent["storage"])
            ent["ref"] = ref_dev.clone()
        bank = ent["bank"]
        if gd.has_pose:  # (a stage-1 model has no pose ControlNet and ignores c_concat)
            pose_map = _one(c["c_concat"])
            gd.hint.copy_(pipe.hint(pose_map.to(pipe.device), frame_key=tensor_key(pose_map), keep_alive=pose_map))
        gd.x.copy_(img.to(device=pipe.device, dtype=torch.float32))
        for i in range(total):
            index = total - i - 1
            bank.wait(index)
            gd.step(index, bank[index])
            if callback:
                callback(i)
            if img_callback:
                img_callback(gd.pred_x0.clone(), i)
            if index % log_every_t == 0 or index == total - 1:
                intermediates["x_inter"].append(gd.x_prev.clone())
                intermediates["pred_x0"].append(gd.pred_x0.clone())
        return gd.x_prev.clone(), intermediates

    def _p_sample_ddim_batched_cfg(self, x, c, t, index, scale, uc):
        """ddim.py:539-566 — the unconditional conditioning carries image_control too (every control_mode other than
        'controlnet_important', test_tiktok.py:237-243): ONE apply_model over the batch [unconditional ; conditional],
        both halves in 'read' mode with their own prompt, pose map and appearance bank.  Not graph-replayed: the
        appearance pass depends on both prompts and runs inside every step, exactly as in the reference."""
        from .. import ops
        pipe = self._pipeline(scale)
        dev = pipe.device
        ref = _one(c["image_control"]).to(dev)
        ref_n = ref if c["wonoise"] else self.model.q_sample(ref, t.to(dev))
        pair = lambda k: torch.cat([_one(uc[k]).to(dev), _one(c[k]).to(dev)])
        x = x.to(device=dev, dtype=torch.float32).contiguous()
        cond_in = {"c_crossattn": [pair("c_crossattn")]}
        if pipe.engine.pose is not None:  # a stage-1 model has no pose ControlNet and ignores c_concat
            cond_in["c_concat"] = [pair("c_concat")]
        eps = self.model.apply_model(torch.cat([x, x]), torch.cat([t, t]).to(dev), cond_in, torch.cat([ref_n, ref_n]))
        e_u, e_c = eps.chunk(2)
        noise = torch.randn_like(x) if float(self.ddim_sigmas[index]) != 0.0 else None
        return ops.cfg_ddim_update(x, e_c.contiguous(), e_u.contiguous(), pipe.coef[index], noise=noise)

    def _rows_identical(self, t):
        """all batch rows of t equal row 0?  One device->host sync per (tensor, version), not per DDIM step: the
        answer is cached with a strong reference to the tensor (its address cannot be recycled meanwhile)."""
        if t.shape[0] == 1:
            return True
        cache = self.model.__dict__.setdefault("_mdb_rows_identical", {})
        key = tensor_key(t)
        hit = cache.get(key)
        if hit is None:
            if len(cache) >= 8:
                cache.clear()
            hit = (bool((t[1:] == t[:1]).all()), t)
            cache[key] = hit
        return hit[0]

    @torch.no_grad()
    def p_sample_ddim(self, x, c, t, index, repeat_noise=False, use_original_steps=False, quantize_denoised=False,
                      temperature=1., noise_dropout=0., score_corrector=None, corrector_kwargs=None,
                      unconditional_guidance_scale=1., unconditional_conditioning=None, dynamic_threshold=None,
                      inpaint=None):
        """ddim.py:518-645.  The branch MagicPose's released scripts take (graph-replayed by ddim_sampling, fused
        here): c carries image_control (+wonoise), the unconditional conditioning does not ('controlnet is more
        important', ddim.py:598-605), so eps = eps_u + s (eps_c - eps_u) with eps_u = apply_model(x, t, c, None,
        uc=True).  The batched branch for the other control modes (ddim.py:539-566) runs eagerly; the no-guidance
        call (ddim.py:536-537, which the reference itself cannot execute for this model: apply_model lacks its
        reference argument) and AnimateDiff overlap sampling (ddim.py:568-594) raise."""
        if (inpaint is not None or use_original_steps or quantize_denoised or score_corrector is not None
                or dynamic_threshold is not None or noise_dropout != 0.0 or temperature != 1.0):
            raise NotImplementedError("option not used by the MagicPose inference scripts")
        if not (isinstance(c, dict) and c.get("image_control") is not None):
            raise NotImplementedError("p_sample_ddim needs cond['image_control'] (the reference image latent)")
        if unconditional_conditioning is None or unconditional_guidance_scale == 1.0:
            raise NotImplementedError("only the classifier-free-guidance path of the scripts is accelerated")
        if unconditional_conditioning.get("image_control") is not None:
            return self._p_sample_ddim_batched_cfg(x, c, t, index, unconditional_guidance_scale, unconditional_conditioning)
        if c.get("overlap_sampling"):
            raise NotImplementedError("overlap_sampling is off in every released script (test_tiktok.py:247)")
        pipe = self._pipeline(unconditional_guidance_scale)
        dev = pipe.device
        x = x.to(device=dev, dtype=torch.float32)
        ref, ctx = _one(c["image_control"]), _one(c["c_crossattn"])
        # the clean reference latent feeds the appearance net (ddim.py:532-533): the bank depends on (reference, t)
        # only.  One reference for the whole batch (the scripts repeat it per sample) is computed once and broadcast
        # in-kernel; the result is cached per timestep for the next frames.
        if c["wonoise"] and self._rows_identical(ref) and self._rows_identical(ctx):
            bank_kv = pipe.reference_bank(ref, ctx, index, first_only=True)
        else:  # per-sample references, or a noised one (ddim.py:535), which depends on fresh noise: not cached
            ref_in = ref if c["wonoise"] else self.model.q_sample(ref, t.to(ref.device))
            bank_kv = pipe.engine.bank_kv(ref_in, pipe.t_dev[index].expand(ref.shape[0]).contiguous(), ctx)
        hint = None
        if pipe.engine.pose is not None:  # a stage-1 model has no pose ControlNet and ignores c_concat
            pose_map = _one(c["c_concat"])
            hint = pipe.hint(pose_map.to(dev), frame_key=tensor_key(pose_map), keep_alive=pose_map)
        noise = None
        if float(self.ddim_sigmas[index]) != 0.0:
            noise = torch.randn_like(x)
        x_prev, pred_x0, _, _ = pipe.step(x, index, ctx.to(dev), hint, bank_kv, noise=noise)
        return x_prev, pred_x0
