"""DDIM step scheduler over the DenoiseEngine: the GPU-side counterpart of
DDIMSampler_ReferenceOnly (model_lib/ControlNet/ldm/models/diffusion/ddim.py:346-730), restricted
to the path MagicPose's inference script drives (test_tiktok.py:261-268): eps-parameterisation,
'controlnet is more important' CFG branch (ddim.py:598-605), wonoise=True (ddim.py:532-533).

What is cached, and why it is legal (SURVEY §8a):
  * text K/V of every attn2            — depends only on the prompt            (per sequence)
  * hint-encoder features              — depend only on the pose map           (per frame)
  * appearance bank K/V per timestep   — with wonoise the appearance net sees (reference latent, t)
                                         only, so it is identical for every frame of a sequence
  * the unconditional call skips the pose ControlNet whose output the reference discards.
Host code here is scheduling only; all tensor math goes through magicdance_b200.ops.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import ops
from .engine import DenoiseEngine, tensor_key


def linear_beta_schedule(n_timestep=1000, linear_start=0.00085, linear_end=0.0120):
    """make_beta_schedule('linear') (ldm/modules/diffusionmodules/util.py:21-28) -> float64 numpy."""
    return np.linspace(linear_start ** 0.5, linear_end ** 0.5, n_timestep, dtype=np.float64) ** 2


def alphas_cumprod_f32(n_timestep=1000, linear_start=0.00085, linear_end=0.0120):
    """DDPM.register_schedule (ddpm.py:120-133): cumprod in float64, stored as a float32 buffer."""
    return np.cumprod(1.0 - linear_beta_schedule(n_timestep, linear_start, linear_end), axis=0).astype(np.float32)


def ddim_timesteps_uniform(num_ddim, num_ddpm=1000):
    """make_ddim_timesteps('uniform') (util.py:45-59): range(0, T, T//S) + 1."""
    return np.asarray(list(range(0, num_ddpm, num_ddpm // num_ddim))) + 1


def ddim_parameters(alphacums, ddim_timesteps, eta):
    """make_ddim_sampling_parameters (util.py:62-73)."""
    alphas = alphacums[ddim_timesteps]
    alphas_prev = np.asarray([alphacums[0]] + alphacums[ddim_timesteps[:-1]].tolist())
    sigmas = eta * np.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
    return sigmas, alphas, alphas_prev


class DenoisePipeline:
    def __init__(self, engine: DenoiseEngine, ddim_steps=50, scale=7.0, eta=0.0, num_ddpm=1000,
                 linear_start=0.00085, linear_end=0.0120, alphas_cumprod=None):
        self.engine = engine
        self.device = engine.device
        self.scale = float(scale)
        acp = alphas_cumprod_f32(num_ddpm, linear_start, linear_end) if alphas_cumprod is None else \
            np.asarray(alphas_cumprod, dtype=np.float32)
        self.alphas_cumprod = acp
        self.make_schedule(ddim_steps, eta)
        self._bank_cache = {}
        self._hint_cache = {}

    def make_schedule(self, ddim_steps, eta=0.0):
        self.ddim_steps = ddim_steps
        self.timesteps = ddim_timesteps_uniform(ddim_steps, self.alphas_cumprod.shape[0])
        sig, a, a_prev = ddim_parameters(self.alphas_cumprod, self.timesteps, eta)
        self.sigmas, self.alphas, self.alphas_prev = sig, a, a_prev
        coef = np.zeros((len(self.timesteps), 8), dtype=np.float32)
        for i in range(len(self.timesteps)):
            coef[i, :6] = [self.scale, math.sqrt(a[i]), math.sqrt(a_prev[i]),
                           math.sqrt(max(1.0 - a_prev[i] - sig[i] ** 2, 0.0)), sig[i], math.sqrt(1.0 - a[i])]
        self.coef = torch.from_numpy(coef).to(self.device)  # row i = coefficients of ddim index i
        self.t_dev = torch.from_numpy(self.timesteps.astype(np.int64)).to(self.device)

    # ---- per-sequence / per-frame preparation --------------------------------------------------
    def reference_bank(self, ref_latent, context, index, first_only=False):
        """Bank K/V for ddim index `index` (appearance 'write' pass + projection), cached per
        (reference tensor, CONTEXT tensor, index): the appearance net runs with the prompt's context
        (cldm.py:1110), so a new prompt with the same reference image needs a new bank.
        first_only: all rows of ref_latent AND of context are the same; compute row 0 and broadcast."""
        seq = (tensor_key(ref_latent), tensor_key(context), bool(first_only))
        if getattr(self, "_bank_seq", None) != seq:
            self._bank_cache.clear()  # a new reference image or prompt: drop the previous sequence's banks (2.3 GB)
            self._bank_seq = seq
            self._bank_keep = (ref_latent, context)  # keep both alive: their addresses key the cache
        hit = self._bank_cache.get(int(index))
        if hit is None:
            src = ref_latent[:1].contiguous() if first_only else ref_latent
            rb = src.shape[0]
            t = self.t_dev[index].expand(rb).contiguous()
            hit = self.engine.bank_kv(src, t, context[:rb])
            self._bank_cache[int(index)] = hit
        return hit

    def clear_caches(self):
        self._bank_cache.clear()
        self._bank_seq = self._bank_keep = None
        self._hint_cache.clear()

    HINT_CACHE_FRAMES = 8

    def hint(self, pose_map, frame_key=None, keep_alive=None):
        """Hint-encoder features of a pose map, cached per caller-supplied frame key.  When the key is derived from
        a tensor's address (the drop-in sampler keys on the caller's pose tensor), pass that tensor as `keep_alive`:
        the entry then holds a strong reference, so the storage cannot be freed and its address handed to the NEXT
        frame's pose map while the entry exists (a recycled address would be a silent stale hit)."""
        if frame_key is None:
            return self.engine.hint_features(pose_map)
        hit = self._hint_cache.get(frame_key)
        if hit is None:
            while len(self._hint_cache) >= self.HINT_CACHE_FRAMES:  # oldest first (dicts keep insertion order)
                self._hint_cache.pop(next(iter(self._hint_cache)))
            hit = (self.engine.hint_features(pose_map), keep_alive)
            self._hint_cache[frame_key] = hit
        return hit[0]

    # ---- one DDIM step ---------------------------------------------------------------------------
    def step(self, x, index, context, hint_feat, bank_kv, noise=None):
        """p_sample_ddim (ddim.py:518-645): eps_c = apply_model(x,t,c,ref), eps_u = apply_model(x,t,c,None,uc),
        CFG combine, DDIM update.  x: fp32 NCHW on the device.  Returns (x_prev, pred_x0, eps_c, eps_u).
        Without a pose ControlNet (stage 1) hint_feat is not read and no residuals are added."""
        eng = self.engine
        t = self.t_dev[index:index + 1]  # one timestep for the whole batch (a view: no kernel)
        pose = None if eng.pose is None else eng.controlnet(x, hint_feat, t, context)
        eps_c, eps_u = eng.unet_forward(x, t, context, bank_kv=bank_kv, pose=pose, cfg_pair=True)
        x_prev, pred_x0 = ops.cfg_ddim_update(x.contiguous(), eps_c.contiguous(), eps_u.contiguous(), self.coef[index],
                                              noise=noise)
        return x_prev, pred_x0, eps_c, eps_u

    @torch.no_grad()
    def sample(self, x_T, context, pose_map, ref_latent, frame_key=None, callback=None):
        """ddim_sampling (ddim.py:460-516) for a batch of frames sharing one reference latent."""
        x = x_T.to(device=self.device, dtype=torch.float32).contiguous()
        context = context.to(self.device)
        ref_latent = ref_latent.to(self.device)
        hint_feat = None if self.engine.pose is None else self.hint(pose_map.to(self.device), frame_key)
        pred_x0 = x
        for i in range(self.ddim_steps):
            index = self.ddim_steps - 1 - i
            bank_kv = self.reference_bank(ref_latent, context, index)
            x, pred_x0, _, _ = self.step(x, index, context, hint_feat, bank_kv)
            if callback:
                callback(i)
        return x, pred_x0


def build_bank_slots(eng: DenoiseEngine, ref_latent, t_vec, context, layout, tokens, out_slots):
    """Appearance 'write' pass for a BATCH of timesteps of one reference latent (the appearance net
    takes per-sample t, cldm.py:469-472) + K/V projection, re-laid out as one contiguous flat slot
    per timestep (parallel.BankLayout with ref_batches=1): out_slots [len(t_vec), layout.numel]."""
    tb = t_vec.shape[0]
    ref = ref_latent[:1].expand(tb, -1, -1, -1).contiguous()
    kv = eng.bank_kv(ref, t_vec, context[:1])
    for (k, vt, n, _), (rows, c), ldv, off in zip(kv, layout.layer_shapes, layout.ldv, layout.offsets):
        # K [tb*n, c] -> slot j rows; V^T [c, tb*ldv] -> slot j [c, ldv]
        out_slots[:, off:off + n * c].view(tb, n, c).copy_(k.view(tb, n, c))
        out_slots[:, off + n * c:off + n * c + c * ldv].view(tb, c, ldv).copy_(vt.view(c, tb, ldv).permute(1, 0, 2))


def plan_bank_chunks(indices, chunk):
    """[(first slot, [ddim indices])]: the sequence's distinct timesteps in the order the steps consume them, cut
    into appearance-pass batches of at most `chunk`."""
    idx = list(dict.fromkeys(int(i) for i in indices))
    return [(s0, idx[s0:s0 + chunk]) for s0 in range(0, len(idx), chunk)]


class GraphedDenoiser:
    """The whole DDIM step and the (timestep-batched) appearance-bank build captured once as CUDA
    graphs and replayed: at batch 1 the step is ~650 small kernels, so launch latency and Python
    would otherwise dominate (SURVEY §7 step 6).  Everything timestep-dependent is read from device
    memory refreshed by tiny copies before each replay (the timestep, the DDIM coefficient row, the
    bank K/V of that timestep), so ONE graph serves every step."""

    def __init__(self, pipe: DenoisePipeline, batch: int, latent_hw, context: torch.Tensor, bank_chunk: int = 10):
        from . import parallel
        self.pipe, self.eng = pipe, pipe.engine
        eng, dev = self.eng, pipe.device
        h, w = latent_hw
        self.batch, self.bank_chunk = batch, bank_chunk
        self.ctx = context.to(dev).contiguous()
        self.x = torch.zeros((batch, 4, h, w), dtype=torch.float32, device=dev)
        self.x_prev = torch.zeros_like(self.x)
        self.pred_x0 = torch.zeros_like(self.x)
        self.ref = torch.zeros((1, 4, h, w), dtype=torch.float32, device=dev)
        self.t_cur = torch.zeros((1,), dtype=torch.int64, device=dev)
        self.t_vec = torch.zeros((bank_chunk,), dtype=torch.int64, device=dev)
        self.coef_cur = torch.zeros((8,), dtype=torch.float32, device=dev)
        self.has_pose = eng.pose is not None  # stage 1 (ControlLDMReferenceOnly) has no pose ControlNet
        self.hint = None
        if self.has_pose:
            self.hint = torch.zeros((batch * h * w, eng.cfg.model_channels), dtype=torch.float16, device=dev)
        geo = eng.attn_geometry(h, w)
        self.tokens = [n for n, _ in geo]
        self.layout = parallel.BankLayout([(n, c) for n, c in geo])
        self.bank_cur = torch.zeros((self.layout.numel,), dtype=torch.float16, device=dev)
        self.bank_built = torch.zeros((bank_chunk, self.layout.numel), dtype=torch.float16, device=dev)
        # timestep path hoisted out of the step: embedding -> time_embed MLP -> all emb_layers depend on t only, so the
        # tables for every ddim index are computed once (capture()) and a step copies its two rows into these buffers
        self.emb_unet = torch.zeros((1, eng.unet.emb_total), dtype=torch.float32, device=dev)
        self.emb_pose = self.side = None
        if self.has_pose:
            self.emb_pose = torch.zeros((1, eng.pose.emb_total), dtype=torch.float32, device=dev)
            self.side = torch.cuda.Stream(device=dev)  # the pose ControlNet's stream (joins the UNet at the middle block)
        self.emb_tab_unet = self.emb_tab_pose = None
        self.g_step = self.g_bank = None
        self.replayed_launches = 0
        # auxiliary streams for independent branches inside a block (engine._fork): lane 0 (UNet pass) -> lane 2,
        # lane 1 (ControlNet pass on the side stream) -> lane 3
        # (kept on THIS object and handed to the engine only for the duration of _step_body: eager calls through the
        # same engine must not inherit the fork/join path and its scratch lanes)
        self.aux_streams = None
        if batch <= 2:
            self.aux_streams = {0: (torch.cuda.Stream(device=dev), 2)}
            if self.has_pose:
                self.aux_streams[1] = (torch.cuda.Stream(device=dev), 3)

    # the two bodies, written against the static buffers only
    def _step_body(self):
        """One DDIM step.  The pose ControlNet and the UNet's encoder half are independent (the pose
        residuals enter at the middle block, cldm.py:93-104), and at one frame per GPU each of their
        kernels fills only part of the 132 SMs, so the ControlNet runs on a second stream (forked and
        joined with events, captured into the same graph) with its own scratch buffers."""
        eng, b = self.eng, self.batch
        prev_aux, eng.aux_streams = eng.aux_streams, self.aux_streams
        try:
            self._step_body_inner(eng, b)
        finally:
            eng.aux_streams = prev_aux

    def _step_body_inner(self, eng, b):
        t = self.t_cur  # one timestep for the whole batch
        bank_kv = self.layout.views(self.bank_cur, self.tokens, 1)
        if not self.has_pose:
            eps_c, eps_u = eng.unet_forward(self.x, t, self.ctx, bank_kv=bank_kv, cfg_pair=True, emb_all=self.emb_unet)
            ops.cfg_ddim_update(self.x, eps_c, eps_u, self.coef_cur, x_prev=self.x_prev, pred_x0=self.pred_x0,
                                update_x=True)
            return
        main = torch.cuda.current_stream()
        self.side.wait_stream(main)
        with torch.cuda.stream(self.side), ops.workspace_lane(1):
            pose = eng.controlnet(self.x, self.hint, t, self.ctx, emb_all=self.emb_pose)
        join = lambda: main.wait_stream(self.side)
        eps_c, eps_u = eng.unet_forward(self.x, t, self.ctx, bank_kv=bank_kv, pose=pose, cfg_pair=True, before_pose=join,
                                        emb_all=self.emb_unet)
        # x advances in place (x_prev and pred_x0 are also kept for the callers)
        ops.cfg_ddim_update(self.x, eps_c, eps_u, self.coef_cur, x_prev=self.x_prev, pred_x0=self.pred_x0, update_x=True)

    def _bank_body(self):
        build_bank_slots(self.eng, self.ref, self.t_vec, self.ctx, self.layout, self.tokens, self.bank_built)

    def capture(self):
        """Warm up eagerly (fills every cache and workspace), then capture both graphs."""
        s = torch.cuda.Stream(device=self.pipe.device)
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            eng, td = self.eng, self.pipe.t_dev
            self.emb_tab_unet = torch.cat([eng.time_bias(eng.unet, td[i:i + 1]) for i in range(td.shape[0])], 0)
            if self.has_pose:
                self.emb_tab_pose = torch.cat([eng.time_bias(eng.pose, td[i:i + 1]) for i in range(td.shape[0])], 0)
            self.emb_unet.copy_(self.emb_tab_unet[-1:])
            if self.has_pose:
                self.emb_pose.copy_(self.emb_tab_pose[-1:])
            for _ in range(2):
                self._bank_body()
                self._step_body()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        n0 = ops.launch_count()
        self.g_bank = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_bank):
            self._bank_body()
        n1 = ops.launch_count()
        self.g_step = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_step, pool=self.g_bank.pool()):
            self._step_body()
        torch.cuda.synchronize()
        # kernels of OUR library inside each graph (the C ABI counts launches at capture time only)
        self.bank_launches, self.step_launches = n1 - n0, ops.launch_count() - n1
        # The graphs hold raw pointers to the text K/V of this context (engine._ctx_cache evicts) — keep those
        # tensors alive for as long as the graphs are; scratch workspaces are never freed (ops._workspace retires).
        self._pinned = list(self.eng._ctx_cache.values())
        return self

    # ---- replay helpers ---------------------------------------------------------------------------
    def build_bank(self, indices, ref_latent, out_slots):
        """bank K/V of the given ddim indices (<= bank_chunk of them) -> out_slots [len(indices), numel]"""
        n = len(indices)
        assert 0 < n <= self.bank_chunk
        self.ref.copy_(ref_latent[:1])
        idx = torch.as_tensor(list(indices) + [indices[-1]] * (self.bank_chunk - n), device=self.pipe.device)
        self.t_vec.copy_(self.pipe.t_dev[idx])
        self.g_bank.replay()
        self.replayed_launches += self.bank_launches
        out_slots.copy_(self.bank_built[:n])

    def step(self, index, bank_flat):
        """one DDIM step on self.x in place (result also in self.x_prev / self.pred_x0)"""
        self.t_cur.copy_(self.pipe.t_dev[index:index + 1])
        self.coef_cur.copy_(self.pipe.coef[index])
        self.emb_unet.copy_(self.emb_tab_unet[index:index + 1])
        if self.has_pose:
            self.emb_pose.copy_(self.emb_tab_pose[index:index + 1])
        self.bank_cur.copy_(bank_flat)
        self.g_step.replay()
        self.replayed_launches += self.step_launches
        return self.x_prev
