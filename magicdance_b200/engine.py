"""Host-side schedule of the denoising hot path over the sm_90a kernels (magicdance_b200.ops).

Implements, for the reference's three networks and their glue:
  ControlledUnetModelAttnPose.forward   model_lib/ControlNet/cldm/cldm.py:59-112
  ControlNetReferenceOnly.forward       cldm.py:469-497   ('write' mode -> attention bank)
  ControlNet.forward                    cldm.py:736-757   (13 pose residuals)
  ControlLDMReferenceOnlyPose.apply_model  cldm.py:1099-1117
built from the blocks of ldm/modules/diffusionmodules/openaimodel.py:79-295 and
ldm/modules/attention.py:50-77,146-385.

Data layout in HBM: activations fp16 channels-last, held as 2-D [B*H*W, C] matrices (the same
buffer is the NHWC image for convolutions and the token matrix for the transformer blocks, so
the reference's `b c h w -> b (h w) c` rearranges vanish); weights fp16 K-major (see pack_*);
norm parameters, biases and the timestep path fp32.

Weights are read from a plain state dict with the reference's key names (SURVEY §8b), repacked
once here.  Nothing in this file computes on the CPU or through torch operators on the per-step
path: torch only allocates buffers, and at levels whose token count is not a multiple of 8 copies the V^T operand's
tokens into their padded layout (ops.pad_tokens).
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

from . import ops

UNET = "model.diffusion_model."
APPEARANCE = "appearance_control_model."
POSE = "pose_control_model."


@dataclass(frozen=True)
class NetConfig:
    """kwargs of the three nets in models/cldm_v15_reference_only_pose.yaml:21-72"""
    in_channels: int = 4
    out_channels: int = 4
    hint_channels: int = 3
    model_channels: int = 320
    attention_resolutions: tuple = (4, 2, 1)
    num_res_blocks: int = 2
    channel_mult: tuple = (1, 2, 4, 4)
    num_heads: int = 8
    context_dim: int = 768

    @staticmethod
    def from_kwargs(**kw):
        keys = NetConfig.__dataclass_fields__.keys()
        d = {k: (tuple(v) if isinstance(v, (list, tuple)) else v) for k, v in kw.items() if k in keys}
        return NetConfig(**d)


def block_plan(cfg: NetConfig):
    """(input_blocks, middle_block, output_blocks) as lists of (kind, index-in-block, cin, cout);
    mirrors how UNetModel.__init__ (openaimodel.py:562-750) lays out its ModuleLists, which fixes
    the state-dict key of every layer."""
    mc = cfg.model_channels
    inp = [[("conv_in", 0, cfg.in_channels, mc)]]
    chans = [mc]
    ch, ds = mc, 1
    for level, mult in enumerate(cfg.channel_mult):
        for _ in range(cfg.num_res_blocks):
            blk = [("res", 0, ch, mult * mc)]
            ch = mult * mc
            if ds in cfg.attention_resolutions:
                blk.append(("attn", 1, ch, ch))
            inp.append(blk)
            chans.append(ch)
        if level != len(cfg.channel_mult) - 1:
            inp.append([("down", 0, ch, ch)])
            chans.append(ch)
            ds *= 2
    mid = [("res", 0, ch, ch), ("attn", 1, ch, ch), ("res", 2, ch, ch)]
    out = []
    for level, mult in list(enumerate(cfg.channel_mult))[::-1]:
        for i in range(cfg.num_res_blocks + 1):
            ich = chans.pop()
            blk = [("res", 0, ch + ich, mult * mc)]
            ch = mult * mc
            if ds in cfg.attention_resolutions:
                blk.append(("attn", len(blk), ch, ch))
            if level and i == cfg.num_res_blocks:
                blk.append(("up", len(blk), ch, ch))
                ds //= 2
            out.append(blk)
    return inp, mid, out


# ------------------------------------------------------------------------------------------------
# weight packing
# ------------------------------------------------------------------------------------------------
def _f16(t, device):
    return t.detach().to(device=device, dtype=torch.float16).contiguous()


def _f32(t, device):
    return t.detach().to(device=device, dtype=torch.float32).contiguous()


def pack_conv3x3(w, device):
    """Conv2d OIHW fp32 -> [O][kh][kw][I] fp16 viewed as [O, 9*I] on `device` (ops.pack_conv_weight)."""
    return ops.pack_conv_weight(w.detach().to(device))


def pack_conv1x1(w, device):
    return _f16(w.detach().reshape(w.shape[0], w.shape[1]), device)


def pack_geglu(w, b, device):
    """GEGLU.proj (attention.py:53-56): rows [0,4C) are values, [4C,8C) gates.  Interleave them in
    blocks of 32 rows [value | gate] so that one GEMM tile holds matching value/gate columns."""
    n = w.shape[0] // 2
    idx = torch.arange(n).reshape(-1, 32)
    order = torch.cat([idx, idx + n], dim=1).reshape(-1)
    return _f16(w.detach()[order], device), _f32(b.detach()[order], device)


def fold_layernorm(w, gamma, beta, bias, device):
    """LayerNorm(x) W^T + b as ONE GEMM over the raw x (ops.gemm(ln_u=...)): returns
    (W diag(gamma) in fp16, u = row sums of that fp16 matrix, v = W beta + b) — u is taken from the ROUNDED weights,
    because it has to cancel exactly what the tensor core sums."""
    w, gamma, beta = w.detach().to(device).float(), gamma.detach().to(device).float(), beta.detach().to(device).float()
    w_ln = (w * gamma[None, :]).to(torch.float16).contiguous()
    u = w_ln.float().sum(dim=1).contiguous()
    v = w @ beta
    if bias is not None:
        v = v + bias.detach().to(device).float()
    return w_ln, u, v.contiguous()


class ResW:
    pass


class AttnW:
    pass


class PackedNet:
    """One network's weights (UNet / appearance twin / pose ControlNet) repacked for the kernels."""

    def __init__(self, sd, prefix, cfg: NetConfig, kind: str, device):
        self.cfg, self.kind, self.prefix, self.device = cfg, kind, prefix, device
        self.inp, self.mid, self.out = block_plan(cfg)
        g = lambda k: sd[prefix + k]
        mc = cfg.model_channels
        self.te0_w, self.te0_b = _f16(g("time_embed.0.weight"), device), _f32(g("time_embed.0.bias"), device)
        self.te2_w, self.te2_b = _f16(g("time_embed.2.weight"), device), _f32(g("time_embed.2.bias"), device)
        self.layers = {}
        emb_w, emb_b, off = [], [], 0
        blocks = [(f"input_blocks.{i}.", b) for i, b in enumerate(self.inp)]
        blocks.append(("middle_block.", self.mid))
        if kind != "controlnet":
            blocks += [(f"output_blocks.{i}.", b) for i, b in enumerate(self.out)]
        for bp, blk in blocks:
            for kind_, j, cin, cout in blk:
                p = f"{bp}{j}."
                if kind_ == "conv_in":
                    self.layers[p] = (pack_conv3x3(g(p + "weight"), device), _f32(g(p + "bias"), device))
                elif kind_ == "res":
                    r = ResW()
                    r.cin, r.cout = cin, cout
                    r.gn1 = (_f32(g(p + "in_layers.0.weight"), device), _f32(g(p + "in_layers.0.bias"), device))
                    r.w1 = pack_conv3x3(g(p + "in_layers.2.weight"), device)
                    r.gn2 = (_f32(g(p + "out_layers.0.weight"), device), _f32(g(p + "out_layers.0.bias"), device))
                    r.w2 = pack_conv3x3(g(p + "out_layers.3.weight"), device)
                    r.b2 = _f32(g(p + "out_layers.3.bias"), device)
                    if (prefix + p + "skip_connection.weight") in sd:
                        r.skip_w = pack_conv1x1(g(p + "skip_connection.weight"), device)
                        r.skip_b = _f32(g(p + "skip_connection.bias"), device)
                    else:
                        r.skip_w = r.skip_b = None
                    # emb_layers Linear (openaimodel.py:238-244) stacked for one skinny GEMM per call;
                    # the first conv's bias is folded into the stacked bias.
                    emb_w.append(g(p + "emb_layers.1.weight").detach())
                    emb_b.append(g(p + "emb_layers.1.bias").detach() + g(p + "in_layers.2.bias").detach())
                    r.emb_off = off
                    off += cout
                    self.layers[p] = r
                elif kind_ == "attn":
                    self.layers[p] = self._pack_attn(g, p, cin, device)
                elif kind_ == "down":
                    self.layers[p] = (pack_conv3x3(g(p + "op.weight"), device), _f32(g(p + "op.bias"), device))
                elif kind_ == "up":
                    self.layers[p] = (pack_conv3x3(g(p + "conv.weight"), device), _f32(g(p + "conv.bias"), device))
        self.emb_w = _f16(torch.cat(emb_w, 0), device)
        self.emb_b = _f32(torch.cat(emb_b, 0), device)
        self.emb_total = off
        if kind == "unet":
            self.out_gn = (_f32(g("out.0.weight"), device), _f32(g("out.0.bias"), device))
            self.out_w, self.out_b = pack_conv3x3(g("out.2.weight"), device), _f32(g("out.2.bias"), device)
        if kind == "controlnet":
            self.hint = []
            for i in range(8):
                w = g(f"input_hint_block.{2 * i}.weight")
                self.hint.append((pack_conv3x3(w, device), _f32(g(f"input_hint_block.{2 * i}.bias"), device),
                                  w.shape[1], w.shape[0]))
            self.zero = []
            for i in range(len(self.inp)):
                self.zero.append((pack_conv1x1(g(f"zero_convs.{i}.0.weight"), device),
                                  _f32(g(f"zero_convs.{i}.0.bias"), device)))
            self.zero.append((pack_conv1x1(g("middle_block_out.0.weight"), device),
                              _f32(g("middle_block_out.0.bias"), device)))

    def _pack_attn(self, g, p, c, device):
        a = AttnW()
        a.c, a.heads, a.d = c, self.cfg.num_heads, c // self.cfg.num_heads
        a.gn = (_f32(g(p + "norm.weight"), device), _f32(g(p + "norm.bias"), device))
        a.pin_w, a.pin_b = pack_conv1x1(g(p + "proj_in.weight"), device), _f32(g(p + "proj_in.bias"), device)
        a.pout_w, a.pout_b = pack_conv1x1(g(p + "proj_out.weight"), device), _f32(g(p + "proj_out.bias"), device)
        t = p + "transformer_blocks.0."
        for i in (1, 3):  # norm2 is folded into attn2.to_q below
            setattr(a, f"ln{i}", (_f32(g(t + f"norm{i}.weight"), device), _f32(g(t + f"norm{i}.bias"), device)))
        # self-attention: q and k projections share one GEMM ([2C, C]); v is produced transposed
        a.wqk = _f16(torch.cat([g(t + "attn1.to_q.weight").detach(), g(t + "attn1.to_k.weight").detach()], 0), device)
        a.wv = _f16(g(t + "attn1.to_v.weight"), device)
        a.wo, a.bo = _f16(g(t + "attn1.to_out.0.weight"), device), _f32(g(t + "attn1.to_out.0.bias"), device)
        a.wq2_ln, a.q2_u, a.q2_v = fold_layernorm(g(t + "attn2.to_q.weight"), g(t + "norm2.weight"), g(t + "norm2.bias"),
                                                  None, device)
        a.wk2 = _f16(g(t + "attn2.to_k.weight"), device)
        a.wv2 = _f16(g(t + "attn2.to_v.weight"), device)
        a.wo2, a.bo2 = _f16(g(t + "attn2.to_out.0.weight"), device), _f32(g(t + "attn2.to_out.0.bias"), device)
        a.wff1, a.bff1 = pack_geglu(g(t + "ff.net.0.proj.weight"), g(t + "ff.net.0.proj.bias"), device)
        a.wff2, a.bff2 = _f16(g(t + "ff.net.2.weight"), device), _f32(g(t + "ff.net.2.bias"), device)
        return a

    def attn_layers(self):
        """AttnW objects in execution order (the order of the attention bank, attention.py:287-298)."""
        order = []
        blocks = [(f"input_blocks.{i}.", b) for i, b in enumerate(self.inp)] + [("middle_block.", self.mid)]
        if self.kind != "controlnet":
            blocks += [(f"output_blocks.{i}.", b) for i, b in enumerate(self.out)]
        for bp, blk in blocks:
            for kind_, j, _, _ in blk:
                if kind_ == "attn":
                    order.append(self.layers[f"{bp}{j}."])
        return order


# ------------------------------------------------------------------------------------------------
# execution
# ------------------------------------------------------------------------------------------------
@dataclass
class Act:
    """fp16 channels-last activation: data is [B*H*W, C]"""
    data: torch.Tensor
    b: int
    h: int
    w: int

    @property
    def c(self):
        return self.data.shape[1]

    @property
    def hw(self):
        return self.h * self.w


def tensor_key(t):
    """identity of a tensor's contents as far as the host can tell without a device sync: storage address, view
    geometry and the in-place version counter.  A cache keyed on it must hold a strong reference to the tensor, so
    that its storage cannot be freed and the address recycled by another tensor while the entry exists."""
    return (t.untyped_storage().data_ptr(), t.storage_offset(), tuple(t.shape), tuple(t.stride()), t._version)


def _igemm_ok(h, w, c):
    """does an h x w x c conv output tile into the implicit-GEMM conv's 128-pixel TMA boxes?  (512x512 and 256x256
    images do at every level.)  Other sizes take the same kernels with TMA im2col loads (ops.conv3x3_igemm)."""
    hw = h * w
    if c % 64:
        return False
    # mirrors pixel_box(..., fwd=true) in csrc/gemm.cu
    return ((128 % w == 0 and hw % 128 == 0) or w % 128 == 0) if hw >= 128 else (128 % hw == 0)


def conv3x3(x: Act, w, bias, *, cout, stride=1, residual=None, bias_batch_stride=0) -> Act:
    """3x3 pad-1 conv, w packed by pack_conv3x3.  Tensor cores (implicit GEMM over TMA boxes where the pixels tile into
    them, over TMA im2col loads at any other size) when cin and cout fit their tiles; the direct conv otherwise (few
    channels in or out: the UNet's conv_in/out, the VAE's ends)."""
    cin = x.c
    ho, wo = (x.h - 1) // stride + 1, (x.w - 1) // stride + 1
    tc = cout % 8 == 0 and cout >= 64 and cin % 64 == 0
    if tc and _igemm_ok(ho, wo, cin):  # stride 2: TMA element strides of 2, no im2col buffer
        y = ops.gemm(x.data, w, bias=bias, bias_batch_stride=bias_batch_stride, rows_per_batch=ho * wo,
                     residual=residual, conv=(x.b, x.h, x.w, cin), conv_stride=stride)
    elif tc:
        # latent sizes whose rows do not tile into 128-pixel TMA boxes (e.g. 96x64 -> 12x8 at the deepest
        # level): the same wgmma kernel, its activation tiles loaded in TMA im2col mode
        y = ops.conv3x3_igemm(x.data, w, conv=(x.b, x.h, x.w, cin), conv_stride=stride, bias=bias,
                              bias_batch_stride=bias_batch_stride, rows_per_batch=ho * wo, residual=residual)
    else:
        assert bias_batch_stride == 0
        y = ops.conv3x3_direct(x.data, w, bias, batch=x.b, h=x.h, w=x.w, cin=cin, cout=cout, stride=stride,
                               residual=residual)
    return Act(y, x.b, ho, wo)


def _vt(wv, x, b, out=None):
    """(V^T = W_v x^T as [C, b*ldv], ldv): each sample's column block starts at a multiple of 8 (ops.pad_tokens)"""
    xp, ldv = ops.pad_tokens(x, b)
    return ops.gemm(wv, xp, out=out), ldv


class _BankComplete(Exception):
    """unwinds appearance_write as soon as the last norm1 state is in the bank"""


class DenoiseEngine:
    """Runs the three networks of ControlLDMReferenceOnlyPose on one GPU (or, built by from_packed without a pose
    ControlNet, the two of the stage-1 ControlLDMReferenceOnly)."""

    def __init__(self, state_dict, cfg: NetConfig | None = None, device="cuda"):
        ops.ensure_device()
        self.cfg = cfg or NetConfig()
        self.device = torch.device(device)
        self.unet = PackedNet(state_dict, UNET, self.cfg, "unet", self.device)
        self.appearance = PackedNet(state_dict, APPEARANCE, self.cfg, "appearance", self.device)
        self.pose = PackedNet(state_dict, POSE, self.cfg, "controlnet", self.device)
        self._ctx_cache = {}

    @classmethod
    def from_packed(cls, unet: "PackedNet", appearance: "PackedNet | None", pose: "PackedNet | None"):
        """Engine over already-packed networks (the drop-in nn.Modules pack themselves lazily)."""
        ops.ensure_device()
        self = cls.__new__(cls)
        first = unet or appearance or pose
        self.cfg, self.device = first.cfg, first.device
        self.unet, self.appearance, self.pose = unet, appearance, pose
        self._ctx_cache = {}
        return self

    # ---- small pieces -------------------------------------------------------------------------
    def time_bias(self, net: PackedNet, t: torch.Tensor, rows=None):
        """timestep_embedding -> time_embed MLP -> all emb_layers of the net (util.py:189-209,
        openaimodel.py:547-551,238-244).  Returns fp32 [rows, sum(cout)] = emb_out + conv1 bias; t may hold fewer
        entries than rows (one timestep for the whole batch; the cond | uncond pair): row b uses t[b % len(t)]."""
        if t.shape[0] == 1:
            rows = 1  # one timestep for the whole batch: ONE bias row, shared by every sample (bias_batch_stride 0)
        e = ops.timestep_embedding(t, self.cfg.model_channels, rows)
        e = ops.skinny_linear(e, net.te0_w, net.te0_b, silu_out=True)
        e = ops.skinny_linear(e, net.te2_w, net.te2_b)
        return ops.skinny_linear(e, net.emb_w, net.emb_b, silu_in=True)

    def context_kv(self, net: PackedNet, ctx16: torch.Tensor, context: torch.Tensor, paired=False):
        """Text keys/values of every attn2 (CrossAttention.to_k/to_v on the CLIP context,
        attention.py:172-174); depends only on the context -> cached per (net, context).  ctx16 is the caller's
        `context` in fp16 on the device, stacked twice when `paired` (the cond | uncond batch of unet_forward)."""
        # (net, storage, offset, shape, stride, version, paired); per PackedNet object: drop-in modules all have an
        # empty key prefix
        ck = (id(net),) + tensor_key(context) + (paired,)
        hit = self._ctx_cache.get(ck)
        if hit is not None:  # the entry's strong reference keeps that storage alive, so the address is still its own
            return hit[0]
        b, n, cd = ctx16.shape
        flat = ctx16.reshape(b * n, cd)
        padded, ldv = ops.pad_tokens(flat, b)  # 77 tokens -> V^T [C, b*80]
        res = []
        for a in net.attn_layers():
            k = ops.gemm(flat, a.wk2)
            vt = ops.gemm(a.wv2, padded)
            res.append((k, vt, n, b, ldv))
        if len(self._ctx_cache) > 8:
            self._ctx_cache.clear()
        self._ctx_cache[ck] = (res, context)  # strong ref to the context tensor
        return res

    # ---- optional intra-network concurrency ---------------------------------------------------------
    # At one or two samples per launch most kernels fill a fraction of the SMs, so independent branches of a
    # block (the 1x1 skip conv of a ResBlock vs its GroupNorm->conv chain; the V^T projection vs the q/k
    # projection) can run on an auxiliary stream.  aux_streams maps the workspace lane of the calling pass to
    # (stream, lane of the auxiliary work); set by pipeline.GraphedDenoiser, captured into the step graph.
    aux_streams = None

    def _fork(self, fn):
        """Run fn() on this lane's auxiliary stream (if any); returns (result, join)."""
        aux = self.aux_streams.get(ops.current_lane()) if self.aux_streams else None
        if aux is None:
            return fn(), (lambda: None)
        stream, lane = aux
        main = torch.cuda.current_stream()
        stream.wait_stream(main)
        with torch.cuda.stream(stream), ops.workspace_lane(lane):
            out = fn()
        return out, (lambda: main.wait_stream(stream))

    # ---- blocks -------------------------------------------------------------------------------
    def _res(self, r: ResW, x: Act, skip: Act | None, emb_all):
        x2 = None if skip is None else skip.data
        if r.skip_w is None:
            assert skip is None
            res, join = x.data, (lambda: None)
        else:
            res, join = self._fork(lambda: ops.gemm(x.data, r.skip_w, bias=r.skip_b, a2=x2))
        h = ops.groupnorm(x.data, *r.gn1, batch=x.b, hw=x.hw, eps=1e-5, silu=True, x2=x2)
        bias = emb_all[:, r.emb_off:r.emb_off + r.cout]
        h = conv3x3(Act(h, x.b, x.h, x.w), r.w1, bias, cout=r.cout,
                    bias_batch_stride=emb_all.stride(0) if emb_all.shape[0] > 1 else 0)
        h2 = ops.groupnorm(h.data, *r.gn2, batch=x.b, hw=x.hw, eps=1e-5, silu=True)
        join()
        return conv3x3(Act(h2, x.b, x.h, x.w), r.w2, r.b2, cout=r.cout, residual=res)

    def _transformer(self, a: AttnW, x: Act, ctx_kv, mode, bank, bank_kv, bank_batches):
        b, n, c = x.b, x.hw, a.c
        h = ops.groupnorm(x.data, *a.gn, batch=b, hw=n, eps=1e-6, silu=False)
        h = ops.gemm(h, a.pin_w, bias=a.pin_b)
        # --- attn1 (self / self + bank) ---
        n1 = ops.layernorm(h, *a.ln1)
        if mode == "write":
            bank.append(n1)
            if bank_batches and len(bank) >= bank_batches:
                # the LAST bank entry has been produced: everything after it in the appearance net (this
                # block's attentions and feed-forward, the rest of the decoder) is dead compute (SURVEY §8a a4)
                raise _BankComplete()
        # V^T [C, B*ldv] from the tokens padded per sample (a copy only where n % 8 != 0, on the auxiliary stream with
        # the GEMM); q and k stay on the unpadded rows
        (vt, ldv), join_v = self._fork(lambda: _vt(a.wv, n1, b))
        qk = ops.gemm(n1, a.wqk)
        join_v()
        kw = {}
        if mode == "read" and bank_kv is not None:
            k1, vt1, nb1, kvb1 = bank_kv
            kw = dict(k1=k1, vt1=vt1, n1=nb1, kv1_batches=kvb1, ldv1_batch=vt1.shape[1] // kvb1,
                      bank_batches=min(bank_batches, b))
        at = ops.attention(qk[:, :c], qk[:, c:], vt, n, heads=a.heads, d=a.d, batch=b, nq=n, ldv0_batch=ldv, **kw)
        h = ops.gemm(at, a.wo, bias=a.bo, residual=h)
        # --- attn2 (text) ---
        # norm2 is folded into the projection: W diag(gamma) on the raw h, row statistics taken by the GEMM's epilogue
        # warps from the staged A tiles, rstd (acc - mean u) + W beta in the epilogue (no LayerNorm kernel, no n2 tensor)
        q2 = ops.gemm(h, a.wq2_ln, bias=a.q2_v, ln_u=a.q2_u, ln_eps=1e-5)
        kt, vtt, nt, kvb, ldv = ctx_kv
        at2 = ops.attention(q2, kt, vtt, nt, heads=a.heads, d=a.d, batch=b, nq=n, kv0_batches=kvb if kvb == b else 1,
                            ldv0_batch=ldv)
        h = ops.gemm(at2, a.wo2, bias=a.bo2, residual=h)
        # --- GEGLU feed-forward ---
        n3 = ops.layernorm(h, *a.ln3)
        ff = ops.gemm(n3, a.wff1, bias=a.bff1, epilogue=ops.EPI_GEGLU)
        h = ops.gemm(ff, a.wff2, bias=a.bff2, residual=h)
        y = ops.gemm(h, a.pout_w, bias=a.pout_b, residual=x.data)
        return Act(y, x.b, x.h, x.w)

    def _run_block(self, net, bp, blk, x: Act, skip, emb_all, ctx_kvs, state):
        for kind, j, cin, cout in blk:
            p = f"{bp}{j}."
            lw = net.layers[p]
            if kind == "conv_in":
                x = conv3x3(x, lw[0], lw[1], cout=cout, residual=state.get("hint"))
            elif kind == "res":
                x = self._res(lw, x, skip, emb_all)
                skip = None
            elif kind == "attn":
                i = state["attn_i"]
                bank_kv = state["bank_kv"][i] if state.get("bank_kv") is not None else None
                x = self._transformer(lw, x, ctx_kvs[i], state["mode"], state.get("bank"), bank_kv,
                                      state.get("bank_batches", 0))
                state["attn_i"] = i + 1
            elif kind == "down":
                x = conv3x3(x, lw[0], lw[1], cout=cout, stride=2)
            elif kind == "up":
                up = ops.upsample2x(x.data, batch=x.b, h=x.h, w=x.w, c=x.c)
                x = conv3x3(Act(up, x.b, 2 * x.h, 2 * x.w), lw[0], lw[1], cout=cout)
        return x

    # ---- the three networks -------------------------------------------------------------------
    def _prep(self, x_nchw, context, copies=1):
        x = x_nchw.to(device=self.device, dtype=torch.float32)
        b, c, h, w = x.shape
        act = Act(ops.nchw_f32_to_nhwc_f16(x, copies=copies), copies * b, h, w)
        ctx16 = context.to(device=self.device, dtype=torch.float16).contiguous()
        return act, ctx16

    def appearance_write(self, ref_latent, t, context):
        """ControlNetReferenceOnly.forward 'write' (cldm.py:469-497): returns the bank, a list of 16
        norm1(x) token matrices [B*N_l, C_l] fp16 (attention.py:287-298).  Layers after the last
        norm1 (dead compute in the reference, SURVEY §8a a4) are skipped."""
        net = self.appearance
        x, ctx16 = self._prep(ref_latent, context)
        ctx_kvs = self.context_kv(net, ctx16, context)
        emb_all = self.time_bias(net, t, x.b)
        n_total = len(net.attn_layers())
        # in write mode `bank_batches` carries the number of bank entries after which the pass may stop
        state = {"mode": "write", "attn_i": 0, "bank": [], "bank_batches": n_total}
        hs = []
        try:
            for i, blk in enumerate(net.inp):
                x = self._run_block(net, f"input_blocks.{i}.", blk, x, None, emb_all, ctx_kvs, state)
                hs.append(x)
            x = self._run_block(net, "middle_block.", net.mid, x, None, emb_all, ctx_kvs, state)
            for i, blk in enumerate(net.out):
                x = self._run_block(net, f"output_blocks.{i}.", blk, x, hs.pop(), emb_all, ctx_kvs, state)
        except _BankComplete:
            pass
        return state["bank"]

    def attn_geometry(self, h, w):
        """(tokens, channels) of every attention layer of the UNet, in bank order, for an h x w latent."""
        net = self.unet
        geo = []
        for blk in net.inp:
            for kind, _, _, cout in blk:
                if kind == "attn":
                    geo.append((h * w, cout))
                elif kind == "down":
                    h, w = h // 2, w // 2
        geo.append((h * w, net.mid[1][3]))
        for blk in net.out:
            for kind, _, _, cout in blk:
                if kind == "attn":
                    geo.append((h * w, cout))
                elif kind == "up":
                    h, w = 2 * h, 2 * w
        return geo

    def project_bank(self, bank, batches, out=None):
        """K/V of the bank under the DENOISING UNet's attn1.to_k/to_v (attention.py:289,307):
        algebraically identical to projecting cat([x_norm1] + bank) (SURVEY §8a semantics 1).
        Returns per layer (K [batches*N, C], V^T [C, batches*ldv], N, batches): each sample's V^T column block is
        ldv = V^T.shape[1] // batches wide (N rounded up to a multiple of 8, ops.pad_tokens), the attention's
        ldv1_batch.  With `out` (a list of such tuples aliasing preallocated storage, see parallel.BankLayout) the
        GEMMs write in place."""
        res = []
        layers = self.unet.attn_layers()
        assert len(layers) == len(bank)
        for i, (a, n1) in enumerate(zip(layers, bank)):
            c = a.c
            rows = n1.shape[0]
            ko, vo = (out[i][0], out[i][1]) if out is not None else (None, None)
            k1 = ops.gemm(n1, a.wqk[c:], out=ko)
            vt1, _ = _vt(a.wv, n1, batches, out=vo)
            res.append((k1, vt1, rows // batches, batches))
        return res

    def bank_kv(self, ref_latent, t, context):
        """project_bank of the appearance bank of ref_latent: the bank_kv argument of unet_forward"""
        return self.project_bank(self.appearance_write(ref_latent, t, context), ref_latent.shape[0])

    def hint_features(self, pose_map):
        """ControlNet.input_hint_block (cldm.py:599-615); depends only on the pose map."""
        net = self.pose
        hint = pose_map.to(device=self.device, dtype=torch.float32)
        b, c, h, w = hint.shape
        x = ops.nchw_f32_to_nhwc_f16(hint)
        strides = (1, 1, 2, 1, 2, 1, 2, 1)
        for i, ((wt, bias, cin, cout), s) in enumerate(zip(net.hint, strides)):
            last = i == len(strides) - 1
            if last and _igemm_ok(h, w, cin):
                x = ops.gemm(x, wt, bias=bias, conv=(b, h, w, cin))
            elif last and cin % 64 == 0:  # pixels that do not tile into TMA boxes: TMA im2col loads
                x = ops.conv3x3_igemm(x, wt, conv=(b, h, w, cin), bias=bias)
            else:
                x = ops.conv3x3_direct(x, wt, bias, batch=b, h=h, w=w, cin=cin, cout=cout, stride=s, silu=not last)
            h, w = (h + 2 - 3) // s + 1, (w + 2 - 3) // s + 1
        return x  # [B*h*w, model_channels]

    def controlnet(self, x_noisy, hint_feat, t, context, emb_all=None):
        """ControlNet.forward (cldm.py:736-757) -> 13 residuals as fp16 [B*H*W, C] matrices.
        emb_all: precomputed time_bias(self.pose, t) (it depends on the timestep only: a sampler computes it once
        per schedule entry instead of once per frame-step)."""
        net = self.pose
        x, ctx16 = self._prep(x_noisy, context)
        ctx_kvs = self.context_kv(net, ctx16, context)
        if emb_all is None:
            emb_all = self.time_bias(net, t, x.b)
        state = {"mode": "plain", "attn_i": 0, "hint": hint_feat}
        outs = []
        for i, blk in enumerate(net.inp):
            x = self._run_block(net, f"input_blocks.{i}.", blk, x, None, emb_all, ctx_kvs, state)
            state["hint"] = None
            zw, zb = net.zero[i]
            outs.append(ops.gemm(x.data, zw, bias=zb))
        x = self._run_block(net, "middle_block.", net.mid, x, None, emb_all, ctx_kvs, state)
        zw, zb = net.zero[-1]
        outs.append(ops.gemm(x.data, zw, bias=zb))
        return outs

    def unet_forward(self, x_noisy, t, context, bank_kv=None, pose=None, uc=False, taps=None, cfg_pair=False,
                     before_pose=None, emb_all=None):
        """ControlledUnetModelAttnPose.forward (cldm.py:59-112).  uc=True: plain SD UNet without bank
        or pose residuals (cldm.py:70-84); otherwise 'read' mode.  bank_kv: project_bank() output.
        Returns eps as NCHW fp32.

        cfg_pair=True runs the conditional AND the unconditional evaluation of p_sample_ddim
        (ddim.py:598-604: same x, t and text for both) as ONE batch of 2B samples: every shared-weight
        layer streams its weights once and sees twice the rows; samples [0,B) read the bank and take the
        pose residuals, samples [B,2B) do neither.  Returns (eps_cond, eps_uncond)."""
        net = self.unet
        x, ctx16 = self._prep(x_noisy, context, copies=2 if cfg_pair else 1)
        b = x_noisy.shape[0]
        assert not (cfg_pair and uc)
        paired = cfg_pair and ctx16.shape[0] > 1  # a single context row is broadcast to both halves as it is
        if paired:
            ctx16 = torch.cat([ctx16, ctx16])
        ctx_kvs = self.context_kv(net, ctx16, context, paired)
        if emb_all is None:  # (else: precomputed time_bias(self.unet, t), one row per distinct timestep)
            emb_all = self.time_bias(net, t, x.b)  # the pair repeats the timesteps: row b uses t[b % B]
        state = {"mode": "plain" if uc else "read", "attn_i": 0}
        pose = None if (uc or pose is None) else list(pose)
        state["bank_kv"] = None if uc else bank_kv
        state["bank_batches"] = b
        hs = []

        def add_pose(act):
            p = pose.pop()
            if cfg_pair:  # in place on the conditional half only
                first = act.data[:b * act.hw]
                ops.add(first, p, batch=b, out=first)
                return act
            return Act(ops.add(act.data, p, batch=b), act.b, act.h, act.w)

        for i, blk in enumerate(net.inp):
            x = self._run_block(net, f"input_blocks.{i}.", blk, x, None, emb_all, ctx_kvs, state)
            hs.append(x)
            if taps is not None:
                taps.append(x)
        x = self._run_block(net, "middle_block.", net.mid, x, None, emb_all, ctx_kvs, state)
        if taps is not None:
            taps.append(x)
        if before_pose is not None:
            before_pose()  # join point for a pose ControlNet running on another stream
        if pose is not None:
            x = add_pose(x)
        for i, blk in enumerate(net.out):
            skip = hs.pop()
            if pose is not None:
                skip = add_pose(skip)
            x = self._run_block(net, f"output_blocks.{i}.", blk, x, skip, emb_all, ctx_kvs, state)
            if taps is not None:
                taps.append(x)
        hn = ops.groupnorm(x.data, *net.out_gn, batch=x.b, hw=x.hw, eps=1e-5, silu=True)
        y = conv3x3(Act(hn, x.b, x.h, x.w), net.out_w, net.out_b, cout=self.cfg.out_channels)
        eps = ops.nhwc_f16_to_nchw_f32(y.data, batch=x.b, c=self.cfg.out_channels, h=x.h, w=x.w)
        if cfg_pair:
            return eps[:b], eps[b:]
        return eps

    # ---- glue ---------------------------------------------------------------------------------
    def apply_model(self, x_noisy, t, context, pose_map, reference_image_noisy, uc=False, hint_feat=None,
                    bank_kv=None, return_parts=False):
        """ControlLDMReferenceOnlyPose.apply_model (cldm.py:1099-1117).  Unlike the reference, the
        unconditional call does not run the pose ControlNet whose output it would discard
        (cldm.py:1112-1114 vs 70-84).  An engine without a pose ControlNet (self.pose None) is the stage-1
        ControlLDMReferenceOnly.apply_model (cldm.py:1067-1077): pose_map is ignored and no residuals are added."""
        t = t.to(device=self.device, dtype=torch.int64)
        bank, pose = None, None
        if not uc:
            if bank_kv is None and reference_image_noisy is not None:
                rb = reference_image_noisy.shape[0]
                bank = self.appearance_write(reference_image_noisy, t[:rb], context[:rb])
                bank_kv = self.project_bank(bank, rb)
            if self.pose is not None:
                if hint_feat is None:
                    hint_feat = self.hint_features(pose_map)
                pose = self.controlnet(x_noisy, hint_feat, t, context)
        else:
            pose, bank_kv = None, None
        taps = [] if return_parts else None
        eps = self.unet_forward(x_noisy, t, context, bank_kv=bank_kv, pose=pose, uc=uc, taps=taps)
        if return_parts:
            return eps, bank, pose, taps
        return eps
