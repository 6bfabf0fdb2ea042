"""Differentiable forward of the three networks on the sm_90a kernels: the training counterpart of
engine.DenoiseEngine.apply_model (uc=False) for ControlLDMReferenceOnlyPose.p_losses (ddpm.py:2165-2212), and of the
two networks of the stage-1 ControlLDMReferenceOnly (no pose ControlNet).

It walks the same engine.block_plan as the inference engine, but every layer is one of the autograd ops of
magicdance_b200.ops (tc_gemm, two_source_attention, group_norm, layer_norm, geglu, direct_conv3x3, skinny_linear_ad,
upsample_2x, add_ad, nchw_to_nhwc / nhwc_to_nchw), so loss.backward() runs the backward kernels.  Where the inference
engine fuses a layer that has no backward kernel, training runs it unfused: norm2 -> attn2.to_q is layer_norm then
tc_gemm, and the GEGLU projection is tc_gemm on ff.net.0.proj in its own row order followed by geglu.  Text K/V are
projected per call (two of the nets train them) and none of the inference caches (text K/V, hint features, bank) is
read or written.

Weights: each kernel reads an fp16 copy in its own layout, passed beside the fp32 tensor that receives the gradient
(w_param / a_param).  Copies of trainable parameters are made once per forward, before any checkpointed region (as
autocast does); copies of frozen ones are cached on the module, keyed on the parameters' storage and version counter.
Stacked weights (attn1 q | k, the emb_layers of a net with the first conv's bias folded in) are torch.cat of the
parameters, so autograd routes their gradients back.

Activation checkpointing (torch.utils.checkpoint, non-reentrant) wraps every ResBlock and SpatialTransformer of a net
whose module has use_checkpoint set, as the reference's CheckpointFunction does (util.py:101-187).  The kernels are
deterministic, so the recompute reproduces the forward bit for bit and the gradients do not depend on the flag.

Gradient range: activation gradients are fp16 in every backward kernel.  The gradient of the loss with respect to eps is
scaled by a power of two at the output boundary (largest element in [1, 2)) and the scale is taken off the fp32
gradients of the parameters and of x_noisy again, exactly; a caller's GradScaler factor passes through unchanged, and
non-finite gradients propagate as they are.
"""
from __future__ import annotations

import torch
from torch.utils.checkpoint import checkpoint

from . import ops
from .engine import Act, _BankComplete, _igemm_ok, block_plan

CUDA_ONLY = ("magicdance_b200: the training forward and backward run only on an sm_90 CUDA device, with no CPU "
             "fallback — move the model to the GPU first")


# ------------------------------------------------------------------------------------------------
# gradient scaling at the boundary
# ------------------------------------------------------------------------------------------------
class GradScale:
    """One power-of-two scale per forward: set by the output's backward from dL/d(eps), divided out at the inputs."""

    def __init__(self):
        self.s = None


class _ScaleOut(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gs):
        ctx.gs = gs
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        amax = g.abs().amax().float()
        ok = torch.isfinite(amax) & (amax > 0)
        e = torch.floor(torch.log2(torch.where(ok, amax, torch.ones_like(amax))))
        s = torch.where(ok, torch.exp2(-e), torch.ones_like(amax))
        ctx.gs.s = s
        return g * s.to(g.dtype), None


class _Unscale(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gs):
        ctx.gs = gs
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        s = ctx.gs.s
        return (g if s is None else g / s.to(g.dtype)), None


def _input(t, gs):
    return _Unscale.apply(t, gs) if t.requires_grad else t


# ------------------------------------------------------------------------------------------------
# weights
# ------------------------------------------------------------------------------------------------
def _mat(w):
    """Linear (out, in) as it is; a 1x1 Conv2d (O, I, 1, 1) viewed as (O, I)"""
    return w.reshape(w.shape[0], -1)


class _Weights:
    """One drop-in network's parameters as the kernels of one training forward see them."""

    def __init__(self, module, gs):
        self.params = dict(module.named_parameters())
        self.cache = module.__dict__.setdefault("_mdb_train_cache", {})
        self.gs = gs
        self.seen = {}

    def p(self, name):
        """the fp32 parameter as the graph sees it (through the gradient unscale when it is trained)"""
        t = self.params[name]
        if not t.requires_grad:
            return t
        if name not in self.seen:
            self.seen[name] = _Unscale.apply(t, self.gs)
        return self.seen[name]

    def packed(self, key, names, source, pack=lambda w: w):
        """(fp16 copy, fp32 source): source(*params) is the tensor that receives the gradient (the parameter itself,
        a view or a torch.cat of several), pack(source) the kernel's layout of it"""
        src = [self.params[n] for n in names]
        if any(t.requires_grad for t in src):
            wp = source(*(self.p(n) for n in names))
            return pack(wp.detach()).to(torch.float16).contiguous(), wp
        ver = tuple((t.data_ptr(), t._version) for t in src)
        hit = self.cache.get(key)
        if hit is None or hit[0] != ver:
            wp = source(*src)
            hit = (ver, pack(wp).to(torch.float16).contiguous(), wp)
            self.cache[key] = hit
        return hit[1], hit[2]

    def conv(self, name):
        return self.packed((name, "conv"), [name], lambda w: w, ops.pack_conv_weight)

    def mat(self, name):
        return self.packed((name, "mat"), [name], _mat)


class _Res:
    pass


class _Attn:
    pass


class TrainNet:
    """One drop-in network (UNetModel subclass) with its weights packed for one training forward."""

    def __init__(self, module, gs):
        self.cfg, self.kind = module.cfg, module._kind
        self.use_checkpoint = bool(getattr(module, "use_checkpoint", False))
        self.inp, self.mid, self.out = block_plan(self.cfg)
        W = _Weights(module, gs)
        self.te0, self.te0_b = W.mat("time_embed.0.weight"), W.p("time_embed.0.bias")
        self.te2, self.te2_b = W.mat("time_embed.2.weight"), W.p("time_embed.2.bias")
        self.layers = {}
        emb_names, emb_b, off = [], [], 0
        for bp, blk in self.blocks():
            for kind, j, cin, cout in blk:
                p = f"{bp}{j}."
                if kind == "conv_in":
                    self.layers[p] = (W.conv(p + "weight"), W.p(p + "bias"))
                elif kind == "res":
                    r = _Res()
                    r.cin, r.cout = cin, cout
                    r.gn1 = (W.p(p + "in_layers.0.weight"), W.p(p + "in_layers.0.bias"))
                    r.w1 = W.conv(p + "in_layers.2.weight")
                    r.gn2 = (W.p(p + "out_layers.0.weight"), W.p(p + "out_layers.0.bias"))
                    r.w2, r.b2 = W.conv(p + "out_layers.3.weight"), W.p(p + "out_layers.3.bias")
                    if p + "skip_connection.weight" in W.params:
                        r.skip, r.skip_b = W.mat(p + "skip_connection.weight"), W.p(p + "skip_connection.bias")
                    else:
                        r.skip = r.skip_b = None
                    emb_names.append(p + "emb_layers.1.weight")
                    emb_b.append(W.p(p + "emb_layers.1.bias") + W.p(p + "in_layers.2.bias"))
                    r.emb_off = off
                    off += cout
                    self.layers[p] = r
                elif kind == "attn":
                    self.layers[p] = self._attn(W, p, cin)
                elif kind == "down":
                    self.layers[p] = (W.conv(p + "op.weight"), W.p(p + "op.bias"))
                elif kind == "up":
                    self.layers[p] = (W.conv(p + "conv.weight"), W.p(p + "conv.bias"))
        # the emb_layers Linear of every ResBlock (openaimodel.py:238-244) stacked for one skinny GEMM per forward
        self.emb = W.packed(("emb", "stack"), emb_names, lambda *ws: torch.cat(ws, 0))
        self.emb_b = torch.cat(emb_b, 0)
        if self.kind == "unet":
            self.out_gn = (W.p("out.0.weight"), W.p("out.0.bias"))
            self.out_w, self.out_b = W.conv("out.2.weight"), W.p("out.2.bias")
        if self.kind == "controlnet":
            self.hint = []
            for i in range(8):
                nm = f"input_hint_block.{2 * i}."
                shape = W.params[nm + "weight"].shape
                self.hint.append((W.conv(nm + "weight"), W.p(nm + "bias"), shape[1], shape[0]))
            self.zero = [(W.mat(f"zero_convs.{i}.0.weight"), W.p(f"zero_convs.{i}.0.bias")) for i in range(len(self.inp))]
            self.zero.append((W.mat("middle_block_out.0.weight"), W.p("middle_block_out.0.bias")))

    def blocks(self):
        bl = [(f"input_blocks.{i}.", b) for i, b in enumerate(self.inp)] + [("middle_block.", self.mid)]
        if self.kind != "controlnet":
            bl += [(f"output_blocks.{i}.", b) for i, b in enumerate(self.out)]
        return bl

    def _attn(self, W, p, c):
        a = _Attn()
        a.c, a.heads, a.d = c, self.cfg.num_heads, c // self.cfg.num_heads
        t = p + "transformer_blocks.0."
        a.gn = (W.p(p + "norm.weight"), W.p(p + "norm.bias"))
        a.pin, a.pin_b = W.mat(p + "proj_in.weight"), W.p(p + "proj_in.bias")
        a.pout, a.pout_b = W.mat(p + "proj_out.weight"), W.p(p + "proj_out.bias")
        for i in (1, 2, 3):
            setattr(a, f"ln{i}", (W.p(t + f"norm{i}.weight"), W.p(t + f"norm{i}.bias")))
        a.wqk = W.packed((t + "attn1.qk", "stack"), [t + "attn1.to_q.weight", t + "attn1.to_k.weight"],
                         lambda q, k: torch.cat([q, k], 0))
        a.wv = W.mat(t + "attn1.to_v.weight")
        a.wo, a.bo = W.mat(t + "attn1.to_out.0.weight"), W.p(t + "attn1.to_out.0.bias")
        a.wq2, a.wk2, a.wv2 = (W.mat(t + f"attn2.to_{x}.weight") for x in "qkv")
        a.wo2, a.bo2 = W.mat(t + "attn2.to_out.0.weight"), W.p(t + "attn2.to_out.0.bias")
        a.wff1, a.bff1 = W.mat(t + "ff.net.0.proj.weight"), W.p(t + "ff.net.0.proj.bias")
        a.wff2, a.bff2 = W.mat(t + "ff.net.2.weight"), W.p(t + "ff.net.2.bias")
        return a

    def n_attn(self):
        return sum(1 for _, blk in self.blocks() for kind, *_ in blk if kind == "attn")


# ------------------------------------------------------------------------------------------------
# layers and blocks
# ------------------------------------------------------------------------------------------------
def check_latent_size(cfg, h, w):
    """The training forward halves the latent at every level but the last and concatenates each output block's input
    with the skip of the same size, so both sides must be divisible by 2^(levels - 1) (8: 64x64, 112x64, 40x24 ...).
    Its tensor-core 3x3 convs run as implicit GEMMs over TMA boxes where the pixels tile into them and over TMA im2col
    loads otherwise, so any such size works."""
    levels = len(cfg.channel_mult)
    if h <= 0 or w <= 0 or h % (1 << (levels - 1)) or w % (1 << (levels - 1)):
        raise ValueError(f"magicdance_b200: the training forward supports latents whose sides are multiples of "
                         f"{1 << (levels - 1)} (one halving per level); {h}x{w} is not")


def _conv3x3(x: Act, w, cout, *, stride=1, bias=None, residual=None, bias_batch_stride=0) -> Act:
    """engine.conv3x3 on the autograd ops (implicit GEMM over TMA boxes or TMA im2col loads, else the direct conv for
    few channels in or out)"""
    w16, wp = w
    cin = x.c
    ho, wo = (x.h - 1) // stride + 1, (x.w - 1) // stride + 1
    if cout % 8 == 0 and cout >= 64 and cin % 64 == 0:
        if _igemm_ok(ho, wo, cin):
            y = ops.tc_gemm(x.data, w16, w_param=wp, bias=bias, bias_batch_stride=bias_batch_stride,
                            rows_per_batch=ho * wo, residual=residual, conv=(x.b, x.h, x.w, cin), conv_stride=stride)
        else:
            y = ops.conv3x3_igemm_ad(x.data, w16, w_param=wp, bias=bias, bias_batch_stride=bias_batch_stride,
                                     rows_per_batch=ho * wo, residual=residual, conv=(x.b, x.h, x.w, cin),
                                     conv_stride=stride)
    else:
        assert bias_batch_stride == 0
        y = ops.direct_conv3x3(x.data, w16, w_param=wp, bias=bias, residual=residual, batch=x.b, h=x.h, w=x.w,
                               cin=cin, cout=cout, stride=stride)
    return Act(y, x.b, ho, wo)


def _vt(w, x, b):
    """V^T = W_v x^T as [C, b*ldv]: each sample's columns start at a multiple of 8 (the attention kernels' V^T
    alignment; the deepest level of a 16x16 latent has 4 tokens), the padding columns are never read"""
    xp, ldv = ops.pad_tokens(x, b)
    return ops.tc_gemm(w[0], xp, a_param=w[1]), ldv


def _ckpt(on, fn, *args):
    return checkpoint(fn, *args, use_reentrant=False) if on else fn(*args)


def _res(net: TrainNet, r: _Res, x: Act, skip: Act | None, emb_all) -> Act:
    """ResBlock (openaimodel.py:275-295); the skip tensor of an output block is the GroupNorm's and the 1x1 skip
    conv's second source (the concat is never materialised)"""
    b, hh, ww = x.b, x.h, x.w

    def fn(xd, sd, emb):
        h = ops.group_norm(xd, *r.gn1, batch=b, hw=hh * ww, eps=1e-5, silu=True, x2=sd)
        bias = emb[:, r.emb_off:r.emb_off + r.cout].contiguous()
        h = _conv3x3(Act(h, b, hh, ww), r.w1, r.cout, bias=bias, bias_batch_stride=r.cout)
        h = ops.group_norm(h.data, *r.gn2, batch=b, hw=hh * ww, eps=1e-5, silu=True)
        if r.skip is None:
            assert sd is None
            res = xd
        else:
            res = ops.tc_gemm(xd, r.skip[0], w_param=r.skip[1], a2=sd, bias=r.skip_b)
        return _conv3x3(Act(h, b, hh, ww), r.w2, r.cout, bias=r.b2, residual=res).data

    return Act(_ckpt(net.use_checkpoint, fn, x.data, None if skip is None else skip.data, emb_all), b, hh, ww)


def _transformer(net: TrainNet, a: _Attn, x: Act, text, mode, bank_n1, stop):
    """SpatialTransformer (attention.py:366-385) around one BasicTransformerBlock (attention.py:278-320).
    mode 'write': returns (y, norm1(x)) — only norm1(x) when `stop` (the appearance net's last bank entry);
    'read': self-attention over [self ; bank] with the bank projected by this net's attn1.to_k / to_v."""
    b, n, c = x.b, x.hw, a.c
    ctx16, ctx_pad, nt, ldv = text

    def fn(xd, ctx, pad, bank):
        h = ops.group_norm(xd, *a.gn, batch=b, hw=n, eps=1e-6, silu=False)
        h = ops.tc_gemm(h, a.pin[0], w_param=a.pin[1], bias=a.pin_b)
        n1 = ops.layer_norm(h, *a.ln1)
        if stop:
            return n1
        # --- attn1: self, or self + bank ---
        qk = ops.tc_gemm(n1, a.wqk[0], w_param=a.wqk[1])
        vt, ldv0 = _vt(a.wv, n1, b)
        kw = {}
        if bank is not None:
            k1 = ops.tc_gemm(bank, a.wqk[0][c:], w_param=a.wqk[1][c:])
            vt1, ldv1 = _vt(a.wv, bank, b)
            kw = dict(k1=k1, vt1=vt1, n1=bank.shape[0] // b, kv1_batches=b, ldv1_batch=ldv1, bank_batches=b)
        at = ops.two_source_attention(qk[:, :c], qk[:, c:], vt, n, heads=a.heads, d=a.d, batch=b, nq=n,
                                      ldv0_batch=ldv0, **kw)
        h = ops.tc_gemm(at, a.wo[0], w_param=a.wo[1], bias=a.bo, residual=h)
        # --- attn2: text, one context per sample ---
        q2 = ops.tc_gemm(ops.layer_norm(h, *a.ln2), a.wq2[0], w_param=a.wq2[1])
        kt = ops.tc_gemm(ctx, a.wk2[0], w_param=a.wk2[1])
        vtt = ops.tc_gemm(a.wv2[0], pad, a_param=a.wv2[1])  # tokens padded to ldv per sample with zero rows
        at2 = ops.two_source_attention(q2, kt, vtt, nt, heads=a.heads, d=a.d, batch=b, nq=n, kv0_batches=b,
                                       ldv0_batch=ldv)
        h = ops.tc_gemm(at2, a.wo2[0], w_param=a.wo2[1], bias=a.bo2, residual=h)
        # --- GEGLU feed-forward ---
        ff = ops.geglu(ops.tc_gemm(ops.layer_norm(h, *a.ln3), a.wff1[0], w_param=a.wff1[1], bias=a.bff1))
        h = ops.tc_gemm(ff, a.wff2[0], w_param=a.wff2[1], bias=a.bff2, residual=h)
        y = ops.tc_gemm(h, a.pout[0], w_param=a.pout[1], bias=a.pout_b, residual=xd)
        return (y, n1) if mode == "write" else y

    return _ckpt(net.use_checkpoint, fn, x.data, ctx16, ctx_pad, bank_n1)


def _run_block(net: TrainNet, bp, blk, x: Act, skip, emb_all, text, st) -> Act:
    for kind, j, cin, cout in blk:
        p = f"{bp}{j}."
        lw = net.layers[p]
        if kind == "conv_in":
            x = _conv3x3(x, lw[0], cout, bias=lw[1], residual=st.get("hint"))
        elif kind == "res":
            x = _res(net, lw, x, skip, emb_all)
            skip = None
        elif kind == "attn":
            i = st["attn_i"]
            st["attn_i"] = i + 1
            if st["mode"] == "write":
                stop = i + 1 == st["n_attn"]
                out = _transformer(net, lw, x, text, "write", None, stop)
                st["bank"].append(out if stop else out[1])
                if stop:  # everything after the last norm1 of the appearance net is dead compute
                    raise _BankComplete()
                x = Act(out[0], x.b, x.h, x.w)
            else:
                bank = st["bank"][i] if st.get("bank") is not None else None
                x = Act(_transformer(net, lw, x, text, st["mode"], bank, False), x.b, x.h, x.w)
        elif kind == "down":
            x = _conv3x3(x, lw[0], cout, stride=2, bias=lw[1])
        elif kind == "up":
            up = ops.upsample_2x(x.data, batch=x.b, h=x.h, w=x.w, c=x.c)
            x = _conv3x3(Act(up, x.b, 2 * x.h, 2 * x.w), lw[0], cout, bias=lw[1])
    return x


# ------------------------------------------------------------------------------------------------
# the three networks
# ------------------------------------------------------------------------------------------------
def _time_bias(net: TrainNet, t, rows):
    """timestep_embedding -> time_embed -> every emb_layers Linear (+ the first conv's bias): fp32 [rows, sum(cout)]"""
    e = ops.timestep_embedding(t, net.cfg.model_channels, rows)
    e = ops.skinny_linear_ad(e, net.te0[0], net.te0_b, w_param=net.te0[1])
    e = ops.skinny_linear_ad(e, net.te2[0], net.te2_b, w_param=net.te2[1], silu_in=True)
    return ops.skinny_linear_ad(e, net.emb[0], net.emb_b, w_param=net.emb[1], silu_in=True)


def _text(context16):
    """(context [B*77, 768], the same padded to a multiple of 8 tokens per sample [B*ldv, 768], tokens, ldv)"""
    b, nt, cd = context16.shape
    flat = context16.reshape(b * nt, cd)
    pad, ldv = ops.pad_tokens(flat, b)
    return flat, pad, nt, ldv


def appearance_write(net: TrainNet, ref16: Act, t, text):
    """ControlNetReferenceOnly.forward 'write' (cldm.py:469-497): the 16 norm1(x) bank entries"""
    emb_all = _time_bias(net, t, ref16.b)
    st = {"mode": "write", "attn_i": 0, "bank": [], "n_attn": net.n_attn()}
    x, hs = ref16, []
    try:
        for i, blk in enumerate(net.inp):
            x = _run_block(net, f"input_blocks.{i}.", blk, x, None, emb_all, text, st)
            hs.append(x)
        x = _run_block(net, "middle_block.", net.mid, x, None, emb_all, text, st)
        for i, blk in enumerate(net.out):
            x = _run_block(net, f"output_blocks.{i}.", blk, x, hs.pop(), emb_all, text, st)
    except _BankComplete:
        pass
    return st["bank"]


def hint_features(net: TrainNet, pose_map):
    """ControlNet.input_hint_block (cldm.py:599-615): 7 direct convs + SiLU, the last conv as an implicit GEMM (over TMA
    boxes, or TMA im2col loads where the latent's pixels do not tile into them)"""
    b, _, h, w = pose_map.shape
    x = ops.nchw_to_nhwc(pose_map)
    strides = (1, 1, 2, 1, 2, 1, 2, 1)
    for i, (((w16, wp), bias, cin, cout), s) in enumerate(zip(net.hint, strides)):
        if i == len(strides) - 1 and _igemm_ok(h, w, cin):
            x = ops.tc_gemm(x, w16, w_param=wp, bias=bias, conv=(b, h, w, cin))
        elif i == len(strides) - 1 and cin % 64 == 0:
            x = ops.conv3x3_igemm_ad(x, w16, w_param=wp, bias=bias, conv=(b, h, w, cin))
        else:
            x = ops.direct_conv3x3(x, w16, w_param=wp, bias=bias, batch=b, h=h, w=w, cin=cin, cout=cout, stride=s,
                                   silu=i != len(strides) - 1)
        h, w = (h - 1) // s + 1, (w - 1) // s + 1
    return x


def controlnet(net: TrainNet, x: Act, hint, t, text):
    """ControlNet.forward (cldm.py:736-757): 13 zero-conv outputs; the hint enters once, through conv_in's residual"""
    emb_all = _time_bias(net, t, x.b)
    st = {"mode": "plain", "attn_i": 0, "hint": hint}
    outs = []
    for i, blk in enumerate(net.inp):
        x = _run_block(net, f"input_blocks.{i}.", blk, x, None, emb_all, text, st)
        st["hint"] = None
        (zw, zp), zb = net.zero[i]
        outs.append(ops.tc_gemm(x.data, zw, w_param=zp, bias=zb))
    x = _run_block(net, "middle_block.", net.mid, x, None, emb_all, text, st)
    (zw, zp), zb = net.zero[-1]
    outs.append(ops.tc_gemm(x.data, zw, w_param=zp, bias=zb))
    return outs


def unet(net: TrainNet, x: Act, t, text, bank, pose):
    """ControlledUnetModelAttnPose.forward (cldm.py:59-112) in 'read' mode: NHWC fp16 [B*H*W, out_channels].
    pose None: ControlledUnetModelAttn.forward (cldm.py:115-161), the stage-1 UNet without residual adds."""
    emb_all = _time_bias(net, t, x.b)
    st = {"mode": "read", "attn_i": 0, "bank": bank}
    pose = None if pose is None else list(pose)
    hs = []
    for i, blk in enumerate(net.inp):
        x = _run_block(net, f"input_blocks.{i}.", blk, x, None, emb_all, text, st)
        hs.append(x)
    x = _run_block(net, "middle_block.", net.mid, x, None, emb_all, text, st)
    if pose is not None:
        x = Act(ops.add_ad(x.data, pose.pop(), batch=x.b), x.b, x.h, x.w)
    for i, blk in enumerate(net.out):
        s = hs.pop()
        if pose is not None:
            s = Act(ops.add_ad(s.data, pose.pop(), batch=s.b), s.b, s.h, s.w)
        x = _run_block(net, f"output_blocks.{i}.", blk, x, s, emb_all, text, st)
    hn = ops.group_norm(x.data, *net.out_gn, batch=x.b, hw=x.hw, eps=1e-5, silu=True)
    return _conv3x3(Act(hn, x.b, x.h, x.w), net.out_w, net.cfg.out_channels, bias=net.out_b)


def apply_model(unet_module, appearance_module, pose_module, x_noisy, t, context, pose_map, reference_latent):
    """ControlLDMReferenceOnlyPose.apply_model (cldm.py:1099-1117, uc=False) as a differentiable function of every
    parameter of the three drop-in networks that requires grad, and of x_noisy (and context) when they do.
    Returns eps as NCHW fp32.  reference_latent: the appearance net's input (the clean latent with wonoise), one per
    sample, or None (no bank).  pose_module None: the stage-1 ControlLDMReferenceOnly.apply_model (cldm.py:1067-1077),
    with no hint path, no pose ControlNet and no residual adds; pose_map is not read."""
    modules = tuple(m for m in (unet_module, appearance_module, pose_module) if m is not None)
    try:
        for dev in {x_noisy.device} | {p.device for m in modules for p in m.parameters()}:
            ops.require_cuda(dev)
    except RuntimeError as e:
        raise NotImplementedError(CUDA_ONLY) from e
    ops.ensure_device()
    dev = x_noisy.device
    b, _, h, w = x_noisy.shape
    check_latent_size(unet_module.cfg, h, w)
    if reference_latent is not None and tuple(reference_latent.shape) != tuple(x_noisy.shape):
        raise ValueError("magicdance_b200: the training forward takes one reference latent per sample, shaped like "
                         "x_noisy")
    gs = GradScale()
    with torch.autocast("cuda", enabled=False):
        # fp16 copies of the trained weights: once per forward, outside every checkpointed region
        un, app = TrainNet(unet_module, gs), TrainNet(appearance_module, gs)
        pose = None if pose_module is None else TrainNet(pose_module, gs)
        t = t.to(device=dev, dtype=torch.int64).reshape(-1)
        if t.shape[0] == 1 and b > 1:
            t = t.expand(b).contiguous()
        ctx = _input(context.to(device=dev, dtype=torch.float32), gs).to(torch.float16)
        if ctx.shape[0] == 1 and b > 1:
            ctx = ctx.expand(b, -1, -1)
        text = _text(ctx.contiguous())
        x16 = Act(ops.nchw_to_nhwc(_input(x_noisy.to(torch.float32), gs)), b, h, w)
        bank = None
        if reference_latent is not None:
            ref = _input(reference_latent.to(device=dev, dtype=torch.float32), gs)
            bank = appearance_write(app, Act(ops.nchw_to_nhwc(ref), b, h, w), t, text)
        residuals = None
        if pose is not None:
            hint = hint_features(pose, _input(pose_map.to(device=dev, dtype=torch.float32), gs).contiguous())
            residuals = controlnet(pose, x16, hint, t, text)
        y = unet(un, x16, t, text, bank, residuals)
        eps = ops.nhwc_to_nchw(y.data, batch=b, c=un.cfg.out_channels, h=h, w=w)
        return _ScaleOut.apply(eps, gs)
