"""First-stage VAE decoder / encoder on the hot path's kernels (SURVEY §8f rank 2).

`decode_first_stage` (ldm/models/diffusion/ddpm.py:2100-2108 -> ldm/models/autoencoder.py:88-91 ->
ldm/modules/diffusionmodules/model.py:619-652) is the step right after the denoising loop, once per frame:
2514.5 GFLOP at 512x512, more than one CFG denoise step.  It is ResnetBlocks (GroupNorm(32, eps 1e-6) -> swish ->
conv3x3, model.py:129-149), three nearest-x2 upsample convs, and ONE single-head attention over all 512 channels in
the middle block (model.py:179-203) — so it maps onto the kernels the denoiser already has:

  conv3x3            engine.conv3x3: wgmma implicit GEMM at every level — a 128-pixel TMA box is whole rows at the
                     64- and 128-pixel levels and a segment of ONE row (x0 = m0 mod w) at 256 and 512; the direct
                     conv for the 3-, 4- and 8-channel ends (conv_in, conv_out, post_quant_conv, quant_conv)
  GroupNorm + swish  ops.groupnorm(eps=1e-6, silu=True) — 4, 8 and 16 channels per group
  1x1 convs          ops.gemm (nin_shortcut, q, k, proj_out); v is produced transposed by swapping operands
  attention (d=512)  ops.gemm (q k^T, scale folded into the q weights) -> ops.softmax_rows -> ops.gemm (P V);
                     the v bias is folded into proj_out's bias (rows of P sum to one)
  post_quant_conv    a 3x3 direct conv whose only non-zero tap is the centre (1x1 conv, 1/scale_factor folded in)

tests/test_vae_gpu.py holds decode / encode to rel-L2 <= 5e-3 against the unmodified reference's goldens
(tests/golden/vae16.npz, vae64.npz) and the pinned oracle (oracle/vae_restatement.py).  The decoder's time per frame is
not measured.
"""
from __future__ import annotations

import torch

from . import ops
from .engine import Act, _f16, _f32, conv3x3, pack_conv1x1, pack_conv3x3

PREFIX = "first_stage_model."
CH_MULT = (1, 2, 4, 4)       # yaml:84-88
NUM_RES_BLOCKS = 2           # yaml:89
SCALE_FACTOR = 0.18215       # yaml:9
GN_EPS = 1e-6                # model.py:45-46


def _taker(state_dict, consumed):
    """take(name): first_stage_model.<name> of the state dict in fp32, its key appended to `consumed`"""
    def take(name):
        key = PREFIX + name
        consumed.append(key)
        return state_dict[key].detach().float()
    return take


def _center_tap(w1x1, input_scale=1.0):
    """[O, I, 1, 1] -> a 3x3 kernel whose only non-zero tap is the centre (a 1x1 conv on the direct-conv kernel),
    applied to its input divided by input_scale"""
    o, i = w1x1.shape[:2]
    w3 = torch.zeros(o, i, 3, 3)
    w3[:, :, 1, 1] = w1x1[:, :, 0, 0] / input_scale
    return w3


class _Res:
    """one ResnetBlock: (gamma1, beta1), conv1, (gamma2, beta2), conv2, optional 1x1 shortcut"""

    def __init__(self, take, name, device):
        self.gn1 = (_f32(take(name + ".norm1.weight"), device), _f32(take(name + ".norm1.bias"), device))
        w1 = take(name + ".conv1.weight")
        self.cin, self.cout = w1.shape[1], w1.shape[0]
        self.w1, self.b1 = pack_conv3x3(w1, device), _f32(take(name + ".conv1.bias"), device)
        self.gn2 = (_f32(take(name + ".norm2.weight"), device), _f32(take(name + ".norm2.bias"), device))
        self.w2, self.b2 = pack_conv3x3(take(name + ".conv2.weight"), device), _f32(take(name + ".conv2.bias"), device)
        self.nin_w = self.nin_b = None
        if self.cin != self.cout:  # model.py:119-127 (conv_shortcut=False in this config)
            self.nin_w = pack_conv1x1(take(name + ".nin_shortcut.weight"), device)
            self.nin_b = _f32(take(name + ".nin_shortcut.bias"), device)


def _pack_mid_attention(p, take, a, c, device):
    """the middle block's single-head attention over all c channels (model.py:152-203) as p.at_gn, p.wq, p.bq, p.wk,
    p.bk, p.wv, p.wp, p.bp: scale folded into q, v bias into proj_out"""
    p.at_gn = (_f32(take(a + ".norm.weight"), device), _f32(take(a + ".norm.bias"), device))
    s = float(c) ** -0.5                                                        # model.py:190
    p.wq = _f16(take(a + ".q.weight").reshape(c, c) * s, device)
    p.bq = _f32(take(a + ".q.bias") * s, device)
    p.wk, p.bk = pack_conv1x1(take(a + ".k.weight"), device), _f32(take(a + ".k.bias"), device)
    p.wv = pack_conv1x1(take(a + ".v.weight"), device)
    bv = take(a + ".v.bias")
    wp = take(a + ".proj_out.weight").reshape(c, c)
    p.wp = _f16(wp, device)
    # softmax rows sum to one: P (V + 1 bv^T) = P V + bv^T, and proj_out(o + bv) = proj_out(o) + Wp bv
    p.bp = _f32(take(a + ".proj_out.bias") + wp @ bv, device)


def _res_block(r: _Res, x: Act) -> Act:
    """ResnetBlock (model.py:129-149)"""
    h = ops.groupnorm(x.data, *r.gn1, batch=x.b, hw=x.hw, eps=GN_EPS, silu=True)
    h = conv3x3(Act(h, x.b, x.h, x.w), r.w1, r.b1, cout=r.cout)
    h2 = ops.groupnorm(h.data, *r.gn2, batch=x.b, hw=x.hw, eps=GN_EPS, silu=True)
    res = x.data if r.nin_w is None else ops.gemm(x.data, r.nin_w, bias=r.nin_b)
    return conv3x3(Act(h2, x.b, x.h, x.w), r.w2, r.b2, cout=r.cout, residual=res)


def _mid_attention(p, x: Act) -> Act:
    """AttnBlock (model.py:152-203) of the middle block, weights as _pack_mid_attention left them on the packer p"""
    n = x.hw
    assert n % 64 == 0, "the P V product runs as a GEMM over the token axis: h*w must be a multiple of 64"
    h = ops.groupnorm(x.data, *p.at_gn, batch=x.b, hw=n, eps=GN_EPS, silu=False)
    q = ops.gemm(h, p.wq, bias=p.bq)                       # already scaled by c^-0.5
    k = ops.gemm(h, p.wk, bias=p.bk)
    o = torch.empty_like(q)
    for b in range(x.b):                                   # one [n, n] score matrix at a time
        rows = slice(b * n, (b + 1) * n)
        vt = ops.gemm(p.wv, h[rows])                       # [c, n] == V^T (bias folded into proj_out)
        s = ops.gemm(q[rows], k[rows])                     # [n, n] = q k^T
        ops.softmax_rows(s)
        ops.gemm(s, vt, out=o[rows])                       # [n, c] = P V
    return Act(ops.gemm(o, p.wp, bias=p.bp, residual=x.data), x.b, x.h, x.w)


class PackedVaeDecoder:
    """fp16 repack of `first_stage_model.{post_quant_conv, decoder.*}` (PyTorch-native layouts in, kernel layouts
    out).  `consumed` lists the state-dict keys read, so a test can check nothing is silently ignored."""

    def __init__(self, state_dict, device="cuda", scale_factor=SCALE_FACTOR):
        """scale_factor: decode() takes the latent as the sampler returns it and divides by this first
        (decode_first_stage, ddpm.py:2107); pass 1.0 to get AutoencoderKL.decode (autoencoder.py:88-91)."""
        self.device = torch.device(device)
        self.consumed = []
        dev = self.device
        take = _taker(state_dict, self.consumed)
        # post_quant_conv (autoencoder.py:34,89) on z / scale_factor (ddpm.py:2107)
        self.pq_w = pack_conv3x3(_center_tap(take("post_quant_conv.weight"), float(scale_factor)), dev)
        self.pq_b = _f32(take("post_quant_conv.bias"), dev)
        self.in_w = pack_conv3x3(take("decoder.conv_in.weight"), dev)               # [512, 36]
        self.in_b = _f32(take("decoder.conv_in.bias"), dev)
        self.c_mid = self.in_w.shape[0]
        self.mid1 = _Res(take, "decoder.mid.block_1", dev)
        self.mid2 = _Res(take, "decoder.mid.block_2", dev)
        _pack_mid_attention(self, take, "decoder.mid.attn_1", self.c_mid, dev)
        # up path, executed from the deepest level (model.py:635-643)
        self.up = {}
        for lvl in reversed(range(len(CH_MULT))):
            blocks = [_Res(take, f"decoder.up.{lvl}.block.{i}", dev) for i in range(NUM_RES_BLOCKS + 1)]
            ups = None
            if lvl != 0:
                ups = (pack_conv3x3(take(f"decoder.up.{lvl}.upsample.conv.weight"), dev),
                       _f32(take(f"decoder.up.{lvl}.upsample.conv.bias"), dev))
            self.up[lvl] = (blocks, ups)
        self.out_gn = (_f32(take("decoder.norm_out.weight"), dev), _f32(take("decoder.norm_out.bias"), dev))
        self.out_w = pack_conv3x3(take("decoder.conv_out.weight"), dev)             # [3, 9*128]
        self.out_b = _f32(take("decoder.conv_out.bias"), dev)
        self.c_out = self.out_w.shape[0]


class VaeDecoder:
    """decode_first_stage(z): latent [B, 4, h, w] fp32 (as the sampler returns it) -> image [B, 3, 8h, 8w] fp32."""

    def __init__(self, packed: PackedVaeDecoder):
        ops.ensure_device()
        self.p = packed

    @torch.no_grad()
    def decode(self, z: torch.Tensor) -> torch.Tensor:
        if not z.is_cuda:
            raise RuntimeError("magicdance_b200.vae: the decoder runs on CUDA kernels only (no CPU fallback)")
        return self._decode(z)

    def _decode(self, z: torch.Tensor) -> torch.Tensor:
        p = self.p
        assert z.dim() == 4 and z.shape[1] == 4, "latent must be [B, 4, h, w]"
        b, _, hh, ww = z.shape
        x = ops.nchw_f32_to_nhwc_f16(z.float())                                         # [b*h*w, 4]
        a = conv3x3(Act(x, b, hh, ww), p.pq_w, p.pq_b, cout=4)                           # post_quant_conv(z / scale)
        a = conv3x3(a, p.in_w, p.in_b, cout=p.c_mid)
        a = _res_block(p.mid1, a)
        a = _mid_attention(p, a)
        a = _res_block(p.mid2, a)
        for lvl in reversed(range(len(CH_MULT))):
            blocks, ups = p.up[lvl]
            for r in blocks:
                a = _res_block(r, a)
            if ups is not None:
                u = ops.upsample2x(a.data, batch=a.b, h=a.h, w=a.w, c=a.c)               # nearest (model.py:62)
                a = conv3x3(Act(u, a.b, 2 * a.h, 2 * a.w), ups[0], ups[1], cout=a.c)
        h = ops.groupnorm(a.data, *p.out_gn, batch=a.b, hw=a.hw, eps=GN_EPS, silu=True)
        y = conv3x3(Act(h, a.b, a.h, a.w), p.out_w, p.out_b, cout=p.c_out)
        return ops.nhwc_f16_to_nchw_f32(y.data, batch=a.b, c=p.c_out, h=a.h, w=a.w)


# =====================================================================================================================
# Encoder (encode_first_stage: ddpm.py:2109-2117 -> autoencoder.py:82-86 -> model.py:518-543) — the reference image is
# encoded once per sequence (1116.7 GFLOP at 512x512).  Same kernels as the decoder plus ops.im2col3x3(pad="br") for the
# Downsample's bottom/right padding.
# =====================================================================================================================
class PackedVaeEncoder:
    """fp16 repack of `first_stage_model.{encoder.*, quant_conv}`; `consumed` lists the keys read."""

    def __init__(self, state_dict, device="cuda"):
        self.device = torch.device(device)
        self.consumed = []
        dev = self.device
        take = _taker(state_dict, self.consumed)
        self.in_w = pack_conv3x3(take("encoder.conv_in.weight"), dev)                # [128, 27]
        self.in_b = _f32(take("encoder.conv_in.bias"), dev)
        self.c0 = self.in_w.shape[0]
        self.down = []
        for lvl in range(len(CH_MULT)):
            blocks = [_Res(take, f"encoder.down.{lvl}.block.{i}", dev) for i in range(NUM_RES_BLOCKS)]
            ds = None
            if lvl != len(CH_MULT) - 1:
                ds = (pack_conv3x3(take(f"encoder.down.{lvl}.downsample.conv.weight"), dev),
                      _f32(take(f"encoder.down.{lvl}.downsample.conv.bias"), dev))
            self.down.append((blocks, ds))
        self.mid1 = _Res(take, "encoder.mid.block_1", dev)
        self.c_mid = self.mid1.cout
        _pack_mid_attention(self, take, "encoder.mid.attn_1", self.c_mid, dev)
        self.mid2 = _Res(take, "encoder.mid.block_2", dev)
        self.out_gn = (_f32(take("encoder.norm_out.weight"), dev), _f32(take("encoder.norm_out.bias"), dev))
        self.out_w = pack_conv3x3(take("encoder.conv_out.weight"), dev)              # [8, 9*512]
        self.out_b = _f32(take("encoder.conv_out.bias"), dev)
        self.c_out = self.out_w.shape[0]
        self.q_w = pack_conv3x3(_center_tap(take("quant_conv.weight")), dev)         # 1x1 conv, autoencoder.py:33,84
        self.q_b = _f32(take("quant_conv.bias"), dev)


class VaeEncoder:
    """encode(x): image [B, 3, H, W] fp32 in [-1, 1] -> the posterior's moments [B, 8, H/8, W/8] fp32 (mean | logvar),
    i.e. what AutoencoderKL.encode wraps in DiagonalGaussianDistribution (autoencoder.py:82-86)."""

    def __init__(self, packed: PackedVaeEncoder):
        ops.ensure_device()
        self.p = packed

    @torch.no_grad()
    def encode(self, x: torch.Tensor) -> torch.Tensor:
        if not x.is_cuda:
            raise RuntimeError("magicdance_b200.vae: the encoder runs on CUDA kernels only (no CPU fallback)")
        return self._encode(x)

    def _encode(self, x: torch.Tensor) -> torch.Tensor:
        p = self.p
        assert x.dim() == 4 and x.shape[1] == 3 and x.shape[2] % 8 == 0 and x.shape[3] % 8 == 0, "image must be [B, 3, 8h, 8w]"
        b, _, hh, ww = x.shape
        t = ops.nchw_f32_to_nhwc_f16(x.float())                                         # [b*H*W, 3]
        a = conv3x3(Act(t, b, hh, ww), p.in_w, p.in_b, cout=p.c0)
        for blocks, ds in p.down:
            for r in blocks:
                a = _res_block(r, a)
            if ds is not None:  # F.pad(x, (0,1,0,1)) + conv(k=3, s=2, p=0)  (model.py:82-84)
                col = ops.im2col3x3(a.data, batch=a.b, h=a.h, w=a.w, c=a.c, stride=2, pad="br")
                a = Act(ops.gemm(col, ds[0], bias=ds[1]), a.b, a.h // 2, a.w // 2)
        a = _res_block(p.mid1, a)
        a = _mid_attention(p, a)
        a = _res_block(p.mid2, a)
        h = ops.groupnorm(a.data, *p.out_gn, batch=a.b, hw=a.hw, eps=GN_EPS, silu=True)
        y = conv3x3(Act(h, a.b, a.h, a.w), p.out_w, p.out_b, cout=p.c_out)
        y = conv3x3(y, p.q_w, p.q_b, cout=p.c_out)                                         # quant_conv
        return ops.nhwc_f16_to_nchw_f32(y.data, batch=a.b, c=p.c_out, h=a.h, w=a.w)


def posterior_sample(moments: torch.Tensor, noise: torch.Tensor | None = None) -> torch.Tensor:
    """DiagonalGaussianDistribution.sample / .mode (distributions.py:27-37,59-60) on the [B, 8, h, w] moments: a
    few elementwise operations on a 128 KB tensor, done with torch on the device the moments live on (off the hot
    path; the reference does the same arithmetic in torch)."""
    mean, logvar = torch.chunk(moments, 2, dim=1)
    if noise is None:
        return mean
    return mean + torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0)) * noise

