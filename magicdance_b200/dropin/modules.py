"""Parameter-holding nn.Module tree with the reference's class names, constructor kwargs and
state-dict keys (SURVEY §8b) for the three networks of the hot path.  The modules own fp32
parameters exactly like the reference's (Conv2d OIHW, Linear (out,in)); their forward()s do not run
PyTorch operators — they hand the tensors to the sm_90a engine (magicdance_b200.engine).

Reference layout being mirrored (paths relative to model_lib/ControlNet/):
  ResBlock / Upsample / Downsample / TimestepEmbedSequential / UNetModel
                                   ldm/modules/diffusionmodules/openaimodel.py:73-295,432-806
  SpatialTransformer / BasicTransformerBlock / CrossAttention / FeedForward / GEGLU
                                   ldm/modules/attention.py:50-77,146-199,253-385
  ControlledUnetModelAttnPose / ControlNetReferenceOnly / ControlNet
                                   cldm/cldm.py:59-112,164-497,500-757
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops
from ..engine import NetConfig, PackedNet, block_plan


def _empty_init(module: nn.Module):
    """Cheap deterministic initial state (weights 0, norm scales 1): the reference's default-init
    model outputs exactly 0 as well (every zero_module tensor), and both are meant to be followed by
    load_state_dict()."""
    return module


def conv_nd(dims, *args, **kwargs):
    assert dims == 2, "only 2-D convolutions are on the hot path"
    return torch.nn.utils.skip_init(nn.Conv2d, *args, **kwargs)


def linear(*args, **kwargs):
    return torch.nn.utils.skip_init(nn.Linear, *args, **kwargs)


def normalization(channels, eps=1e-5):
    """GroupNorm32 (util.py:252-265): 32 groups, fp32 statistics."""
    return torch.nn.utils.skip_init(nn.GroupNorm, 32, channels, eps=eps)


def zero_module(module):
    return module


class TimestepBlock(nn.Module):
    pass


class TimestepEmbedSequential(nn.Sequential, TimestepBlock):
    """Container only: the dispatch the reference performs here (openaimodel.py:79-108) is done by the
    engine's block schedule."""


class Upsample(nn.Module):
    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=1):
        super().__init__()
        self.channels, self.out_channels, self.use_conv, self.dims = channels, out_channels or channels, use_conv, dims
        if use_conv:
            self.conv = conv_nd(dims, self.channels, self.out_channels, 3, padding=padding)


class Downsample(nn.Module):
    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=1):
        super().__init__()
        self.channels, self.out_channels, self.use_conv, self.dims = channels, out_channels or channels, use_conv, dims
        assert use_conv, "the hot path only uses the strided-conv downsample"
        self.op = conv_nd(dims, self.channels, self.out_channels, 3, stride=2, padding=padding)


class ResBlock(TimestepBlock):
    def __init__(self, channels, emb_channels, dropout, out_channels=None, use_conv=False, use_scale_shift_norm=False,
                 dims=2, use_checkpoint=False, up=False, down=False):
        super().__init__()
        assert not (up or down or use_scale_shift_norm), "resblock_updown / scale-shift norm are not used by MagicPose"
        self.channels, self.emb_channels, self.dropout = channels, emb_channels, dropout
        self.out_channels = out_channels or channels
        self.use_checkpoint = use_checkpoint
        self.in_layers = nn.Sequential(normalization(channels), nn.SiLU(),
                                       conv_nd(dims, channels, self.out_channels, 3, padding=1))
        self.emb_layers = nn.Sequential(nn.SiLU(), linear(emb_channels, self.out_channels))
        self.out_layers = nn.Sequential(normalization(self.out_channels), nn.SiLU(), nn.Dropout(p=dropout),
                                        zero_module(conv_nd(dims, self.out_channels, self.out_channels, 3, padding=1)))
        if self.out_channels == channels:
            self.skip_connection = nn.Identity()
        elif use_conv:
            self.skip_connection = conv_nd(dims, channels, self.out_channels, 3, padding=1)
        else:
            self.skip_connection = conv_nd(dims, channels, self.out_channels, 1)


class CrossAttention(nn.Module):
    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64, dropout=0., checkpoint=True):
        super().__init__()
        inner = dim_head * heads
        context_dim = query_dim if context_dim is None else context_dim
        self.scale, self.heads = dim_head ** -0.5, heads
        self.to_q = linear(query_dim, inner, bias=False)
        self.to_k = linear(context_dim, inner, bias=False)
        self.to_v = linear(context_dim, inner, bias=False)
        self.to_out = nn.Sequential(linear(inner, query_dim), nn.Dropout(dropout))


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = linear(dim_in, dim_out * 2)


class FeedForward(nn.Module):
    def __init__(self, dim, dim_out=None, mult=4, glu=False, dropout=0.):
        super().__init__()
        assert glu, "the SD transformer block uses the gated feed-forward"
        inner = int(dim * mult)
        self.net = nn.Sequential(GEGLU(dim, inner), nn.Dropout(dropout), linear(inner, dim_out or dim))


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim, n_heads, d_head, dropout=0., context_dim=None, gated_ff=True, checkpoint=True,
                 disable_self_attn=False):
        super().__init__()
        assert not disable_self_attn
        self.attn1 = CrossAttention(query_dim=dim, heads=n_heads, dim_head=d_head, dropout=dropout, checkpoint=checkpoint)
        self.ff = FeedForward(dim, dropout=dropout, glu=gated_ff)
        self.attn2 = CrossAttention(query_dim=dim, context_dim=context_dim, heads=n_heads, dim_head=d_head,
                                    dropout=dropout, checkpoint=checkpoint)
        self.norm1 = torch.nn.utils.skip_init(nn.LayerNorm, dim)
        self.norm2 = torch.nn.utils.skip_init(nn.LayerNorm, dim)
        self.norm3 = torch.nn.utils.skip_init(nn.LayerNorm, dim)


class SpatialTransformer(nn.Module):
    def __init__(self, in_channels, n_heads, d_head, depth=1, dropout=0., context_dim=None, disable_self_attn=False,
                 use_linear=False, use_checkpoint=True):
        super().__init__()
        assert depth == 1 and not use_linear, "SD1.5: transformer_depth 1 with 1x1-conv projections"
        if context_dim is not None and not isinstance(context_dim, (list, tuple)):
            context_dim = [context_dim]
        inner = n_heads * d_head
        self.in_channels = in_channels
        self.norm = normalization(in_channels, eps=1e-6)  # Normalize(), attention.py:89-90
        self.proj_in = conv_nd(2, in_channels, inner, 1)
        self.transformer_blocks = nn.ModuleList([
            BasicTransformerBlock(inner, n_heads, d_head, dropout=dropout, context_dim=context_dim[0],
                                  checkpoint=use_checkpoint)])
        self.proj_out = zero_module(conv_nd(2, inner, in_channels, 1))


def _reset(module: nn.Module):
    """weights 0, norm scales 1 (see _empty_init)"""
    with torch.no_grad():
        for m in module.modules():
            if isinstance(m, (nn.GroupNorm, nn.LayerNorm)):
                m.weight.fill_(1.0)
                m.bias.zero_()
            elif isinstance(m, (nn.Conv2d, nn.Linear)):
                m.weight.zero_()
                if m.bias is not None:
                    m.bias.zero_()


class UNetModel(nn.Module):
    """Module tree of openaimodel.py:432-806 for the configuration MagicPose uses (spatial transformer,
    num_heads given, no class conditioning).  `_kind` selects which parts exist: the appearance twin has
    no `out` head but a (dead) hint block, the ControlNet has no decoder but zero convs."""

    _kind = "unet"

    def __init__(self, image_size=32, in_channels=4, model_channels=320, out_channels=4, num_res_blocks=2,
                 attention_resolutions=(4, 2, 1), dropout=0, channel_mult=(1, 2, 4, 4), conv_resample=True, dims=2,
                 num_classes=None, use_checkpoint=False, use_fp16=False, num_heads=-1, num_head_channels=-1,
                 num_heads_upsample=-1, use_scale_shift_norm=False, resblock_updown=False,
                 use_new_attention_order=False, use_spatial_transformer=False, transformer_depth=1, context_dim=None,
                 n_embed=None, legacy=True, disable_self_attentions=None, num_attention_blocks=None,
                 disable_middle_self_attn=False, use_linear_in_transformer=False, hint_channels=3, **kwargs):
        super().__init__()
        assert use_spatial_transformer and context_dim is not None and num_heads != -1 and num_classes is None
        assert not resblock_updown and dims == 2 and transformer_depth == 1
        self.image_size, self.in_channels, self.model_channels, self.out_channels = image_size, in_channels, model_channels, out_channels
        self.num_res_blocks = num_res_blocks if not isinstance(num_res_blocks, int) else len(channel_mult) * [num_res_blocks]
        self.attention_resolutions, self.channel_mult = tuple(attention_resolutions), tuple(channel_mult)
        self.dropout, self.conv_resample, self.use_checkpoint = dropout, conv_resample, use_checkpoint
        self.dtype = torch.float32  # parameters stay fp32 (openaimodel.py:540); the kernels use fp16 copies
        self.num_heads, self.context_dim = num_heads, context_dim
        self.cfg = NetConfig(in_channels=in_channels, out_channels=out_channels or 4, hint_channels=hint_channels,
                             model_channels=model_channels, attention_resolutions=tuple(attention_resolutions),
                             num_res_blocks=num_res_blocks, channel_mult=tuple(channel_mult), num_heads=num_heads,
                             context_dim=context_dim)
        ted = model_channels * 4
        self.time_embed = nn.Sequential(linear(model_channels, ted), nn.SiLU(), linear(ted, ted))
        inp, mid, out = block_plan(self.cfg)

        def build(blk):
            layers = []
            for kind, _, cin, cout in blk:
                if kind == "conv_in":
                    layers.append(conv_nd(dims, cin, cout, 3, padding=1))
                elif kind == "res":
                    layers.append(ResBlock(cin, ted, dropout, out_channels=cout, dims=dims, use_checkpoint=use_checkpoint))
                elif kind == "attn":
                    layers.append(SpatialTransformer(cin, num_heads, cin // num_heads, depth=1, context_dim=context_dim,
                                                     use_checkpoint=use_checkpoint))
                elif kind == "down":
                    layers.append(Downsample(cin, conv_resample, dims=dims, out_channels=cout))
                elif kind == "up":
                    layers.append(Upsample(cin, conv_resample, dims=dims, out_channels=cout))
            return TimestepEmbedSequential(*layers)

        self.input_blocks = nn.ModuleList([build(b) for b in inp])
        self.middle_block = build(mid)
        if self._kind != "controlnet":
            self.output_blocks = nn.ModuleList([build(b) for b in out])
        if self._kind == "unet":
            self.out = nn.Sequential(normalization(model_channels), nn.SiLU(),
                                     zero_module(conv_nd(dims, model_channels, out_channels, 3, padding=1)))
        if self._kind in ("appearance", "controlnet"):
            chans = [hint_channels, 16, 16, 32, 32, 96, 96, 256, model_channels]
            strides = [1, 1, 2, 1, 2, 1, 2, 1]
            layers = []
            for i, s in enumerate(strides):
                layers.append(conv_nd(dims, chans[i], chans[i + 1], 3, padding=1, stride=s))
                if i != len(strides) - 1:
                    layers.append(nn.SiLU())
            self.input_hint_block = TimestepEmbedSequential(*layers)
        if self._kind == "controlnet":
            self.zero_convs = nn.ModuleList([
                TimestepEmbedSequential(conv_nd(dims, b[-1][3], b[-1][3], 1, padding=0)) for b in inp])
            self.middle_block_out = TimestepEmbedSequential(conv_nd(dims, mid[-1][3], mid[-1][3], 1, padding=0))
        _reset(self)
        self._packed = None
        self._packed_params, self._packed_key = [], ()
        self.register_load_state_dict_post_hook(lambda mod, keys: mod.invalidate())

    # ---- engine plumbing ---------------------------------------------------------------------------
    def invalidate(self):
        """Drop the repacked fp16 weights.  packed() notices in-place updates of the parameters by their version
        counters; an update that bypasses them (`p.data.copy_`, an in-place collective) needs this call."""
        self._packed = None

    def packed(self, device=None) -> PackedNet:
        """The inference packing of the current weights: the same object for as long as no parameter changes (so
        that captured graphs stay valid), rebuilt after an optimizer step or a load.  The check reads the version
        counters of the parameter list taken at packing time (walking the module tree costs milliseconds)."""
        dev = torch.device(device) if device is not None else next(self.parameters()).device
        ops.require_cuda(dev)
        if (self._packed is None or self._packed.device != dev
                or tuple(p._version for p in self._packed_params) != self._packed_key):
            self._packed_params = list(self.parameters())
            self._packed_key = tuple(p._version for p in self._packed_params)
            self._packed = PackedNet(self.state_dict(), "", self.cfg, self._kind, dev)
        return self._packed
