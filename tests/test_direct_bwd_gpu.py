"""Direct-conv / skinny-Linear / upsample backward on the GPU: per-shape gradient numerics (tests/direct_bwd_cases.py),
bit-reproducibility, and three pieces of the networks differentiated end to end through library kernels against the
fp32 restatement (oracle/restatement.py): the pose hint path into conv_in, the timestep MLP into a ResBlock, and the
UNet head with an output-block upsample."""
import pytest
import torch
import torch.nn.functional as F

from oracle import restatement as R
from tests import direct_bwd_cases as N
from tests.kernel_cases import _rand
from tests.kernel_guard import rel

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", N.CASES, ids=[N.case_id(c) for c in N.CASES])
def test_backward_matches_torch_fp64(case):
    fn, kw = case
    err, tol, desc = fn(**kw)
    torch.cuda.synchronize()
    print(desc)
    assert err <= tol, f"{desc}: error {err:.3e} > {tol:.1e}"


def test_backward_is_bit_reproducible():
    """every output of a repeated call is bit-equal (fixed-order reductions, no atomics)"""
    from magicdance_b200 import ops
    outs = []
    for _ in range(2):
        run = []
        for cin, cout, stride, hw in ((3, 16, 1, 256), (16, 32, 2, 256), (96, 96, 1, 64), (4, 320, 1, 64),
                                      (320, 4, 1, 64)):
            x, _, wt, b, dy, _, _ = N._conv_inputs(2, hw, hw, cin, cout, stride, True, seed=cin + cout)
            run += ops.conv3x3_direct_backward(x, wt, dy, batch=2, h=hw, w=hw, cin=cin, cout=cout, stride=stride,
                                               bias=b, silu=cin != 320)
        x, w, dy = _rand(20, 1280, seed=1), _rand(20160, 1280, seed=2, scale=0.03).half(), _rand(20, 20160, seed=3)
        run += ops.skinny_linear_backward(x, w, dy, silu_in=True)
        run.append(ops.upsample2x_backward(_rand(2 * 1024, 1280, seed=4).half(), batch=2, h=16, w=16, c=1280))
        outs.append(run)
    torch.cuda.synchronize()
    for a, b_ in zip(*outs):
        assert torch.equal(a, b_)


def _params(spec, seed):
    """{name: fp32 tensor on the GPU, rounded through fp16} for (name, shape, scale) — scale None: 1 + 0.2 N(0, 1)
    (norm weights)"""
    sd = {}
    for i, (nm, shape, scale) in enumerate(spec):
        t = 1 + 0.2 * _rand(*shape, seed=seed + i) if scale is None else _rand(*shape, seed=seed + i, scale=scale)
        sd[nm] = t.half().float()
    return sd


def _leaves(sd):
    return {k: v.clone().requires_grad_() for k, v in sd.items()}


def _nhwc(t):
    """NCHW -> [B*H*W, C]"""
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def _check(errs, sd, p, r):
    for k in sd:
        assert p[k].grad.shape == r[k].grad.shape and p[k].grad.dtype == torch.float32, k
        errs[k] = rel(p[k].grad, r[k].grad)
    print({k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) <= 1e-2, errs


def test_pose_hint_path_backward():
    """pose map (NCHW fp32) -> the hint encoder's 7 direct convs + SiLU and the 256 -> 320 GEMM conv -> conv_in 4 -> 320
    of x_noisy with the hint as its residual: all 16 hint parameters, conv_in's weight and bias and dx_noisy against
    R.hint_block + conv2d in fp32"""
    with torch.enable_grad():  # other tests switch autograd off process-wide
        _pose_hint_path()


def _pose_hint_path():
    from magicdance_b200 import ops
    b, s, lat = 2, 128, 16
    chans = [3, 16, 16, 32, 32, 96, 96, 256, 320]
    strides = (1, 1, 2, 1, 2, 1, 2, 1)
    spec = []
    for i in range(8):
        cin, cout = chans[i], chans[i + 1]
        spec += [(f"input_hint_block.{2 * i}.weight", (cout, cin, 3, 3), (9 * cin) ** -0.5 * 1.5),
                 (f"input_hint_block.{2 * i}.bias", (cout,), 0.1)]
    spec += [("input_blocks.0.0.weight", (320, 4, 3, 3), 36 ** -0.5), ("input_blocks.0.0.bias", (320,), 0.1)]
    sd = _params(spec, seed=30)
    pose = _rand(b, 3, s, s, seed=1).half().float()
    x_noisy = _rand(b, 4, lat, lat, seed=2).half().float()
    g = _rand(b * lat * lat, 320, seed=3)

    p = _leaves(sd)
    xn = x_noisy.clone().requires_grad_()
    h = ops.nchw_to_nhwc(pose)
    hh = s
    for i in range(7):
        cin, cout, st = chans[i], chans[i + 1], strides[i]
        wp = p[f"input_hint_block.{2 * i}.weight"]
        h = ops.direct_conv3x3(h, ops.pack_conv_weight(wp), w_param=wp, bias=p[f"input_hint_block.{2 * i}.bias"], batch=b,
                               h=hh, w=hh, cin=cin, cout=cout, stride=st, silu=True)
        hh = (hh - 1) // st + 1
    wl = p["input_hint_block.14.weight"]
    hint = ops.tc_gemm(h, ops.pack_conv_weight(wl), w_param=wl, bias=p["input_hint_block.14.bias"], conv=(b, hh, hh, 256))
    wc = p["input_blocks.0.0.weight"]
    out = ops.direct_conv3x3(ops.nchw_to_nhwc(xn), ops.pack_conv_weight(wc), w_param=wc, bias=p["input_blocks.0.0.bias"],
                             residual=hint, batch=b, h=lat, w=lat, cin=4, cout=320)
    (out.float() * g).sum().backward()

    r = _leaves(sd)
    rx = x_noisy.clone().requires_grad_()
    ref = R._conv(r, "input_blocks.0.0", rx) + R.hint_block(r, "", pose)
    (_nhwc(ref) * g).sum().backward()
    _check({"dx_noisy": rel(xn.grad, rx.grad)}, sd, p, r)


def test_time_path_into_resblock_backward():
    """t -> timestep embedding -> time_embed.0 -> SiLU -> time_embed.2 -> SiLU -> the stacked emb_layers (torch.cat of
    two blocks' fp32 parameters) -> this block's slice + in_layers.2.bias as the per-sample bias of a 320 -> 320
    ResBlock's first conv: every time_embed.*, emb_layers.1.* and ResBlock gradient against R.time_embed + R.resblock,
    with one timestep per sample and with one shared timestep"""
    with torch.enable_grad():
        _time_path(torch.tensor([999, 17], dtype=torch.int64, device="cuda"))
        _time_path(torch.tensor([500], dtype=torch.int64, device="cuda"))


def _time_path(t):
    from magicdance_b200 import ops
    b, hh, ww, c, mc, te = 2, 16, 16, 320, 320, 1280
    hw = hh * ww
    pre = "rb."
    sd = _params([("time_embed.0.weight", (te, mc), mc ** -0.5), ("time_embed.0.bias", (te,), 0.1),
                  ("time_embed.2.weight", (te, te), te ** -0.5), ("time_embed.2.bias", (te,), 0.1),
                  (pre + "in_layers.0.weight", (c,), None), (pre + "in_layers.0.bias", (c,), 0.2),
                  (pre + "in_layers.2.weight", (c, c, 3, 3), (9 * c) ** -0.5), (pre + "in_layers.2.bias", (c,), 0.1),
                  (pre + "emb_layers.1.weight", (c, te), te ** -0.5), (pre + "emb_layers.1.bias", (c,), 0.1),
                  (pre + "out_layers.0.weight", (c,), None), (pre + "out_layers.0.bias", (c,), 0.2),
                  (pre + "out_layers.3.weight", (c, c, 3, 3), (9 * c) ** -0.5), (pre + "out_layers.3.bias", (c,), 0.1)],
                 seed=50)
    other = _leaves(_params([("w", (640, te), te ** -0.5), ("b", (640,), 0.1)], seed=70))  # another block's emb layer
    x = _rand(b * hw, c, seed=1).half()
    g = _rand(b * hw, c, seed=2)

    p = _leaves(sd)
    xs = x.clone().requires_grad_()
    e = ops.timestep_embedding(t, mc, rows=b)
    w0, w2 = p["time_embed.0.weight"], p["time_embed.2.weight"]
    e = ops.skinny_linear_ad(e, w0.detach().half(), p["time_embed.0.bias"], w_param=w0)
    e = ops.skinny_linear_ad(e, w2.detach().half(), p["time_embed.2.bias"], w_param=w2, silu_in=True)
    emb_w = torch.cat([p[pre + "emb_layers.1.weight"], other["w"]])
    emb_b = torch.cat([p[pre + "emb_layers.1.bias"], other["b"]])
    emb_all = ops.skinny_linear_ad(e, emb_w.detach().half(), emb_b, w_param=emb_w, silu_in=True)
    bias = (emb_all[:, :c] + p[pre + "in_layers.2.bias"]).contiguous()
    a = ops.group_norm(xs, p[pre + "in_layers.0.weight"], p[pre + "in_layers.0.bias"], batch=b, hw=hw, eps=1e-5,
                       silu=True)
    a = ops.tc_gemm(a, ops.pack_conv_weight(p[pre + "in_layers.2.weight"]), w_param=p[pre + "in_layers.2.weight"], bias=bias,
                    bias_batch_stride=c, rows_per_batch=hw, conv=(b, hh, ww, c))
    a = ops.group_norm(a, p[pre + "out_layers.0.weight"], p[pre + "out_layers.0.bias"], batch=b, hw=hw, eps=1e-5,
                       silu=True)
    out = ops.tc_gemm(a, ops.pack_conv_weight(p[pre + "out_layers.3.weight"]), w_param=p[pre + "out_layers.3.weight"],
                      bias=p[pre + "out_layers.3.bias"], residual=xs, conv=(b, hh, ww, c))
    (out.float() * g).sum().backward()
    assert not other["w"].grad.any() and not other["b"].grad.any()  # the other block's slice gets exactly zero

    r = _leaves(sd)
    rx = x.float().view(b, hh, ww, c).permute(0, 3, 1, 2).contiguous().requires_grad_()
    emb = R.time_embed(r, "", t.expand(b) if t.numel() == 1 else t, mc)
    ref = R.resblock(r, pre, rx, emb)
    (_nhwc(ref) * g).sum().backward()
    _check({"dx": rel(xs.grad.float(), _nhwc(rx.grad))}, sd, p, r)


def test_unet_head_and_upsample_backward():
    """group_norm + SiLU -> the 320 -> 4 out conv (dx only, as for the frozen UNet), and upsample_2x -> the Upsample's
    3x3 conv: dh, du and the parameter gradients against R._gn / R._conv / F.interpolate(nearest)"""
    with torch.enable_grad():
        _head_and_upsample()


def _head_and_upsample():
    from magicdance_b200 import ops
    b, hh, c, cu, lo = 2, 16, 320, 640, 8
    sd = _params([("out.0.weight", (c,), None), ("out.0.bias", (c,), 0.2),
                  ("up.conv.weight", (cu, cu, 3, 3), (9 * cu) ** -0.5), ("up.conv.bias", (cu,), 0.1)], seed=90)
    w_out = _rand(4, c, 3, 3, seed=91, scale=(9 * c) ** -0.5).half().float()  # frozen: no gradient wanted
    h = _rand(b * hh * hh, c, seed=1).half()
    u = _rand(b * lo * lo, cu, seed=2).half()
    g1, g2 = _rand(b * hh * hh, 4, seed=3), _rand(b * hh * hh, cu, seed=4)

    p = _leaves(sd)
    hs, us = h.clone().requires_grad_(), u.clone().requires_grad_()
    a = ops.group_norm(hs, p["out.0.weight"], p["out.0.bias"], batch=b, hw=hh * hh, eps=1e-5, silu=True)
    eps_out = ops.direct_conv3x3(a, ops.pack_conv_weight(w_out), batch=b, h=hh, w=hh, cin=c, cout=4)
    up = ops.upsample_2x(us, batch=b, h=lo, w=lo, c=cu)
    y = ops.tc_gemm(up, ops.pack_conv_weight(p["up.conv.weight"]), w_param=p["up.conv.weight"], bias=p["up.conv.bias"],
                    conv=(b, hh, hh, cu))
    ((eps_out.float() * g1).sum() + (y.float() * g2).sum()).backward()

    r = _leaves(sd)
    rh = h.float().view(b, hh, hh, c).permute(0, 3, 1, 2).contiguous().requires_grad_()
    ru = u.float().view(b, lo, lo, cu).permute(0, 3, 1, 2).contiguous().requires_grad_()
    r["out.2.weight"] = w_out
    ref1 = R._conv(r, "out.2", F.silu(R._gn(r, "out.0", rh, 1e-5)))
    ref2 = R._conv(r, "up.conv", F.interpolate(ru, scale_factor=2, mode="nearest"))
    ((_nhwc(ref1) * g1).sum() + (_nhwc(ref2) * g2).sum()).backward()
    _check({"dh": rel(hs.grad.float(), _nhwc(rh.grad)), "du": rel(us.grad.float(), _nhwc(ru.grad))}, sd, p, r)
