"""Split-K on the GPU at the skinny shapes of a one-frame step: every count from 1 to 16 (2 ... 8 reduce inside a
thread-block cluster, more through the fp32 workspace), the automatic plan of the 8x8 and 16x16 levels, every epilogue
through the cluster reduction, bit-equal repeats, graph replays and two streams.  Outputs go into poisoned, guarded
buffers and are compared with torch fp32 (tests/kernel_cases.py)."""
import pytest
import torch

from magicdance_b200 import ops
from tests import igemm_cases as I
from tests import kernel_cases as K

pytestmark = pytest.mark.gpu


def _ok(res):
    err, tol, desc = res
    torch.cuda.synchronize()
    print(desc)
    assert err <= tol, f"{desc}: error {err:.3e} > {tol:.1e}"


@pytest.mark.parametrize("splits", list(range(1, 17)))
def test_every_split_count(splits):
    """K = 1280 (20 chunks): 3, 6 and 7 give uneven last splits; 12 ... 16 round down to fewer (no empty split)"""
    _ok(K.case_gemm(128, 1280, 1280, bias=True, residual=True, splits=splits))


@pytest.mark.parametrize("m", [64, 77, 128, 224, 512])
@pytest.mark.parametrize("n", [1280, 200])
def test_automatic_plan_at_skinny_m(m, n):
    """at K = 5120 the skinny plan picks 80-wide tiles (N % 160 == 0) or 128-wide ones (ragged N = 200) and up to 8
    splits"""
    _ok(K.case_gemm(m, n, 5120, bias=True, residual=True, splits=0))


@pytest.mark.parametrize("splits", [3, 5, 7])
def test_odd_counts_with_per_batch_bias_and_dual_source(splits):
    _ok(K.case_gemm_batch_bias(2, 64, 1280, 1280, splits=splits))
    _ok(K.case_gemm_dual(128, 1280, 1280, 1280, splits=splits))


@pytest.mark.parametrize("splits", [0, 3, 6])
def test_box_conv_8x8(splits):
    _ok(K.case_conv(2, 8, 8, 1280, 1280, bias=True, residual=True, splits=splits, batch_bias=True))


@pytest.mark.parametrize("kw", [dict(nb=2, h=14, w=8, cin=1280, cout=1280, splits=0, bias="batch", residual=True),
                                dict(nb=2, h=14, w=8, cin=1280, cout=1280, splits=5, bias="row"),
                                dict(nb=1, h=14, w=8, cin=2560, cout=1280, c2=1280, splits=7, residual=True),
                                dict(nb=2, h=16, w=16, cin=1280, cout=1280, stride=2, splits=0, bias="row"),
                                dict(nb=1, h=28, w=16, cin=640, cout=640, stride=2, splits=6, bias="batch")],
                         ids=I.case_id)
def test_im2col_conv(kw):
    _ok(I.case_fwd(**kw))


def _skinny_layer(seed):
    a = K._rand(128, 5120, seed=seed).half()
    w = K._rand(1280, 5120, seed=seed + 1, scale=5120 ** -0.5).half()
    b = K._rand(1280, seed=seed + 2).float()
    r = K._rand(128, 1280, seed=seed + 3).half()
    return a, w, b, r


def test_graph_replays_equal_eager():
    """20 replays of a captured automatic-plan GEMM (16 tiles x 6 splits) are bit-equal to the eager call"""
    a, w, b, r = _skinny_layer(0)
    eager = ops.gemm(a, w, bias=b, residual=r)
    out = K.poison_(torch.empty_like(eager))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.gemm(a, w, bias=b, residual=r, out=out)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.gemm(a, w, bias=b, residual=r, out=out)
    for i in range(20):
        K.poison_(out)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager), f"replay {i} differs from the eager call"


def test_two_streams_with_separate_lanes():
    """two skinny split-K GEMMs running concurrently on two streams, each with its own scratch lane, give the results
    they give alone"""
    l0, l1 = _skinny_layer(0), _skinny_layer(10)
    ref0, ref1 = ops.gemm(*l0[:2], bias=l0[2], residual=l0[3]), ops.gemm(*l1[:2], bias=l1[2], residual=l1[3])
    outs = [[K.poison_(torch.empty_like(ref0)) for _ in range(8)] for _ in range(2)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for i in range(8):
        for lane, (layer, st) in enumerate(zip((l0, l1), streams)):
            with torch.cuda.stream(st), ops.workspace_lane(lane):
                ops.gemm(*layer[:2], bias=layer[2], residual=layer[3], out=outs[lane][i])
    torch.cuda.synchronize()
    for i in range(8):
        assert torch.equal(outs[0][i], ref0) and torch.equal(outs[1][i], ref1), f"concurrent launch {i} differs"
