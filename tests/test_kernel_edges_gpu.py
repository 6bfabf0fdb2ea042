"""Edge cases of the small kernels (tests/kernel_edge_cases.py) against float64 / bit-exact references (GPU)."""
import pytest
import torch

from tests import kernel_edge_cases as E

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fn,args", E.EDGE_CASES,
                         ids=[f"{f.__name__}-{'-'.join(str(x) for x in a)}" for f, a in E.EDGE_CASES])
def test_kernel_edge_matches_reference(fn, args):
    err, tol, desc = fn(*args)
    torch.cuda.synchronize()
    assert err <= tol, f"{desc}: error {err:.3e} > {tol:.1e}"
