"""GPU parity of the wgmma implicit-GEMM kernels, one op at a time, through the C ABI (vsb_debug_conv) against a plain
PyTorch fp32 reference of the same op on the same fp16-rounded operands.  Tolerances: fp16 outputs 2e-2*max(1,|ref|max)
(one fp16 rounding of O(1..10) values plus fp32 accumulation-order noise), fp32 outputs 5e-3*max(1,|ref|max)."""
import pytest

from tests.conv_cases import CASES

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", list(CASES))
def test_conv_case(built_lib, name):
    from tests.conv_cases import run_case
    res = run_case(name)
    assert res["ok"], res
