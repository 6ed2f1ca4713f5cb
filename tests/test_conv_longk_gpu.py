"""GPU parity of the 256-row long-K tensor-core kernel, one op at a time, through the C ABI (vsb_debug_conv) against the fp32
PyTorch reference of the same op on the same fp16-rounded operands (tolerance of tests/test_conv_gemm_gpu.py for fp16 outputs), with the
kernel the library selected checked per case and one forced 128-row vs 256-row comparison that must be bit-identical."""
import pytest

from tests.conv_longk_cases import CASES

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", list(CASES))
def test_conv_longk_case(built_lib, name):
    from tests.conv_longk_cases import run_case
    res = run_case(name)
    assert res["ok"], res
