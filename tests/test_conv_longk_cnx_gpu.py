"""GPU parity of the ConvNeXt pointwise GEMMs on the 256-row long-K kernel, one op at a time through the C ABI (vsb_debug_conv):
the library selects the kernel the case names by itself, the result matches the fp32 PyTorch reference, and where the 256-row
kernel ran, g, the GRN partial rows and the fp32 residual stream (and its fp16 copy) are bit-identical to the forced 128-row
kernel on the same operands."""
import pytest

from tests.conv_longk_cnx_cases import CASES


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_conv_longk_cnx_case(built_lib, name):
    from tests.conv_longk_cnx_cases import run_case
    res = run_case(name)
    assert res["ok"], f"{name}: {res}"
