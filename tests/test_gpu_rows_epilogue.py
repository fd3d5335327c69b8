"""Halo-row 3x3 kernel (umma_conv3x3.cu) with its epilogue taken from the accumulator registers: shapes that exercise two
halo stages over several items per CTA (odd batch at 256x256), a bf16 mask and a residual read from global memory, a
filter ring at C = 128, a ragged last 64-channel chunk (Cout = 96, clipped by the TMA store) and a launch with fewer work
items than SMs.  Same check and tolerance as test_gpu_shapes.test_conv_fprop_epilogue_cases: fp32 torch on the CPU with the
same bf16 operands, 8e-3."""
import pytest

pytestmark = pytest.mark.gpu

from test_gpu_shapes import test_conv_fprop_epilogue_cases as _fprop_case  # noqa: E402

# id: (B, H, W, Cin, Cout, KH, KW, bias, relu, residual, res_up2, bf16 mask, fp32 output)
ROWS_CASES = {
    "rows c64-64 256x256 relu B=3": (3, 256, 256, 64, 64, 3, 3, 1, 1, 0, 0, 0, 0),
    "rows c64-64 128x256 mask":     (1, 128, 256, 64, 64, 3, 3, 0, 0, 0, 0, 1, 0),
    "rows c128-128 256x128 res":    (1, 256, 128, 128, 128, 3, 3, 1, 1, 1, 0, 0, 0),
    "rows c64-96 ragged chunk":     (1, 128, 128, 64, 96, 3, 3, 1, 1, 1, 1, 0, 0),
    "rows c128-64 few items":       (1, 8, 128, 128, 64, 3, 3, 1, 0, 0, 0, 1, 0),
}


@pytest.mark.parametrize("B,H,W,Cin,Cout,KH,KW,bias,relu,res,up2,mask,fp32", list(ROWS_CASES.values()), ids=list(ROWS_CASES))
def test_conv3x3_rows_register_epilogue_cases(B, H, W, Cin, Cout, KH, KW, bias, relu, res, up2, mask, fp32):
    _fprop_case(B, H, W, Cin, Cout, KH, KW, bias, relu, res, up2, mask, fp32)
