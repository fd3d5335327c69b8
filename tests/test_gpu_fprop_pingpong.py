"""Generic conv kernel (umma_conv.cu) on its ping-pong schedule: each consumer warpgroup owns whole tiles, runs its epilogue
straight from the accumulator registers and stores the tile as two 64-row half boxes.  The cases add what the entries of
test_gpu_shapes.FPROP_CASES do not already cover on that path: the (128, 1, 1) -> (64, 1, 1) half box at 256x256 with an odd
number of tiles per CTA, a bf16 mask through the aux ring at 256x256, the quarter-size residual box at 64x64 (tile (64, 2, 1),
split along h), a linear layer with B = 256 (tile (1, 1, 128), split along the batch), a ragged 17x17 1x7 layer with a
variant epilogue, a K > 640 3x3 layer with a ragged Cout = 192 and an aux residual, and a K > 640 3x3 layer with Cout = 96 on
the general kernel's TMA-store epilogue.  Same check and tolerance as test_gpu_shapes.test_conv_fprop_epilogue_cases: fp32
torch on the CPU with the same bf16 operands, 8e-3."""
import pytest

pytestmark = pytest.mark.gpu

from test_gpu_shapes import test_conv_fprop_epilogue_cases as _fprop_case  # noqa: E402

# id: (B, H, W, Cin, Cout, KH, KW, bias, relu, residual, res_up2, bf16 mask, fp32 output)
PINGPONG_CASES = {
    "pp 1x1 c128-64 256x256 bias":       (1, 256, 256, 128, 64, 1, 1, 1, 0, 0, 0, 0, 0),
    "pp 1x1 c64-64 256x256 mask":        (1, 256, 256, 64, 64, 1, 1, 0, 0, 0, 0, 1, 0),
    "pp 1x1 c64-128 64x64 up2res":       (2, 64, 64, 64, 128, 1, 1, 1, 0, 1, 1, 0, 0),
    "pp linear 256-512 B=256 bias/relu": (256, 1, 1, 256, 512, 1, 1, 1, 1, 0, 0, 0, 0),
    "pp 1x7 c64-128 17x17 ragged":       (2, 17, 17, 64, 128, 1, 7, 1, 1, 0, 0, 0, 0),
    "pp 3x3 c128-192 16x16 res K>640":   (2, 16, 16, 128, 192, 3, 3, 1, 0, 1, 0, 0, 0),
    "3x3 c256-96 16x16 b/r/res K>640":   (1, 16, 16, 256, 96, 3, 3, 1, 1, 1, 0, 0, 0),
}


@pytest.mark.parametrize("B,H,W,Cin,Cout,KH,KW,bias,relu,res,up2,mask,fp32", list(PINGPONG_CASES.values()), ids=list(PINGPONG_CASES))
def test_conv_fprop_pingpong_epilogue_cases(B, H, W, Cin, Cout, KH, KW, bias, relu, res, up2, mask, fp32):
    _fprop_case(B, H, W, Cin, Cout, KH, KW, bias, relu, res, up2, mask, fp32)
