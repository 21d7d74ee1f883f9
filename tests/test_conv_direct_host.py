"""Host checks (no GPU) of the domain of the direct-convolution kernels (ops.conv_direct_ok, the
C entry sb_conv_direct_ok): which conv layers past the first skip the patch matrix and which stay
on im2col + GEMM."""
import pytest


@pytest.mark.parametrize("Fi,Ci,Co,kh,kw,s", [
    (37, 32, 32, 5, 8, 2),     # the benchmark's (and the WSJ / RNN-T recipes') second layer
    (12, 16, 8, 2, 3, 3),      # stride 3
    (37, 8, 8, 5, 8, 2),       # Ci = 8: a 16-wide k-chunk spans two taps
    (34, 8, 8, 6, 11, 2),      # 66 taps per output pixel
    (21, 16, 24, 3, 4, 1),     # stride 1, Co = 24
])
def test_direct_domain_accepts(Fi, Ci, Co, kh, kw, s):
    from speech_b200 import ops
    assert ops.conv_direct_ok(Fi, Ci, Co, kh, kw, s)


@pytest.mark.parametrize("Fi,Ci,Co,kh,kw,s,why", [
    (65, 32, 32, 5, 32, 1, "TIMIT's [32, 5, 32, 1]: 32 x 5120 bf16 weights (320 KB) do not fit"),
    (37, 32, 40, 5, 8, 2, "more than 32 output channels"),
    (37, 32, 64, 5, 8, 2, "more than 32 output channels"),
    (37, 12, 32, 5, 8, 2, "input channels not a multiple of 8"),
    (37, 4, 32, 5, 8, 2, "fewer than 8 input channels"),
    (6, 32, 32, 5, 8, 2, "kernel wider than the input"),
])
def test_direct_domain_falls_back(Fi, Ci, Co, kh, kw, s, why):
    from speech_b200 import ops
    assert not ops.conv_direct_ok(Fi, Ci, Co, kh, kw, s), why
