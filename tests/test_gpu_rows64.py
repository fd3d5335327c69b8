"""The halo-row conv kernel (conv3x3_rows_kernel, csrc/umma_conv3x3.cu) on 64-pixel-wide maps, segment S = 64: a work item is
4 output rows x 64 pixels x one output-channel tile, staged as 6 halo rows of 66 pixels per 64-channel K block, and Cin up to
256 streams its filter through the ring (pytest -m gpu).

The layers are the flagship's 3x3 convolutions at 64x64 (D stage 2, G stage 3: 256 -> 256; G stage 4: 128 -> 128), forward
and through the dgrad pack, at B = 16, where the 256-pixel items fill every SM.  Below one item per SM the generic kernel keeps
the layer (its 128-pixel tiles occupy twice as many SMs); both sides of that rule are launched.  Each case checks the kernel
that ran (torch.profiler) and the output against float64 with the tolerances of test_gpu_conv_fused: one rounding plus the
fp32-accumulation atol, ReLU bit planes exactly wherever |pre-ReLU reference| > atol, and every channel of a wider output
tensor outside the written slice unchanged bit for bit.  The last test runs every 3x3 geometry of the flagship networks at the
micro-batch B = 128 and checks that the launch class conv_fprop accounts the call to (sgb200/kernels.py) names the kernel
that ran.  As in test_gpu_resfamily_shapes, a torch.profiler session that records no CUDA kernel at all is repeated once, and
if it records nothing again the kernel identity is reported as unchecked (a warning) while the numbers are still checked."""
import warnings

import pytest
import torch

from test_gpu_conv_fused import (SENTINEL, _bf16_weight, _check_fprop, _d_blocks, _flags, _g_blocks, _launch, _launched, _pack,
                                 _pack_bits, _wide, flagship)  # noqa: F401  (flagship: module fixture)
from test_gpu_norm_shapes import _act, _cuda
from test_gpu_resfamily_shapes import _launched_checked

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16
B64 = 16          # 16 images x 16 row groups x 1 or 2 channel tiles: 256 / 512 items, past one per SM

# id -> (variant, B, Cin, Cout, options).  Options as in test_gpu_conv_fused.FUSED_CASES (bias, relu, bits, mask, x / y / m
# slices, fp32, zero_rows) plus dgrad: the launch reads the dgrad pack of a Cout x Cin layer (input gradient), as the
# backward of ConvFn does.
CASES = {
    "Full|Bias 256->256 (G stage 3 conv2d2)":                 ("Full|Bias", B64, 256, 256, {"bias": 1}),
    "Full|Bias|Relu 256->256 (D stage 2 conv2d2, no grad)":   ("Full|Bias|Relu", B64, 256, 256, {"bias": 1, "relu": 1}),
    "Full|Bias|Relu|BitsOut 256->256 (D stage 2 conv2d2)":    ("Full|Bias|Relu|BitsOut", B64, 256, 256, {"bias": 1, "relu": 1, "bits": 1}),
    "Full|Mask|MaskBits 256->256":                            ("Full|Mask|MaskBits", B64, 256, 256, {"mask": "bits"}),
    "Full 256->256":                                          ("Full", B64, 256, 256, {}),
    "Full|Bias 128->128 (G stage 4 conv2d2)":                 ("Full|Bias", B64, 128, 128, {"bias": 1}),
    "Full|Bias|Relu 128->128":                                ("Full|Bias|Relu", B64, 128, 128, {"bias": 1, "relu": 1}),
    "Full|Bias|Relu|BitsOut 128->128":                        ("Full|Bias|Relu|BitsOut", B64, 128, 128, {"bias": 1, "relu": 1, "bits": 1}),
    "Full|Mask|MaskBits 128->128":                            ("Full|Mask|MaskBits", B64, 128, 128, {"mask": "bits"}),
    "Full 128->128":                                          ("Full", B64, 128, 128, {}),
    "dgrad Full|Mask|MaskBits 256->256 (D stage 2 conv2d3)":  ("Full|Mask|MaskBits", B64, 256, 256, {"mask": "bits", "dgrad": 1}),
    "dgrad Full 256->256 (G stage 3 conv2d3)":                ("Full", B64, 256, 256, {"dgrad": 1}),
    "dgrad Full|Mask|MaskBits 128->128":                      ("Full|Mask|MaskBits", B64, 128, 128, {"mask": "bits", "dgrad": 1}),
    "dgrad Full 128->128 (G stage 4 conv2d3)":                ("Full", B64, 128, 128, {"dgrad": 1}),
    "Full|Bias 256->256, x at channel 128 of 512, y at 64 of 384":
        ("Full|Bias", B64, 256, 256, {"bias": 1, "x": (128, 512), "y": (64, 384)}),
    "Full|Bias|Relu|BitsOut 128->128, x at channel 64 of 256, y at 128 of 384":
        ("Full|Bias|Relu|BitsOut", B64, 128, 128, {"bias": 1, "relu": 1, "bits": 1, "x": (64, 256), "y": (128, 384)}),
    "Full|Mask 256->256, bf16 mask at channel 64 of 384":     ("Full|Mask", B64, 256, 256, {"mask": "bf16", "m": (64, 384)}),
    "general 128->128, fp32 output (staged-row epilogue)":    ("general", B64, 128, 128, {"bias": 1, "fp32": 1}),
    "general 256->8 (8 packed channels, N = 16 tile)":        ("general", B64, 256, 8, {"bias": 1, "zero_rows": 5}),
}


def _setup64(case, dev, variant, B, Cin, Cout, o):
    """Operands of one 64x64 launch in the dictionary layout of test_gpu_conv_fused._setup / _launch / _check_fprop.  With
    dgrad, w is the effective forward weight of the launch (the layer's weight rotated by 180 degrees, in / out swapped) and
    wf the layer's dgrad pack."""
    from sgb200 import kernels as K
    H = W = 64
    gen = torch.Generator(device=dev).manual_seed(sum(map(ord, case)))
    s = {"o": o, "k": 3, "Cout": Cout}
    xo, xt = o.get("x", (0, Cin))
    s["x"], s["xbuf"] = _wide(gen, B, Cin, H, W, dev, xo, xt)
    yo, yt = o.get("y", (0, Cout))
    dt = torch.float32 if o.get("fp32") else bf16
    s["ybuf"] = torch.full((B, H, W, yt), SENTINEL, device=dev, dtype=dt).permute(0, 3, 1, 2)
    s["y"] = s["ybuf"][:, yo:yo + Cout]
    if o.get("dgrad"):
        layer = _bf16_weight(gen, Cin, Cout, 3, dev)                       # the layer: Cout_launch -> Cin_launch
        s["w"] = layer.flip(2, 3).transpose(0, 1)
        s["wf"] = K.weight_pack(layer.float(), None, Cin, Cout, 9, False, True)[1]
    else:
        s["w"] = _bf16_weight(gen, Cout, Cin, 3, dev, o.get("zero_rows", 0))
        s["wf"] = _pack(s["w"])
    s["bias"] = 0.5 * torch.randn(Cout, generator=gen, device=dev) if o.get("bias") else None
    if o.get("bias") and o.get("zero_rows"):
        s["bias"][Cout - o["zero_rows"]:] = 0
    s["alpha"], s["alpha_ptr"], s["res"] = 1.0, None, None
    s["mask"] = s["mask_bits"] = s["mask_bool"] = None
    if o.get("mask") == "bf16":
        mo, mt = o.get("m", (0, Cout))
        s["mask"] = _wide(gen, B, Cout, H, W, dev, mo, mt)[0]
        s["mask_bool"] = s["mask"] > 0
    elif o.get("mask") == "bits":
        s["mask_bool"] = torch.rand((B, Cout, H, W), generator=gen, device=dev) < 0.6
        s["mask_bits"] = _pack_bits(s["mask_bool"])
    s["before"] = s["ybuf"].clone()
    return s


def _run_and_check(case, variant, B, Cin, Cout, o, kern):
    dev = _cuda()
    s = _setup64(case, dev, variant, B, Cin, Cout, o)
    y = _launched_checked(lambda: _launch(s), {(kern, _flags(variant))})
    assert y.data_ptr() == s["y"].data_ptr()
    worst = _check_fprop(s, y)
    print("%s: %.3g of one rounding" % (case, worst))
    assert worst <= 1.0


@pytest.mark.parametrize("case", list(CASES))
def test_rows64_vs_float64(case):
    """Each case must run conv3x3_rows_kernel<F> of its variant and match float64 within one rounding."""
    variant, B, Cin, Cout, o = CASES[case]
    _run_and_check(case, variant, B, Cin, Cout, o, "rows")


def _wave_batches(C):
    """(largest B that leaves a C -> C 3x3 @64x64 on the generic kernel, smallest B that moves it to the halo-row kernel):
    the halo-row kernel takes it once its items (16 row groups x channel tiles per image) number at least the SMs."""
    sms = torch.cuda.get_device_properties(_cuda()).multi_processor_count
    per_image = 16 * (C // 128)
    stay = -(-sms // per_image) - 1
    return stay, stay + 1


@pytest.mark.parametrize("C", [256, 128])
def test_rows64_wave_rule(C):
    """Both sides of the occupancy rule: the largest batch below one item per SM stays on conv_fprop_kernel, the next one
    runs conv3x3_rows_kernel; both within one rounding of float64."""
    stay, move = _wave_batches(C)
    assert stay >= 1
    for B, kern in ((stay, "fprop"), (move, "rows")):
        case = "wave rule %d->%d B=%d" % (C, C, B)
        _run_and_check(case, "Full|Bias|Relu", B, C, C, {"bias": 1, "relu": 1}, kern)


def _flagship_3x3(G, D):
    """Distinct (Cin, Cout, resolution) of every 3x3 convolution of the flagship networks, forward and input gradient (padded
    to the 8-channel granularity of the packs, as the model launches them)."""
    pad8 = lambda c: (c + 7) // 8 * 8   # noqa: E731
    shapes = set()
    for b, R, _, _ in _d_blocks(D):
        for m in (b.conv2d2, b.conv2d3):
            shapes |= {(m.in_channels, m.out_channels, R), (m.out_channels, m.in_channels, R)}
    for b, R in _g_blocks(G):
        Ru = 2 * R if b.upsample else R
        for m in (b.conv2d2, b.conv2d3):
            shapes |= {(m.in_channels, m.out_channels, Ru), (m.out_channels, m.in_channels, Ru)}
    for m in (G.conv2d5, D.input_conv):
        shapes |= {(pad8(m.in_channels), pad8(m.out_channels), 256), (pad8(m.out_channels), pad8(m.in_channels), 256)}
    return sorted(shapes, key=lambda s: (s[2], s[0], s[1]))


def test_accounting_class_names_the_kernel_that_ran(flagship):
    """Every 3x3 geometry of the flagship at the micro-batch B = 128: the class in conv_fprop's accounting tag (which the
    ledger and bench.py's roofline read) is conv3x3_rows exactly when conv3x3_rows_kernel ran; the 64x64 layers run it."""
    from sgb200 import _lib as L
    from sgb200 import kernels as K
    dev = _cuda()
    G, D = flagship
    gen = torch.Generator(device=dev).manual_seed(61)
    shapes = _flagship_3x3(G, D)
    assert (256, 256, 64) in shapes and (128, 128, 64) in shapes
    rows_at_64 = set()
    for Cin, Cout, R in shapes:
        x = _act(gen, 128, Cin, R, R, dev)
        wf = _pack(_bf16_weight(gen, Cout, Cin, 3, dev))
        bias = torch.zeros(Cout, device=dev)
        for _ in range(2):          # a profiler session that recorded no CUDA kernel at all is repeated once
            L.PROFILE["events"] = []
            L.PROFILE["enabled"] = True
            try:
                seen, names, _ = _launched(lambda: K.conv_fprop(x, wf, Cout, 3, 3, 1, 1, bias=bias))
            finally:
                L.PROFILE["enabled"] = False
            if any("kernel" in n for n in names):
                break
        tags = [e[0] for e in L.PROFILE["events"] if e[0].startswith("conv")]
        L.PROFILE["events"] = []
        if not any("kernel" in n for n in names):
            warnings.warn("torch.profiler recorded no CUDA kernels: the kernel of 3x3 %d->%d @%d not checked" % (Cin, Cout, R))
            continue
        assert len(tags) == 1 and len(seen) == 1, (tags, seen)
        kern = next(iter(seen))[0]
        print("3x3 %d->%d @%d B=128: %s, accounted as %s" % (Cin, Cout, R, kern, tags[0]))
        assert (kern == "rows") == tags[0].startswith("conv3x3_rows "), (tags[0], seen)
        if R == 64:
            rows_at_64.add(kern == "rows")
        del x
    assert False not in rows_at_64
