"""The conv engine's epilogue variants and the fused BigGAN-Deep block ops at flagship shapes, against float64 (pytest -m gpu).

The flagship is BigGAN-Deep 256x256 (configs/BigGAN-Deep-256res.yaml: conv_dim 128, depth 2, spectral norm, attention after
D stage 1 and G stage 3).  Three parts:
1. One or more launches of every compiled epilogue variant: the 15 ``FpropCompiled`` variants of conv_fprop_kernel
   (csrc/umma_conv.cu), the 6 halo-row variants of conv3x3_rows_kernel (csrc/umma_conv3x3.cu) and the run-time general
   kernel (F = -1) of each.  Each case is a flagship layer geometry and sets the options the model sets there: res_scale 0.25
   with res_up2, mask bits together with a residual, bit planes written with a residual on the aux ring, operands that are
   channel slices of wider tensors (the concat-skip buffer, the generator's x[:, :out] skip), plus the ABI options the model
   does not use (res_after_mask, alpha_ptr).  The variants actually launched are read from a torch.profiler trace and must
   equal the declared set.
2. The fused discriminator / generator block ops (DEntryConvFn, ConcatSkipFn, ConvFn with premasked / mask_input, AvgPoolFn,
   SplitResidualFn and the sliced res_up2 skip of GenBlock.conv2d4) at every distinct flagship block geometry, forward and
   backward, with the spectral norm run the way the model runs it (batched pass, sn_cache); and every DiscBlock as a whole,
   block(x, in_relu, out_relu), against the reference block arithmetic restated in float64.
3. conv_wgrad at the flagship micro-batch B = 128: every distinct (Cin, Cout, k, H, W) of the D and G block convolutions, the
   fused bias gradient and the second micro-batch (accumulate=True into non-zero dw / dbias).

References: plain float64 torch on the GPU, on the same bf16 operands and bf16 packed weights the kernel reads, chunked over
images so that no temporary is much larger than one activation.  Nothing on the reference side calls the library.

Tolerances (bf16 keeps 8 significant bits: one round-to-nearest moves a value by at most 2^-8 of itself):
* "one rounding": |got - ref| <= 2^-8 |ref| + atol per element.  atol covers the fp32 accumulation of bf16 products in the
  tensor cores: atol = 2^-14 * alpha * (|x| (*) |w|), the same convolution on absolute values in float64 (an estimate: a
  K-term fp32 sum is expected within ~sqrt(K) 2^-24 of its terms' magnitude, and K <= 2304 here gives 3e-6; the bound leaves
  20x).  Everything after the accumulator (alpha, bias, fmaf of the residual, ReLU, mask) is exact or one fp32 rounding.
  fp32 outputs (no bf16 rounding): |got - ref| <= 2^-22 |ref| + atol (a few fp32 roundings after the accumulator).
* Bit planes must equal (pre-ReLU reference > 0) wherever |pre-ReLU reference| > atol: set above atol, clear below -atol.
* Outputs are stored into channel slices of sentinel-filled tensors: every channel outside the slice must be unchanged, bit
  for bit.  2x2 average pooling (one fp32 sum of four bf16 values, times 0.25, one rounding) is checked bit for bit.
* Attention softmax P = softmax(theta phi^T): atol = P * (2 * 2^-14 * max_row(|theta| |phi|^T) + 2^-18) (the logit error
  enters P twice, through its own exponent and through the row sum; ex2.approx adds 2^-22; an estimate), plus 2^-126
  absolute: ex2.approx.ftz flushes probabilities below the smallest normal fp32 to zero.  dS = P * (dP - delta)
  with delta given: atol = P * 2^-14 (|do| |g|^T).
* Weight gradients (fp32 tensor-core accumulation over B*H*W pixels, split-K partial sums added with fp32 atomics in any
  order): |dw - ref| <= 2^-18 * (|x| (*) |dy|) per weight, the same sum on absolute values (an estimate: the partial sums
  are each within ~sqrt(n) 2^-24 of their terms, and the atomics add log-many more roundings; 2^-18 = 64 ulps of fp32);
  the bias gradient the same with sum |dy|.
* Block composition (block(x, in_relu, out_relu) against the reference block in float64): relative L2 bounds on the
  output, dx and every parameter gradient, estimated in BLOCK_L2 below.
* Block ops: each op's output is held to one rounding of the float64 op on the bf16 tensors the product passed it (atol as
  above); input gradients likewise (one rounding, atol from the absolute-value transposed convolution); parameter gradients
  to the weight-gradient bound, with W / sigma from one float64 power iteration on the saved u.
"""
import copy
import os
import re

import pytest
import torch
import torch.nn.functional as F

from test_gpu_norm_shapes import PKG, _Err, _act, _cuda, _rounding_ratio

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16
ACC_REL = 2.0 ** -14          # fp32 accumulation of a forward / dgrad conv, relative to (|x| (*) |w|)
WGRAD_REL = 2.0 ** -18        # weight / bias gradient, relative to the absolute-value sum
FP32_REL = 2.0 ** -22        # fp32 output: alpha, bias and residual add a few fp32 roundings after the accumulator
SENTINEL = -65536.0           # exact in bf16, never produced by these layers

# epilogue flag bits of csrc/conv_epilogue.cuh
FLAG = {"Bias": 1, "Relu": 2, "ResPre": 4, "ResPost": 8, "Mask": 16, "Full": 32, "MaskBits": 64, "AuxRes": 128,
        "AuxMask": 256, "BitsOut": 512, "SmStats": 1024, "SmApply": 2048, "SmBwd": 4096}


def _flags(s):
    return -1 if s == "general" else sum(FLAG[t] for t in s.split("|"))


# The compiled variants (FpropCompiled in csrc/umma_conv.cu, RowsCompiled in csrc/umma_conv3x3.cu).
FPROP_VARIANTS = {_flags(s) for s in (
    "Full", "Full|Bias", "Full|Bias|Relu", "Full|Bias|Relu|BitsOut", "Full|ResPre|AuxRes", "Full|Bias|ResPre|AuxRes",
    "Full|Bias|Relu|ResPre|AuxRes", "Full|Bias|Relu|ResPre|AuxRes|BitsOut", "Full|Mask|MaskBits",
    "Full|Mask|MaskBits|ResPre|AuxRes", "Full|Mask|AuxMask", "Full|Mask|ResPre|AuxMask", "Full|SmStats", "Full|SmApply",
    "Full|SmBwd", "general")}
ROWS_VARIANTS = {_flags(s) for s in ("Full|Bias", "Full|Bias|Relu", "Full|Bias|Relu|BitsOut", "Full|Mask", "Full|Mask|MaskBits",
                                     "Full", "general")}
_KERNEL_RE = re.compile(r"(conv_fprop_kernel|conv3x3_rows_kernel)<(-?\d+)>")


def _launched(fn):
    """Run fn() under torch.profiler; returns ({(kernel, F)} of the conv fprop kernels it launched, kernel names, fn())."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    seen = set()
    for n in names:
        m = _KERNEL_RE.search(n)
        if m:
            seen.add(("fprop" if m.group(1) == "conv_fprop_kernel" else "rows", int(m.group(2))))
    return seen, names, out


def _bf16_weight(gen, Cout, Cin, k, dev, zero_rows=0):
    w = (torch.randn((Cout, Cin, k, k), generator=gen, device=dev) / (Cin * k * k) ** 0.5).to(bf16)
    if zero_rows:
        w[Cout - zero_rows:] = 0
    return w


def _pack(w):
    """The fprop pack [Cout][taps][Cin] of an already bf16-valued weight (sigma = 1: the values are copied unchanged)."""
    from sgb200 import kernels as K
    Cout, Cin, KH, KW = w.shape
    return K.weight_pack(w.float(), None, Cout, Cin, KH * KW, True, False)[0]


def _pack_bits(m):
    """bool [B, C, H, W] -> the bit-plane layout uint8 [B, H, W, C / 8] (bit j of byte k = channel 8k + j)."""
    B, C, H, W = m.shape
    sh = torch.arange(8, device=m.device, dtype=torch.uint8)
    return (m.permute(0, 2, 3, 1).reshape(B, H, W, C // 8, 8).to(torch.uint8) << sh).sum(-1, dtype=torch.uint8)


def _unpack_bits(bits, C):
    B, H, W, _ = bits.shape
    sh = torch.arange(8, device=bits.device, dtype=torch.uint8)
    return ((bits[..., None] >> sh) & 1).reshape(B, H, W, C).permute(0, 3, 1, 2).bool()


def _up2(t):
    return t.repeat_interleave(2, 2).repeat_interleave(2, 3)


def _conv64(x, w, pad):
    """float64 stride-1 convolution [b, Cin, H, W] (*) [Cout, Cin, k, k] -> [b, Cout, H, W] as one matmul per tap (float64
    GEMMs; the float64 convolution kernels are far slower at these sizes).  pad = k - 1 - pad' gives the transposed conv."""
    b, Cin, H, W = x.shape
    Cout, _, k, _ = w.shape
    Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
    xp = F.pad(x.double().permute(0, 2, 3, 1), (0, 0, pad, pad, pad, pad))
    w = w.double()
    y = torch.zeros((b, Ho, Wo, Cout), device=x.device, dtype=torch.float64)
    for t in range(k * k):
        y += xp[:, t // k:t // k + Ho, t % k:t % k + Wo] @ w[:, :, t // k, t % k].t()
    return y.permute(0, 3, 1, 2)


def _dgrad64(dz, w, pad):
    """float64 input gradient of a stride-1 conv with weight w [Cout, Cin, k, k]: the conv of dz with the flipped, transposed w."""
    k = w.shape[2]
    return _conv64(dz, w.flip(2, 3).transpose(0, 1), k - 1 - pad)


def _wide(gen, B, C, H, W, dev, off, total):
    """bf16 activation [B, C, H, W] = channels [off, off + C) of a [B, total, H, W] NHWC tensor (and that tensor)."""
    full = _act(gen, B, total, H, W, dev)
    return full[:, off:off + C], full


# ------------------------------------------------------------------------------------------------ 1. epilogue variants
# id -> (kernel, variant, B, H, W, Cin, Cout, k, options).  Options: bias, relu, bits (want_relu_bits), res ("full" | "up2"),
# res_scale, res_after, mask ("bf16" | "bits"), alpha_ptr, fp32, zero_rows (padded output channels of the weight),
# x / y / res / mask slices as (channel offset, channels of the wider tensor), concat (y is the channel slice after x of
# x's own buffer, as ConcatSkipFn writes it), x_in_res (x and the residual are slices of one buffer, as its backward reads them).
FUSED_CASES = {
    "fprop Full: D stage 0 conv2d4 dgrad 1x1 256->64 @128x128":
        ("fprop", "Full", 2, 128, 128, 256, 64, 1, {}),
    "fprop Full|Bias: G stage 3 conv2d1 1x1 1024->256 @32x32, alpha_ptr, y at channel 64 of 384":
        ("fprop", "Full|Bias", 8, 32, 32, 1024, 256, 1, {"bias": 1, "alpha_ptr": 1, "y": (64, 384)}),
    "fprop Full|Bias: D stage 1 concat-skip conv2d0 1x1 256->256 @64x64 into skip[:, 256:]":
        ("fprop", "Full|Bias", 4, 64, 64, 256, 256, 1, {"bias": 1, "concat": 1}),
    "fprop Full|Bias: G stage 2 conv2d2 3x3 256->256 @32x32":
        ("fprop", "Full|Bias", 4, 32, 32, 256, 256, 3, {"bias": 1}),
    "fprop Full|Bias|Relu: D stage 2 conv2d2 3x3 256->256 @64x64 (no-grad pass)":
        ("fprop", "Full|Bias|Relu", 2, 64, 64, 256, 256, 3, {"bias": 1, "relu": 1}),
    "fprop Full|Bias|Relu|BitsOut: D stage 3 conv2d1 1x1 1024->256 @32x32":
        ("fprop", "Full|Bias|Relu|BitsOut", 8, 32, 32, 1024, 256, 1, {"bias": 1, "relu": 1, "bits": 1}),
    "fprop Full|ResPre|AuxRes: D stage 1 concat-skip dgrad 1x1 256->256 @64x64, x = dskip[:, 256:], res = dskip[:, :256]":
        ("fprop", "Full|ResPre|AuxRes", 4, 64, 64, 256, 256, 1, {"res": "full", "x_in_res": 1}),
    "fprop Full|Bias|ResPre|AuxRes: G stage 2 block 1 conv2d4 1x1 256->512 @32x32 + up2 skip x[:, :512] of 1024":
        ("fprop", "Full|Bias|ResPre|AuxRes", 4, 32, 32, 256, 512, 1, {"bias": 1, "res": "up2", "r": (0, 1024)}),
    "fprop Full|Bias|ResPre|AuxRes: D stage 3 block 1 conv2d4 1x1 256->1024 @32x32 + skip at channel 128 of 1280":
        ("fprop", "Full|Bias|ResPre|AuxRes", 4, 32, 32, 256, 1024, 1, {"bias": 1, "res": "full", "r": (128, 1280)}),
    "fprop Full|Bias|Relu|ResPre|AuxRes: D stage 4 block 1 conv2d4 1x1 512->2048 @16x16 + skip, out_relu (no-grad pass)":
        ("fprop", "Full|Bias|Relu|ResPre|AuxRes", 16, 16, 16, 512, 2048, 1, {"bias": 1, "relu": 1, "res": "full"}),
    "fprop Full|Bias|Relu|ResPre|AuxRes|BitsOut: D stage 2 block 0 conv2d4 1x1 256->1024 @32x32 + concat skip, out_relu":
        ("fprop", "Full|Bias|Relu|ResPre|AuxRes|BitsOut", 4, 32, 32, 256, 1024, 1, {"bias": 1, "relu": 1, "bits": 1, "res": "full"}),
    "fprop Full|Mask|MaskBits: D stage 2 conv2d3 dgrad 3x3 256->256 @64x64, mask bits":
        ("fprop", "Full|Mask|MaskBits", 2, 64, 64, 256, 256, 3, {"mask": "bits"}),
    "fprop Full|Mask|MaskBits|ResPre|AuxRes: D stage 2 entry dgrad 1x1 256->512 @64x64, mask bits + up2 dpx x 0.25":
        ("fprop", "Full|Mask|MaskBits|ResPre|AuxRes", 4, 64, 64, 256, 512, 1, {"mask": "bits", "res": "up2", "res_scale": 0.25}),
    "fprop Full|Mask|AuxMask: D stage 3 conv2d2 dgrad 3x3 256->256 @32x32, bf16 mask at channel 64 of 384":
        ("fprop", "Full|Mask|AuxMask", 4, 32, 32, 256, 256, 3, {"mask": "bf16", "m": (64, 384)}),
    "fprop Full|Mask|ResPre|AuxMask: D stage 2 entry dgrad after the attention 1x1 256->512 @64x64, bf16 a0 + up2 dpx x 0.25":
        ("fprop", "Full|Mask|ResPre|AuxMask", 4, 64, 64, 256, 512, 1, {"mask": "bf16", "res": "up2", "res_scale": 0.25}),
    "fprop general: 1x1 256->512 @32x32, bf16 mask then res_after_mask, alpha_ptr":
        ("fprop", "general", 4, 32, 32, 256, 512, 1, {"bias": 1, "relu": 1, "mask": "bf16", "res": "full", "res_after": 1,
                                                      "alpha_ptr": 1}),
    "fprop general: G cBN gain linear 256->2048, fp32 output, B=128":
        ("fprop", "general", 128, 1, 1, 256, 2048, 1, {"fp32": 1}),
    "rows Full|Bias: G stage 4 block 1 conv2d2 3x3 128->128 @128x128, alpha_ptr, y at channel 64 of 256":
        ("rows", "Full|Bias", 2, 128, 128, 128, 128, 3, {"bias": 1, "alpha_ptr": 1, "y": (64, 256)}),
    "rows Full|Bias|Relu: D stage 1 conv2d2 3x3 128->128 @128x128 (no-grad pass)":
        ("rows", "Full|Bias|Relu", 2, 128, 128, 128, 128, 3, {"bias": 1, "relu": 1}),
    "rows Full|Bias|Relu|BitsOut: D stage 0 conv2d2 3x3 64->64 @256x256, B=3":
        ("rows", "Full|Bias|Relu|BitsOut", 3, 256, 256, 64, 64, 3, {"bias": 1, "relu": 1, "bits": 1}),
    "rows Full|Mask: D stage 1 conv2d3 dgrad 3x3 128->128 @128x128, bf16 mask at channel 128 of 384":
        ("rows", "Full|Mask", 2, 128, 128, 128, 128, 3, {"mask": "bf16", "m": (128, 384)}),
    "rows Full|Mask|MaskBits: D stage 0 conv2d3 dgrad 3x3 64->64 @256x256, mask bits":
        ("rows", "Full|Mask|MaskBits", 2, 256, 256, 64, 64, 3, {"mask": "bits"}),
    "rows Full: G stage 5 conv2d3 dgrad 3x3 64->64 @256x256, x at channel 64 of 192":
        ("rows", "Full", 1, 256, 256, 64, 64, 3, {"x": (64, 192)}),
    "rows general: G conv2d5 3x3 128->3 (8 packed channels) @256x256":
        ("rows", "general", 2, 256, 256, 128, 8, 3, {"bias": 1, "zero_rows": 5}),
}


def _setup(case, dev):
    """Operands of one case (product side): everything conv_fprop is called with, plus the wider buffers."""
    kern, _, B, H, W, Cin, Cout, k, o = FUSED_CASES[case]
    gen = torch.Generator(device=dev).manual_seed(sum(map(ord, case)))
    s = {"o": o, "k": k, "Cout": Cout}
    if o.get("concat"):            # skip buffer [px | conv0(px)]: x = skip[:, :Cin], y = skip[:, Cin:]
        s["x"], s["ybuf"] = _wide(gen, B, Cin, H, W, dev, 0, Cin + Cout)
        s["ybuf"][:, Cin:] = SENTINEL
        s["y"] = s["ybuf"][:, Cin:]
    else:
        xo, xt = (Cout, Cin + Cout) if o.get("x_in_res") else o.get("x", (0, Cin))    # dskip = [d_lo | d_hi]: x = d_hi
        s["x"], s["xbuf"] = _wide(gen, B, Cin, H, W, dev, xo, xt)
        yo, yt = o.get("y", (0, Cout))
        dt = torch.float32 if o.get("fp32") else bf16
        s["ybuf"] = torch.full((B, H, W, yt), SENTINEL, device=dev, dtype=dt).permute(0, 3, 1, 2)
        s["y"] = s["ybuf"][:, yo:yo + Cout]
    s["w"] = _bf16_weight(gen, Cout, Cin, k, dev, o.get("zero_rows", 0))
    s["wf"] = _pack(s["w"])
    s["bias"] = 0.5 * torch.randn(Cout, generator=gen, device=dev) if o.get("bias") else None
    if o.get("bias") and o.get("zero_rows"):
        s["bias"][Cout - o["zero_rows"]:] = 0
    s["alpha"] = 0.5 if o.get("alpha_ptr") else 1.0
    s["alpha_ptr"] = torch.tensor([1.5], device=dev) if o.get("alpha_ptr") else None      # 0.5 * 1.5 = 0.75 exactly in fp32
    s["res"] = None
    if o.get("res"):
        Hr, Wr = (H // 2, W // 2) if o["res"] == "up2" else (H, W)
        if o.get("x_in_res"):
            s["res"] = s["xbuf"][:, :Cout]
        else:
            ro, rt = o.get("r", (0, Cout))
            s["res"] = _wide(gen, B, Cout, Hr, Wr, dev, ro, rt)[0]
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


def _launch(s):
    from sgb200 import kernels as K
    o, k = s["o"], s["k"]
    return K.conv_fprop(s["x"], s["wf"], s["Cout"], k, k, k // 2, k // 2, bias=s["bias"], residual=s["res"],
                        res_up2=o.get("res") == "up2", res_after_mask=bool(o.get("res_after")), mask=s["mask"],
                        mask_bits=s["mask_bits"], relu=bool(o.get("relu")), alpha=s["alpha"], alpha_ptr=s["alpha_ptr"],
                        out=s["y"], res_scale=o.get("res_scale", 1.0), want_relu_bits=bool(o.get("bits")))


def _fprop_reference(s, b0, b1):
    """(pre-ReLU reference, final reference, atol) in float64 for images b0:b1, in the kernel's order."""
    o, k = s["o"], s["k"]
    x = s["x"][b0:b1].double()
    w = s["w"].double()
    alpha = s["alpha"] * (1.5 if o.get("alpha_ptr") else 1.0)
    z = alpha * _conv64(x, w, k // 2)
    atol = ACC_REL * alpha * _conv64(x.abs(), w.abs(), k // 2)
    if s["bias"] is not None:
        z = z + s["bias"].double().view(1, -1, 1, 1)
    r = None
    if s["res"] is not None:
        r = o.get("res_scale", 1.0) * s["res"][b0:b1].double()
        if o["res"] == "up2":
            r = _up2(r)
    if r is not None and not o.get("res_after"):
        z = z + r
    pre = z
    if o.get("relu"):
        z = z.clamp(min=0)
    if s["mask_bool"] is not None:
        z = torch.where(s["mask_bool"][b0:b1], z, torch.zeros((), device=z.device, dtype=z.dtype))
    if r is not None and o.get("res_after"):
        z = z + r
    return pre, z, atol


def _check_fprop(s, y):
    """Worst one-rounding ratio over the output; asserts the bit planes and the untouched neighbour channels."""
    o = s["o"]
    B = s["x"].shape[0]
    per = max(1, (1 << 24) // max(1, s["y"][0].numel()))
    worst = 0.0
    for b0 in range(0, B, per):
        b1 = min(B, b0 + per)
        pre, ref, atol = _fprop_reference(s, b0, b1)
        if o.get("fp32"):        # fp32 output: the accumulation bound plus a few fp32 roundings, no bf16 rounding
            worst = max(worst, float(((y[b0:b1].double() - ref).abs() / (FP32_REL * ref.abs() + atol + 1e-30)).max()))
        else:
            worst = max(worst, _rounding_ratio(y[b0:b1], ref, atol + 1e-30))
        if o.get("bits"):        # both ways: set where the pre-ReLU reference is > atol, clear where it is < -atol
            got = _unpack_bits(y._sgb_relu_bits[b0:b1], s["Cout"])
            sure = pre.abs() > atol
            assert torch.equal(got[sure], (pre > 0)[sure]), "ReLU bit planes differ from (reference > 0)"
            assert bool((~got[pre < -atol]).all()) and bool(got[pre > atol].all())
    # every channel of the wider output tensor outside the slice is untouched
    yb, yo = s["ybuf"], s["y"]
    off = (yo.data_ptr() - yb.data_ptr()) // yb.element_size()
    assert torch.equal(yb[:, :off], s["before"][:, :off])
    assert torch.equal(yb[:, off + s["Cout"]:], s["before"][:, off + s["Cout"]:])
    return worst


@pytest.mark.parametrize("case", list(FUSED_CASES))
def test_epilogue_variant_vs_float64(case):
    """One flagship launch per epilogue variant: the kernel its id names must run, and y (with the ReLU bit planes where
    written) must be within one rounding of the float64 epilogue."""
    dev = _cuda()
    kern, variant = FUSED_CASES[case][:2]
    s = _setup(case, dev)
    seen, _, y = _launched(lambda: _launch(s))
    assert seen == {(kern, _flags(variant))}, "%s ran %s" % (case, seen)
    assert y.data_ptr() == s["y"].data_ptr()
    worst = _check_fprop(s, y)
    print("%s: %.3g of one rounding" % (case, worst))
    assert worst <= 1.0


# attention at the flagship's 64x64 map (D after stage 1, 512 channels): N = 4096 queries, M = 1024 keys, c8 = 64, c2 = 256
ATTN = (128, 64, 64, 256)


def _attention_operands(dev):
    B, S, c8, c2 = ATTN
    gen = torch.Generator(device=dev).manual_seed(41)
    theta = _act(gen, B, c8, S, S, dev)
    phi = _act(gen, B, c8, S // 2, S // 2, dev)
    g = _act(gen, B, c2, S // 2, S // 2, dev)
    do = _act(gen, B, c2, S, S, dev)
    return theta, phi, g, do


def _attention_fwd(theta, phi):
    """P = softmax(theta . phi^T): the statistics pass, then the apply pass of the same GEMM."""
    from sgb200 import kernels as K
    M = phi.shape[2] * phi.shape[3]
    P, stats = K.conv_fprop(theta, phi, M, 1, 1, 0, 0, w_mode=1, sm_mode=1)
    K.conv_fprop(theta, phi, M, 1, 1, 0, 0, w_mode=1, sm_mode=2, sm_stats=stats, out=P)
    return P


def _attention_bwd(do, g, P, delta):
    """dS = P * (do . g^T - delta)."""
    from sgb200 import kernels as K
    return K.conv_fprop(do, g, P.shape[1], 1, 1, 0, 0, w_mode=1, sm_mode=3, sm_delta=delta, sm_p=P)


def _rows(t):
    """[b, C, h, w] NHWC activation -> float64 [b, h*w, C]."""
    b, C = t.shape[:2]
    return t.double().permute(0, 2, 3, 1).reshape(b, -1, C)


def test_attention_softmax_variants_at_flagship_shape_vs_float64():
    """The three softmax epilogues (statistics, apply, backward) at B = 128, N = 4096, M = 1024, c8 = 64, c2 = 256.
    delta (an input of the backward GEMM) is rowsum(P * dP) of the kernel's P, as the model forms it from do . o."""
    dev = _cuda()
    theta, phi, g, do = _attention_operands(dev)
    B = theta.shape[0]
    seen, _, P = _launched(lambda: _attention_fwd(theta, phi))
    assert seen == {("fprop", _flags("Full|SmStats")), ("fprop", _flags("Full|SmApply"))}, seen
    delta = torch.empty(B * theta.shape[2] * theta.shape[3], device=dev, dtype=torch.float32)
    per = 8
    for b0 in range(0, B, per):
        b1 = min(B, b0 + per)
        dP = _rows(do[b0:b1]) @ _rows(g[b0:b1]).transpose(1, 2)
        delta.view(B, -1)[b0:b1] = (_rows(P[b0:b1]) * dP).sum(-1).float()
    seen, _, dS = _launched(lambda: _attention_bwd(do, g, P, delta))
    assert seen == {("fprop", _flags("Full|SmBwd"))}, seen
    wp = wd = 0.0
    for b0 in range(0, B, per):
        b1 = min(B, b0 + per)
        q, kk = _rows(theta[b0:b1]), _rows(phi[b0:b1])
        logits, labs = q @ kk.transpose(1, 2), q.abs() @ kk.abs().transpose(1, 2)
        Pref = torch.softmax(logits, -1)
        atol = Pref * (2 * ACC_REL * labs.amax(-1, keepdim=True) + 2.0 ** -18) + 2.0 ** -126
        wp = max(wp, _rounding_ratio(_rows(P[b0:b1]), Pref, atol))
        dP = _rows(do[b0:b1]) @ _rows(g[b0:b1]).transpose(1, 2)
        dabs = _rows(do[b0:b1]).abs() @ _rows(g[b0:b1]).abs().transpose(1, 2)
        Pk = _rows(P[b0:b1])
        dref = Pk * (dP - delta.view(B, -1)[b0:b1].double()[..., None])
        wd = max(wd, _rounding_ratio(_rows(dS[b0:b1]), dref, Pk * ACC_REL * dabs + 1e-30))
    print("attention softmax: P %.3g dS %.3g of one rounding" % (wp, wd))
    assert wp <= 1.0 and wd <= 1.0


def test_every_compiled_epilogue_variant_is_launched():
    """The table above, launched once under torch.profiler: the set of (kernel, F) seen must equal the compiled set plus the
    two general kernels.  A dispatch change that moves a launch to another variant fails here instead of dropping coverage."""
    dev = _cuda()

    def run_all():
        for case in FUSED_CASES:
            _launch(_setup(case, dev))
        theta, phi, g, do = _attention_operands(dev)
        P = _attention_fwd(theta[:2], phi[:2])
        _attention_bwd(do[:2], g[:2], P, torch.zeros(2 * theta.shape[2] * theta.shape[3], device=dev))

    seen, _, _ = _launched(run_all)
    want = {("fprop", f) for f in FPROP_VARIANTS} | {("rows", f) for f in ROWS_VARIANTS}
    print("variants seen:", sorted(seen))
    assert seen == want, "missing %s, unexpected %s" % (sorted(want - seen), sorted(seen - want))
    assert len(FPROP_VARIANTS) == 16 and len(ROWS_VARIANTS) == 7


# ------------------------------------------------------------------------------------------------ flagship geometry
@pytest.fixture(scope="module")
def flagship():
    """(G, D) of configs/BigGAN-Deep-256res.yaml (conv_dim 128, depth 2, spectral norm, attention), built once for this
    module and released after it."""
    from sgb200 import config as C
    from sgb200.models import model as M
    dev = _cuda()
    cfgs = C.Configurations(os.path.join(PKG, "configs", "BigGAN-Deep-256res.yaml"))
    MODEL = copy.copy(cfgs.MODEL)
    MODEL.apply_g_ema = False
    torch.manual_seed(0)
    G, _, _, D, _, _, _, _ = M.load_generator_discriminator(cfgs.DATA, cfgs.OPTIMIZATION, MODEL, cfgs.STYLEGAN, cfgs.MODULES,
                                                           cfgs.RUN, dev, None)
    gen = torch.Generator(device=dev).manual_seed(1)
    with torch.no_grad():      # the initialisation zeroes the conv biases: give the epilogues a bias to add
        for m in list(G.modules()) + list(D.modules()):
            if isinstance(m, torch.nn.Conv2d) and m.bias is not None:
                m.bias.copy_(0.3 * torch.randn(m.bias.shape, generator=gen, device=dev))
    yield G.train(), D.train()
    del G, D
    torch.cuda.empty_cache()


def _d_blocks(D):
    """[(block, R, in_relu, out_relu)] in forward order: R = input resolution; the ReLU hand-over of Discriminator.forward."""
    from sgb200.models.big_resnet_deep_legacy import DiscBlock
    seq = [b for bl in D.blocks for b in bl]
    out, R, relu_in = [], 256, isinstance(seq[0], DiscBlock)
    for i, b in enumerate(seq):
        if isinstance(b, DiscBlock):
            nxt = seq[i + 1] if i + 1 < len(seq) else None
            relu_out = nxt is None or isinstance(nxt, DiscBlock)
            out.append((b, R, relu_in, relu_out))
            relu_in = relu_out
            R = R // 2 if b.downsample else R
        else:
            relu_in = False
    return out


def _g_blocks(G):
    """[(block, R)] in forward order: R = input resolution (the generator starts at 4x4)."""
    from sgb200.models.big_resnet_deep_legacy import GenBlock
    out, R = [], 4
    for b in (b for bl in G.blocks for b in bl):
        if isinstance(b, GenBlock):
            out.append((b, R))
            R = 2 * R if b.upsample else R
    return out


def _wgrad_shapes(G, D):
    """Distinct (Cin, Cout, k, H, W) of the block convolutions of both networks."""
    shapes = set()
    for b, R, _, _ in _d_blocks(D):
        Ro = R // 2 if b.downsample else R
        hid, out = b.conv2d1.out_channels, b.conv2d4.out_channels
        shapes |= {(b.conv2d1.in_channels, hid, 1, R), (hid, hid, 3, R), (hid, out, 1, Ro)}
        if b.learnable_sc:
            shapes.add((b.conv2d0.in_channels, b.conv2d0.out_channels, 1, Ro))
    for b, R in _g_blocks(G):
        Ru = 2 * R if b.upsample else R
        hid = b.conv2d1.out_channels
        shapes |= {(b.conv2d1.in_channels, hid, 1, R), (hid, hid, 3, Ru), (hid, b.conv2d4.out_channels, 1, Ru)}
    return sorted(shapes, key=lambda s: (s[3], s[2], s[0], s[1]))


# ------------------------------------------------------------------------------------------------ 3. weight gradients
def _wgrad_ref(x, dy, k, co):
    """float64 sum over images and pixels of dy[co] (x) x-shifted-by-tap: ([len(co), k*k, Cin], the same on |x|, |dy|),
    in the fprop-pack layout.  Chunked over images (<= 2^25 elements of x per chunk)."""
    B, Cin, H, W = x.shape
    p = k // 2
    ref = torch.zeros((len(co), k * k, Cin), device=x.device, dtype=torch.float64)
    rabs = torch.zeros_like(ref)
    per = max(1, (1 << 25) // ((H + 2 * p) * (W + 2 * p) * Cin))
    for b0 in range(0, B, per):
        b1 = min(B, b0 + per)
        xp = F.pad(x[b0:b1].double().permute(0, 2, 3, 1), (0, 0, p, p, p, p))       # [b, H + 2p, W + 2p, Cin]
        d = dy[b0:b1][:, co].double().permute(0, 2, 3, 1).reshape(-1, len(co))
        for t in range(k * k):
            xs = xp[:, t // k:t // k + H, t % k:t % k + W].reshape(-1, Cin)
            ref[:, t] += d.t() @ xs
            rabs[:, t] += d.abs().t() @ xs.abs()
    return ref, rabs


def _wgrad_worst(dw, ref, rabs):
    return float(((dw.double() - ref).abs() / (WGRAD_REL * rabs + 1e-30)).max())


def _channels(C):
    """Output channels checked: all up to 128, else the first, a middle and the last 64-channel tile."""
    idx = torch.arange(C)
    return idx if C <= 128 else torch.cat([idx[:64], idx[C // 2:C // 2 + 64], idx[-64:]])


def test_conv_wgrad_every_flagship_layer_at_micro_batch(flagship):
    """conv_wgrad (with the fused bias gradient) on every distinct block-conv geometry of the flagship D and G.  B = 128 up
    to 64x64; at 128x128 and 256x256 B = 4 (B = 3 for the first such shape), except one B = 130 launch at 256x256 per
    kernel: the 64-channel 3x3 kernel (D stage 0 conv2d2 / conv2d3) and the generic kernel (D stage 0 conv2d1, whose x of
    130 x 128 channels x 256^2 is 2.18 GB: its last images lie past 2^31 bytes).  Shapes up
    to 32x32 also run a second micro-batch: accumulate=True into the non-zero dw and, through dbias_acc, the non-zero
    bias gradient of the first."""
    from sgb200 import kernels as K
    dev = _cuda()
    G, D = flagship
    shapes = _wgrad_shapes(G, D)
    assert (64, 64, 3, 256) in shapes and (128, 64, 1, 256) in shapes
    gen = torch.Generator(device=dev).manual_seed(51)
    worst, worst_db, odd_done, kernels = 0.0, 0.0, False, set()
    for Cin, Cout, k, R in shapes:
        if R <= 64:
            B = 128
        elif (Cin, Cout, k, R) in ((64, 64, 3, 256), (128, 64, 1, 256)):
            B = 130
        else:
            B, odd_done = (4 if odd_done else 3), True
        x, dy = _act(gen, B, Cin, R, R, dev), _act(gen, B, Cout, R, R, dev)
        seen, names, (dw, db) = _launched(lambda: K.conv_wgrad(x, dy, k, k, k // 2, k // 2, want_dbias=True))
        kernels |= {n for n in names if "wgrad" in n and "kernel" in n}
        co = _channels(Cout)
        ref, rabs = _wgrad_ref(x, dy, k, co.to(dev))
        e = _wgrad_worst(dw[co.to(dev)], ref, rabs)
        dref = dy.double().sum((0, 2, 3))
        edb = float(((db.double() - dref).abs() / (WGRAD_REL * dy.double().abs().sum((0, 2, 3)))).max())
        if R <= 32:         # second micro-batch into the first one's dw / bias gradient
            x2, dy2 = _act(gen, B, Cin, R, R, dev), _act(gen, B, Cout, R, R, dev)
            _, done = K.conv_wgrad(x2, dy2, k, k, k // 2, k // 2, dw=dw, accumulate=True, dbias_acc=db)
            assert done is True
            r2, a2 = _wgrad_ref(x2, dy2, k, co.to(dev))
            e = max(e, _wgrad_worst(dw[co.to(dev)], ref + r2, rabs + a2))
            dref2 = dref + dy2.double().sum((0, 2, 3))
            dabs = dy.double().abs().sum((0, 2, 3)) + dy2.double().abs().sum((0, 2, 3))
            edb = max(edb, float(((db.double() - dref2).abs() / (WGRAD_REL * dabs)).max()))
        print("wgrad %dx%d %d->%d @%d B=%d: dw %.3g db %.3g" % (k, k, Cin, Cout, R, B, e, edb))
        worst, worst_db = max(worst, e), max(worst_db, edb)
        assert e <= 1.0 and edb <= 1.0, (Cin, Cout, k, R)
        del x, dy, dw, db, ref, rabs
    print("wgrad: %d shapes, worst dw %.3g db %.3g; kernels %s" % (len(shapes), worst, worst_db, sorted(kernels)))
    assert any("wgrad3x3_c64_kernel" in n for n in kernels) and any("conv_wgrad_kernel" in n for n in kernels)


def test_attention_per_image_weight_gradient_at_flagship_shape():
    """The per-image gradient of the attention keys: dphi[b] = dS[b]^T theta[b] at B = 128, N = 4096, M = 1024, c8 = 64
    (conv_wgrad per_image=True), against a float64 per-image product."""
    from sgb200 import kernels as K
    dev = _cuda()
    B, S, c8, _ = ATTN
    M = (S // 2) ** 2
    gen = torch.Generator(device=dev).manual_seed(52)
    theta, dS = _act(gen, B, c8, S, S, dev), _act(gen, B, M, S, S, dev)
    got = K.conv_wgrad(theta, dS, 1, 1, 0, 0, per_image=True).view(B, M, c8)
    worst = 0.0
    for b0 in range(0, B, 16):
        b1 = min(B, b0 + 16)
        t, d = _rows(theta[b0:b1]), _rows(dS[b0:b1])
        ref, rabs = d.transpose(1, 2) @ t, d.abs().transpose(1, 2) @ t.abs()
        worst = max(worst, float(((got[b0:b1].double() - ref).abs() / (WGRAD_REL * rabs)).max()))
    print("attention per-image wgrad: %.3g" % worst)
    assert worst <= 1.0


# ------------------------------------------------------------------------------------------------ 2. fused block ops
def _packed_weight(m):
    """The bf16 W / sigma the kernels read: the fprop pack of the batched spectral-norm pass, as [Cout, Cin, k, k]."""
    Cout, Cin, k = m.out_channels, m.in_channels, m.kernel_size[0]
    return m._sn_cache[0][:Cout, :, :Cin].reshape(Cout, k, k, Cin).permute(0, 3, 1, 2)


def _sn_ref(m, u0):
    """float64 (W [Cout, Cin, k, k], u, v, sigma) of one power iteration from the saved u."""
    from sgb200.utils import ops
    W = ops._w(m).detach().double()
    Wm = W.reshape(W.shape[0], -1)
    v = F.normalize(Wm.t() @ u0.double(), dim=0, eps=ops.SN_EPS)
    s = Wm @ v
    u = F.normalize(s, dim=0, eps=ops.SN_EPS)
    return W, u, v, float(u @ s)


def _param_grad_worst(m, u0, x, dz):
    """Weight and bias gradient of the SN conv m given its input x and output gradient dz (both [B, ., H, W] bf16): the
    float64 chain rule dW = (G - <G, W / sigma> u v^T) / sigma on G = sum dz (x) x, against the weight-gradient bound."""
    from sgb200.utils import ops
    k = m.kernel_size[0]
    W, u, v, sig = _sn_ref(m, u0)
    G, Gabs = _wgrad_ref(x, dz, k, torch.arange(m.out_channels, device=x.device))
    Cout, Cin = m.out_channels, m.in_channels
    G, Gabs = (t.view(Cout, k, k, Cin).permute(0, 3, 1, 2) for t in (G, Gabs))
    uv = torch.outer(u, v).view_as(W)
    ref = (G - float((G * W).sum()) / sig * uv) / sig
    bound = WGRAD_REL * (Gabs + float((Gabs * W.abs()).sum()) / sig * uv.abs()) / sig
    e = float(((ops._w(m).grad.double() - ref).abs() / (bound + 1e-30)).max())
    dref, dabs = dz.double().sum((0, 2, 3)), dz.double().abs().sum((0, 2, 3))
    eb = float(((m.bias.grad.double() - dref).abs() / (WGRAD_REL * dabs + 1e-30)).max())
    return max(e, eb)


def _images(B):
    """Images whose per-element outputs are compared (a conv output depends on its own image only): all up to 8, else the
    first and the last four."""
    return list(range(B)) if B <= 8 else [0, 1, 2, 3, B - 4, B - 3, B - 2, B - 1]


def _conv_ratio(got, x, w, pad, bias=None, res=None, relu=False, mask=None, idx=None):
    """One-rounding ratio of a conv op's output on the images idx: [mask] relu(conv(x, w) + bias + res)."""
    x = x[idx]
    z = _conv64(x, w, pad)
    atol = ACC_REL * _conv64(x.abs(), w.abs(), pad) + 1e-30
    if bias is not None:
        z = z + bias.detach().double().view(1, -1, 1, 1)
    if res is not None:
        z = z + res[idx].double()
    if relu:
        z = z.clamp(min=0)
    if mask is not None:
        z = z * (mask[idx] > 0)
    return _rounding_ratio(got[idx], z, atol)


def _dgrad_ratio(got, dz, w, pad, mask=None, res=None, res_scale=1.0, res_up2=False, idx=None):
    """One-rounding ratio of an input gradient on the images idx: [mask > 0] (dgrad(dz, w) + res_scale [up2] res)."""
    dz = dz[idx]
    z = _dgrad64(dz, w.double(), pad)
    atol = ACC_REL * _dgrad64(dz.abs(), w.double().abs(), pad) + 1e-30
    if res is not None:
        r = res_scale * res[idx].double()
        z = z + (_up2(r) if res_up2 else r)
    if mask is not None:
        z = z * (mask[idx] > 0)
    return _rounding_ratio(got[idx], z, atol)


def _pool_bits(t, scale):
    """2x2 pooling as the kernels compute it: ((a + b) + c) + d in fp32, times scale, one rounding to bf16."""
    f = t.float()
    s = ((f[..., 0::2, 0::2] + f[..., 0::2, 1::2]) + f[..., 1::2, 0::2]) + f[..., 1::2, 1::2]
    return (s * scale).to(bf16)


CBN_REL, CBN_L2 = 8e-3, 3e-3     # cBN + ReLU outputs: max-norm relative to the largest element, and relative L2


def _cbn_err(y, x, cbn, affine, up2):
    """cBN + ReLU output y against float64 batch norm (batch statistics, eps of the layer) of the bf16 input x, with
    gain / bias = affine . W^T from the packs of the cBN linears, chunked over channels."""
    B, C, H, W = x.shape
    K = affine.shape[1]
    a = affine.view(B, K).double()
    gain = a @ cbn.gain._sn_cache[0][:C, 0, :K].double().t()
    bias = a @ cbn.bias._sn_cache[0][:C, 0, :K].double().t()
    e = _Err()
    cc = max(1, min(C, (1 << 24) // (B * H * W)))
    for c0 in range(0, C, cc):
        sl = slice(c0, min(C, c0 + cc))
        xc = x[:, sl].double()
        mu, var = xc.mean((0, 2, 3), keepdim=True), xc.var((0, 2, 3), unbiased=False, keepdim=True)
        z = ((xc - mu) * (var + cbn.bn.eps).rsqrt() * (1 + gain[:, sl, None, None]) + bias[:, sl, None, None]).clamp(min=0)
        e.add(y[:, sl, ::2, ::2] if up2 else y[:, sl], z)
        if up2:
            for i, j in ((0, 1), (1, 0), (1, 1)):
                assert torch.equal(y[:, sl, i::2, j::2], y[:, sl, ::2, ::2])
    return e


def _relu_input(gen, B, C, R, dev, in_relu):
    """Block input: with in_relu, a0 = relu(.) carrying the producer's bit planes (as a relu conv epilogue leaves it)."""
    x = _act(gen, B, C, R, R, dev)
    if in_relu:
        x = x.clamp(min=0)
        x._sgb_relu_bits = _pack_bits(x > 0)
    return x.requires_grad_(True)


def _d_block_ops(blk, x, in_relu, out_relu):
    """DiscBlock.forward, op by op, returning every intermediate."""
    from sgb200 import autograd_ops as A
    from sgb200.utils import ops
    t = {"x": x}
    t["a0"] = x if in_relu else A.ReluPassFn.call(x)
    c1 = blk.conv2d1
    t["h1"], t["px"] = A.DEntryConvFn.call(t["a0"], ops._w(c1), c1.bias,
                                           {"downsample": blk.downsample, "sn": c1._sn, "do_power_iteration": True,
                                            "sn_cache": c1._sn_cache, "sn_pass": c1._sn_pass,
                                            "skip_channels": blk.conv2d4.out_channels if blk.learnable_sc else 0})
    t["h2"] = blk.conv2d2(t["h1"], relu=True, premasked=True, mask_input=True)
    t["h3"] = blk.conv2d3(t["h2"], relu=True, premasked=True, mask_input=True)
    t["hp"] = A.AvgPoolFn.call(t["h3"], True) if blk.downsample else t["h3"]
    t["skip"] = t["px"]
    if blk.learnable_sc:
        c0 = blk.conv2d0
        t["skip"] = A.ConcatSkipFn.call(t["px"], ops._w(c0), c0.bias, {"sn": c0._sn, "do_power_iteration": True,
                                                                         "sn_cache": c0._sn_cache, "sn_pass": c0._sn_pass})
    t["out"] = blk.conv2d4(t["hp"], residual=t["skip"], mask_input=not blk.downsample, relu=out_relu, premasked=out_relu)
    return t


def _check_d_block(blk, R, in_relu, out_relu, B, dev, u0):
    gen = torch.Generator(device=dev).manual_seed(R * 7 + blk.conv2d4.out_channels + B)
    x = _relu_input(gen, B, blk.conv2d1.in_channels, R, dev, in_relu)
    t = _d_block_ops(blk, x, in_relu, out_relu)
    idx = _images(B)
    W1, W2, W3, W4 = (_packed_weight(m) for m in (blk.conv2d1, blk.conv2d2, blk.conv2d3, blk.conv2d4))
    a0, h1, h2, h3, hp, px, skip, out = (t[n].detach() for n in ("a0", "h1", "h2", "h3", "hp", "px", "skip", "out"))
    r = {}
    if not in_relu:
        assert torch.equal(a0, x.detach().clamp(min=0))
    r["h1"] = _conv_ratio(h1, a0, W1, 0, blk.conv2d1.bias, relu=True, idx=idx)
    assert torch.equal(_unpack_bits(t["h1"]._sgb_relu_bits, h1.shape[1]), h1 > 0)
    r["h2"] = _conv_ratio(h2, h1, W2, 1, blk.conv2d2.bias, relu=True, idx=idx)
    r["h3"] = _conv_ratio(h3, h2, W3, 1, blk.conv2d3.bias, relu=True, idx=idx)
    if blk.downsample:
        assert torch.equal(px, _pool_bits(a0, 0.25)) and torch.equal(hp, _pool_bits(h3, 0.25))
    if blk.learnable_sc:
        Cin = px.shape[1]
        assert px.data_ptr() == skip.data_ptr() and torch.equal(skip[:, :Cin], px)     # pooled straight into the concat buffer
        r["skip"] = _conv_ratio(skip[:, Cin:], px, _packed_weight(blk.conv2d0), 0, blk.conv2d0.bias, idx=idx)
    r["out"] = _conv_ratio(out, hp, W4, 0, blk.conv2d4.bias, res=skip, relu=out_relu, idx=idx)
    if out_relu:
        assert torch.equal(_unpack_bits(t["out"]._sgb_relu_bits, out.shape[1]), out > 0)
    # backward from a seeded bf16 gradient; a premasked output (out_relu) receives it already masked, as its consumer sends it
    for n in ("h1", "h2", "h3", "hp", "px", "skip"):
        t[n].retain_grad()
    dout = _act(gen, *out.shape, dev)
    if out_relu:
        dout = dout * (out > 0)
    for p in blk.parameters():
        p.grad = None
    t["out"].backward(dout)
    g = {n: t[n].grad for n in ("h1", "h2", "h3", "hp", "px", "skip")}
    assert torch.equal(g["skip"], dout)
    r["d_hp"] = _dgrad_ratio(g["hp"], dout, W4, 0, mask=None if blk.downsample else hp, idx=idx)
    if blk.downsample:      # average-pool backward into a post-ReLU input: 0.25 dy where h3 > 0, bit for bit
        assert torch.equal(g["h3"], (_up2(g["hp"].float()) * 0.25 * (h3 > 0)).to(bf16))
    r["d_h2"] = _dgrad_ratio(g["h2"], g["h3"], W3, 1, mask=h2, idx=idx)
    r["d_h1"] = _dgrad_ratio(g["h1"], g["h2"], W2, 1, mask=h1, idx=idx)
    dpx = g["px"]
    if blk.learnable_sc:
        Cin = px.shape[1]
        r["d_px"] = _dgrad_ratio(dpx, g["skip"][:, Cin:], _packed_weight(blk.conv2d0), 0, res=g["skip"][:, :Cin], idx=idx)
    # DEntryConvFn: dx = [a0 > 0] (dgrad1(dh1) + 0.25 up2(dpx)) in one launch (ReluPassFn passes it through)
    r["dx"] = _dgrad_ratio(x.grad, g["h1"], W1, 0, mask=a0, res=dpx, res_scale=0.25 if blk.downsample else 1.0,
                           res_up2=blk.downsample, idx=idx)
    r["dW4"] = _param_grad_worst(blk.conv2d4, u0[blk.conv2d4], hp, dout)
    r["dW1"] = _param_grad_worst(blk.conv2d1, u0[blk.conv2d1], a0, g["h1"])
    r["dW2"] = _param_grad_worst(blk.conv2d2, u0[blk.conv2d2], h1, g["h2"])
    r["dW3"] = _param_grad_worst(blk.conv2d3, u0[blk.conv2d3], h2, g["h3"])
    if blk.learnable_sc:
        r["dW0"] = _param_grad_worst(blk.conv2d0, u0[blk.conv2d0], px, g["skip"][:, px.shape[1]:])
    return r


def _sn_run(net):
    """The batched spectral-norm pass of the model's forward; returns the u of every layer before it (the saved u)."""
    u0 = {m: m.weight_u.clone() for m in net.modules() if hasattr(m, "weight_u")}
    with torch.enable_grad():
        net._snb.run()
    return u0


def test_discriminator_block_ops_every_flagship_geometry_vs_float64(flagship):
    """Every DiscBlock of the flagship (12 distinct geometries, including the block before the 64x64 attention, out_relu =
    False, and the one after it, which takes ReluPassFn): the ops of DiscBlock.forward forward and backward.  B = 128 for the
    blocks at 64x64 and below, B = 3 at 256x256 and B = 4 at 128x128.  Per-element outputs and input gradients are compared on
    the first and last four images of the batch; the weight and bias gradients of every conv over the whole batch."""
    dev = _cuda()
    _, D = flagship
    blocks = _d_blocks(D)
    assert len(blocks) == 12 and any(not o for _, _, _, o in blocks) and any(not i for _, _, i, _ in blocks)
    u0 = _sn_run(D)
    worst = {}
    try:
        for blk, R, in_relu, out_relu in blocks:
            B = 128 if R <= 64 else (3 if R == 256 else 4)
            r = _check_d_block(blk, R, in_relu, out_relu, B, dev, u0)
            print("D %d->%d @%d B=%d in_relu=%d out_relu=%d: %s" % (blk.conv2d1.in_channels, blk.conv2d4.out_channels, R, B,
                                                                   in_relu, out_relu, {k: round(v, 3) for k, v in r.items()}))
            for k, v in r.items():
                worst[k] = max(worst.get(k, 0.0), v)
            torch.cuda.empty_cache()
    finally:
        D._snb.clear()
    print("D block ops worst:", worst)
    assert max(worst.values()) <= 1.0, worst


def test_discriminator_entry_at_256_past_2_31_bytes(flagship):
    """DEntryConvFn of D stage 0 at B = 130 (a0 and its gradient: 130 x 128 channels x 256^2 bf16 = 2.18 GB, so images 128
    and 129 lie past 2^31 bytes): h1, the pooled skip source in the concat buffer, and the fused input gradient with mask
    bits and the up-sampled pooled-skip gradient, compared on images on both sides of the boundary."""
    from sgb200 import autograd_ops as A
    from sgb200.utils import ops
    dev = _cuda()
    _, D = flagship
    blk, R, in_relu, _ = _d_blocks(D)[0]
    assert R == 256 and in_relu and blk.downsample and blk.learnable_sc
    _sn_run(D)
    try:
        c1 = blk.conv2d1
        gen = torch.Generator(device=dev).manual_seed(61)
        B = 130
        a0 = _relu_input(gen, B, c1.in_channels, R, dev, True)
        assert a0.numel() * a0.element_size() > 2 ** 31
        h1, px = A.DEntryConvFn.call(a0, ops._w(c1), c1.bias, {"downsample": True, "sn": c1._sn, "do_power_iteration": True,
                                                               "sn_cache": c1._sn_cache, "sn_pass": c1._sn_pass,
                                                               "skip_channels": blk.conv2d4.out_channels})
        W1 = _packed_weight(c1)
        idx = [0, 1, 64, 127, 128, B - 1]
        r = {"h1": _conv_ratio(h1.detach(), a0.detach(), W1, 0, c1.bias, relu=True, idx=idx)}
        assert torch.equal(px.detach()[idx], _pool_bits(a0.detach()[idx], 0.25))
        dh1 = _act(gen, *h1.shape, dev) * (h1.detach() > 0)
        dpx = _act(gen, *px.shape, dev)
        torch.autograd.backward([h1, px], [dh1, dpx])
        r["dx"] = _dgrad_ratio(a0.grad, dh1, W1, 0, mask=a0.detach(), res=dpx, res_scale=0.25, res_up2=True, idx=idx)
        print("D stage 0 entry at B=130:", r)
        assert max(r.values()) <= 1.0
    finally:
        D._snb.clear()


def test_generator_block_ops_every_flagship_geometry_vs_float64(flagship):
    """Every distinct GenBlock of the flagship: SplitResidualFn, the cBN + ReLU (+ x2) BNActFn launches, the four ConvFn
    launches and conv2d4's skip x[:, :out] (res_up2 in the up-sampling blocks, read from the wider block input), forward
    and backward.  The conv outputs and input gradients are held to one rounding of float64 on the bf16 tensors the ops
    passed each other; the four cBN + ReLU outputs (bn2 with the x2 up-sample) against float64 batch norm with the gains of
    the cBN linears' packs; the skip gradient is the 2x2 sum of conv2d4's output gradient (pool2_fwd mode 2) and is added in
    place into the first channels of the main-branch gradient, both bit for bit; the weight / bias gradients of every conv
    over the whole batch.  B = 128 where the block's
    largest map is at most 64x64, B = 4 at 128x128 and B = 3 at 256x256."""
    from sgb200 import autograd_ops as A
    from sgb200.utils import ops
    dev = _cuda()
    G, _ = flagship
    seen, worst = set(), {}
    u0 = _sn_run(G)
    try:
        for blk, R in _g_blocks(G):
            Ru = 2 * R if blk.upsample else R
            geo = (blk.in_channels, blk.out_channels, R, blk.upsample)
            if geo in seen:
                continue
            seen.add(geo)
            B = 128 if Ru <= 64 else (4 if Ru == 128 else 3)
            gen = torch.Generator(device=dev).manual_seed(R * 13 + blk.in_channels + B)
            x = _act(gen, B, blk.in_channels, R, R, dev).requires_grad_(True)
            affine = (0.5 * torch.randn((B, G.affine_input_dim, 1, 1), generator=gen, device=dev)).to(bf16)
            t = {}
            t["main"], t["skip"] = A.SplitResidualFn.call(x, blk.out_channels)
            assert t["skip"].data_ptr() == x.data_ptr() and t["skip"].shape[1] == blk.out_channels
            t["a1"] = blk.bn1(t["main"], affine, relu=True)
            t["h1"] = blk.conv2d1(t["a1"])
            t["a2"] = blk.bn2(t["h1"], affine, relu=True, up2=blk.upsample)
            t["h2"] = blk.conv2d2(t["a2"])
            t["a3"] = blk.bn3(t["h2"], affine, relu=True)
            t["h3"] = blk.conv2d3(t["a3"])
            t["a4"] = blk.bn4(t["h3"], affine, relu=True)
            t["out"] = blk.conv2d4(t["a4"], residual=t["skip"], res_up2=blk.upsample)
            d = {n: v.detach() for n, v in t.items()}
            idx = _images(B)
            Ws = [_packed_weight(m) for m in (blk.conv2d1, blk.conv2d2, blk.conv2d3, blk.conv2d4)]
            r = {"h1": _conv_ratio(d["h1"], d["a1"], Ws[0], 0, blk.conv2d1.bias, idx=idx),
                 "h2": _conv_ratio(d["h2"], d["a2"], Ws[1], 1, blk.conv2d2.bias, idx=idx),
                 "h3": _conv_ratio(d["h3"], d["a3"], Ws[2], 1, blk.conv2d3.bias, idx=idx)}
            skip_in = _up2(d["skip"][idx]) if blk.upsample else d["skip"][idx]
            sk = torch.zeros_like(d["out"][:, :1]).expand(-1, d["out"].shape[1], -1, -1).clone()
            sk[idx] = skip_in
            r["out"] = _conv_ratio(d["out"], d["a4"], Ws[3], 0, blk.conv2d4.bias, res=sk, idx=idx)
            for n, src, bn, up in (("a1", "main", blk.bn1, False), ("a2", "h1", blk.bn2, blk.upsample), ("a3", "h2", blk.bn3, False),
                                   ("a4", "h3", blk.bn4, False)):
                e = _cbn_err(d[n], d[src], bn, affine, up)
                r[n + " rel"], r[n + " l2"] = e.rel / CBN_REL, e.l2 / CBN_L2
            for n in ("h1", "h2", "h3", "a1", "a2", "a3", "a4"):
                t[n].retain_grad()
            split_in = {}            # the gradients SplitResidualFn receives, before its in-place add
            t["main"].register_hook(lambda g_: split_in.__setitem__("main", g_.clone()))
            t["skip"].register_hook(lambda g_: split_in.__setitem__("skip", g_.clone()))
            for p in blk.parameters():
                p.grad = None
            dout = _act(gen, *d["out"].shape, dev)
            t["out"].backward(dout)
            gr = {n: t[n].grad for n in ("h1", "h2", "h3", "a1", "a2", "a3", "a4")}
            gr.update(split_in)
            # the skip gradient: the 2x2 sum of dout (pool2_fwd mode 2) in the up-sampling blocks, dout itself otherwise
            assert torch.equal(gr["skip"], _pool_bits(dout, 1.0) if blk.upsample else dout)
            r["d_a4"] = _dgrad_ratio(gr["a4"], dout, Ws[3], 0, idx=idx)
            r["d_a3"] = _dgrad_ratio(gr["a3"], gr["h3"], Ws[2], 1, idx=idx)
            r["d_a2"] = _dgrad_ratio(gr["a2"], gr["h2"], Ws[1], 1, idx=idx)
            r["d_a1"] = _dgrad_ratio(gr["a1"], gr["h1"], Ws[0], 0, idx=idx)
            # SplitResidualFn: dx = d_main with d_skip added into its first channels (one fp32 add, one rounding)
            c = blk.out_channels
            want = gr["main"].clone()
            want[:, :c] = (gr["main"][:, :c].float() + gr["skip"].float()).to(bf16)
            assert torch.equal(x.grad, want)
            r["dW1"] = _param_grad_worst(blk.conv2d1, u0[blk.conv2d1], d["a1"], gr["h1"])
            r["dW2"] = _param_grad_worst(blk.conv2d2, u0[blk.conv2d2], d["a2"], gr["h2"])
            r["dW3"] = _param_grad_worst(blk.conv2d3, u0[blk.conv2d3], d["a3"], gr["h3"])
            r["dW4"] = _param_grad_worst(blk.conv2d4, u0[blk.conv2d4], d["a4"], dout)
            print("G %d->%d @%d up=%d B=%d: %s" % (blk.in_channels, blk.out_channels, R, blk.upsample, B,
                                                   {k: round(v, 3) for k, v in r.items()}))
            for k, v in r.items():
                worst[k] = max(worst.get(k, 0.0), v)
            del t, d, gr, x
            torch.cuda.empty_cache()
    finally:
        G._snb.clear()
    print("G block ops worst:", worst)
    assert len(seen) == 12 and max(worst.values()) <= 1.0, worst


# Block composition: relative L2 of the block output, dx and every parameter gradient against the float64 reference block.
# Estimates.  The output carries a chain of four bf16-stored convs and the bf16 W / sigma packs, each ~2^-9 relative: 1e-2.
# The gradients also pass the four ReLU masks, which the two computations form from their own forward values: an element
# whose pre-activation lies within the forward error (e ~ 2^-9 relative) of zero falls on different sides in the two, and
# carries its whole gradient on one side only.  A flip fraction ~e per mask adds ~sqrt(e) ~ 4e-2 to the relative L2 of
# what is computed from the masked gradients: 5e-2 for dx; the parameter gradients, sums over the batch of those masked
# gradients times activations, add their own masks' flips: 1.5e-1.
BLOCK_L2 = {"out": 1e-2, "dx": 5e-2, "param": 1.5e-1}


def _ref_disc_block(blk, x, dout, in_relu, out_relu, P):
    """The reference DiscBlock.forward in float64 on images x (bf16 values): x0 = x; relu(x) in place (so the skip path
    carries relu(x)); conv2d1 .. conv2d3 each after a ReLU; ReLU; avgpool; conv2d4; skip = [avgpool](x0), cat([x0,
    conv2d0(x0)]) with a learnable shortcut; out = h + skip (and the next block's ReLU with out_relu).  P: conv -> (W / sigma,
    bias) with autograd to the float64 parameters.  Returns (out, dx) after backpropagating dout."""
    xin = x.double().requires_grad_(True)
    a0 = torch.relu(xin)
    h = a0
    for m in (blk.conv2d1, blk.conv2d2, blk.conv2d3):
        W, b = P[m]
        h = torch.relu(_conv64(h, W, m.padding[0]) + b.view(1, -1, 1, 1))
    x0 = a0
    if blk.downsample:
        h, x0 = F.avg_pool2d(h, 2), F.avg_pool2d(a0, 2)
    W, b = P[blk.conv2d4]
    h = _conv64(h, W, 0) + b.view(1, -1, 1, 1)
    if blk.learnable_sc:
        W, b = P[blk.conv2d0]
        x0 = torch.cat([x0, _conv64(x0, W, 0) + b.view(1, -1, 1, 1)], 1)
    out = h + x0
    if out_relu:
        out = torch.relu(out)
    out.backward(dout.double())
    return out.detach(), xin.grad


def test_discriminator_block_composition_vs_float64_reference_block(flagship):
    """block(x, in_relu, out_relu) of every flagship DiscBlock, forward and backward, against the reference block arithmetic
    restated in float64 (_ref_disc_block), with W / sigma from one float64 power iteration on the saved u (sigma = u W v with
    u, v held constant, as the spectral norm's gradient treats them).  The flagship's hand-over cases are all here: blocks
    between blocks (in_relu = out_relu = True), the block before the 64x64 attention (out_relu = False) and the one after it
    (in_relu = False: ReluPassFn).  A premasked output (out_relu) receives its gradient masked, as its consumer sends it.
    B = 128 at 64x64 and below, B = 4 at 128x128, B = 3 at 256x256; the reference runs over chunks of images and
    accumulates the parameter gradients."""
    from sgb200.utils import ops
    dev = _cuda()
    _, D = flagship
    blocks = _d_blocks(D)
    assert {(i, o) for _, _, i, o in blocks} == {(True, True), (True, False), (False, True)}
    u0 = _sn_run(D)
    worst = {"out": 0.0, "dx": 0.0, "param": 0.0}
    try:
        for blk, R, in_relu, out_relu in blocks:
            B = 128 if R <= 64 else (3 if R == 256 else 4)
            gen = torch.Generator(device=dev).manual_seed(R * 11 + blk.conv2d4.out_channels + B)
            x = _relu_input(gen, B, blk.conv2d1.in_channels, R, dev, in_relu)
            convs = [blk.conv2d1, blk.conv2d2, blk.conv2d3, blk.conv2d4] + ([blk.conv2d0] if blk.learnable_sc else [])
            for p in blk.parameters():
                p.grad = None
            out = blk(x, in_relu=in_relu, out_relu=out_relu)
            dout = _act(gen, *out.shape, dev)
            if out_relu:
                dout = dout * (out.detach() > 0)
            out.backward(dout)
            leaves = {}
            for m in convs:
                W, u, v, _ = _sn_ref(m, u0[m])
                leaves[m] = (W.requires_grad_(True), u, v, m.bias.detach().double().requires_grad_(True))
            e_out, e_dx = _Err(), _Err()
            per = max(1, (1 << 25) // (blk.conv2d1.in_channels * R * R))
            for b0 in range(0, B, per):
                b1 = min(B, b0 + per)
                P = {m: (W / (u @ (W.reshape(W.shape[0], -1) @ v)), b) for m, (W, u, v, b) in leaves.items()}
                ro, rdx = _ref_disc_block(blk, x.detach()[b0:b1], dout[b0:b1], in_relu, out_relu, P)
                e_out.add(out.detach()[b0:b1], ro)
                e_dx.add(x.grad[b0:b1], rdx)
            r = {"out": e_out.l2, "dx": e_dx.l2, "param": 0.0}
            for m, (W, _, _, b) in leaves.items():
                for got, ref in ((ops._w(m).grad, W.grad), (m.bias.grad, b.grad)):
                    e = _Err()
                    e.add(got, ref)
                    r["param"] = max(r["param"], e.l2)
            print("D block %d->%d @%d B=%d in_relu=%d out_relu=%d: out %.3g dx %.3g params %.3g (relative L2)" % (
                blk.conv2d1.in_channels, blk.conv2d4.out_channels, R, B, in_relu, out_relu, r["out"], r["dx"], r["param"]))
            for k in worst:
                worst[k] = max(worst[k], r[k])
            del x, out, dout, leaves
            torch.cuda.empty_cache()
    finally:
        D._snb.clear()
    print("D block composition worst:", {k: "%.3g of %.3g" % (v, BLOCK_L2[k]) for k, v in worst.items()})
    assert all(worst[k] <= BLOCK_L2[k] for k in worst), worst
