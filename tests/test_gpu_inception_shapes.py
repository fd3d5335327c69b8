"""The FID InceptionV3 feature extractor (metrics/inception_net.py) launch by launch at the batches of the FID-50k
evaluation, against float64 (pytest -m gpu).

bench.py evaluates FID-50k with min(256, per-rank batch), the per-rank batch capped at 128 for BigGAN-Deep, and its
reference-statistics pass ends on a short batch.  So the Inception batches that run are B = 128 (every batch at one and
two GPUs), 80 (the last reference batch at one and two GPUs: 50 000 - 390 * 128), 64 (four GPUs), 32 (eight GPUs) and
16 (the last reference batch of a rank at four and eight GPUs).  Inputs are 256x256 images, resized to 299 by the
"legacy" resizer: generated ones (fp32 in [-1, 1], quantize=True) at B = 128, 64 and 32, reference ones
(integer-valued 0..255, quantize=False) at B = 80 and 16.  Weights are seeded_state_dict(0), as in bench.py.  The images
are smooth (bilinearly upsampled low-resolution noise through tanh), so that the deep layers see activation statistics
like those of real images rather than of per-pixel noise.

Four parts:
1. quantize_resize_normalize from 256x256 to 299 at B = 128 and 80 in both input modes, with generated inputs outside
   [-1, 1] and on the quantiser's .5 boundaries: the normalised image and the [B, 149, 149, 32] patch tensor the first
   convolution reads.
2. Every launch of InceptionV3.forward at each B, one at a time: the 94 convolutions and the fc layer (conv_fprop), the
   13 3x3 pools (pool3x3) and the feature sum (sum_hw), each against float64 on the bf16 input it actually received.
   These are the conv engine paths the training step never takes: the run-time-flag kernel (F = -1) with TMA stores at
   Cout % 64 != 0 (48, 80, 96, 160), the one-row-per-thread epilogue (Cout 32, the four stride-2 convolutions and the
   fp32 fc output), "valid" convolutions, asymmetric pads and 1x7 / 7x1 / 1x3 / 3x1 / 5x5 filters, K blocks past Cin,
   ragged pixel tiles and image-pair tiles.  Wrappers replace kernels.conv_fprop / pool3x3 / sum_hw / empty_nhwc for
   one forward.  Every tensor empty_nhwc allocates (block outputs, branch intermediates, the patch tensor, the fc
   output) starts filled with SENTINEL, so an element no kernel stores is seen: no op may read one, no op output may
   keep one, and none may be left once the forward has run.  A launch that writes a channel slice of a block tensor
   (out=) must leave every other channel of that tensor bit-identical (stride-2 stores on odd positions, TMA boxes
   spilling past Cout into the next branch, wrong nested slice offsets in the E blocks).  The launch counts (95
   conv_fprop, 13 pool3x3, 1 sum_hw) are pinned, so a forward routed around the wrappers fails instead of checking
   less, and a torch.profiler trace must show both the run-time-flag conv_fprop_kernel and a compiled variant.
3. The forward as a whole at each B against O.fid_inception_forward on the torchvision module (O.fid_inception, batch
   norms not folded, in float64): an independent statement of the topology that catches what a per-op check cannot
   see -- branch order inside _cat, the pool mode of each block, which tensor feeds which branch.
4. The FID moments at FID-50k's N: 50 000 non-negative 2048-d features (per-dimension mean ~3x the standard deviation,
   like pooled post-ReLU features, where the one-pass sum f f^T - n mu mu^T of moments_finalize_kernel cancels most)
   through MomentsAccumulator as the evaluation folds them (390 updates of 128 rows, then 80) and through
   calculate_moments' 4096-row blocks.

References: plain float64 torch on the GPU, on the same bf16 operands and packed bf16 weights the kernels read (a conv's
weight is unpacked from the [Cout_p][taps][Cin_p] pack it was handed).  Per-element outputs are compared on the images
_images(B), the first four and the last four, so the last pixel and image tiles of every launch are inside the check;
the sentinel and slice checks cover the whole batch.  Nothing on the reference side calls the library.

Tolerances (bf16 keeps 8 significant bits: one round-to-nearest moves a value by at most 2^-8 of itself):
* pre-processing: the image within 5e-5 of O.eval_preprocess (fp32 bilinear weights; a quantised value one grey level
  off would be 7.8e-3 away); the patch tensor one bf16 rounding of the reference's 3x3 / stride-2 unfold plus that
  5e-5; channels 27..31 exactly zero.
* convolutions with a bf16 output: one bf16 rounding plus atol = ACC_REL (2^-14) of the absolute-value convolution, the
  rule of test_gpu_conv_fused.py; the fc layer (fp32 output, no ReLU): FP32_REL (2^-22) |ref| + the same atol.
* max pools bit for bit.  Average pools (count_include_pad=False): one bf16 rounding plus 2^-20 of the window's mean
  |x|: the kernel adds <= 9 values in fp32 (<= 8 roundings, each <= 2^-24 of a partial sum of non-negative values) and
  multiplies by an fp32 1 / cnt (two more roundings): <= 10 * 2^-24 of the mean |x|.
* sum_hw: 2^-20 of sum |x| over the 8x8 map, i.e. of the mean |x| after the division by 64.  The kernel adds chunks of
  <= 13 pixels in fp32 and up to 32 chunk sums (at B = 16) with fp32 atomics in any order; the worst case of ~45
  roundings would reach ~2^-18.5, but independent roundings add up to a standard deviation of ~2^-23 of the total and
  the largest of 2048 * B such errors stays near 2^-21 (an estimate).
* the forward as a whole (WHOLE_L2): relative L2 per image, not pooled over the batch, <= 3e-2 on the pool features and
  on the logits, the bound of test_gpu_eval.py's golden comparison.  Estimate: every stored activation is rounded to
  bf16 (relative RMS error ~0.4 * 2^-8 ~ 1.6e-3 per store), and a path from the image to the features crosses 18 (the
  1x1 and pooling branches) to 49 (the double 7x7 branches) such stores, one more to the logits; with independent
  errors and gains ~1 through the He-scaled layers that is sqrt(18..50) * 1.6e-3 ~ 7e-3..1.1e-2.
* moments: the bounds of test_gpu_eval.py against a float64 two-pass mean and covariance (np.cov's arithmetic):
  mu rtol / atol 1e-12, sigma rtol 1e-9, atol 1e-10.
"""
import warnings

import pytest
import torch
import torch.nn.functional as F

from oracle import studiogan_oracle as O
from test_gpu_conv_fused import ACC_REL, FP32_REL, SENTINEL, _images, _launched
from test_gpu_norm_shapes import _cuda, _rounding_ratio

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16
# B -> input mode of the batches of that size in the FID-50k evaluation
BATCHES = {128: "generated", 80: "reference", 64: "generated", 32: "generated", 16: "reference"}
IMG_TOL = 5e-5
POOL_REL = 2.0 ** -20
WHOLE_L2 = 3e-2
LAUNCHES = {"conv_fprop": 95, "pool3x3": 13, "sum_hw": 1}


def _images_for(B, mode, edges=False):
    """B smooth 256x256 images (CPU fp32) of the input mode and its quantize flag.  Two octaves of bilinearly upsampled
    noise (8x8 and 32x32) through tanh, gain and shift drawn per image.  generated: values in (-1, 1); with edges, the
    first half of the batch is scaled by 1.25 (the quantiser clamps) and five rows of every channel carry the values at
    and 1-2 ulps around each of the quantiser's 255 .5 boundaries.  reference: round(127.5 (t + 1)), integers 0..255."""
    g = torch.Generator().manual_seed(1000 + B + (7 if mode == "reference" else 0))
    up = lambda r: F.interpolate(torch.randn(B, 3, r, r, generator=g), size=(256, 256), mode="bilinear",  # noqa: E731
                                 align_corners=False)
    gain = 0.8 + 1.2 * torch.rand(B, 1, 1, 1, generator=g)
    shift = 0.6 * torch.rand(B, 1, 1, 1, generator=g) - 0.3
    t = torch.tanh((up(8) + 0.35 * up(32)) * gain + shift)
    if mode == "reference":
        return torch.round((t + 1.0) * 127.5).clamp(0, 255), False
    if edges:
        t[:B // 2] *= 1.25
        # 255 (x + 1) / 2 + 0.5 = k exactly at x = (2k - 1) / 255 - 1, k = 1..255: the nearest fp32 and its neighbours
        x = ((2.0 * torch.arange(1, 256, dtype=torch.float64) - 1.0) / 255.0 - 1.0).float()
        up1, dn1 = torch.nextafter(x, torch.tensor(2.0)), torch.nextafter(x, torch.tensor(-2.0))
        up2, dn2 = torch.nextafter(up1, torch.tensor(2.0)), torch.nextafter(dn1, torch.tensor(-2.0))
        t[:, :, 120:125, :255] = torch.stack([x, up1, dn1, up2, dn2])
    return t, True


# ------------------------------------------------------------------------------------------------ 1. pre-processing
@pytest.mark.parametrize("B,mode", [(128, "generated"), (128, "reference"), (80, "generated"), (80, "reference")])
def test_preprocess_at_eval_size_vs_reference(B, mode, monkeypatch):
    from sgb200 import kernels as K
    dev = _cuda()
    real_empty = K.empty_nhwc

    def empty_nhwc(*a, **kw):                      # the patch tensor starts as SENTINEL: channels 27..31 must be stored
        return real_empty(*a, **kw).fill_(SENTINEL)
    monkeypatch.setattr(K, "empty_nhwc", empty_nhwc)
    img, quantize = _images_for(B, mode, edges=True)
    ref = O.eval_preprocess(img, 299, quantize).to(dev)
    got, col = K.quantize_resize_normalize(img.to(dev), 299, quantize=quantize, want_image=True, want_col=True)
    assert got.shape == (B, 3, 299, 299) and col.shape == (B, 32, 149, 149)
    img_err = float((got - ref).abs().max())
    c = col.permute(0, 2, 3, 1)                    # [B, 149, 149, 32], k = tap * 3 + channel
    unf = F.unfold(ref.double(), kernel_size=3, stride=2).view(B, 3, 9, 149, 149).permute(0, 3, 4, 2, 1).reshape(B, 149, 149, 27)
    ratio = _rounding_ratio(c[..., :27], unf, IMG_TOL)
    print("preprocess B=%d %s: image %.3g (bound %.0e), patches %.3f" % (B, mode, img_err, IMG_TOL, ratio))
    assert img_err <= IMG_TOL
    assert ratio <= 1.0
    assert bool((c[..., 27:] == 0).all())


# ------------------------------------------------------------------------------------------------ 2. every launch
def _conv64(x, w, ph, pw, stride):
    """float64 convolution of [b, Cin, Hin, Win] with [Cout, Cin, KH, KW], pads (ph, pw), on the stride-1 output grid
    Hin + 2 ph - KH + 1 (same or valid); stride 2 keeps its even positions.  One float64 matmul per tap; returns
    (conv(x, w), conv(|x|, |w|))."""
    b, Cin, Hin, Win = x.shape
    Cout, _, KH, KW = w.shape
    H, W = Hin + 2 * ph - KH + 1, Win + 2 * pw - KW + 1
    Ho, Wo = (H + 1) // 2 if stride == 2 else H, (W + 1) // 2 if stride == 2 else W
    xp = F.pad(x.double().permute(0, 2, 3, 1), (0, 0, pw, pw, ph, ph))
    w = w.double()
    y = torch.zeros((b, Ho, Wo, Cout), device=x.device, dtype=torch.float64)
    ya = torch.zeros_like(y)
    for kh in range(KH):
        for kw in range(KW):
            xt = xp[:, kh:kh + H:stride, kw:kw + W:stride]
            wt = w[:, :, kh, kw].t()
            y += xt @ wt
            ya += xt.abs() @ wt.abs()
    return y.permute(0, 3, 1, 2), ya.permute(0, 3, 1, 2)


class _Launches:
    """Wrappers over kernels.conv_fprop / pool3x3 / sum_hw / empty_nhwc for one forward, and what they measured.
    worst: part -> (largest ratio to its bound, label of that launch); faults: labels of failed exact checks."""

    def __init__(self, K, B, monkeypatch):
        self.real = {n: getattr(K, n) for n in ("conv_fprop", "pool3x3", "sum_hw", "empty_nhwc")}
        self.idx = _images(B)
        self.allocated, self.faults, self.worst = [], [], {}
        self.counts = {n: 0 for n in LAUNCHES}
        for n in self.real:
            monkeypatch.setattr(K, n, getattr(self, n))

    def _note(self, part, ratio, label):
        if ratio > self.worst.get(part, (-1.0, None))[0]:
            self.worst[part] = (ratio, label)

    def _clean(self, t, what, label):
        if bool((t == SENTINEL).any()):
            self.faults.append("%s holds SENTINEL: %s" % (what, label))

    def empty_nhwc(self, B, C, H, W, device, dtype=bf16):
        t = self.real["empty_nhwc"](B, C, H, W, device, dtype).fill_(SENTINEL)
        self.allocated.append(t)
        return t

    def _slice(self, out):
        """(block tensor holding the channel slice out, channel offset, its channels before the launch) or None."""
        if out is None:
            return None
        base = [t for t in self.allocated if t.untyped_storage().data_ptr() == out.untyped_storage().data_ptr()]
        assert len(base) == 1 and base[0].stride() == out.stride(), "out= is not a channel slice of one allocated tensor"
        off = (out.data_ptr() - base[0].data_ptr()) // out.element_size()
        assert 0 <= off and off + out.shape[1] <= base[0].shape[1]
        return base[0], off, base[0].permute(0, 2, 3, 1).clone()

    def _after(self, snap, y, label):
        """Output checks common to conv and pool: no SENTINEL left in it, and outside its slice the block tensor unchanged."""
        self._clean(y, "output", label)
        if snap is None:
            return
        base, off, before = snap
        now, before = base.permute(0, 2, 3, 1).view(torch.int16), before.view(torch.int16)
        C = y.shape[1]
        if not (torch.equal(now[..., :off], before[..., :off]) and torch.equal(now[..., off + C:], before[..., off + C:])):
            self.faults.append("channels outside [%d, %d) of the block tensor changed: %s" % (off, off + C, label))

    def conv_fprop(self, x, w, Cout, KH, KW, pad_h, pad_w, **kw):
        assert set(kw) <= {"bias", "relu", "out", "same_size", "stride", "out_fp32"}, sorted(kw)
        n = self.counts["conv_fprop"] = self.counts["conv_fprop"] + 1
        B, Cin, Hin, Win = x.shape
        stride, relu, bias, fp32 = kw.get("stride", 1), kw.get("relu", False), kw.get("bias"), kw.get("out_fp32", False)
        label = "conv %d: %d->%d %dx%d pad (%d, %d) stride %d at %dx%d" % (n, Cin, Cout, KH, KW, pad_h, pad_w, stride, Hin, Win)
        self._clean(x, "input", label)
        snap = self._slice(kw.get("out"))
        y = self.real["conv_fprop"](x, w, Cout, KH, KW, pad_h, pad_w, **kw)
        self._after(snap, y, label)
        # the pack [Cout_p][taps][Cin_p] the kernel read; its rows are Cin long (the tensor map's row length)
        assert w.shape[0] >= Cout and w.shape[1] == KH * KW and w.shape[2] == Cin, (label, tuple(w.shape))
        wt = w[:Cout].reshape(Cout, KH, KW, Cin).permute(0, 3, 1, 2)
        z, za = _conv64(x[self.idx], wt, pad_h, pad_w, stride)
        assert y.shape == (B, Cout) + tuple(z.shape[2:]), (label, tuple(y.shape))
        if bias is not None:
            z = z + bias.double().view(1, -1, 1, 1)
        if relu:
            z = z.clamp(min=0)
        got, atol = y[self.idx], ACC_REL * za + 1e-30
        if fp32:
            self._note("fc (fp32)", float(((got.double() - z).abs() / (FP32_REL * z.abs() + atol)).max()), label)
        else:
            self._note("conv", _rounding_ratio(got, z, atol), label)
        return y

    def pool3x3(self, x, stride, pad, mode, out=None):
        n = self.counts["pool3x3"] = self.counts["pool3x3"] + 1
        label = "pool %d: %s stride %d pad %d, %d ch at %dx%d" % (n, "max" if mode == 1 else "avg", stride, pad, x.shape[1],
                                                                  x.shape[2], x.shape[3])
        self._clean(x, "input", label)
        snap = self._slice(out)
        y = self.real["pool3x3"](x, stride, pad, mode, out=out)
        self._after(snap, y, label)
        xi = x[self.idx].double()
        got = y[self.idx]
        if mode == 1:
            ref = F.max_pool2d(xi, 3, stride, pad)
            if got.shape != ref.shape or not torch.equal(got.double(), ref):
                self.faults.append("max pool not bit-exact: " + label)
        else:
            ref = F.avg_pool2d(xi, 3, stride, pad, count_include_pad=False)
            assert got.shape == ref.shape, label
            atol = POOL_REL * F.avg_pool2d(xi.abs(), 3, stride, pad, count_include_pad=False) + 1e-30
            self._note("avg pool", _rounding_ratio(got, ref, atol), label)
        return y

    def sum_hw(self, x, relu):
        self.counts["sum_hw"] += 1
        self._clean(x, "input", "sum_hw")
        h = self.real["sum_hw"](x, relu)
        xd = x.double()
        ref = (xd.clamp(min=0) if relu else xd).sum((2, 3))
        self._note("sum_hw", float(((h.double() - ref).abs() / (POOL_REL * xd.abs().sum((2, 3)) + 1e-30)).max()), "sum_hw")
        return h


@pytest.fixture(scope="module")
def inception():
    """(product InceptionV3, torchvision Inception3 in float64 on the GPU) with seeded_state_dict(0)."""
    from sgb200.metrics.inception_net import InceptionV3, seeded_state_dict
    dev = _cuda()
    sd = seeded_state_dict(0)
    nets = InceptionV3(sd, dev), O.fid_inception(sd).double().to(dev)
    yield nets
    del nets
    torch.cuda.empty_cache()


@pytest.mark.parametrize("B", list(BATCHES))
def test_every_inception_launch_at_fid50k_batch_vs_float64(inception, B, monkeypatch):
    from sgb200 import kernels as K
    dev = _cuda()
    net = inception[0]
    img, quantize = _images_for(B, BATCHES[B])
    img = img.to(dev)
    rec = _Launches(K, B, monkeypatch)
    seen, names, (pool, logits) = _launched(lambda: net.forward(img, quantize=quantize))
    monkeypatch.undo()
    for t in rec.allocated:
        rec._clean(t, "tensor after the forward", "%s %s" % (tuple(t.shape), t.dtype))
    print("B=%d launches %s, worst %s" % (B, rec.counts, {k: "%.3f (%s)" % v for k, v in rec.worst.items()}))
    assert rec.counts == LAUNCHES
    assert not rec.faults, rec.faults[:10]
    assert set(rec.worst) == {"conv", "fc (fp32)", "avg pool", "sum_hw"}
    for part, (ratio, label) in rec.worst.items():
        assert ratio <= 1.0, (part, ratio, label)
    assert pool.shape == (B, 2048) and logits.shape == (B, 1008)
    if any("kernel" in n for n in names):
        assert ("fprop", -1) in seen and any(F_ >= 0 for _, F_ in seen), sorted(seen)
    else:
        warnings.warn("torch.profiler recorded no CUDA kernels: conv kernel identity not checked")


# ------------------------------------------------------------------------------------------------ 3. the whole forward
@pytest.mark.parametrize("B", list(BATCHES))
def test_inception_forward_at_fid50k_batch_vs_float64_torchvision(inception, B):
    dev = _cuda()
    net, onet = inception
    img, quantize = _images_for(B, BATCHES[B])
    pool, logits = net.forward(img.to(dev), quantize=quantize)
    x = O.eval_preprocess(img, 299, quantize)
    worst = {}
    for b0 in range(0, B, 32):
        op, ol = O.fid_inception_forward(onet, x[b0:b0 + 32].to(dev, torch.float64))
        for name, got, ref in (("pool", pool[b0:b0 + 32], op), ("logits", logits[b0:b0 + 32], ol)):
            e = ((got.double() - ref).norm(dim=1) / ref.norm(dim=1)).max()
            worst[name] = max(worst.get(name, 0.0), float(e))
    print("B=%d whole forward, worst relative L2 per image: %s (bound %.0e)" % (B, worst, WHOLE_L2))
    for name, e in worst.items():
        assert e <= WHOLE_L2, (name, e)


# ------------------------------------------------------------------------------------------------ 4. FID moments
def test_fid_moments_at_fid50k_n_vs_float64_two_pass():
    from sgb200.metrics import fid
    dev = _cuda()
    N, D = 50000, 2048
    g = torch.Generator(device=dev).manual_seed(11)
    std = 0.5 + torch.rand(D, generator=g, device=dev)
    shared = torch.randn(N, 32, generator=g, device=dev)          # 32 common factors: correlated dimensions
    z = 0.6 * torch.randn(N, D, generator=g, device=dev) + 0.8 * shared[:, torch.arange(D, device=dev) % 32]
    f = (std * (3.0 + z.clamp(min=-3.0))).float()                 # >= 0, mean ~3 std
    del shared, z
    acc = fid.MomentsAccumulator(D, dev)
    for s in range(0, N, 128):                                    # 390 batches of 128, then 80
        acc.update(f[s:s + 128])
    assert acc.n == N
    f64 = f.double()
    mu = f64.mean(0)
    fc = f64 - mu
    sigma = fc.t() @ fc / (N - 1)
    del f64, fc
    for name, (m, s) in (("accumulator", acc.finalize()), ("calculate_moments", fid.calculate_moments(f))):
        em = float(((m - mu).abs() / (1e-12 + 1e-12 * mu.abs())).max())
        es = float(((s - sigma).abs() / (1e-10 + 1e-9 * sigma.abs())).max())
        print("moments N=%d (%s): mu %.3g, sigma %.3g of the bound" % (N, name, em, es))
        assert em <= 1.0 and es <= 1.0, name
