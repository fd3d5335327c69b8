"""Batch-norm, spectral-norm and streaming kernels at the shapes the benchmark configurations run (pytest -m gpu).

The conv kernels are tested at bench shapes in test_gpu_shapes.py / test_gpu_rows_epilogue.py.  This file does the same
for the other kernels of a training step: bn.cu (statistics, finalize, apply, backward, gradient-penalty tangent), sn.cu
(batched power iteration, weight packs, batched chain rule) and the ew.cu kernels around them.  Sizes are chosen to
reach the branches the small tests never take: one pixel row per block at C >= 2048, two kChunkC channel chunks,
grid.y = B = 128 with small pixel chunks, several tangent channel groups (blockIdx.y > 0), the pseudo-tile pack of
4x4 filters, the unstaged spectral-norm backward (taps * Cin_p > 8192) and a layer with more power-iteration tiles
than the 4096-block grid.

References: plain float64 torch on the same bf16 / fp32 operands the kernel reads, computed on the GPU and chunked over
channels so that no temporary is much larger than one activation.  Nothing here calls the library for a reference.

Tolerances (bf16 has an 8-bit significand: one round-to-nearest changes a value by at most 2^-8 of itself):
* bit-exact where the kernel is a fixed sequence of fp32 operations on bf16 / fp32 values that torch can replay in the same
  order: ReLU, max, layouts, casts, zero-stuffing, the replicated x2 upsample, the spectral-norm weight packs, an in-place
  call against the same call out of place.
* "one bf16 rounding": |got - ref| <= 2^-8 |ref| + atol per element, where atol covers the fp32 error of what the kernel
  computes before rounding (stated per test; these atol values are estimates, not measurements).
* fp32 accumulation: max-norm error relative to the largest reference element (``rel``), and relative L2 (``l2``).
  Batch norm: mean within 1e-5 (|mean| + std), rstd 1e-4 relative (estimate for fp32 sums over up to 2 M pixels per
  channel), y one rounding + 2e-4 absolute, dx max-norm 4e-3 (one output rounding, 2^-9 of the largest element, plus fp32
  terms) and L2 2e-3, per-image / per-channel gain and bias gradients 1e-4 (fp32 sums, no output rounding).
  Large-mean statistics (|mean| / std up to 16, 4 M pixels per channel): bn_stats forms var = E[x^2] - mean^2 in fp32,
  so the cancellation scales its error by (mean / std)^2; rstd 1e-3 relative (an estimate, not a measurement).
  Tangent kernels: dx max-norm 8e-3 / L2 4e-3 (a sum of three products of fp32 channel sums, one output rounding),
  da 4e-3 / 2e-3 (one rounding), dgamma 2e-4 (fp32 sums, a [C] torch expression).
  Spectral norm: u, v 1e-4 max-norm, sigma 1e-5 relative (fp32 dot products of up to 16384 terms: ~1e-6 expected);
  the eval-mode sigma = u . W v of a stale u, v cancels, so its 1e-5 is relative to |W v|; chain rule dW 1e-5 of
  max |dW_before| + max |G| / sigma (three fp32 roundings per element plus an fp32 <G, W> sum whose terms cancel).
"""
import copy
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import studiogan_oracle as O
from test_gpu_parity import bfr, rel_err

pytestmark = pytest.mark.gpu

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pytorch-studiogan_b200")
BF16_REL = 2.0 ** -8
bf16 = torch.bfloat16


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


class _Err:
    """Max-norm and L2 error of a kernel output against a float64 reference, accumulated over chunks on the device."""

    def __init__(self):
        self.dmax = self.rmax = self.d2 = self.r2 = 0.0

    def add(self, got, ref):
        d = got.double() - ref
        self.dmax = max(self.dmax, float(d.abs().max()))
        self.rmax = max(self.rmax, float(ref.abs().max()))
        self.d2 += float((d * d).sum())
        self.r2 += float((ref * ref).sum())

    @property
    def rel(self):
        return self.dmax / (self.rmax + 1e-30)

    @property
    def l2(self):
        return self.d2 ** 0.5 / (self.r2 ** 0.5 + 1e-30)


def _rounding_ratio(got, ref, atol):
    """max |got - ref| / (2^-8 |ref| + atol): <= 1 means at most one bf16 rounding (plus atol) per element."""
    return float(((got.double() - ref).abs() / (BF16_REL * ref.abs() + atol)).max())


def _act(gen, B, C, H, W, dev, mean=None, std=None, cpad=0):
    """bf16 activation [B, C, H, W], NHWC in memory with channel stride C + cpad, drawn on the device as N(mean_c, std_c^2)."""
    t = torch.randn((B, H, W, C + cpad), generator=gen, device=dev)
    if std is not None:
        t[..., :C].mul_(std)
    if mean is not None:
        t[..., :C].add_(mean)
    return t.to(bf16).permute(0, 3, 1, 2)[:, :C]


def _chunk(C, per_channel, limit=1 << 25):
    return max(1, min(C, limit // max(per_channel, 1)))


# ------------------------------------------------------------------------------------------------ 1. batch norm
# id: (B, C, H, W, mode (0 cBN, 1 affine, 2 plain), relu, up2, extra)
BN_CASES = {
    "cbn_c2048_4x4_up2": (128, 2048, 4, 4, 0, True, True, {}),
    "cbn_c1024_8x8": (128, 1024, 8, 8, 0, True, False, {}),
    "cbn_c512_16x16_up2": (128, 512, 16, 16, 0, True, True, {}),
    "cbn_c256_32x32": (128, 256, 32, 32, 0, True, False, {}),
    "cbn_c256_64x64_up2": (64, 256, 64, 64, 0, True, True, {}),
    "cbn_c128_256x256": (32, 128, 256, 256, 0, True, False, {}),
    "affine_c64_128x128": (128, 64, 128, 128, 1, True, False, {}),         # BN discriminator of the WGAN-GP 128x128 config
    "cbn_c2560_4x4_two_chunks": (128, 2560, 4, 4, 0, True, False, {}),
    "plain_c8_128x128": (32, 8, 128, 128, 2, False, False, {}),
    "affine_c24_128x128": (32, 24, 128, 128, 1, True, False, {}),
    "cbn_channel_slice": (64, 200, 16, 16, 0, True, False, {"cpad": 56}),  # x = X[:, :200] of a 256-channel tensor
    "cbn_affine_ld_up2": (128, 512, 8, 8, 0, True, True, {"affine_ld": 1536}),
    "eval_cbn_c512_16x16": (128, 512, 16, 16, 0, True, False, {"eval": True}),
    "eval_affine_c256_32x32": (64, 256, 32, 32, 1, False, False, {"eval": True}),
    "clamp_eps_affine_c256_64x64": (64, 256, 64, 64, 1, True, False, {"clamp": True}),
}


@pytest.mark.parametrize("case", list(BN_CASES))
def test_bn_act_at_benchmark_shapes_vs_float64(case):
    """BNActFn forward / backward and the K.bn_stats / K.bn_finalize statistics against float64 batch norm.
    cBN gains are per image (1 + gain[b, c]); with affine_ld they are column slices of one wider [B, K] matrix, as
    snbatch.cbn_affine_all hands them over.  The reference ReLU mask is the kernel's own (y > 0, which is its fp32
    pre-activation > 0): an element with |z| ~ 1e-7 may fall on either side, and its whole gradient with it."""
    from sgb200 import autograd_ops as A
    from sgb200 import kernels as K
    B, C, H, W, mode, relu, up2, ex = BN_CASES[case]
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(11)
    train, clamp = not ex.get("eval", False), ex.get("clamp", False)
    eps = 0.5 if clamp else 1e-4
    if clamp:     # channel variances on both sides of eps = 0.5, none within 7 % of it
        std = torch.linspace(0.2, 2.0, C, device=dev)
        std = torch.where((std > 0.68) & (std < 0.74), std * 1.12, std)
    else:
        std = 0.5 + 1.5 * torch.rand(C, generator=gen, device=dev)
    mean = 0.3 * torch.randn(C, generator=gen, device=dev)
    x = _act(gen, B, C, H, W, dev, mean, std, ex.get("cpad", 0))
    Ho, Wo = (2 * H, 2 * W) if up2 else (H, W)
    dy = _act(gen, B, C, Ho, Wo, dev)
    aff = None
    if mode == 0:
        ld = ex.get("affine_ld")
        if ld:
            aff = (0.3 * torch.randn(B, ld, generator=gen, device=dev)).requires_grad_(True)
            gain, bias = aff[:, 256:256 + C], aff[:, ld - C:]
        else:
            gain = (0.3 * torch.randn(B, C, generator=gen, device=dev)).requires_grad_(True)
            bias = (0.3 * torch.randn(B, C, generator=gen, device=dev)).requires_grad_(True)
    elif mode == 1:
        gain = (0.5 + torch.rand(C, generator=gen, device=dev)).requires_grad_(True)
        bias = (0.3 * torch.randn(C, generator=gen, device=dev)).requires_grad_(True)
    else:
        gain = bias = None
    rm0 = 0.2 * torch.randn(C, generator=gen, device=dev)
    rv0 = 0.5 + torch.rand(C, generator=gen, device=dev)
    rm, rv = rm0.clone(), rv0.clone()
    cfg = {"mode": mode, "relu": relu, "up2": up2, "use_batch_stats": train, "track": True, "momentum": 0.1, "eps": eps, "group": None}
    if clamp:
        cfg["clamp_eps"] = True
    x.requires_grad_(True)
    y = A.BNActFn.apply(x, gain, bias, rm, rv, cfg)
    y.backward(dy)
    N = B * H * W
    ubs = (2 if clamp else 1) if train else 0
    stats = K.bn_stats(x.detach()) if train else None
    mean_k, rstd_k, _, _ = K.bn_finalize(stats, N, rm0.clone(), rv0.clone(), 0.1, eps, ubs, True, 2, None, None, 1, C, dev)
    if mode == 0:
        gsrc = aff.grad[:, 256:256 + C] if aff is not None else gain.grad
        bsrc = aff.grad[:, ex["affine_ld"] - C:] if aff is not None else bias.grad
    elif mode == 1:
        gsrc, bsrc = gain.grad, bias.grad
    e_dx, e_dg, e_db = _Err(), _Err(), _Err()
    worst_y = worst_mean = worst_rstd = worst_rm = worst_rv = 0.0
    cc = _chunk(C, B * Ho * Wo)
    for c0 in range(0, C, cc):
        sl = slice(c0, min(C, c0 + cc))
        xc = x.detach()[:, sl].double()
        if train:
            mu, var = xc.mean((0, 2, 3)), xc.var((0, 2, 3), unbiased=False)
            rs = (var.clamp(min=eps) if clamp else var + eps).rsqrt()
            scale_ref = (mu.abs() + var.sqrt())
            worst_mean = max(worst_mean, float(((mean_k[sl].double() - mu).abs() / scale_ref).max()))
            rm_ref, rv_ref = 0.9 * rm0[sl].double() + 0.1 * mu, 0.9 * rv0[sl].double() + 0.1 * var * N / (N - 1)
            worst_rm = max(worst_rm, float(((rm[sl].double() - rm_ref).abs() / (scale_ref + rm_ref.abs())).max()))
            worst_rv = max(worst_rv, float(((rv[sl].double() - rv_ref).abs() / rv_ref).max()))
        else:
            mu, var = rm0[sl].double(), rv0[sl].double()
            rs = (var + eps).rsqrt()
            assert torch.equal(mean_k[sl], rm0[sl]) and torch.equal(rm[sl], rm0[sl]) and torch.equal(rv[sl], rv0[sl])
        worst_rstd = max(worst_rstd, float(((rstd_k[sl].double() - rs).abs() / rs).max()))
        bc = lambda t: t[:, None, None]      # noqa: E731  [c] -> [c, 1, 1]
        xh = (xc - bc(mu)) * bc(rs)
        if mode == 0:
            g, be = 1 + gain.detach()[:, sl].double()[:, :, None, None], bias.detach()[:, sl].double()[:, :, None, None]
        elif mode == 1:
            g, be = bc(gain.detach()[sl].double()), bc(bias.detach()[sl].double())
        else:
            g, be = 1.0, 0.0
        z = xh * g + be
        yref = z.clamp(min=0) if relu else z
        yk = y.detach()[:, sl]
        if up2:
            for i, j in ((0, 1), (1, 0), (1, 1)):
                assert torch.equal(yk[..., i::2, j::2], yk[..., ::2, ::2])
            yk = yk[..., ::2, ::2]
        worst_y = max(worst_y, _rounding_ratio(yk, yref, 2e-4))
        dz = dy[:, sl].double()
        if up2:
            dz = dz.reshape(B, -1, H, 2, W, 2).sum((3, 5))
        d = dz * (yk > 0) if relu else dz
        dxh = d * g
        if train:
            m1, m2 = dxh.mean((0, 2, 3), keepdim=True), (dxh * xh).mean((0, 2, 3), keepdim=True)
            if clamp:       # clamped channels: inv_std is a constant, the variance term vanishes
                m2 = m2 * (var >= eps).double().view(1, -1, 1, 1)
            dxr = bc(rs) * (dxh - m1 - xh * m2)
        else:
            dxr = bc(rs) * dxh
        e_dx.add(x.grad[:, sl], dxr)
        if mode in (0, 1):
            db, dg = d.sum((2, 3)), (d * xh).sum((2, 3))
            if mode == 1:
                db, dg = db.sum(0), dg.sum(0)
            e_dg.add(gsrc[..., sl], dg)
            e_db.add(bsrc[..., sl], db)
    print("%s: y %.3g (<= 1) mean %.3g rstd %.3g rm %.3g rv %.3g dx %.3g/%.3g dgain %.3g/%.3g dbias %.3g/%.3g" % (
        case, worst_y, worst_mean, worst_rstd, worst_rm, worst_rv, e_dx.rel, e_dx.l2, e_dg.rel, e_dg.l2, e_db.rel, e_db.l2))
    assert worst_y <= 1.0
    assert worst_mean <= 1e-5 and worst_rm <= 1e-5
    assert worst_rstd <= (1e-4 if train else 1e-6) and worst_rv <= 2e-4
    assert e_dx.rel <= 4e-3 and e_dx.l2 <= 2e-3
    if mode in (0, 1):
        assert e_dg.rel <= 1e-4 and e_dg.l2 <= 1e-4
        assert e_db.rel <= 1e-4 and e_db.l2 <= 1e-4
    if aff is not None:       # columns of the wider matrix that are neither gain nor bias get no gradient
        ld = ex["affine_ld"]
        assert float(aff.grad[:, :256].abs().max()) == 0.0 and float(aff.grad[:, 256 + C:ld - C].abs().max()) == 0.0


def test_bn_stats_large_mean_to_std_ratio():
    """Per-channel |mean| / std from 0 to 16 at 4 M pixels per channel (B=64, C=64, 256x256).  bn_stats accumulates sum
    and sum of squares in fp32 and bn_finalize forms var = E[x^2] - mean^2: the relative error of E[x^2] is multiplied
    by (1 + (mean / std)^2) = 257 at the top of the range."""
    from sgb200 import kernels as K
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(12)
    B, C, H, W = 64, 64, 256, 256
    std = 0.5 + 1.5 * torch.rand(C, generator=gen, device=dev)
    mean = 16.0 * torch.linspace(-1.0, 1.0, C, device=dev) * std
    x = _act(gen, B, C, H, W, dev, mean, std)
    N = B * H * W
    rm0, rv0 = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    rm, rv = rm0.clone(), rv0.clone()
    mean_k, rstd_k, _, _ = K.bn_finalize(K.bn_stats(x), N, rm, rv, 0.1, 1e-4, 1, True, 2, None, None, 1, C, dev)
    worst_mean = worst_rstd = worst_rv = 0.0
    cc = _chunk(C, N)
    for c0 in range(0, C, cc):
        sl = slice(c0, min(C, c0 + cc))
        xc = x[:, sl].double()
        mu, var = xc.mean((0, 2, 3)), xc.var((0, 2, 3), unbiased=False)
        worst_mean = max(worst_mean, float(((mean_k[sl].double() - mu).abs() / (mu.abs() + var.sqrt())).max()))
        worst_rstd = max(worst_rstd, float(((rstd_k[sl].double() * (var + 1e-4).sqrt()) - 1).abs().max()))
        rv_ref = 0.9 + 0.1 * var * N / (N - 1)
        worst_rv = max(worst_rv, float(((rv[sl].double() - rv_ref).abs() / rv_ref).max()))
    print("large mean: mean %.3g rstd %.3g running var %.3g" % (worst_mean, worst_rstd, worst_rv))
    assert worst_mean <= 1e-5
    assert worst_rstd <= 1e-3 and worst_rv <= 2e-3


# ------------------------------------------------------------------------------------------------ 2. BN tangent kernels
@pytest.mark.parametrize("B,C,H,W", [(128, 512, 16, 16), (128, 512, 8, 8), (128, 1024, 16, 16), (128, 1024, 8, 8),
                                     (64, 264, 16, 16)])       # 264 = 33 channel groups: a partial last blockIdx.y group
def test_bn_tangent_backward_at_discriminator_shapes_vs_float64(B, C, H, W):
    """BNTangentFn (bn_bwd_reduce / bn_bwd_apply forward, bn_tangent_bwd_reduce / bn_tangent_bwd_apply backward) against
    the oracle's closed forms in float64.  The tangent a and the cotangent c are correlated with x and with each other, so
    that every one of the five channel sums is far from zero."""
    from sgb200 import autograd_ops as A
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(13)
    eps = 1e-4
    std = 0.5 + 1.5 * torch.rand(C, generator=gen, device=dev)
    mean = 0.3 * torch.randn(C, generator=gen, device=dev)
    x = _act(gen, B, C, H, W, dev, mean, std)
    xf = x.float()
    a = (torch.randn(xf.shape, generator=gen, device=dev).to(memory_format=torch.channels_last) + 0.5 * xf + 0.2).to(bf16)
    c = (torch.randn(xf.shape, generator=gen, device=dev).to(memory_format=torch.channels_last) + 0.3 * a.float() + 0.1).to(bf16)
    del xf
    gamma = 0.5 + torch.rand(C, generator=gen, device=dev)
    x64 = x.double()
    mu, var = x64.mean((0, 2, 3)), x64.var((0, 2, 3), unbiased=False)
    del x64
    mean32, rstd32 = mu.float(), (var + eps).rsqrt().float()
    cfg = {"count": float(B * H * W), "use_batch_stats": True, "group": None}
    xd, ad, gd = x.detach().requires_grad_(True), a.detach().requires_grad_(True), gamma.clone().requires_grad_(True)
    t = A.BNTangentFn.apply(xd, ad, gd, mean32, rstd32, cfg)
    t.backward(c)
    e_t, e_dx, e_da, e_dg = _Err(), _Err(), _Err(), _Err()
    cc = _chunk(C, B * H * W, 1 << 24)
    for c0 in range(0, C, cc):
        sl = slice(c0, min(C, c0 + cc))
        xs, as_, cs, gs = x[:, sl].double(), a[:, sl].double(), c[:, sl].double(), gamma[sl].double()
        e_t.add(t.detach()[:, sl], O.bn_tangent(xs, as_, gs, eps))
        dx, da, dgamma = O.bn_tangent_backward(xs, as_, cs, gs, eps)
        e_dx.add(xd.grad[:, sl], dx)
        e_da.add(ad.grad[:, sl], da)
        e_dg.add(gd.grad[sl], dgamma)
    print("tangent B%d C%d %dx%d: t %.3g/%.3g dx %.3g/%.3g da %.3g/%.3g dgamma %.3g" % (
        B, C, H, W, e_t.rel, e_t.l2, e_dx.rel, e_dx.l2, e_da.rel, e_da.l2, e_dg.rel))
    assert e_t.rel <= 4e-3 and e_t.l2 <= 2e-3
    assert e_dx.rel <= 8e-3 and e_dx.l2 <= 4e-3
    assert e_da.rel <= 4e-3 and e_da.l2 <= 2e-3
    assert e_dg.rel <= 2e-4


# ------------------------------------------------------------------------------------------------ 3. spectral norm
def _geom(m):
    from sgb200.utils import ops
    W = ops._w(m).detach()
    Cout = W.shape[0]
    taps = W.shape[2] * W.shape[3] if W.dim() == 4 else 1
    Cin = W.numel() // (Cout * taps)
    return W.reshape(Cout, Cin, taps), Cout, Cin, taps, getattr(m, "_perm_S", 1)


def _pack_rows(Cout, S, dev):
    """Packed row of each output channel: perm_S > 1 (linear0) stores row c*S + s at s*C + c."""
    co = torch.arange(Cout, device=dev)
    return (co % S) * (Cout // S) + co // S if S > 1 else co


def _check_packs(wf, wd, W3, S, sigma):
    """Both packs must be bf16(W * (1 / sigma)) bit for bit ((1 / sigma) in fp32), zero-padded."""
    from sgb200 import kernels as K
    Cout, Cin, taps = W3.shape
    inv = (torch.ones(1) / sigma.detach().float().cpu()).to(W3.device) if sigma is not None else torch.ones(1, device=W3.device)
    Wb = (W3 * inv).to(bf16)
    rows = _pack_rows(Cout, S, W3.device)
    ef = torch.zeros((K.pad8(Cout), taps, K.pad8(Cin)), device=W3.device, dtype=bf16)
    ef[rows, :, :Cin] = Wb.permute(0, 2, 1)
    assert torch.equal(wf, ef)
    if wd is not None:
        ed = torch.zeros((K.pad8(Cin), taps, K.pad8(Cout)), device=W3.device, dtype=bf16)
        ed[:Cin, :, rows] = Wb.permute(1, 2, 0).flip(1)
        assert torch.equal(wd, ed)


def _sn_forward_checks(net, label):
    """Eval call (sigma = u . W v, no update), then two train calls, each against float64 from the state before it."""
    from sgb200.utils import ops
    snb = net._snb
    net.eval()
    with torch.no_grad():
        snb.run()
    mods = snb.mods
    worst = {"u": 0.0, "v": 0.0, "sigma": 0.0, "sigma_eval": 0.0}
    state = [(m.weight_u.clone(), m.weight_v.clone()) if hasattr(m, "_sn") else None for m in mods]
    for m, st in zip(mods, state):
        W3, Cout, Cin, taps, S = _geom(m)
        sig = m._sn_cache[2]
        if st is not None:     # u . s with u, s far from aligned cancels: the bound is relative to |u| |s| = |s|
            s = W3.reshape(Cout, -1).double() @ st[1].double()
            worst["sigma_eval"] = max(worst["sigma_eval"], abs(float(sig) - float(st[0].double() @ s)) / float(s.norm()))
        _check_packs(m._sn_cache[0], m._sn_cache[1], W3, S, sig)
    net.train()
    for call in range(2):
        with torch.enable_grad():
            snb.run()
        for m, st in zip(mods, state):
            W3, Cout, Cin, taps, S = _geom(m)
            sig = m._sn_cache[2]
            _check_packs(m._sn_cache[0], m._sn_cache[1], W3, S, sig)
            if st is None:
                assert sig is None
                continue
            Wm = W3.reshape(Cout, -1).double()
            v = F.normalize(Wm.t() @ st[0].double(), dim=0, eps=ops.SN_EPS)
            s = Wm @ v
            u = F.normalize(s, dim=0, eps=ops.SN_EPS)
            worst["u"] = max(worst["u"], rel_err(m.weight_u, u))
            worst["v"] = max(worst["v"], rel_err(m.weight_v, v))
            worst["sigma"] = max(worst["sigma"], abs(float(sig) - float(u @ s)) / float(u @ s))
        state = [(m.weight_u.clone(), m.weight_v.clone()) if hasattr(m, "_sn") else None for m in mods]
    print("%s forward (%d layers): %s" % (label, len(mods), worst))
    assert worst["u"] <= 1e-4 and worst["v"] <= 1e-4
    assert worst["sigma"] <= 1e-5 and worst["sigma_eval"] <= 1e-5


def _sn_backward_checks(net, label, per_layer):
    """sgb_sn_backward_batch (through the pass's flush) on every layer: dW += (G - <G, W/sigma> u v^T) / sigma, with G
    in the fprop-pack layout holding a rank-one part along u v^T (so that the <G, W/sigma> term is not negligible) and
    noise in its padding (which the kernel must not read).  Then per-layer K.sn_backward on the layers in ``per_layer``."""
    from sgb200 import kernels as K
    snb = net._snb
    dev = next(net.parameters()).device
    gen = torch.Generator(device=dev).manual_seed(14)
    net.train()
    with torch.enable_grad():
        snb.run()
    cur = snb.mods[0]._sn_pass[0]
    assert snb.bwd_table() is not None
    for p in snb.params:
        p.grad.copy_(torch.randn(p.shape, generator=gen, device=dev))     # the kernel accumulates: start from non-zero
    dW0 = [p.grad.clone() for p in snb.params]
    g_flat = torch.randn(snb.total_f, generator=gen, device=dev)
    Gs = []
    for i, m in enumerate(snb.mods):
        W3, Cout, Cin, taps, S = _geom(m)
        of, _, nf, shf, _, su, sv = snb.slices[i]
        G = torch.randn((Cout, Cin, taps), generator=gen, device=dev)
        if su is not None:
            G += 2.0 * (Cout * Cin * taps) ** 0.5 * torch.outer(cur.us[su[0]:su[1]], cur.vs[sv[0]:sv[1]]).view(Cout, Cin, taps)
        g_flat[of:of + nf].view(shf)[_pack_rows(Cout, S, dev), :, :Cin] = G.permute(0, 2, 1)
        Gs.append(G)
    cur.g_flat = g_flat
    cur.flush()
    worst, worst_single = 0.0, 0.0

    def ref_delta(i, m, W3, G):
        """(G - <G, W/sigma> u v^T) / sigma in float64, and max |G| / sigma: the rank-one part of G cancels in the result,
        so errors are measured against the size of the terms, not of the difference."""
        su, sv = snb.slices[i][5], snb.slices[i][6]
        if su is None:
            return G.double(), float(G.abs().max())
        s = float(cur.sigma[i])
        uv = torch.outer(cur.us[su[0]:su[1]].double(), cur.vs[sv[0]:sv[1]].double()).view(G.shape)
        return (G.double() - float((G.double() * W3.double()).sum()) / s * uv) / s, float(G.abs().max()) / s

    for i, (m, p, G) in enumerate(zip(snb.mods, snb.params, Gs)):
        W3 = _geom(m)[0]
        delta, size = ref_delta(i, m, W3, G)
        ref = dW0[i].reshape(W3.shape).double() + delta
        e = float((p.grad.reshape(W3.shape).double() - ref).abs().max()) / (size + float(dW0[i].abs().max()))
        worst = max(worst, e)
    for i in per_layer:
        m = snb.mods[i]
        W3, Cout, Cin, taps, S = _geom(m)
        of, _, nf, shf, _, su, sv = snb.slices[i]
        has = su is not None
        dW = K.sn_backward(g_flat[of:of + nf].view(shf), W3, cur.us[su[0]:su[1]] if has else None, cur.vs[sv[0]:sv[1]] if has else None,
                           cur.sigma[i:i + 1] if has else None, Cout, Cin, taps, S)
        ref, size = ref_delta(i, m, W3, Gs[i])
        worst_single = max(worst_single, float((dW.reshape(W3.shape).double() - ref).abs().max()) / size)
    print("%s chain rule: batched %.3g, per-layer %.3g" % (label, worst, worst_single))
    assert worst <= 1e-5 and worst_single <= 1e-5


def _one_iteration(W3, u0):
    """float64 power iteration from u0: (u, v, sigma)."""
    from sgb200.utils import ops
    Wm = W3.reshape(W3.shape[0], -1).double()
    v = F.normalize(Wm.t() @ u0.double(), dim=0, eps=ops.SN_EPS)
    s = Wm @ v
    u = F.normalize(s, dim=0, eps=ops.SN_EPS)
    return u, v, float(u @ s)


def _sn_per_layer_checks(net, label):
    """The per-layer entry points on every layer: K.sn_power_iter from a fresh workspace, called twice (its tickets and
    accumulator must reset), each call against float64 from the state before it; then both K.weight_pack packs."""
    from sgb200 import kernels as K
    from sgb200.utils import ops
    worst = {"u": 0.0, "v": 0.0, "sigma": 0.0}
    for m in net._snb.mods:
        W3, Cout, Cin, taps, S = _geom(m)
        W = ops._w(m).detach()
        sigma = None
        if hasattr(m, "_sn"):
            u, v = m.weight_u.clone(), m.weight_v.clone()
            ws = K.sn_workspace(Cout, Cin * taps, W.device)
            sigma = torch.empty(1, device=W.device)
            for call in range(2):
                u_ref, v_ref, s_ref = _one_iteration(W3, u)
                K.sn_power_iter(W, u, v, sigma, ws, ops.SN_EPS, True)
                worst["u"] = max(worst["u"], rel_err(u, u_ref))
                worst["v"] = max(worst["v"], rel_err(v, v_ref))
                worst["sigma"] = max(worst["sigma"], abs(float(sigma) - s_ref) / s_ref)
        wf, wd = K.weight_pack(W, sigma, Cout, Cin, taps, True, True, S)
        _check_packs(wf, wd, W3, S, sigma)
    print("%s per-layer power iteration: %s" % (label, worst))
    assert worst["u"] <= 1e-4 and worst["v"] <= 1e-4 and worst["sigma"] <= 1e-5


def _flagship_nets(dev):
    """Generator and discriminator of configs/BigGAN-Deep-256res.yaml (without the EMA copy), and the configuration."""
    from sgb200 import config as C
    from sgb200.models import model as M
    cfgs = C.Configurations(os.path.join(PKG, "configs", "BigGAN-Deep-256res.yaml"))
    MODEL = copy.copy(cfgs.MODEL)
    MODEL.apply_g_ema = False
    torch.manual_seed(0)
    G, _, _, D, _, _, _, _ = M.load_generator_discriminator(cfgs.DATA, cfgs.OPTIMIZATION, MODEL, cfgs.STYLEGAN, cfgs.MODULES,
                                                           cfgs.RUN, dev, None)
    return G, D, cfgs


def _attach_arena(net):
    from sgb200.utils.optim import ArenaAdam
    opt = ArenaAdam(net, lr=2e-4, betas=(0.0, 0.999), eps=1e-6)
    opt.zero_grad()
    return opt


def test_spectral_norm_every_flagship_layer_vs_float64():
    """BigGAN-Deep 256x256 (configs/BigGAN-Deep-256res.yaml, conv_dim 128, 1000 classes, depth 2, attention): all 150
    generator and 56 discriminator layers of the batched spectral norm -- u, v, sigma, both weight packs (including the
    perm_S = 16 row order of linear0), a second call (tickets and workspace reset), an eval call, and the batched
    chain rule."""
    dev = _cuda()
    G, D, _ = _flagship_nets(dev)
    for net, label, n in ((G, "G", 150), (D, "D", 56)):
        _attach_arena(net)
        _sn_forward_checks(net, label)
        mods = net._snb.mods
        assert len(mods) == n
        perm = [i for i, m in enumerate(mods) if getattr(m, "_perm_S", 1) > 1]
        assert label == "D" or perm            # linear0 of the generator
        pick = sorted(set([0, len(mods) // 2, len(mods) - 1] + perm + [i for i, m in enumerate(mods) if _geom(m)[3] == 9][:1]))
        _sn_backward_checks(net, label, pick)
        net._snb.clear()


def test_no_grad_attention_generator_iterates_each_layer_once():
    """A gradient-free forward of the flagship generator in evaluation mode as misc.make_GAN_untrainable sets it (eval(),
    then the convs / linears back in train mode so that the power iteration runs, as in the reference): FID / IS / PRDC
    sampling and standing statistics.  The attention convs must take one power iteration per forward like every other
    layer.  Their weights are re-drawn from N(0, 1): for the orthogonal initialisation u is a fixed point of the iteration,
    and a second iteration would not show."""
    from sgb200.utils import misc, ops
    dev = _cuda()
    G, _, cfgs = _flagship_nets(dev)
    G.eval()
    G.apply(misc.set_deterministic_op_trainable)
    attn = [c for sa in G.modules() if isinstance(sa, ops.SelfAttention)
            for c in (sa.conv1x1_theta, sa.conv1x1_phi, sa.conv1x1_g, sa.conv1x1_attn)]
    assert attn and all(hasattr(c, "_sn") for c in attn)
    gen = torch.Generator(device=dev).manual_seed(15)
    with torch.no_grad():
        for c in attn:
            ops._w(c).copy_(torch.randn(ops._w(c).shape, generator=gen, device=dev))
    before = [(_geom(c)[0], c.weight_u.clone()) for c in attn]
    z = torch.randn((2, cfgs.MODEL.z_dim), generator=gen, device=dev)
    y = torch.randint(0, cfgs.DATA.num_classes, (2,), generator=gen, device=dev)
    with torch.no_grad():
        G(z, y, eval=True)
    worst = {"u": 0.0, "v": 0.0}
    for c, (W3, u0) in zip(attn, before):
        u_ref, v_ref, _ = _one_iteration(W3, u0)
        worst["u"] = max(worst["u"], rel_err(c.weight_u, u_ref))
        worst["v"] = max(worst["v"], rel_err(c.weight_v, v_ref))
    print("no-grad attention generator (%d convs): %s" % (len(attn), worst))
    assert worst["u"] <= 1e-4 and worst["v"] <= 1e-4


class _EdgeLayers(nn.Module):
    def __init__(self):
        from sgb200.snbatch import SNBatch
        from sgb200.utils import ops
        super().__init__()
        self.c4 = ops.snconv2d(40, 72, 4, 2, 1)          # 4x4 (DCGAN down-sampling conv): 16 taps, pseudo-tile packs
        self.odd = ops.snconv2d(13, 29, 3, 1, 1)         # Cin, Cout not multiples of 8 or 32: padded packs
        self.odd1 = ops.snconv2d(100, 45, 1)
        self.wide = ops.snconv2d(1040, 24, 3, 1, 1)      # taps * Cin_p = 9360 > 8192: unstaged chain rule
        self.plain = ops.conv2d(64, 40, 3, 1, 1)         # no spectral norm: sigma = 1 packing, G passed through
        self.perm = ops.snlinear(20, 48)
        self.perm._perm_S = 16
        self.big = ops.snlinear(16384, 4160)             # 64 x 65 = 4160 power-iteration tiles > the 4096-block grid
        self._snb = SNBatch(self)


def test_spectral_norm_edge_layers_vs_float64():
    """Layers the flagship does not have: pseudo tiles, odd channel counts, the unstaged backward, a layer without
    spectral norm and a layer with more Wt.u tiles than blocks in the batched power iteration; batched and per-layer."""
    dev = _cuda()
    torch.manual_seed(5)
    net = _EdgeLayers().to(dev)
    _attach_arena(net)
    _sn_forward_checks(net, "edge")
    _sn_per_layer_checks(net, "edge")
    _sn_backward_checks(net, "edge", list(range(len(net._snb.mods))))
    net._snb.clear()


# ------------------------------------------------------------------------------------------------ 4. streaming kernels
@pytest.mark.parametrize("B,C,H,W,cpad", [(128, 256, 64, 64, 0), (3, 24, 6, 10, 8)])
def test_relu_pool2_bit_exact(B, C, H, W, cpad):
    from sgb200 import kernels as K
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(21)
    x = _act(gen, B, C, H, W, dev, cpad=cpad)
    a0, y = K.relu_pool2(x)
    r = x.float().clamp(min=0)
    assert torch.equal(a0, r.to(bf16))
    ref = 0.25 * (((r[..., 0::2, 0::2] + r[..., 0::2, 1::2]) + r[..., 1::2, 0::2]) + r[..., 1::2, 1::2])
    assert torch.equal(y, ref.to(bf16))


@pytest.mark.parametrize("rows,n", [(65536, 1024), (37, 72)])
def test_softmax_bwd_rows_vs_float64_and_in_place(rows, n):
    """ds = p * (dp - <p, dp>) per row: fp32 dot, one output rounding (atol 1e-6 max|ds| for the fp32 dot);
    the in-place call (ds = dp) must equal the out-of-place one bit for bit."""
    from sgb200 import kernels as K
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(22)
    p = torch.softmax(3 * torch.randn((rows, n), generator=gen, device=dev), -1).to(bf16)
    dp = torch.randn((rows, n), generator=gen, device=dev).to(bf16)
    ds = K.softmax_bwd_rows(p, dp, n)
    p64, dp64 = p.double(), dp.double()
    ref = p64 * (dp64 - (p64 * dp64).sum(-1, keepdim=True))
    r = _rounding_ratio(ds, ref, 1e-6 * float(ref.abs().max()))
    print("softmax_bwd_rows %dx%d: %.3g" % (rows, n, r))
    assert r <= 1.0
    K.softmax_bwd_rows(p, dp, n, out=dp)
    assert torch.equal(dp, ds)


@pytest.mark.parametrize("B,C,H,W,relu,cpad", [(128, 2048, 4, 4, True, 0), (3, 40, 5, 7, False, 24)])
def test_sum_hw_and_backward(B, C, H, W, relu, cpad):
    """sum_hw: fp32 sum of H*W values (1e-6 of the sum of magnitudes); sum_hw_bwd: bit-exact broadcast with the ReLU mask."""
    from sgb200 import kernels as K
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(23)
    x = _act(gen, B, C, H, W, dev, cpad=cpad)
    h = K.sum_hw(x, relu)
    xr = x.double().clamp(min=0) if relu else x.double()
    assert float(((h.double() - xr.sum((2, 3))).abs() / (xr.abs().sum((2, 3)) + 1e-30)).max()) <= 1e-6
    dh = torch.randn((B, C), generator=gen, device=dev)
    dx = K.sum_hw_bwd(dh, x, relu)
    ref = dh[:, :, None, None].expand(B, C, H, W)
    if relu:
        ref = torch.where(x.float() > 0, ref, torch.zeros_like(ref))
    assert torch.equal(dx, ref.to(bf16))


@pytest.mark.parametrize("n", [128 * 3 * 256 * 256, 296])
def test_dot_vs_float64(n):
    from sgb200 import kernels as K
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(24)
    x = torch.randn(n, generator=gen, device=dev).to(bf16)
    y = (torch.randn(n, generator=gen, device=dev) + 0.1).to(bf16)
    got = float(K.dot(x, y))
    p = x.double() * y.double()
    assert abs(got - float(p.sum())) <= 1e-6 * float(p.abs().sum())


@pytest.mark.parametrize("B,C,H,W,Cp", [(128, 3, 256, 256, 8), (2, 3, 5, 7, 16)])
def test_img_grad_to_nhwc(B, C, H, W, Cp):
    """Without tanh a bit-exact re-layout; with it d * (1 - y^2) with one output rounding (atol 1e-6: 1 - y^2 in fp32 loses
    up to 6e-8 absolute where |y| -> 1, times |d| <= 16)."""
    from sgb200 import kernels as K
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(25)
    d = torch.randn((B, C, H, W), generator=gen, device=dev)
    yt = torch.tanh(2 * torch.randn((B, C, H, W), generator=gen, device=dev))
    out = K.img_grad_to_nhwc(d, None, Cp)
    assert out.shape == (B, Cp, H, W) and torch.equal(out[:, :C], d.to(bf16)) and float(out[:, C:].abs().max()) == 0.0
    out = K.img_grad_to_nhwc(d, yt, Cp)
    assert float(out[:, C:].abs().max()) == 0.0
    assert _rounding_ratio(out[:, :C], d.double() * (1 - yt.double() ** 2), 1e-6) <= 1.0


def _col27_ref(xb):
    """[B, 3, H, W] (bf16 values, float64) -> [B, 32, H, W]: channel t*3 + c = x[c] shifted by tap t, 27..31 zero."""
    B, _, H, W = xb.shape
    u = F.unfold(xb, 3, padding=1).view(B, 3, 9, H, W).permute(0, 2, 1, 3, 4).reshape(B, 27, H, W)
    return torch.cat([u, torch.zeros((B, 5, H, W), device=xb.device, dtype=xb.dtype)], 1)


@pytest.mark.parametrize("B,H,W", [(32, 256, 256), (2, 5, 7)])
def test_col27_and_adjoint(B, H, W):
    """col27 from NCHW fp32 and from a channel-strided NHWC bf16 activation: bit-exact gather.  col27_bwd: fp32 sum of
    nine bf16 values (1e-6 of the sum of magnitudes); <col27(x), y> = <x, col27_bwd(y)> to the same bound."""
    from sgb200 import kernels as K
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(26)
    img = torch.rand((B, 3, H, W), generator=gen, device=dev) * 2 - 1
    xb = bfr(img).double()
    ref = _col27_ref(xb)
    assert torch.equal(K.col27(img).double(), ref)
    act = _act(gen, B, 3, H, W, dev, cpad=13)          # channel stride 16
    assert torch.equal(K.col27(act).double(), _col27_ref(act.double()))
    dcol = K.empty_nhwc(B, 32, H, W, dev)
    dcol.copy_(torch.randn((B, 32, H, W), generator=gen, device=dev))
    dimg = K.col27_bwd(dcol)
    fold = lambda t: F.fold(t[:, :27].reshape(B, 9, 3, H * W).permute(0, 2, 1, 3).reshape(B, 27, H * W), (H, W), 3, padding=1)   # noqa: E731
    dref, dabs = fold(dcol.double()), fold(dcol.double().abs())
    assert float(((dimg.double() - dref).abs() - 1e-6 * dabs).max()) <= 0.0
    lhs = float((ref * dcol.double()).sum())
    rhs = float((xb * dimg.double()).sum())
    assert abs(lhs - rhs) <= 1e-6 * float((xb.abs() * dabs).sum())


@pytest.mark.parametrize("B,C,H,W,cpad", [(64, 128, 64, 64, 0), (2, 24, 3, 5, 8)])
def test_zero_stuff2_bit_exact(B, C, H, W, cpad):
    from sgb200 import kernels as K
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(27)
    x = _act(gen, B, C, H, W, dev, cpad=cpad)
    y = K.zero_stuff2(x)
    ref = torch.zeros((B, C, 2 * H, 2 * W), device=dev, dtype=bf16)
    ref[..., ::2, ::2] = x
    assert torch.equal(y, ref)


@pytest.mark.parametrize("n", [50_000_003, 5])
def test_casts_bit_exact(n):
    from sgb200 import kernels as K
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(28)
    x = torch.randn(n, generator=gen, device=dev) * 3
    s = torch.tensor(0.37, dtype=torch.float32)
    assert torch.equal(K.cast_f32_to_bf16(x, float(s)), (x * s.to(dev)).to(bf16))
    xb = x.to(bf16)
    assert torch.equal(K.cast_bf16_to_f32(xb), xb.float())


@pytest.mark.parametrize("n,decay", [(55_736_708, 0.9999), (1001, 0.3)])
def test_ema_lerp_vs_float64(n, decay):
    """ema = p + decay * (ema - p): three fp32 roundings (or a fused multiply-add): 4e-7 (|p| + |ema|)."""
    from sgb200 import kernels as K
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(29)
    p = torch.randn(n, generator=gen, device=dev)
    e = p + 0.01 * torch.randn(n, generator=gen, device=dev)
    ref = p.double() + decay * (e.double() - p.double())
    bound = 4e-7 * (p.double().abs() + e.double().abs())
    K.ema_lerp(e, p, decay)
    assert float(((e.double() - ref).abs() - bound).max()) <= 0.0


@pytest.mark.parametrize("B,C,H,W,cpad", [(128, 256, 32, 32, 0), (3, 40, 5, 7, 8)])
def test_axpby_device_scale_mask_relu(B, C, H, W, cpad):
    """out = mask > 0 ? relu(a * a_dev * x + b * y) : 0: zeros bit-exact, the rest one output rounding (atol 1e-6 for the
    fp32 product / fused add before it)."""
    from sgb200 import kernels as K
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(30)
    x, y, mask = (_act(gen, B, C, H, W, dev, cpad=cpad) for _ in range(3))
    a_dev = torch.tensor([1.7], device=dev)
    f32 = lambda v: torch.tensor(v, dtype=torch.float32)    # noqa: E731
    out = K.axpby(x, y, a=0.7, b=-1.3, a_dev=a_dev, mask=mask, relu=True)
    a32, b32 = float(f32(0.7) * f32(1.7)), float(f32(-1.3))
    ref = (a32 * x.double() + b32 * y.double()).clamp(min=0) * (mask.float() > 0)
    assert float(out.float()[mask.float() <= 0].abs().max()) == 0.0
    assert _rounding_ratio(out, ref, 1e-6) <= 1.0
