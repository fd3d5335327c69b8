"""The ResNet-family blocks (models/_resblocks.py), CIFAR attention and the WGAN-GP gradient penalty at the shapes of the
three other benchmark workloads, against float64 (pytest -m gpu).

Configurations (built from the yaml files, geometries enumerated from the built modules):
* SNGAN-CIFAR10-b256: G 256 channels 4 -> 32 with cBN on a 10-wide one-hot, no spectral norm in G; D with spectral norm,
  128 channels; B = 256.
* BigGAN-CIFAR10-b512: G 384 channels, cBN on [shared 128, z chunk 20] (K = 148), attention after G block 2 (384 ch at
  16x16: c8 = 48, c2 = 192); D 192 channels, attention after D block 1 (192 ch at 16x16: c8 = 24, c2 = 96); spectral norm
  in both; B = 512 per rank (and 128 at four ranks for the attention).
* WGAN-GP-128res: plain batch norm in both nets, G 1024 -> 64 channels 4 -> 128, D 64 -> 1024 channels 128 -> 4; B = 128.
Five parts:
1. Every DiscBlock, op by op, forward and backward: the spectral-norm variant (ReluFn, ForkFn, conv2d1 with ReLU and bit
   planes, conv2d0 or the identity skip, conv2d2 with the residual and mask_input, PoolFn) and the batch-norm variant
   (bn1, conv2d1, bn2, bn0 + conv2d0, conv2d2 with the residual).
2. Every distinct GenBlock, op by op (ForkFn, bn1 + ReLU + x2, conv2d1, bn2 + ReLU, the low-resolution skip conv2d0
   added through res_up2 in conv2d2), and linear0 (z -> 4x4, perm_S = 16).
3. The image edges: DiscOptBlock in both variants (the col27 3x3 input conv as a K = 32 GEMM, ImageInFn into the 1x1
   skip, bn0 on the pooled image) and the generator output conv C -> 3 (8 packed channels) with ImageOutFn, including the
   col27 input gradient of ConvFn.backward's Cout <= 3 path.
4. The BigGAN-CIFAR attention at B = 512 and 128 in both geometries: the three softmax epilogues, o = P . g, dtheta, the
   two per-image weight gradients, and SelfAttentionFn as a whole.
5. conv_wgrad on every distinct (Cin, Cout, k, R) of the three configurations at their per-rank batch (with the fused
   bias gradient and a second accumulate=True micro-batch), and the WGAN-GP penalty through the 128x128 discriminator.

References: plain float64 torch on the GPU, on the same bf16 operands and bf16 packed weights the kernels read; per-element
outputs are compared on the images _images(B), parameter gradients over the whole batch.  Nothing on the reference side
calls the library.  Layers without spectral norm are packed by the same batched pass with sigma = 1, so every conv's and
linear's packed weight is read from its ``_sn_cache``.

Tolerances (the rules of test_gpu_conv_fused.py / test_gpu_norm_shapes.py):
* per element: one bf16 rounding plus the fp32-accumulation atol (2^-14 of the absolute-value convolution); ReLU bit
  planes, pooled outputs, the fork's summed gradient, the pooling / up-sampling gradients and the padded channels exact.
* weight and bias gradients: 2^-18 of the absolute-value sum, through the float64 spectral-norm chain rule where it is on
  (conv_wgrad on independent operands, part 5).  Inside a block (parts 1-3) the two operands of a weight gradient are
  correlated (a post-ReLU input and the gradient of the op after it, through the same ReLU mask or batch norm), so the
  fp32 partial sums grow like the absolute-value sum instead of cancelling, and their rounding error with them: ~sqrt(n)
  2^-24 of the absolute-value sum per partial sum of n MMA steps, n ~ 1000 at these batches: 2^-19 expected.  Bound 2^-17
  there (BLOCK_WGRAD = 2 in units of 2^-18).
* batch-norm outputs: max-norm 8e-3 of the largest element and relative L2 3e-3 against float64 batch norm (CBN_REL, CBN_L2).
* ATTN_L2 (SelfAttentionFn as a whole against O.self_attention on the same bf16 input and packs; estimates): the
  attention branch x -> sigma conv(P g) passes about five bf16 stores (theta, phi, g, P, o), each ~2^-9 relative, and the
  softmax turns an absolute logit error into a relative P error, with logits of magnitude ~1-3 here: ~5e-3 expected,
  bound 2e-2 for the branch of the output (out - x) and for dsigma = <dout, t> (whose error, against a random dout, is
  held to ||dout|| ||t||).  The input gradient's branch (dx - dout) also passes
  the two 2x2 max-pool backwards, which route each gradient to the arg-max of its window: the product picks it among
  bf16-rounded phi / g values, the reference among exact ones, so windows whose two largest values lie within a
  rounding (~2^-8 relative: a few percent of the windows) send their whole gradient elsewhere, ~sqrt(few %) of relative
  L2: bound 1e-1.
* GP_BOUND (penalty through the WGAN-GP discriminator against the float64 double backward; an estimate, see the test):
  the penalty value is a function of the per-image input-gradient norms, each a sum over 49 k pixels of gradients that
  passed six bf16 blocks and five batch norms: 2e-2 relative.  The parameter gradients are second-order, carried in
  bf16 through both passes and the tangent pass, and pass the ReLU masks of both networks' forward values (see BLOCK_L2
  in test_gpu_conv_fused.py): relative L2 per parameter tensor <= 0.35, median <= 0.15, the bounds test_gpu_parity.py
  holds the batch-norm golden penalty to.  Biases whose constant a later batch norm removes (conv2d1 before bn2, and
  everything before the next block's bn0 / bn1) do not change the penalty: their exact gradient is zero, and the
  product's, bf16 rounding noise of the tangent pass, must stay below 2e-2 of the gradient of the weight beside them.  A reference in which the batch-norm statistics are detached (the mean and variance terms of the
  tangent dropped) is computed beside it; the test requires it to lie outside these bounds, so that a broken
  BNTangentFn mean term cannot pass.
"""
import copy
import os
import warnings

import pytest
import torch
import torch.nn.functional as F

from oracle import studiogan_oracle as O
from test_gpu_conv_fused import (ACC_REL, CBN_L2, CBN_REL, WGRAD_REL, _attention_bwd, _attention_fwd, _cbn_err,
                                 _conv_ratio, _dgrad_ratio, _flags, _images, _launched,
                                 _packed_weight, _param_grad_worst, _pool_bits, _rows, _sn_ref, _sn_run, _unpack_bits,
                                 _up2, _wgrad_ref, _wgrad_worst)
from test_gpu_norm_shapes import PKG, _act, _cuda, _Err, _rounding_ratio

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16

# tag -> (yaml, per-rank batch, (DiscOptBlock + DiscBlocks, GenBlocks, attention layers))
CONFIGS = {"sngan": ("SNGAN-CIFAR10-b256.yaml", 256, (4, 3, 0)),
           "biggan": ("BigGAN-CIFAR10-b512.yaml", 512, (4, 3, 2)),
           "wgan_gp": ("WGAN-GP-128res.yaml", 128, (6, 5, 0))}
BLOCK_WGRAD = 2.0
ATTN_L2 = {"out": 2e-2, "dx": 1e-1, "dsigma": 2e-2}
GP_BOUND = {"penalty": 2e-2, "worst": 0.35, "median": 0.15}


@pytest.fixture(scope="module")
def resfamily():
    """tag -> (G, D, cfgs) of the configuration, built on first use and kept for this module (without the EMA copy).
    Conv and linear biases and the batch-norm affine parameters are drawn from a seed: the initialisation zeroes them."""
    from sgb200 import config as C
    from sgb200.models import model as M
    from sgb200.utils import ops
    dev = _cuda()
    built = {}

    def get(tag):
        if tag not in built:
            cfgs = C.Configurations(os.path.join(PKG, "configs", CONFIGS[tag][0]))
            MODEL = copy.copy(cfgs.MODEL)
            MODEL.apply_g_ema = False
            torch.manual_seed(0)
            G, _, _, D, _, _, _, _ = M.load_generator_discriminator(cfgs.DATA, cfgs.OPTIMIZATION, MODEL, cfgs.STYLEGAN,
                                                                   cfgs.MODULES, cfgs.RUN, dev, None)
            gen = torch.Generator(device=dev).manual_seed(2)
            with torch.no_grad():
                for m in list(G.modules()) + list(D.modules()):
                    if isinstance(m, (torch.nn.Conv2d, torch.nn.Linear)) and m.bias is not None:
                        m.bias.copy_(0.3 * torch.randn(m.bias.shape, generator=gen, device=dev))
                    if isinstance(m, ops.BatchNorm2d) and m.affine:
                        m.weight.copy_(0.5 + torch.rand(m.weight.shape, generator=gen, device=dev))
                        m.bias.copy_(0.3 * torch.randn(m.bias.shape, generator=gen, device=dev))
            built[tag] = (G.train(), D.train(), cfgs)
        return built[tag]

    yield get
    built.clear()
    torch.cuda.empty_cache()


def _layout(G, D, img):
    """([(DiscOptBlock | DiscBlock, input resolution)], [(GenBlock, input resolution)], [(SelfAttention, resolution, net)])
    in forward order."""
    from sgb200.models._resblocks import DiscBlock, DiscOptBlock, GenBlock
    from sgb200.utils import ops
    d, g, attn, R = [], [], [], img
    for b in (b for bl in D.blocks for b in bl):
        if isinstance(b, ops.SelfAttention):
            attn.append((b, R, D))
        else:
            assert isinstance(b, (DiscOptBlock, DiscBlock))
            d.append((b, R))
            R = R // 2 if isinstance(b, DiscOptBlock) or b.downsample else R
    R = 4
    for b in (b for bl in G.blocks for b in bl):
        if isinstance(b, ops.SelfAttention):
            attn.append((b, R, G))
        else:
            assert isinstance(b, GenBlock)
            g.append((b, R))
            R *= 2
    assert R == img
    return d, g, attn


def _nets(resfamily, tag):
    G, D, cfgs = resfamily(tag)
    img, B = cfgs.DATA.img_size, CONFIGS[tag][1]
    d, g, attn = _layout(G, D, img)
    assert (len(d), len(g), len(attn)) == CONFIGS[tag][2], (tag, len(d), len(g), len(attn))
    return G, D, img, B, d, g, attn


def _grads_worst(m, u0, x, dz):
    """Weight and bias gradient of conv m given its input x and output gradient dz: through the spectral-norm chain rule
    (_param_grad_worst) where it is on, else against the raw float64 sum."""
    from sgb200.utils import ops
    if hasattr(m, "_sn"):
        return _param_grad_worst(m, u0[m], x, dz)
    k, Cout, Cin = m.kernel_size[0], m.out_channels, m.in_channels
    G, Gabs = _wgrad_ref(x, dz, k, torch.arange(Cout, device=x.device))
    G, Gabs = (t.view(Cout, k, k, Cin).permute(0, 3, 1, 2) for t in (G, Gabs))
    e = _wgrad_worst(ops._w(m).grad, G, Gabs)
    dref, dabs = dz.double().sum((0, 2, 3)), dz.double().abs().sum((0, 2, 3))
    return max(e, float(((m.bias.grad.double() - dref).abs() / (WGRAD_REL * dabs + 1e-30)).max()))


def _bn_err(y, x, bn, relu, up2=False):
    """Affine batch norm [+ ReLU] [+ x2] output y against float64 batch norm (batch statistics, eps of the layer) of the
    bf16 input x, chunked over channels."""
    B, C, H, W = x.shape
    e = _Err()
    cc = max(1, min(C, (1 << 24) // (B * H * W)))
    for c0 in range(0, C, cc):
        sl = slice(c0, min(C, c0 + cc))
        xc = x[:, sl].double()
        mu, var = xc.mean((0, 2, 3), keepdim=True), xc.var((0, 2, 3), unbiased=False, keepdim=True)
        z = (xc - mu) * (var + bn.eps).rsqrt() * bn.weight.detach()[sl].double().view(1, -1, 1, 1) + \
            bn.bias.detach()[sl].double().view(1, -1, 1, 1)
        if relu:
            z = z.clamp(min=0)
        yk = y[:, sl]
        if up2:
            for i, j in ((0, 1), (1, 0), (1, 1)):
                assert torch.equal(yk[..., i::2, j::2], yk[..., ::2, ::2])
            yk = yk[..., ::2, ::2]
        e.add(yk, z)
    return e


def _bn_ratio(r, name, e):
    r[name + " rel"], r[name + " l2"] = e.rel / CBN_REL, e.l2 / CBN_L2


def _fork_sum(g1, g2):
    """ForkFn's backward: one fp32 add of the two bf16 gradients, one rounding."""
    return (g1.float() + g2.float()).to(bf16)


def _launched_checked(fn, want):
    """_launched(fn) and the assertion that the conv kernels it ran are ``want``.  A torch.profiler session that recorded
    no CUDA kernel at all (the profiler failing, not the dispatch) is repeated once; if it records nothing again the
    launch identity is reported as unchecked, the numbers are still checked."""
    for _ in range(2):
        seen, names, out = _launched(fn)
        if any("kernel" in n for n in names):
            assert seen == want, (seen, want)
            return out
    warnings.warn("torch.profiler recorded no CUDA kernels: conv kernel identity %s not checked" % sorted(want))
    return out


def _merge(worst, r):
    for k, v in r.items():
        worst[k] = max(worst.get(k, 0.0), v)


def _block_ok(r):
    """Per-element ratios <= 1; weight / bias gradients of correlated block operands <= BLOCK_WGRAD (module docstring)."""
    return all(v <= (BLOCK_WGRAD if k.startswith("dW") else 1.0) for k, v in r.items())


# ------------------------------------------------------------------------------------------------ 1. discriminator blocks
def _check_d_block_sn(blk, R, B, dev, u0):
    from sgb200 import autograd_ops as A
    gen = torch.Generator(device=dev).manual_seed(R * 7 + blk.conv2d2.out_channels + B)
    has_sc = blk.downsample or blk.ch_mismatch
    x = _act(gen, B, blk.conv2d1.in_channels, R, R, dev).requires_grad_(True)
    t = {"a": A.ReluFn.call(x)}
    t["main"], t["side"] = A.ForkFn.call(t["a"])
    t["h1"] = blk.conv2d1(t["main"], relu=True, premasked=True)
    t["skip"] = blk.conv2d0(t["side"]) if has_sc else t["side"]
    t["h2"] = blk.conv2d2(t["h1"], residual=t["skip"], mask_input=True)
    t["out"] = A.PoolFn.call(t["h2"]) if blk.downsample else t["h2"]
    d = {n: v.detach() for n, v in t.items()}
    idx = _images(B)
    W0 = _packed_weight(blk.conv2d0) if has_sc else None
    W1, W2 = _packed_weight(blk.conv2d1), _packed_weight(blk.conv2d2)
    assert torch.equal(d["a"], x.detach().clamp(min=0))
    r = {"h1": _conv_ratio(d["h1"], d["a"], W1, 1, blk.conv2d1.bias, relu=True, idx=idx)}
    assert torch.equal(_unpack_bits(t["h1"]._sgb_relu_bits, d["h1"].shape[1]), d["h1"] > 0)
    if has_sc:
        r["skip"] = _conv_ratio(d["skip"], d["a"], W0, 0, blk.conv2d0.bias, idx=idx)
    r["h2"] = _conv_ratio(d["h2"], d["h1"], W2, 1, blk.conv2d2.bias, res=d["skip"], idx=idx)
    if blk.downsample:
        assert torch.equal(d["out"], _pool_bits(d["h2"], 0.25))
    for n in ("a", "main", "side", "h1", "skip", "h2"):
        t[n].retain_grad()
    for p in blk.parameters():
        p.grad = None
    dout = _act(gen, *d["out"].shape, dev)
    t["out"].backward(dout)
    g = {n: t[n].grad for n in ("a", "main", "side", "h1", "skip", "h2")}
    assert torch.equal(g["h2"], (_up2(dout.float()) * 0.25).to(bf16) if blk.downsample else dout)
    assert torch.equal(g["skip"], g["h2"])
    r["d_h1"] = _dgrad_ratio(g["h1"], g["h2"], W2, 1, mask=d["h1"], idx=idx)
    r["d_main"] = _dgrad_ratio(g["main"], g["h1"], W1, 1, idx=idx)
    if has_sc:
        r["d_side"] = _dgrad_ratio(g["side"], g["skip"], W0, 0, idx=idx)
    assert torch.equal(g["a"], _fork_sum(g["main"], g["side"]))
    assert torch.equal(x.grad, torch.where(d["a"] > 0, g["a"], torch.zeros((), device=dev, dtype=bf16)))
    r["dW1"] = _grads_worst(blk.conv2d1, u0, d["a"], g["h1"])
    r["dW2"] = _grads_worst(blk.conv2d2, u0, d["h1"], g["h2"])
    if has_sc:
        r["dW0"] = _grads_worst(blk.conv2d0, u0, d["a"], g["skip"])
    return r


def _check_d_block_bn(blk, R, B, dev, u0):
    from sgb200 import autograd_ops as A
    gen = torch.Generator(device=dev).manual_seed(R * 7 + blk.conv2d2.out_channels + B)
    has_sc = blk.downsample or blk.ch_mismatch
    x = _act(gen, B, blk.conv2d1.in_channels, R, R, dev).requires_grad_(True)
    t = {}
    t["main"], t["side"] = A.ForkFn.call(x)
    t["b1"] = blk.bn1(t["main"], relu=True)
    t["h1"] = blk.conv2d1(t["b1"])
    t["b2"] = blk.bn2(t["h1"], relu=True)
    if has_sc:
        t["b0"] = blk.bn0(t["side"])
        t["skip"] = blk.conv2d0(t["b0"])
    else:
        t["skip"] = t["side"]
    t["h2"] = blk.conv2d2(t["b2"], residual=t["skip"])
    t["out"] = A.PoolFn.call(t["h2"]) if blk.downsample else t["h2"]
    d = {n: v.detach() for n, v in t.items()}
    idx = _images(B)
    W1, W2 = _packed_weight(blk.conv2d1), _packed_weight(blk.conv2d2)
    r = {}
    _bn_ratio(r, "b1", _bn_err(d["b1"], x.detach(), blk.bn1, True))
    r["h1"] = _conv_ratio(d["h1"], d["b1"], W1, 1, blk.conv2d1.bias, idx=idx)
    _bn_ratio(r, "b2", _bn_err(d["b2"], d["h1"], blk.bn2, True))
    if has_sc:
        W0 = _packed_weight(blk.conv2d0)
        _bn_ratio(r, "b0", _bn_err(d["b0"], x.detach(), blk.bn0, False))
        r["skip"] = _conv_ratio(d["skip"], d["b0"], W0, 0, blk.conv2d0.bias, idx=idx)
    r["h2"] = _conv_ratio(d["h2"], d["b2"], W2, 1, blk.conv2d2.bias, res=d["skip"], idx=idx)
    if blk.downsample:
        assert torch.equal(d["out"], _pool_bits(d["h2"], 0.25))
    names = ["main", "side", "b1", "h1", "b2", "h2"] + (["b0", "skip"] if has_sc else [])
    for n in names:
        t[n].retain_grad()
    for p in blk.parameters():
        p.grad = None
    dout = _act(gen, *d["out"].shape, dev)
    t["out"].backward(dout)
    g = {n: t[n].grad for n in names}
    g["skip"] = g.get("skip", g["side"])
    assert torch.equal(g["h2"], (_up2(dout.float()) * 0.25).to(bf16) if blk.downsample else dout)
    assert torch.equal(g["skip"], g["h2"])
    r["d_b2"] = _dgrad_ratio(g["b2"], g["h2"], W2, 1, idx=idx)
    r["d_b1"] = _dgrad_ratio(g["b1"], g["h1"], W1, 1, idx=idx)
    if has_sc:
        r["d_b0"] = _dgrad_ratio(g["b0"], g["skip"], W0, 0, idx=idx)
    assert torch.equal(x.grad, _fork_sum(g["main"], g["side"]))
    r["dW1"] = _grads_worst(blk.conv2d1, u0, d["b1"], g["h1"])
    r["dW2"] = _grads_worst(blk.conv2d2, u0, d["b2"], g["h2"])
    if has_sc:
        r["dW0"] = _grads_worst(blk.conv2d0, u0, d["b0"], g["skip"])
    return r


@pytest.mark.parametrize("tag", list(CONFIGS))
def test_discriminator_block_ops_vs_float64(resfamily, tag):
    """Every DiscBlock of the configuration at its per-rank batch, op by op, forward and backward: conv outputs and input
    gradients within one rounding on _images(B); bit planes, pooled outputs, the pooling gradient, the identity skip and
    the fork's summed gradient exact; batch-norm outputs against float64; every weight and bias gradient over the batch."""
    from sgb200.models._resblocks import DiscBlock
    dev = _cuda()
    G, D, img, B, dblocks, _, _ = _nets(resfamily, tag)
    blocks = [(b, R) for b, R in dblocks if isinstance(b, DiscBlock)]
    assert len(blocks) == len(dblocks) - 1
    assert any(not (b.downsample or b.ch_mismatch) for b, _ in blocks)      # an identity skip
    u0 = _sn_run(D)
    worst = {}
    try:
        for blk, R in blocks:
            r = (_check_d_block_sn if blk.apply_d_sn else _check_d_block_bn)(blk, R, B, dev, u0)
            print("%s D %d->%d @%d down=%d B=%d: %s" % (tag, blk.conv2d1.in_channels, blk.conv2d2.out_channels, R,
                                                        blk.downsample, B, {k: round(v, 3) for k, v in r.items()}))
            _merge(worst, r)
            torch.cuda.empty_cache()
    finally:
        D._snb.clear()
    print("%s D block ops worst: %s" % (tag, {k: round(v, 3) for k, v in worst.items()}))
    assert _block_ok(worst), worst


# ------------------------------------------------------------------------------------------------ 2. generator blocks
def _affine(G, tag, B, gen, dev):
    """The conditioning activation the generator hands every cBN layer: ToBF16Fn of the one-hot label (SNGAN) or of
    [shared embedding, z chunk] (BigGAN); None for plain batch norm."""
    from sgb200 import autograd_ops as A
    if tag == "sngan":
        y = torch.randint(0, G.num_classes, (B,), generator=gen, device=dev)
        return A.ToBF16Fn.call(F.one_hot(y, G.num_classes).float())
    if tag == "biggan":
        return A.ToBF16Fn.call(torch.randn((B, G.affine_input_dim), generator=gen, device=dev))
    return None


def _check_g_block(G, blk, R, B, affine, dev, u0):
    from sgb200 import autograd_ops as A
    gen = torch.Generator(device=dev).manual_seed(R * 13 + blk.conv2d1.in_channels + B)
    x = _act(gen, B, blk.conv2d1.in_channels, R, R, dev).requires_grad_(True)
    cond = blk.conditional
    t = {}
    t["main"], t["side"] = A.ForkFn.call(x)
    t["a1"] = blk.bn1(t["main"], affine, relu=True, up2=True) if cond else blk.bn1(t["main"], relu=True, up2=True)
    t["h1"] = blk.conv2d1(t["a1"])
    t["a2"] = blk.bn2(t["h1"], affine, relu=True) if cond else blk.bn2(t["h1"], relu=True)
    t["skip"] = blk.conv2d0(t["side"])
    t["out"] = blk.conv2d2(t["a2"], residual=t["skip"], res_up2=True)
    d = {n: v.detach() for n, v in t.items()}
    idx = _images(B)
    W0, W1, W2 = (_packed_weight(m) for m in (blk.conv2d0, blk.conv2d1, blk.conv2d2))
    r = {}
    for n, src, bn, up in (("a1", x.detach(), blk.bn1, True), ("a2", d["h1"], blk.bn2, False)):
        _bn_ratio(r, n, _cbn_err(d[n], src, bn, affine, up) if cond else _bn_err(d[n], src, bn, True, up))
    r["h1"] = _conv_ratio(d["h1"], d["a1"], W1, 1, blk.conv2d1.bias, idx=idx)
    r["skip"] = _conv_ratio(d["skip"], x.detach(), W0, 0, blk.conv2d0.bias, idx=idx)
    r["out"] = _conv_ratio(d["out"][idx], d["a2"][idx], W2, 1, blk.conv2d2.bias, res=_up2(d["skip"][idx]), idx=slice(None))
    for n in ("main", "side", "a1", "h1", "a2", "skip"):
        t[n].retain_grad()
    for p in blk.parameters():
        p.grad = None
    dout = _act(gen, *d["out"].shape, dev)
    t["out"].backward(dout)
    g = {n: t[n].grad for n in ("main", "side", "a1", "h1", "a2", "skip")}
    assert torch.equal(g["skip"], _pool_bits(dout, 1.0))      # the 2x2 sum of conv2d2's output gradient
    r["d_a2"] = _dgrad_ratio(g["a2"], dout, W2, 1, idx=idx)
    r["d_a1"] = _dgrad_ratio(g["a1"], g["h1"], W1, 1, idx=idx)
    r["d_side"] = _dgrad_ratio(g["side"], g["skip"], W0, 0, idx=idx)
    assert torch.equal(x.grad, _fork_sum(g["main"], g["side"]))
    r["dW1"] = _grads_worst(blk.conv2d1, u0, d["a1"], g["h1"])
    r["dW2"] = _grads_worst(blk.conv2d2, u0, d["a2"], dout)
    r["dW0"] = _grads_worst(blk.conv2d0, u0, x.detach(), g["skip"])
    return r


def _check_linear0(G, B, dev, u0):
    """linear0 (z -> [B, 16 C] in NHWC order, perm_S = 16): output feature s*C + c is row c*16 + s of the weight.  The
    forward against the pack it read, z's gradient, and the weight / bias gradients in the module's row order."""
    from sgb200 import kernels as K
    from sgb200.utils import ops
    m = G.linear0
    S = m._perm_S
    N, Kd = m.out_features, m.in_features
    C = N // S
    gen = torch.Generator(device=dev).manual_seed(N + B)
    z = torch.randn((B, Kd), generator=gen, device=dev).requires_grad_(True)
    out = m(z, perm_S=S)
    assert out.shape == (B, N, 1, 1)
    Wp = m._sn_cache[0][:N, 0, :Kd].double()                  # rows in output order
    zb = z.detach().to(bf16).double()
    bias = m.bias.detach().double().view(C, S).t().reshape(-1)
    ref = zb @ Wp.t() + bias
    r = {"out": _rounding_ratio(out.reshape(B, N), ref, ACC_REL * (zb.abs() @ Wp.abs().t()) + 1e-30)}
    dout = _act(gen, B, N, 1, 1, dev)
    for p in m.parameters():
        p.grad = None
    out.backward(dout)
    dy = dout.reshape(B, N).double()
    r["dz"] = _rounding_ratio(z.grad, dy @ Wp, ACC_REL * (dy.abs() @ Wp.abs()) + 1e-30)
    rows = torch.arange(N, device=dev)
    col = (rows % S) * C + rows // S                           # output feature of weight row r = c*S + s
    Gm, Gabs = dy[:, col].t() @ zb, dy[:, col].abs().t() @ zb.abs()
    got = ops._w(m).grad.double()
    if hasattr(m, "_sn"):
        W, u, v, sig = _sn_ref(m, u0[m])
        uv = torch.outer(u, v)
        refw = (Gm - float((Gm * W).sum()) / sig * uv) / sig
        bound = WGRAD_REL * (Gabs + float((Gabs * W.abs()).sum()) / sig * uv.abs()) / sig
    else:
        refw, bound = Gm, WGRAD_REL * Gabs
    r["dW"] = float(((got - refw).abs() / (bound + 1e-30)).max())
    r["db"] = float(((m.bias.grad.double() - dy[:, col].sum(0)).abs() / (WGRAD_REL * dy[:, col].abs().sum(0) + 1e-30)).max())
    assert K.pad8(Kd) == m._sn_cache[0].shape[2]
    return r


@pytest.mark.parametrize("tag", list(CONFIGS))
def test_generator_block_ops_vs_float64(resfamily, tag):
    """Every distinct GenBlock of the configuration at its per-rank batch, op by op, forward and backward: conv outputs and
    input gradients within one rounding on _images(B); (c)BN + ReLU (+ x2) outputs against float64 batch norm with the
    gains of the cBN linears' packs; the skip gradient (2x2 sum) and the fork's summed gradient exact; every weight and
    bias gradient over the batch.  Then linear0."""
    dev = _cuda()
    G, D, img, B, _, gblocks, _ = _nets(resfamily, tag)
    seen, worst = set(), {}
    u0 = _sn_run(G)
    try:
        affine = _affine(G, tag, B, torch.Generator(device=dev).manual_seed(71), dev)
        for blk, R in gblocks:
            geo = (blk.conv2d1.in_channels, blk.conv2d2.out_channels, R)
            if geo in seen:
                continue
            seen.add(geo)
            r = _check_g_block(G, blk, R, B, affine, dev, u0)
            print("%s G %d->%d @%d B=%d: %s" % (tag, geo[0], geo[1], R, B, {k: round(v, 3) for k, v in r.items()}))
            _merge(worst, r)
            torch.cuda.empty_cache()
        r = _check_linear0(G, B, dev, u0)
        print("%s G linear0 %d->%d B=%d: %s" % (tag, G.linear0.in_features, G.linear0.out_features, B,
                                                {k: round(v, 3) for k, v in r.items()}))
        assert max(r.values()) <= 1.0, r                     # independent operands: the 2^-18 bound
        _merge(worst, {"linear0 " + k: v for k, v in r.items()})
    finally:
        G._snb.clear()
    print("%s G block ops worst: %s" % (tag, {k: round(v, 3) for k, v in worst.items()}))
    assert len(seen) == len(gblocks) and _block_ok(worst), worst


# ------------------------------------------------------------------------------------------------ 3. image edges
def _image_weight(m):
    """The bf16 [Cout, 3, 3, 3] weight the col27 GEMM of an image conv reads: W / sigma formed by torch in fp32 as
    ops._sn_divided forms it (sigma = u . W v of the iterated u, v), or W."""
    W = m.weight_orig if hasattr(m, "_sn") else m.weight
    W = W.detach()
    if hasattr(m, "_sn"):
        W = W / torch.dot(m.weight_u, torch.mv(W.reshape(W.shape[0], -1), m.weight_v))
    return W.to(bf16)


def _check_opt_block(blk, R, B, dev, u0):
    """DiscOptBlock.forward op by op on a seeded image (no input gradient, as in a D step)."""
    from sgb200 import autograd_ops as A
    gen = torch.Generator(device=dev).manual_seed(R + blk.conv2d1.out_channels + B)
    img = torch.rand((B, 3, R, R), generator=gen, device=dev) * 2 - 1
    sn = blk.apply_d_sn
    t = {"col": A.ImageColFn.call(img)}
    t["h1"] = blk.conv2d1(t["col"], relu=sn, premasked=sn)
    if sn:
        t["h2"] = blk.conv2d2(t["h1"], mask_input=True)
    else:
        t["b1"] = blk.bn1(t["h1"], relu=True)
        t["h2"] = blk.conv2d2(t["b1"])
    t["hp"] = A.PoolFn.call(t["h2"])
    x0 = F.avg_pool2d(img, 2)
    if not sn:
        bn0 = blk.bn0
        x0 = F.batch_norm(x0, bn0.running_mean, bn0.running_var, bn0.weight, bn0.bias, bn0.training, bn0.momentum, bn0.eps)
    t["xi"] = A.ImageInFn.call(x0)
    t["s"] = blk.conv2d0(t["xi"])
    t["out"] = A.AddFn.call(t["hp"], t["s"])
    d = {n: v.detach() for n, v in t.items()}
    idx = _images(B)
    ib = img.to(bf16)
    W1 = _image_weight(blk.conv2d1)
    W0, W2 = _packed_weight(blk.conv2d0), _packed_weight(blk.conv2d2)
    assert d["col"].shape[1] == 32 and float(d["col"][:, 27:].abs().max()) == 0.0
    r = {"h1": _conv_ratio(d["h1"], ib, W1, 1, blk.conv2d1.bias, relu=sn, idx=idx)}
    a1 = d["h1"]
    if sn:
        assert torch.equal(_unpack_bits(t["h1"]._sgb_relu_bits, a1.shape[1]), a1 > 0)
    else:
        _bn_ratio(r, "b1", _bn_err(d["b1"], d["h1"], blk.bn1, True))
        a1 = d["b1"]
    r["h2"] = _conv_ratio(d["h2"], a1, W2, 1, blk.conv2d2.bias, idx=idx)
    assert torch.equal(d["hp"], _pool_bits(d["h2"], 0.25))
    # ImageInFn: the pooled (and batch-normalised) image as bf16 in channels 0..2 of 8, the rest zero
    p = F.avg_pool2d(img.double(), 2)
    if not sn:
        mu, var = p.mean((0, 2, 3), keepdim=True), p.var((0, 2, 3), unbiased=False, keepdim=True)
        p = (p - mu) * (var + blk.bn0.eps).rsqrt() * blk.bn0.weight.detach().double().view(1, -1, 1, 1) + \
            blk.bn0.bias.detach().double().view(1, -1, 1, 1)
    r["xi"] = _rounding_ratio(d["xi"][:, :3], p, 2e-4 if not sn else 1e-6)
    assert d["xi"].shape[1] == 8 and float(d["xi"][:, 3:].abs().max()) == 0.0
    r["s"] = _conv_ratio(d["s"], d["xi"][:, :3], W0, 0, blk.conv2d0.bias, idx=idx)
    assert torch.equal(d["out"], _fork_sum(d["hp"], d["s"]))
    names = ["h1", "h2", "hp", "s"] + ([] if sn else ["b1"])
    for n in names:
        t[n].retain_grad()
    for prm in blk.parameters():
        prm.grad = None
    dout = _act(gen, *d["out"].shape, dev)
    t["out"].backward(dout)
    g = {n: t[n].grad for n in names}
    assert torch.equal(g["hp"], dout) and torch.equal(g["s"], dout)
    assert torch.equal(g["h2"], (_up2(dout.float()) * 0.25).to(bf16))
    if sn:
        r["d_h1"] = _dgrad_ratio(g["h1"], g["h2"], W2, 1, mask=d["h1"], idx=idx)
    else:
        r["d_b1"] = _dgrad_ratio(g["b1"], g["h2"], W2, 1, idx=idx)
    # the image conv's weight gradient back in the [Cout, 3, 3, 3] layout (K = 27 of the col27 GEMM, Cin_p = 32)
    r["dW1"] = _grads_worst(blk.conv2d1, u0, ib, g["h1"])
    r["dW2"] = _grads_worst(blk.conv2d2, u0, a1, g["h2"])
    r["dW0"] = _grads_worst(blk.conv2d0, u0, d["xi"][:, :3], dout)
    return r


def _check_output_conv(G, img, B, dev, u0):
    """bn4 + ReLU -> conv2d5 (C -> 3, 8 packed channels) -> ImageOutFn, forward and backward.  Returns (ratios, the conv
    kernels conv2d5's forward launched)."""
    from sgb200 import autograd_ops as A
    m = G.conv2d5
    C = m.in_channels
    gen = torch.Generator(device=dev).manual_seed(C + img + B)
    x = _act(gen, B, C, img, img, dev).requires_grad_(True)
    a = G.bn4(x, relu=True)
    want = {("rows" if img == 128 else "fprop", _flags("general"))}
    y = _launched_checked(lambda: m(a), want)
    out = A.ImageOutFn.call(y, 3)
    idx = _images(B)
    W5 = _packed_weight(m)                                     # [3, C, 3, 3]
    r = {}
    _bn_ratio(r, "bn4", _bn_err(a.detach(), x.detach(), G.bn4, True))
    yd = y.detach()
    assert yd.shape[1] == 8 and float(yd[:, 3:].abs().max()) == 0.0
    r["y"] = _conv_ratio(yd[:, :3], a.detach(), W5, 1, m.bias, idx=idx)
    r["img"] = float((out.detach().double() - torch.tanh(yd[:, :3].double())).abs().max()) / 2.0 ** -20
    a.retain_grad()
    y.retain_grad()
    for p in m.parameters():
        p.grad = None
    dimg = torch.randn(out.shape, generator=gen, device=dev)
    out.backward(dimg)
    dz = y.grad
    assert dz.shape[1] == 8 and float(dz[:, 3:].abs().max()) == 0.0
    r["dz"] = _rounding_ratio(dz[:, :3], dimg.double() * (1 - out.detach().double() ** 2), 1e-6)
    # the Cout <= 3 input gradient: col27(dz) times the [C, 27] re-ordered bf16(W / sigma) (torch's fp32 division)
    sigma = m._sn_cache[2]
    Wd = (m.weight_orig.detach() / sigma if sigma is not None else m.weight.detach()).to(bf16)
    r["d_a"] = _dgrad_ratio(a.grad, dz[:, :3], Wd, 1, idx=idx)
    r["dW5"] = _grads_worst(m, u0, a.detach(), dz[:, :3])
    return r, want


@pytest.mark.parametrize("tag", list(CONFIGS))
def test_image_edges_vs_float64(resfamily, tag):
    """DiscOptBlock (the col27 3x3 input conv as a K = 32 GEMM against a float64 3x3 conv of the bf16 image, its weight
    gradient in the [Cout, 3, 3, 3] layout; ImageInFn into the 1x1 skip; bn0 on the pooled image in the batch-norm variant)
    and the generator output conv C -> 3 with ImageOutFn and the col27 input gradient, at the per-rank batch.  The output
    conv runs the direct-store general kernel at 32x32 and the halo-row general kernel at 128x128."""
    from sgb200.models._resblocks import DiscOptBlock
    dev = _cuda()
    G, D, img, B, dblocks, _, _ = _nets(resfamily, tag)
    blk, R = dblocks[0]
    assert isinstance(blk, DiscOptBlock) and R == img
    uD = _sn_run(D)
    try:
        r = _check_opt_block(blk, R, B, dev, uD)
    finally:
        D._snb.clear()
    print("%s DiscOptBlock 3->%d @%d B=%d: %s" % (tag, blk.conv2d1.out_channels, R, B, {k: round(v, 3) for k, v in r.items()}))
    uG = _sn_run(G)
    try:
        r2, seen = _check_output_conv(G, img, B, dev, uG)
    finally:
        G._snb.clear()
    print("%s G output conv %d->3 @%d B=%d: %s; kernels %s" % (tag, G.conv2d5.in_channels, img, B,
                                                               {k: round(v, 3) for k, v in r2.items()}, sorted(seen)))
    assert _block_ok(r) and _block_ok(r2), (r, r2)


# ------------------------------------------------------------------------------------------------ 4. CIFAR attention
def _attn_operands(B, c8, c2, dev):
    gen = torch.Generator(device=dev).manual_seed(B + c8)
    return (_act(gen, B, c8, 16, 16, dev), _act(gen, B, c8, 8, 8, dev), _act(gen, B, c2, 8, 8, dev),
            _act(gen, B, c2, 16, 16, dev))


def _check_attention_gemms(B, c8, c2, dev):
    """Softmax epilogues, o = P . g, dtheta = dS . phi, dg = P^T do and dphi = dS^T theta (per image) at N = 256, M = 64."""
    from sgb200 import kernels as K
    theta, phi, g, do = _attn_operands(B, c8, c2, dev)
    P = _launched_checked(lambda: _attention_fwd(theta, phi), {("fprop", _flags("Full|SmStats")), ("fprop", _flags("Full|SmApply"))})
    Bn = B * 256
    delta = torch.empty(Bn, device=dev, dtype=torch.float32)
    per = 64
    for b0 in range(0, B, per):
        b1 = min(B, b0 + per)
        dP = _rows(do[b0:b1]) @ _rows(g[b0:b1]).transpose(1, 2)
        delta.view(B, -1)[b0:b1] = (_rows(P[b0:b1]) * dP).sum(-1).float()
    dS = _launched_checked(lambda: _attention_bwd(do, g, P, delta), {("fprop", _flags("Full|SmBwd"))})
    o = K.conv_fprop(P, g, c2, 1, 1, 0, 0, w_mode=2)
    dtheta = K.conv_fprop(dS, phi, c8, 1, 1, 0, 0, w_mode=2)
    dg = K.conv_wgrad(do, P, 1, 1, 0, 0, per_image=True).view(B, 64, c2)
    dphi = K.conv_wgrad(theta, dS, 1, 1, 0, 0, per_image=True).view(B, 64, c8)
    r = dict.fromkeys(("P", "dS", "o", "dtheta", "dg", "dphi"), 0.0)

    def up(k, v):
        r[k] = max(r[k], v)
    for b0 in range(0, B, per):
        b1 = min(B, b0 + per)
        q, kk, gv, dov = _rows(theta[b0:b1]), _rows(phi[b0:b1]), _rows(g[b0:b1]), _rows(do[b0:b1])
        Pk, dSk = _rows(P[b0:b1]), _rows(dS[b0:b1])
        logits, labs = q @ kk.transpose(1, 2), q.abs() @ kk.abs().transpose(1, 2)
        Pref = torch.softmax(logits, -1)
        up("P", _rounding_ratio(Pk, Pref, Pref * (2 * ACC_REL * labs.amax(-1, keepdim=True) + 2.0 ** -18) + 2.0 ** -126))
        dP, dabs = dov @ gv.transpose(1, 2), dov.abs() @ gv.abs().transpose(1, 2)
        dref = Pk * (dP - delta.view(B, -1)[b0:b1].double()[..., None])
        up("dS", _rounding_ratio(dSk, dref, Pk * ACC_REL * dabs + 1e-30))
        up("o", _rounding_ratio(_rows(o[b0:b1]), Pk @ gv, ACC_REL * (Pk.abs() @ gv.abs()) + 1e-30))
        up("dtheta", _rounding_ratio(_rows(dtheta[b0:b1]), dSk @ kk, ACC_REL * (dSk.abs() @ kk.abs()) + 1e-30))
        up("dg", float(((dg[b0:b1].double() - Pk.transpose(1, 2) @ dov).abs() /
                        (WGRAD_REL * (Pk.abs().transpose(1, 2) @ dov.abs()) + 1e-30)).max()))
        up("dphi", float(((dphi[b0:b1].double() - dSk.transpose(1, 2) @ q).abs() /
                          (WGRAD_REL * (dSk.abs().transpose(1, 2) @ q.abs()) + 1e-30)).max()))
    return r


def _check_self_attention(sa, B, dev):
    """SelfAttentionFn forward and backward against O.self_attention in float64 on the same bf16 input and packs: relative
    L2 of the attention branch of the output and of the input gradient, and the error of dsigma relative to ||dout|| ||t||."""
    gen = torch.Generator(device=dev).manual_seed(B + sa.in_channels + 5)
    C = sa.in_channels
    x = _act(gen, B, C, 16, 16, dev).requires_grad_(True)
    with torch.no_grad():
        sa.sigma.fill_(0.7)
    sa.sigma.grad = None
    out = sa(x)
    dout = _act(gen, *out.shape, dev)
    out.backward(dout)
    sd = {n + ".weight": _packed_weight(getattr(sa, n)).double() for n in ("conv1x1_theta", "conv1x1_phi", "conv1x1_g",
                                                                         "conv1x1_attn")}
    sd["sigma"] = sa.sigma.detach().double().clone().requires_grad_(True)
    e_out, e_dx = _Err(), _Err()
    for b0 in range(0, B, 64):
        b1 = min(B, b0 + 64)
        xr = x.detach()[b0:b1].double().requires_grad_(True)
        ref = O.self_attention(sd, "", xr, training=False)
        ref.backward(dout[b0:b1].double())
        e_out.add(out.detach()[b0:b1].double() - xr.detach(), ref.detach() - xr.detach())
        e_dx.add(x.grad[b0:b1].double() - dout[b0:b1].double(), xr.grad - dout[b0:b1].double())
    # dsigma = <dout, t> with a random dout cancels: its error is measured against ||dout|| ||t|| (Cauchy-Schwarz)
    ds = abs(float(sa.sigma.grad) - float(sd["sigma"].grad)) / (float(dout.double().norm()) * e_out.r2 ** 0.5 / 0.7)
    with torch.no_grad():
        sa.sigma.zero_()
    return {"out": e_out.l2, "dx": e_dx.l2, "dsigma": ds}


@pytest.mark.parametrize("B", [512, 128])
def test_biggan_cifar_attention_vs_float64(resfamily, B):
    """The BigGAN-CIFAR attention layers (D: 192 channels, c8 = 24, c2 = 96; G: 384 channels, c8 = 48, c2 = 192; both at
    16x16: N = 256 queries, M = 64 keys) at the per-rank batch of one and of four ranks: the softmax statistics / apply /
    backward epilogues, the w_mode-2 GEMMs o = P . g (Cout = c2) and dtheta = dS . phi (Cout = c8), the per-image weight
    gradients dg (Cin = c2) and dphi (Cin = c8), per element; SelfAttentionFn as a whole in relative L2 (ATTN_L2)."""
    dev = _cuda()
    G, D, _, _, _, _, attn = _nets(resfamily, "biggan")
    assert sorted((sa.in_channels, R) for sa, R, _ in attn) == [(192, 16), (384, 16)]
    worst = {}
    for sa, R, net in attn:
        C = sa.in_channels
        r = _check_attention_gemms(B, C // 8, C // 2, dev)
        u0 = _sn_run(net)
        try:
            l2 = _check_self_attention(sa, B, dev)
        finally:
            net._snb.clear()
        del u0
        print("attention C=%d c8=%d c2=%d B=%d: %s; SelfAttentionFn rel L2 %s" % (
            C, C // 8, C // 2, B, {k: round(v, 3) for k, v in r.items()}, {k: "%.3g" % v for k, v in l2.items()}))
        assert max(r.values()) <= 1.0, r
        assert all(l2[k] <= ATTN_L2[k] for k in l2), l2
        _merge(worst, r)
        torch.cuda.empty_cache()
    print("attention B=%d worst: %s" % (B, {k: round(v, 3) for k, v in worst.items()}))


# ------------------------------------------------------------------------------------------------ 5. weight gradients
def _wgrad_shapes(G, D, dblocks, gblocks, attn, img):
    """Distinct (Cin, Cout, k, R) of every conv / linear weight-gradient launch of one configuration (R = 1: linears)."""
    from sgb200.models._resblocks import DiscOptBlock
    from sgb200 import kernels as K
    from sgb200.utils import ops
    s = set()
    for b, R in dblocks:
        Cout = b.conv2d2.out_channels
        if isinstance(b, DiscOptBlock):    # col27 GEMM (K = 32), conv2d2, the 1x1 skip on the 8-channel pooled image
            s |= {(32, Cout, 1, R), (Cout, Cout, 3, R), (8, Cout, 1, R // 2)}
        else:
            s |= {(b.conv2d1.in_channels, Cout, 3, R), (Cout, Cout, 3, R)}
            if b.downsample or b.ch_mismatch:
                s.add((b.conv2d0.in_channels, Cout, 1, R))
    for b, R in gblocks:
        Cin, Cout = b.conv2d1.in_channels, b.conv2d2.out_channels
        s |= {(Cin, Cout, 3, 2 * R), (Cout, Cout, 3, 2 * R), (Cin, Cout, 1, R)}
    for sa, R, _ in attn:
        C = sa.in_channels
        s |= {(C, C // 8, 1, R), (C, C // 2, 1, R), (C // 2, C, 1, R)}
    s.add((G.conv2d5.in_channels, 8, 3, img))
    for m in G.modules():
        if isinstance(m, ops._LinearBase):
            s.add((K.pad8(m.in_features), m.out_features, 1, 1))
    return s


def test_conv_wgrad_every_resfamily_layer_at_per_rank_batch(resfamily):
    """conv_wgrad with the fused bias gradient on every distinct weight-gradient geometry of the three configurations at
    their per-rank batch, then a second micro-batch (accumulate=True into the non-zero dw and, through dbias_acc, the
    bias gradient), against float64 over the whole batch and every output channel.  Covers Cin = 8 (image skip) and 32
    (col27), Cout = 8 (output conv), 24 (attention theta / phi) and 192 / 384 (a partial second 128-row tile)."""
    from sgb200 import kernels as K
    dev = _cuda()
    cases = set()
    for tag in CONFIGS:
        G, D, img, B, dblocks, gblocks, attn = _nets(resfamily, tag)
        cases |= {sh + (B,) for sh in _wgrad_shapes(G, D, dblocks, gblocks, attn, img)}
    cases = sorted(cases, key=lambda c: (c[3], c[2], c[0], c[1], c[4]))
    assert {c[0] for c in cases} >= {8, 32} and {c[1] for c in cases} >= {8, 24, 192, 384}
    gen = torch.Generator(device=dev).manual_seed(81)
    worst, worst_db = 0.0, 0.0
    for Cin, Cout, k, R, B in cases:
        x, dy = _act(gen, B, Cin, R, R, dev), _act(gen, B, Cout, R, R, dev)
        dw, db = K.conv_wgrad(x, dy, k, k, k // 2, k // 2, want_dbias=True)
        assert db is not None
        co = torch.arange(Cout, device=dev)
        ref, rabs = _wgrad_ref(x, dy, k, co)
        e = _wgrad_worst(dw, ref, rabs)
        dref, dabs = dy.double().sum((0, 2, 3)), dy.double().abs().sum((0, 2, 3))
        edb = float(((db.double() - dref).abs() / (WGRAD_REL * dabs)).max())
        x2, dy2 = _act(gen, B, Cin, R, R, dev), _act(gen, B, Cout, R, R, dev)
        _, done = K.conv_wgrad(x2, dy2, k, k, k // 2, k // 2, dw=dw, accumulate=True, dbias_acc=db)
        assert done is True
        r2, a2 = _wgrad_ref(x2, dy2, k, co)
        e = max(e, _wgrad_worst(dw, ref + r2, rabs + a2))
        dref, dabs = dref + dy2.double().sum((0, 2, 3)), dabs + dy2.double().abs().sum((0, 2, 3))
        edb = max(edb, float(((db.double() - dref).abs() / (WGRAD_REL * dabs)).max()))
        print("wgrad %dx%d %d->%d @%d B=%d: dw %.3g db %.3g" % (k, k, Cin, Cout, R, B, e, edb))
        worst, worst_db = max(worst, e), max(worst_db, edb)
        assert e <= 1.0 and edb <= 1.0, (Cin, Cout, k, R, B)
        del x, dy, x2, dy2, dw, db, ref, rabs, r2, a2
    print("wgrad: %d shapes, worst dw %.3g db %.3g" % (len(cases), worst, worst_db))


# ------------------------------------------------------------------------------------------------ 5. gradient penalty
def _bn_detached_stats(sd, prefix, x, training=True, track=True, affine=False):
    """O.batch_norm with the batch mean and variance held constant (no gradient through them)."""
    mean, var = x.mean(dim=(0, 2, 3)).detach(), x.var(dim=(0, 2, 3), unbiased=False).detach()
    y = (x - mean[None, :, None, None]) * torch.rsqrt(var[None, :, None, None] + O.BN_EPS)
    if affine:
        y = y * sd[prefix + "weight"][None, :, None, None] + sd[prefix + "bias"][None, :, None, None]
    return y


def _gp_reference(sd0, names, real, fake, alpha, labels):
    """O.grad_penalty through O.res_discriminator in float64 (create_graph double backward): (P, {name: dP/dparam})."""
    sd = {k: v.clone().requires_grad_(k in names) for k, v in sd0.items()}
    pen = O.grad_penalty(lambda x: O.res_discriminator(sd, x, labels, 128, 64, cond="W/O")[0], real, fake, alpha)
    pen.backward()
    return float(pen.detach()), {n: sd[n].grad for n in names}


def _gp_distance(got, ref, names):
    """Per-parameter relative L2 of got against ref: (worst, median, worst name)."""
    e = {}
    for n in names:
        a, b = got[n].double(), ref[n]
        e[n] = float((a - b).norm() / (b.norm() + 1e-30))
    vals = sorted(e.values())
    name = max(e, key=e.get)
    return e[name], vals[len(vals) // 2], name


def test_wgan_gp_penalty_vs_float64_double_backward(resfamily, monkeypatch):
    """losses.cal_grad_penalty (primal pass, input-gradient pass, tangent replay through BNTangentFn and ConvFn.tangent)
    through the WGAN-GP 128x128 batch-norm discriminator at B = 64 with a fixed alpha, against O.grad_penalty over
    O.res_discriminator in float64 on the product's state dict: the penalty value and every parameter's gradient.  A
    second float64 reference with the batch-norm statistics detached must lie outside the bounds (GP_BOUND)."""
    from sgb200.utils import losses
    dev = _cuda()
    G, D, img, _, dblocks, _, _ = _nets(resfamily, "wgan_gp")
    assert img == 128 and max(b.conv2d2.out_channels for b, _ in dblocks) == 1024
    B = 64
    gen = torch.Generator(device=dev).manual_seed(91)
    real = torch.rand((B, 3, img, img), generator=gen, device=dev) * 2 - 1
    fake = torch.tanh(torch.randn((B, 3, img, img), generator=gen, device=dev))
    alpha = torch.rand((B, 1), generator=torch.Generator().manual_seed(92))
    labels = torch.zeros(B, dtype=torch.long, device=dev)
    names = [n for n, _ in D.named_parameters()]
    sd0 = {k: v.detach().double().clone() for k, v in D.state_dict().items()}
    for p in D.parameters():
        p.grad = None
    pen = losses.cal_grad_penalty(real_images=real, real_labels=labels, fake_images=fake, discriminator=D, device=dev,
                                  alpha=alpha)
    pen.backward()
    got = {n: (p.grad if p.grad is not None else torch.zeros_like(p)) for n, p in D.named_parameters()}
    a64 = alpha.double().to(dev)
    pen_ref, g_ref = _gp_reference(sd0, names, real.double(), fake.double(), a64, labels)
    with monkeypatch.context() as mp:
        mp.setattr(O, "batch_norm", _bn_detached_stats)
        pen_det, g_det = _gp_reference(sd0, names, real.double(), fake.double(), a64, labels)
    # the penalty does not depend on the head bias: no gradient in the reference, none (or zero) in the product
    free = [n for n in names if g_ref[n] is None]
    assert free == ["linear1.bias"] and float(got["linear1.bias"].abs().max()) == 0.0, free
    names = [n for n in names if n not in free]
    # biases whose constant is removed by a later batch norm do not change the penalty: zero gradient in exact arithmetic
    top = max(float(g_ref[n].norm()) for n in names)
    zero = [n for n in names if float(g_ref[n].norm()) <= 1e-9 * top]
    assert zero and all(n.endswith("bias") for n in zero) and "blocks.0.0.conv2d1.bias" in zero, zero
    zero_ratio = max(float(got[n].norm() / got[n[:-4] + "weight"].norm()) for n in zero)
    names = [n for n in names if n not in zero]
    e_pen = abs(float(pen.detach()) - pen_ref) / abs(pen_ref)
    d_pen = abs(pen_det - pen_ref) / abs(pen_ref)
    worst, median, wname = _gp_distance(got, g_ref, names)
    dworst, dmedian, dname = _gp_distance(g_det, g_ref, names)
    print("WGAN-GP penalty B=%d @%d: P %.6g (float64 %.6g, detached statistics %.6g)" % (B, img, float(pen.detach()), pen_ref,
                                                                                         pen_det))
    print("  product:  penalty %.3g, parameter grads rel L2 worst %.3g (%s) median %.3g; %d zero-gradient biases %.3g of their weight" % (
        e_pen, worst, wname, median, len(zero), zero_ratio))
    print("  detached: penalty %.3g, parameter grads rel L2 worst %.3g (%s) median %.3g" % (d_pen, dworst, dname, dmedian))
    assert e_pen <= GP_BOUND["penalty"] and worst <= GP_BOUND["worst"] and median <= GP_BOUND["median"]
    assert zero_ratio <= 2e-2
    # the bounds must be able to tell a tangent without the batch-statistics terms from the exact one
    assert dworst > GP_BOUND["worst"] and dmedian > GP_BOUND["median"]
