"""ORACLE — test infrastructure only.  Nothing under sgb200/ (the product) may import this file.

A CPU restatement, in plain PyTorch fp32/fp64 tensor algebra and numpy, of the arithmetic on StudioGAN's BigGAN /
BigGAN-Deep hot path.  It is *state-dict driven*: every function takes the flat ``{key: tensor}`` dictionary that the
reference modules (and the sgb200 modules, which keep the same keys) produce, so the same oracle checks both sides.
Each function cites the reference lines it restates (paths relative to the reference checkout; ``torch/`` = PyTorch).

Pinning: tests/golden/make_golden.py imports the real reference in the build container, runs it on seeded inputs and
stores inputs/outputs in tests/golden/*.npz; tests/test_oracle_golden.py (CPU) checks this file against those vectors.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this module.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

SN_EPS = 1e-6
BN_EPS = 1e-4
BN_MOMENTUM = 0.1


# ---------------------------------------------------------------------------------------------------------------------
# spectral norm  (torch/nn/utils/spectral_norm.py:62-114; installed by src/utils/ops.py:195-224, eps 1e-6, 1 iteration)
# ---------------------------------------------------------------------------------------------------------------------
def sn_weight(sd, prefix, training=True, update=True):
    """Returns W / sigma (differentiable w.r.t. sd[prefix+'weight_orig']); updates u, v in ``sd`` like the hook does."""
    W = sd[prefix + "weight_orig"]
    u, v = sd[prefix + "weight_u"], sd[prefix + "weight_v"]
    Wm = W.reshape(W.shape[0], -1)
    if training:
        with torch.no_grad():
            v = F.normalize(torch.mv(Wm.t(), u), dim=0, eps=SN_EPS)
            u = F.normalize(torch.mv(Wm, v), dim=0, eps=SN_EPS)
        if update:
            sd[prefix + "weight_u"], sd[prefix + "weight_v"] = u.clone(), v.clone()
    sigma = torch.dot(u, torch.mv(Wm, v))
    return W / sigma


def weight(sd, prefix, training=True):
    """Weight of a (possibly spectrally-normalised) layer."""
    if prefix + "weight_orig" in sd:
        return sn_weight(sd, prefix, training)
    return sd[prefix + "weight"]


def conv(sd, prefix, x, padding, training=True):
    return F.conv2d(x, weight(sd, prefix, training), sd.get(prefix + "bias"), stride=1, padding=padding)


def linear(sd, prefix, x, training=True):
    return F.linear(x, weight(sd, prefix, training), sd.get(prefix + "bias"))


# ---------------------------------------------------------------------------------------------------------------------
# batch norm  (src/utils/ops.py:227-228 -> nn.BatchNorm2d eps 1e-4 momentum 0.1; F.batch_norm semantics)
# ---------------------------------------------------------------------------------------------------------------------
def batch_norm(sd, prefix, x, training=True, track=True, affine=False):
    if training:
        mean = x.mean(dim=(0, 2, 3))
        var = x.var(dim=(0, 2, 3), unbiased=False)
        if track:
            n = x.numel() / x.shape[1]
            with torch.no_grad():
                sd[prefix + "running_mean"] = (1 - BN_MOMENTUM) * sd[prefix + "running_mean"] + BN_MOMENTUM * mean
                sd[prefix + "running_var"] = (1 - BN_MOMENTUM) * sd[prefix + "running_var"] + BN_MOMENTUM * var * n / (n - 1)
                if prefix + "num_batches_tracked" in sd:
                    sd[prefix + "num_batches_tracked"] = sd[prefix + "num_batches_tracked"] + 1
    else:
        mean, var = sd[prefix + "running_mean"], sd[prefix + "running_var"]
    y = (x - mean[None, :, None, None]) * torch.rsqrt(var[None, :, None, None] + BN_EPS)
    if affine:
        y = y * sd[prefix + "weight"][None, :, None, None] + sd[prefix + "bias"][None, :, None, None]
    return y


def cbn(sd, prefix, x, y, training=True, track=True):
    """ops.ConditionalBatchNorm2d.forward (src/utils/ops.py:24-28)."""
    gain = (1 + linear(sd, prefix + "gain.", y, training)).view(y.size(0), -1, 1, 1)
    bias = linear(sd, prefix + "bias.", y, training).view(y.size(0), -1, 1, 1)
    return batch_norm(sd, prefix + "bn.", x, training, track) * gain + bias


# ---------------------------------------------------------------------------------------------------------------------
# self attention  (src/utils/ops.py:83-103)
# ---------------------------------------------------------------------------------------------------------------------
def self_attention(sd, prefix, x, training=True):
    B, ch, h, w = x.shape
    theta = conv(sd, prefix + "conv1x1_theta.", x, 0, training).view(-1, ch // 8, h * w)
    phi = F.max_pool2d(conv(sd, prefix + "conv1x1_phi.", x, 0, training), 2, 2).view(-1, ch // 8, h * w // 4)
    attn = torch.softmax(torch.bmm(theta.permute(0, 2, 1), phi), dim=-1)
    g = F.max_pool2d(conv(sd, prefix + "conv1x1_g.", x, 0, training), 2, 2).view(-1, ch // 2, h * w // 4)
    attn_g = torch.bmm(g, attn.permute(0, 2, 1)).view(-1, ch // 2, h, w)
    attn_g = conv(sd, prefix + "conv1x1_attn.", attn_g, 0, training)
    return x + sd[prefix + "sigma"] * attn_g


def softmax_from_partials(scores, part_width):
    """nn.Softmax(dim=-1) of src/utils/ops.py:95 computed the way the GEMM epilogues do (csrc/conv_epilogue.cuh, sm_mode 1 / 2):
    the key axis is cut into parts of ``part_width`` columns, every part keeps (max, sum exp(. - max)) of its columns, and the
    second pass merges the partials of a row into (m, l) and writes exp(s - m) / l.  Algebraically identical to the softmax."""
    N, M = scores.shape[-2:]
    parts = scores.split(part_width, dim=-1)
    m_t = torch.stack([p.max(-1).values for p in parts], -1)                       # [..., N, parts]
    l_t = torch.stack([(p - p.max(-1, keepdim=True).values).exp().sum(-1) for p in parts], -1)
    m = m_t.max(-1, keepdim=True).values
    l = (l_t * (m_t - m).exp()).sum(-1, keepdim=True)
    return (scores - m).exp() / l


def softmax_backward_with_delta(P, dO, V):
    """Backward of ``P = softmax(S); O = P @ V`` w.r.t. S as the dP GEMM's epilogue forms it (sm_mode 3):
    dS = P * (dP - delta) with dP = dO @ V^T and delta = rowsum(dO * O) -- equal to rowsum(P * dP), so dP need not exist."""
    O = P @ V
    delta = (dO * O).sum(-1, keepdim=True)
    return P * (dO @ V.transpose(-1, -2) - delta)


def relu_bit_planes(y_nhwc):
    """(y > 0) of a post-ReLU NHWC tensor as the conv epilogues store it (sgb_conv_desc.relu_bits): one little-endian 64-bit word
    per (pixel, 64-channel chunk), bit j = channel 64 * chunk + j, i.e. numpy's packbits(bitorder='little') over the channels."""
    return np.packbits(np.asarray(y_nhwc) > 0, axis=-1, bitorder="little")


# ---------------------------------------------------------------------------------------------------------------------
# BigGAN-Deep (legacy)  (src/models/big_resnet_deep_legacy.py)
# ---------------------------------------------------------------------------------------------------------------------
G_IN = {"32": [4, 4, 4], "64": [16, 8, 4, 2], "128": [16, 16, 8, 4, 2], "256": [16, 16, 8, 8, 4, 2]}
G_OUT = {"32": [4, 4, 4], "64": [8, 4, 2, 1], "128": [16, 8, 4, 2, 1], "256": [16, 8, 8, 4, 2, 1]}
D_IN = {"32": [4, 4, 4], "64": [1, 2, 4, 8], "128": [1, 2, 4, 8, 16], "256": [1, 2, 4, 8, 8, 16]}
D_OUT = {"32": [4, 4, 4], "64": [2, 4, 8, 16], "128": [2, 4, 8, 16, 16], "256": [2, 4, 8, 8, 16, 16]}
D_DOWN = {"32": [True, True, False, False], "64": [True, True, True, True, False],
          "128": [True, True, True, True, True, False], "256": [True, True, True, True, True, True, False]}


def deep_gen_block(sd, p, x, affine, out_channels, upsample, training=True, track=True):
    """GenBlock.forward (src/models/big_resnet_deep_legacy.py:49-73); with a ``conv2d0`` in the state dict it is the
    StudioGAN flavour (src/models/big_resnet_deep_studiogan.py:57-78): learnable 1x1 skip applied after the up-sampling."""
    studiogan = _has(sd, p + "conv2d0.")
    x0 = x if studiogan else (x[:, :out_channels] if x.shape[1] != out_channels else x)
    h = conv(sd, p + "conv2d1.", F.relu(cbn(sd, p + "bn1.", x, affine, training, track)), 0, training)
    h = F.relu(cbn(sd, p + "bn2.", h, affine, training, track))
    if upsample:
        h = F.interpolate(h, scale_factor=2, mode="nearest")
    h = conv(sd, p + "conv2d2.", h, 1, training)
    h = conv(sd, p + "conv2d3.", F.relu(cbn(sd, p + "bn3.", h, affine, training, track)), 1, training)
    h = conv(sd, p + "conv2d4.", F.relu(cbn(sd, p + "bn4.", h, affine, training, track)), 0, training)
    if upsample:
        x0 = F.interpolate(x0, scale_factor=2, mode="nearest")
    if studiogan:
        x0 = conv(sd, p + "conv2d0.", x0, 0, training)
    return h + x0


def deep_generator(sd, z, label, img_size, g_conv_dim, g_depth, attn_g_loc=(), apply_attn=False, training=True, track=True,
                   conditional=True):
    """Generator.forward (src/models/big_resnet_deep_legacy.py:153-184); ``sd`` is mutated like module buffers are."""
    key = str(img_size)
    in_dims = [g_conv_dim * m for m in G_IN[key]]
    out_dims = [g_conv_dim * m for m in G_OUT[key]]
    if conditional:
        z = torch.cat([F.embedding(label, sd["shared.weight"]), z], 1)
    affine = z
    act = linear(sd, "linear0.", z, training).view(-1, in_dims[0], 4, 4)
    bi = 0
    for index in range(len(in_dims)):
        for g_index in range(g_depth):
            oc = in_dims[index] if g_index == 0 else out_dims[index]
            act = deep_gen_block(sd, "blocks.%d.0." % bi, act, affine, oc, g_index == g_depth - 1, training, track)
            bi += 1
        if (index + 1) in attn_g_loc and apply_attn:
            act = self_attention(sd, "blocks.%d.0." % bi, act, training)
            bi += 1
    act = F.relu(batch_norm(sd, "bn4.", act, training, track, affine=True))
    return torch.tanh(conv(sd, "conv2d5.", act, 1, training))


def deep_disc_block(sd, p, x, downsample, training=True):
    """DiscBlock.forward (src/models/big_resnet_deep_legacy.py:210-229).

    NOTE the reference quirk: MODULES.d_act_fn is nn.ReLU(inplace=True) (src/config.py:486), so ``self.activation(x)``
    at :213 also rectifies ``x0`` (same storage).  The skip path therefore carries relu(x), not x."""
    x = F.relu(x)
    x0 = x
    h = conv(sd, p + "conv2d1.", x, 0, training)
    h = conv(sd, p + "conv2d2.", F.relu(h), 1, training)
    h = conv(sd, p + "conv2d3.", F.relu(h), 1, training)
    h = F.relu(h)
    if downsample:
        h = F.avg_pool2d(h, 2)
    h = conv(sd, p + "conv2d4.", h, 0, training)
    if downsample:
        x0 = F.avg_pool2d(x0, 2)
    if (p + "conv2d0.weight_orig") in sd or (p + "conv2d0.weight") in sd:
        x0 = torch.cat([x0, conv(sd, p + "conv2d0.", x0, 0, training)], 1)
    return h + x0


def deep_disc_block_studiogan(sd, p, x, downsample, optblock, training=True):
    """DiscBlock.forward of the StudioGAN flavour (src/models/big_resnet_deep_studiogan.py:233-253): pooling before the
    last activation, skip = conv2d0 (pool first in the opt block, conv first otherwise); the in-place activation
    rectifies the aliased skip tensor exactly as in the legacy variant."""
    x = F.relu(x)
    x0 = x
    h = conv(sd, p + "conv2d1.", x, 0, training)
    h = conv(sd, p + "conv2d2.", F.relu(h), 1, training)
    h = conv(sd, p + "conv2d3.", F.relu(h), 1, training)
    if downsample:
        h = F.avg_pool2d(h, 2)
    h = conv(sd, p + "conv2d4.", F.relu(h), 0, training)
    if optblock:
        x0 = conv(sd, p + "conv2d0.", F.avg_pool2d(x0, 2), 0, training)
    elif _has(sd, p + "conv2d0."):
        x0 = conv(sd, p + "conv2d0.", x0, 0, training)
        if downsample:
            x0 = F.avg_pool2d(x0, 2)
    return h + x0


def disc_head_pd(sd, h, label, training=True, cond="PD"):
    """Sum-pooled features -> adversarial logit (+ projection) (src/models/big_resnet_deep_legacy.py:344-372)."""
    adv = torch.squeeze(linear(sd, "linear1.", h, training))
    if cond == "PD":
        adv = adv + torch.sum(F.embedding(label, weight(sd, "embedding.", training)) * h, 1)
    return adv


def deep_discriminator(sd, x, label, img_size, d_conv_dim, d_depth, attn_d_loc=(), apply_attn=False, training=True,
                       cond="PD", studiogan=False):
    """Discriminator.forward (src/models/big_resnet_deep_legacy.py:334-413; studiogan=True: the same loop of
    src/models/big_resnet_deep_studiogan.py:345-424 with its block); returns (adv_output, h)."""
    key = str(img_size)
    in_dims = [d_conv_dim * m for m in D_IN[key]]
    down = D_DOWN[key]
    h = conv(sd, "input_conv.", x, 1, training)
    bi = 0
    for index in range(len(in_dims)):
        for d_index in range(d_depth):
            if studiogan:
                h = deep_disc_block_studiogan(sd, "blocks.%d.0." % bi, h, bool(down[index] and d_index == 0),
                                              index == 0 and d_index == 0, training)
            else:
                h = deep_disc_block(sd, "blocks.%d.0." % bi, h, bool(down[index] and d_index == 0), training)
            bi += 1
        if (index + 1) in attn_d_loc and apply_attn:
            h = self_attention(sd, "blocks.%d.0." % bi, h, training)
            bi += 1
    h = torch.sum(F.relu(h), dim=[2, 3])
    return disc_head_pd(sd, h, label, training, cond), h


# ---------------------------------------------------------------------------------------------------------------------
# losses  (src/utils/losses.py:197-239, 268-275, 301-316)
# ---------------------------------------------------------------------------------------------------------------------
def d_hinge(d_logit_real, d_logit_fake, DDP=False):
    return torch.mean(F.relu(1. - d_logit_real)) + torch.mean(F.relu(1. + d_logit_fake))


def g_hinge(d_logit_fake, DDP=False):
    return -torch.mean(d_logit_fake)


def d_wasserstein(d_logit_real, d_logit_fake, DDP=False):
    return torch.mean(d_logit_fake - d_logit_real)


def g_wasserstein(d_logit_fake, DDP=False):
    return -torch.mean(d_logit_fake)


def d_vanilla(d_logit_real, d_logit_fake, DDP=False):
    return torch.mean(F.softplus(-d_logit_real)) + torch.mean(F.softplus(d_logit_fake))


def g_vanilla(d_logit_fake, DDP=False):
    return torch.mean(F.softplus(-d_logit_fake))


def grad_penalty(disc_fn, real, fake, alpha):
    """cal_grad_penalty (src/utils/losses.py:301-316) with the CPU-drawn alpha passed in ([B,1] uniform)."""
    B, c, h, w = real.shape
    a = alpha.expand(B, real.nelement() // B).contiguous().view(B, c, h, w)
    interp = (a * real + (1 - a) * fake).detach().requires_grad_(True)
    out = disc_fn(interp)
    grads = torch.autograd.grad(outputs=out, inputs=interp, grad_outputs=torch.ones_like(out), create_graph=True,
                                retain_graph=True, only_inputs=True)[0]
    grads = grads.view(len(grads), -1)
    return ((grads.norm(2, dim=1) - 1) ** 2).mean() + interp[:, 0, 0, 0].mean() * 0


def bn_tangent(x, a, gamma, eps):
    """Tangent (JVP) of training-mode batch norm y = gamma * xhat + beta along a: gamma * r * (a - mean a - xhat * mean(xhat a)).
    (Jacobian of torch's native_batch_norm; identical to its backward map since the Jacobian is symmetric.)"""
    dims = (0, 2, 3)
    mu = x.mean(dims, keepdim=True)
    r = torch.rsqrt(x.var(dims, unbiased=False, keepdim=True) + eps)
    xh = (x - mu) * r
    g = gamma.view(1, -1, 1, 1) if gamma is not None else 1.0
    return g * r * (a - a.mean(dims, keepdim=True) - xh * (xh * a).mean(dims, keepdim=True))


def bn_tangent_backward(x, a, c, gamma, eps):
    """Derivatives of <c, bn_tangent(x, a, gamma)> w.r.t. (x, a, gamma): torch's batchnorm_double_backward
    (tools/autograd/templates/Functions.cpp) with gO := a, ggI := c, written with per-channel sums
    Sa, Sc, Sxa = sum xhat a, Sxc = sum xhat c, Sac = sum a c over M = B*H*W elements."""
    dims = (0, 2, 3)
    M = x.numel() // x.shape[1]
    mu = x.mean(dims, keepdim=True)
    r = torch.rsqrt(x.var(dims, unbiased=False, keepdim=True) + eps)
    xh = (x - mu) * r
    g = gamma.view(1, -1, 1, 1) if gamma is not None else torch.ones_like(r)
    Sa, Sc = a.sum(dims, keepdim=True), c.sum(dims, keepdim=True)
    Sxa, Sxc = (xh * a).sum(dims, keepdim=True), (xh * c).sum(dims, keepdim=True)
    Sac = (a * c).sum(dims, keepdim=True)
    T = Sa * Sc / M - Sac + 3.0 * Sxa * Sxc / M
    dx = g * r * r / M * (xh * T + Sxc * (Sa / M - a) + Sxa * (Sc / M - c))
    da = g * r * (c - Sc / M - xh * Sxc / M)
    dgamma = (r * (Sac - (Sa * Sc + Sxa * Sxc) / M)).reshape(-1)
    return dx, da, dgamma


# ---------------------------------------------------------------------------------------------------------------------
# EMA / Adam  (src/utils/ema.py:27-40; src/config.py:541-563 -> torch.optim.Adam, eps 1e-6)
# ---------------------------------------------------------------------------------------------------------------------
def ema_update(src_sd, ema_sd, decay, step, start_iter):
    d = 0.0 if step < start_iter else decay
    for k in src_sd:
        if k.endswith("num_batches_tracked"):
            ema_sd[k] = src_sd[k].clone()
        else:
            ema_sd[k] = src_sd[k] + d * (ema_sd[k] - src_sd[k])   # torch.lerp(src, ema, d)


def adam_step(p, g, m, v, step, lr, beta1, beta2, eps=1e-6):
    m = beta1 * m + (1 - beta1) * g
    v = beta2 * v + (1 - beta2) * g * g
    bc1, bc2 = 1 - beta1 ** step, 1 - beta2 ** step
    p = p - (lr / bc1) * m / (v.sqrt() / math.sqrt(bc2) + eps)
    return p, m, v


# ---------------------------------------------------------------------------------------------------------------------
# evaluation arithmetic  (src/utils/ops.py:251-263, src/utils/resize.py:83-91, src/metrics/{fid,ins,prdc}.py)
# ---------------------------------------------------------------------------------------------------------------------
def quantize_images(x):
    """ops.quantize_images (src/utils/ops.py:251-255): float [-1,1] -> uint8 with +0.5 and truncation."""
    x = (x + 1) / 2
    x = (255.0 * x + 0.5).clamp(0.0, 255.0)
    return x.detach().cpu().numpy().astype(np.uint8)


def resize_legacy(x_uint8_nchw, size=299):
    """'legacy' resizer (src/utils/resize.py:83-91): per-image F.interpolate bilinear align_corners=False, clip 0..255."""
    x = torch.from_numpy(x_uint8_nchw.astype(np.float32))
    x = F.interpolate(x, size=(size, size), mode="bilinear", align_corners=False)
    return x.clamp(0, 255)


def _pil_taps(in_size, out_size):
    """Pillow Resample.c::precompute_coeffs for the triangle ("bilinear", support 1) filter: per output coordinate the first
    source index and the normalised float64 weights."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = 1.0 * fs
    taps = []
    for o in range(out_size):
        center = (o + 0.5) * scale
        lo = max(int(center - support + 0.5), 0)
        hi = min(int(center + support + 0.5), in_size)
        w = np.array([max(0.0, 1.0 - abs((x + lo - center + 0.5) / fs)) for x in range(hi - lo)], dtype=np.float64)
        if w.sum() != 0.0:
            w = w / w.sum()
        taps.append((lo, w))
    return taps


def resize_friendly(x_uint8_nchw, size=299):
    """'friendly' resizer for InceptionV3_tf (src/utils/resize.py:50-53,72-82): PIL bilinear on every channel as a float32
    'F'-mode image.  Pillow's algorithm restated (ImagingResampleHorizontal_32bpc then ...Vertical_32bpc): separable,
    horizontal pass first, float64 accumulation of float32 pixels with float64 weights, float32 storage after each pass;
    the filter support grows with the down-scaling factor (anti-aliasing)."""
    x = np.asarray(x_uint8_nchw).astype(np.float32)
    B, C, H, W = x.shape
    tx, ty = _pil_taps(W, size), _pil_taps(H, size)
    hor = np.empty((B, C, H, size), dtype=np.float32)
    for o, (lo, w) in enumerate(tx):
        hor[..., o] = (x[..., lo:lo + len(w)].astype(np.float64) * w).sum(-1).astype(np.float32)
    out = np.empty((B, C, size, size), dtype=np.float32)
    for o, (lo, w) in enumerate(ty):
        out[:, :, o, :] = (hor[:, :, lo:lo + len(w), :].astype(np.float64) * w[None, None, :, None]).sum(2).astype(np.float32)
    return torch.from_numpy(out)


def normalize_for_inception(x255):
    """resize_images tail (src/utils/ops.py:262): x/255, (x-0.5)/0.5 for InceptionV3_tf."""
    return (x255 / 255.0 - 0.5) / 0.5


def calculate_kl_div(ps, splits=1):
    """ins.calculate_kl_div (src/metrics/ins.py:28-42)."""
    ps = np.asarray(ps, dtype=np.float64)
    scores = []
    n = ps.shape[0]
    for j in range(splits):
        part = ps[(j * n // splits):((j + 1) * n // splits), :]
        kl = part * (np.log(part) - np.log(np.mean(part, 0, keepdims=True)))
        scores.append(np.exp(np.mean(np.sum(kl, 1))))
    with np.errstate(all="ignore"):
        std = float(np.std(scores, ddof=1)) if len(scores) > 1 else float("nan")   # torch.std is unbiased: NaN for splits=1
    return float(np.mean(scores)), std


def moments(feats):
    """fid.calculate_moments tail (src/metrics/fid.py:96-97): mean and np.cov(rowvar=False)."""
    feats = np.asarray(feats)
    return np.mean(feats, axis=0), np.cov(feats, rowvar=False)


def frechet_distance(mu1, sigma1, mu2, sigma2, eps=1e-6):
    """fid.frechet_inception_distance (src/metrics/fid.py:34-62)."""
    from scipy import linalg
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    sigma1, sigma2 = np.atleast_2d(sigma1), np.atleast_2d(sigma2)
    diff = mu1 - mu2
    covmean = linalg.sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = linalg.sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError("Imaginary component {}".format(np.max(np.abs(covmean.imag))))
        covmean = covmean.real
    return float(diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean))


def prdc(real, fake, nearest_k=5):
    """prdc.compute_prdc (src/metrics/prdc.py:129-168): euclidean distances, k-th NN radii (self included)."""
    real, fake = np.asarray(real, dtype=np.float64), np.asarray(fake, dtype=np.float64)

    def dist(a, b):
        d2 = (a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2 * a @ b.T
        return np.sqrt(np.maximum(d2, 0))

    def kth(d, k):
        return np.partition(d, k, axis=-1)[:, k]     # (k+1)-th smallest, k = nearest_k because self-distance is 0

    rr, ff, rf = dist(real, real), dist(fake, fake), dist(real, fake)
    r_real, r_fake = kth(rr, nearest_k), kth(ff, nearest_k)
    precision = (rf < r_real[:, None]).any(axis=0).mean()
    recall = (rf < r_fake[None, :]).any(axis=1).mean()
    density = (1. / float(nearest_k)) * (rf < r_real[:, None]).sum(axis=0).mean()
    coverage = (rf.min(axis=1) < r_real).mean()
    return dict(precision=float(precision), recall=float(recall), density=float(density), coverage=float(coverage))


# ---------------------------------------------------------------------------------------------------------------------
# BigGAN (src/models/big_resnet.py) and ResNetGAN / SNGAN / WGAN-GP (src/models/resnet.py): shared block arithmetic
# ---------------------------------------------------------------------------------------------------------------------
R_G_IN = {"32": [4, 4, 4], "64": [16, 8, 4, 2], "128": [16, 16, 8, 4, 2], "256": [16, 16, 8, 8, 4, 2]}
R_G_OUT = {"32": [4, 4, 4], "64": [8, 4, 2, 1], "128": [16, 8, 4, 2, 1], "256": [16, 8, 8, 4, 2, 1]}
R_D_IN = {"32": [2, 2, 2], "64": [1, 2, 4, 8], "128": [1, 2, 4, 8, 16], "256": [1, 2, 4, 8, 8, 16]}
R_D_OUT = {"32": [2, 2, 2, 2], "64": [1, 2, 4, 8, 16], "128": [1, 2, 4, 8, 16, 16], "256": [1, 2, 4, 8, 8, 16, 16]}


def _gen_bn(sd, p, x, affine, training, track):
    if (p + "gain.weight_orig") in sd or (p + "gain.weight") in sd:
        return cbn(sd, p, x, affine, training, track)
    return batch_norm(sd, p, x, training, track, affine=True)


def res_gen_block(sd, p, x, affine, training=True, track=True):
    """GenBlock.forward (src/models/big_resnet.py:28-42 == src/models/resnet.py:35-59)."""
    x0 = x
    h = F.relu(_gen_bn(sd, p + "bn1.", x, affine, training, track))
    h = F.interpolate(h, scale_factor=2, mode="nearest")
    h = conv(sd, p + "conv2d1.", h, 1, training)
    h = F.relu(_gen_bn(sd, p + "bn2.", h, affine, training, track))
    h = conv(sd, p + "conv2d2.", h, 1, training)
    x0 = F.interpolate(x0, scale_factor=2, mode="nearest")
    x0 = conv(sd, p + "conv2d0.", x0, 0, training)
    return h + x0


def biggan_generator(sd, z, label, img_size, g_conv_dim, attn_g_loc=(), apply_attn=False, training=True, track=True):
    """Generator.forward of BigGAN (src/models/big_resnet.py:122-158): z chunks, cBN on [shared, chunk]."""
    key = str(img_size)
    in_dims = [g_conv_dim * m for m in R_G_IN[key]]
    nb = len(in_dims)
    chunk = z.shape[1] // (nb + 1)
    zs = torch.split(z, chunk, 1)
    shared = F.embedding(label, sd["shared.weight"])
    affines = [torch.cat([shared, item], 1) for item in zs[1:]]
    act = linear(sd, "linear0.", zs[0], training).view(-1, in_dims[0], 4, 4)
    bi, counter = 0, 0
    for index in range(nb):
        act = res_gen_block(sd, "blocks.%d.0." % bi, act, affines[counter], training, track)
        bi += 1
        counter += 1
        if (index + 1) in attn_g_loc and apply_attn:
            act = self_attention(sd, "blocks.%d.0." % bi, act, training)
            bi += 1
    act = F.relu(batch_norm(sd, "bn4.", act, training, track, affine=True))
    return torch.tanh(conv(sd, "conv2d5.", act, 1, training))


def resnet_generator(sd, z, label, img_size, g_conv_dim, num_classes, conditional=True, attn_g_loc=(), apply_attn=False,
                     training=True, track=True):
    """Generator.forward of ResNetGAN (src/models/resnet.py:137-169): cBN conditioned on one-hot labels, or plain BN."""
    key = str(img_size)
    in_dims = [g_conv_dim * m for m in R_G_IN[key]]
    affine = F.one_hot(label, num_classes=num_classes).to(torch.float32) if conditional else None
    act = linear(sd, "linear0.", z, training).view(-1, in_dims[0], 4, 4)
    bi = 0
    for index in range(len(in_dims)):
        act = res_gen_block(sd, "blocks.%d.0." % bi, act, affine, training, track)
        bi += 1
        if (index + 1) in attn_g_loc and apply_attn:
            act = self_attention(sd, "blocks.%d.0." % bi, act, training)
            bi += 1
    act = F.relu(batch_norm(sd, "bn4.", act, training, track, affine=True))
    return torch.tanh(conv(sd, "conv2d5.", act, 1, training))


def _has(sd, key):
    return (key + "weight_orig") in sd or (key + "weight") in sd


def res_disc_opt_block(sd, p, x, training=True):
    """DiscOptBlock.forward (src/models/big_resnet.py:177-192 == src/models/resnet.py:189-204)."""
    sn = (p + "bn1.weight") not in sd
    x0 = x
    h = conv(sd, p + "conv2d1.", x, 1, training)
    if not sn:
        h = batch_norm(sd, p + "bn1.", h, training, True, affine=True)
    h = conv(sd, p + "conv2d2.", F.relu(h), 1, training)
    h = F.avg_pool2d(h, 2)
    x0 = F.avg_pool2d(x0, 2)
    if not sn:
        x0 = batch_norm(sd, p + "bn0.", x0, training, True, affine=True)
    return h + conv(sd, p + "conv2d0.", x0, 0, training)


def res_disc_block(sd, p, x, downsample, training=True):
    """DiscBlock.forward (src/models/big_resnet.py:223-242 == src/models/resnet.py:233-254).  With spectral norm the
    in-place ReLU (src/config.py:486) also rectifies the aliased skip input; with BN in between it does not."""
    sn = (p + "bn1.weight") not in sd
    if sn:
        x = F.relu(x)
        x0 = x
        h = x
    else:
        x0 = x
        h = F.relu(batch_norm(sd, p + "bn1.", x, training, True, affine=True))
    h = conv(sd, p + "conv2d1.", h, 1, training)
    if not sn:
        h = batch_norm(sd, p + "bn2.", h, training, True, affine=True)
    h = conv(sd, p + "conv2d2.", F.relu(h), 1, training)
    if downsample:
        h = F.avg_pool2d(h, 2)
    if _has(sd, p + "conv2d0."):
        if not sn:
            x0 = batch_norm(sd, p + "bn0.", x0, training, True, affine=True)
        x0 = conv(sd, p + "conv2d0.", x0, 0, training)
        if downsample:
            x0 = F.avg_pool2d(x0, 2)
    return h + x0


def res_discriminator(sd, x, label, img_size, d_conv_dim, attn_d_loc=(), apply_attn=False, training=True, cond="PD"):
    """Discriminator.forward of BigGAN / ResNetGAN (src/models/big_resnet.py:349-428, src/models/resnet.py:363-442)."""
    key = str(img_size)
    n = len(R_D_IN[key]) + 1
    down = D_DOWN[key]
    h = x
    bi = 0
    for index in range(n):
        if index == 0:
            h = res_disc_opt_block(sd, "blocks.%d.0." % bi, h, training)
        else:
            h = res_disc_block(sd, "blocks.%d.0." % bi, h, down[index], training)
        bi += 1
        if (index + 1) in attn_d_loc and apply_attn:
            h = self_attention(sd, "blocks.%d.0." % bi, h, training)
            bi += 1
    h = torch.sum(F.relu(h), dim=[2, 3])
    return disc_head_pd(sd, h, label, training, cond), h


# ---------------------------------------------------------------------------------------------------------------------
# FID InceptionV3  (src/metrics/inception_net.py:16-249) on top of torchvision's module definitions (the reference builds
# on torchvision.models.inception_v3 too, :117) with the TF-compatible pooling of FIDInceptionA/C/E_1/E_2 restated here.
# ---------------------------------------------------------------------------------------------------------------------
def _fid_a(m, x):
    b1 = m.branch1x1(x)
    b5 = m.branch5x5_2(m.branch5x5_1(x))
    d = m.branch3x3dbl_3(m.branch3x3dbl_2(m.branch3x3dbl_1(x)))
    bp = m.branch_pool(F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False))
    return torch.cat([b1, b5, d, bp], 1)


def _fid_c(m, x):
    b1 = m.branch1x1(x)
    s = m.branch7x7_3(m.branch7x7_2(m.branch7x7_1(x)))
    d = m.branch7x7dbl_5(m.branch7x7dbl_4(m.branch7x7dbl_3(m.branch7x7dbl_2(m.branch7x7dbl_1(x)))))
    bp = m.branch_pool(F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False))
    return torch.cat([b1, s, d, bp], 1)


def _fid_e(m, x, use_max):
    b1 = m.branch1x1(x)
    t = m.branch3x3_1(x)
    b3 = torch.cat([m.branch3x3_2a(t), m.branch3x3_2b(t)], 1)
    t = m.branch3x3dbl_2(m.branch3x3dbl_1(x))
    d = torch.cat([m.branch3x3dbl_3a(t), m.branch3x3dbl_3b(t)], 1)
    pooled = F.max_pool2d(x, kernel_size=3, stride=1, padding=1) if use_max else \
        F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False)
    return torch.cat([b1, b3, d, m.branch_pool(pooled)], 1)


def fid_inception(state_dict):
    """torchvision Inception3(1008 classes, no aux) in eval mode carrying ``state_dict`` (torchvision key layout)."""
    import torchvision
    net = torchvision.models.inception_v3(num_classes=1008, aux_logits=False, weights=None, init_weights=False)
    net.load_state_dict(state_dict)
    return net.eval()


@torch.no_grad()
def fid_inception_forward(net, x):
    """InceptionV3.forward (src/metrics/inception_net.py:81-107) with resize_input=False, normalize_input=False:
    x is the normalised 299x299 batch; returns (pool [B,2048], logits [B,1008])."""
    x = net.Conv2d_2b_3x3(net.Conv2d_2a_3x3(net.Conv2d_1a_3x3(x)))
    x = F.max_pool2d(x, kernel_size=3, stride=2)
    x = net.Conv2d_4a_3x3(net.Conv2d_3b_1x1(x))
    x = F.max_pool2d(x, kernel_size=3, stride=2)
    x = _fid_a(net.Mixed_5b, x)
    x = _fid_a(net.Mixed_5c, x)
    x = _fid_a(net.Mixed_5d, x)
    x = net.Mixed_6a(x)
    for name in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
        x = _fid_c(getattr(net, name), x)
    x = net.Mixed_7a(x)
    x = _fid_e(net.Mixed_7b, x, False)
    x = _fid_e(net.Mixed_7c, x, True)
    x = torch.flatten(F.adaptive_avg_pool2d(x, (1, 1)), 1)
    return x, net.fc(x)


def eval_preprocess(images, size=299, quantize=True):
    """LoadEvalModel.get_outputs pre-processing for InceptionV3_tf with the default 'legacy' resizer
    (src/metrics/preparation.py:103-108, src/utils/ops.py:251-263): returns the normalised [B,3,size,size] batch."""
    q = quantize_images(images) if quantize else images.detach().cpu().numpy().astype(np.uint8)
    return normalize_for_inception(resize_legacy(q, size))


# ---------------------------------------------------------------------------------------------------------------------
# DCGAN (src/models/deep_conv.py) -- BASELINE config 1, the reference's CPU-only case.  Oracle level only: the product
# has no sm_90a kernel for the 4x4 / stride-2 (transposed) convolutions (DESIGN.md, out of scope).
# ---------------------------------------------------------------------------------------------------------------------
def dcgan_generator(sd, z, label=None, training=True, track=True):
    """Generator.forward (src/models/deep_conv.py:96-126), unconditional (g_cond_mtd W/O, info N/A):
    linear0 -> [B,512,4,4] -> 3 x (ConvTranspose 4x4 s2 p1 -> BN -> ReLU) -> conv3x3 -> tanh."""
    act = linear(sd, "linear0.", z, training).view(-1, 512, 4, 4)
    for i in range(3):
        p = "blocks.%d.0." % i
        w = sd[p + "deconv0.weight"]                                   # [Cin, Cout, 4, 4]
        act = F.conv_transpose2d(act, w, sd.get(p + "deconv0.bias"), stride=2, padding=1)
        act = F.relu(batch_norm(sd, p + "bn0.", act, training, track, affine=True))
    return torch.tanh(conv(sd, "conv4.", act, 1, training))


def dcgan_discriminator(sd, x, label=None, training=True):
    """Discriminator.forward (src/models/deep_conv.py:233-...): 3 x (conv3x3 -> BN -> ReLU -> conv4x4 s2 p1 -> BN -> ReLU),
    conv3x3 256->512 -> BN -> ReLU -> sum over (H, W) -> linear1.  Returns (adv_output, h)."""
    h = x
    for i in range(3):
        p = "blocks.%d.0." % i
        h = F.relu(batch_norm(sd, p + "bn0.", conv(sd, p + "conv0.", h, 1, training), training, True, affine=True))
        h = F.conv2d(h, weight(sd, p + "conv1.", training), sd.get(p + "conv1.bias"), stride=2, padding=1)
        h = F.relu(batch_norm(sd, p + "bn1.", h, training, True, affine=True))
    h = F.relu(batch_norm(sd, "bn1.", conv(sd, "conv1.", h, 1, training), training, True, affine=True))
    h = torch.sum(h, dim=[2, 3])
    return torch.squeeze(linear(sd, "linear1.", h, training)), h


def diffaug_closed_form(x, params, color=True, translation=True, cutout=True):
    """DiffAugment "color,translation,cutout" (src/utils/diffaug.py:47-100) for given per-sample parameters
    params[b] = (brightness offset, saturation factor, contrast factor, shift_h, shift_w, cut_h0, cut_w0): the reference's seven
    passes restated as the closed form the device kernel evaluates (differentiable w.r.t. x through torch autograd)."""
    B, C, H, W = x.shape
    p = params.to(x.dtype)
    y = x
    if color:
        y = y + p[:, 0].view(B, 1, 1, 1)
        m1 = y.mean(dim=1, keepdim=True)
        y = (y - m1) * p[:, 1].view(B, 1, 1, 1) + m1
        m2 = y.mean(dim=[1, 2, 3], keepdim=True)
        y = (y - m2) * p[:, 2].view(B, 1, 1, 1) + m2
    hh = torch.arange(H).view(1, H, 1)
    ww = torch.arange(W).view(1, 1, W)
    if translation:
        hs = hh + p[:, 3].long().view(B, 1, 1)
        ws = ww + p[:, 4].long().view(B, 1, 1)
        inside = ((hs >= 0) & (hs < H) & (ws >= 0) & (ws < W)).unsqueeze(1)
        idx_b = torch.arange(B).view(B, 1, 1).expand(B, H, W)
        g = y.permute(0, 2, 3, 1)[idx_b, hs.clamp(0, H - 1).expand(B, H, W), ws.clamp(0, W - 1).expand(B, H, W)].permute(0, 3, 1, 2)
        y = g * inside.to(x.dtype)
    if cutout:
        ch, cw = int(H * 0.5 + 0.5), int(W * 0.5 + 0.5)
        h0 = (p[:, 5].long() - ch // 2).view(B, 1, 1)
        w0 = (p[:, 6].long() - cw // 2).view(B, 1, 1)
        box = (hh >= h0.clamp(min=0)) & (hh <= (h0 + ch - 1).clamp(max=H - 1)) & (ww >= w0.clamp(min=0)) & (ww <= (w0 + cw - 1).clamp(max=W - 1))
        y = y * (~box).unsqueeze(1).to(x.dtype)
    return y


def cr_aug_closed_form(x, flip, tx, ty):
    """cr.apply_cr_aug (src/utils/cr.py:13-50) for given draws: mirror along w where ``flip``, then read at
    (reflect(h + tx), reflect(w + ty))."""
    B, C, H, W = x.shape

    def refl(i, n):
        i = i.abs()
        return torch.where(i >= n, 2 * (n - 1) - i, i)
    xf = torch.where(flip.view(B, 1, 1, 1).bool(), x.flip(3), x)
    hs = refl(torch.arange(H).view(1, H, 1) + tx.long().view(B, 1, 1), H).expand(B, H, W)
    ws = refl(torch.arange(W).view(1, 1, W) + ty.long().view(B, 1, 1), W).expand(B, H, W)
    idx_b = torch.arange(B).view(B, 1, 1).expand(B, H, W)
    return xf.permute(0, 2, 3, 1)[idx_b, hs, ws].permute(0, 3, 1, 2)


def seeded_state(keys_shapes, seed):
    """Deterministic weights for a (key, shape) list: used for the DCGAN fixture, whose 6.4 M parameters are regenerated
    from the seed on both sides instead of being stored (conv / linear weights ~ N(0, 0.05^2), BN weight 1 + 0.1 N,
    biases 0.1 N, running_mean 0.1 N, running_var 1 + 0.2 U, counters 0)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in keys_shapes:
        shape = tuple(int(v) for v in shape)
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.zeros(shape, dtype=torch.long)
        elif k.endswith("running_var"):
            sd[k] = 1.0 + 0.2 * torch.rand(shape, generator=g)
        elif k.endswith("running_mean") or k.endswith("bias"):
            sd[k] = 0.1 * torch.randn(shape, generator=g)
        elif ".bn" in k or k.startswith("bn"):
            sd[k] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif k.startswith("linear1."):
            # small output head: keeps the logits O(1).  With saturated logits every sample gets the same loss gradient and
            # the BatchNorm backward (dy - mean(dy) - ...) cancels catastrophically -- the reference's own fp32 gradients
            # are then only good to ~1e-2, which would make the fixture a noise comparison.
            sd[k] = 0.001 * torch.randn(shape, generator=g)
        else:
            sd[k] = 0.05 * torch.randn(shape, generator=g)
    return sd
