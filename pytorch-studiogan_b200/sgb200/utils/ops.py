"""Operator library behind ``cfgs.MODULES`` — same factory names, signatures and state_dict keys as the reference
``src/utils/ops.py`` (conv2d / snconv2d / linear / snlinear / embedding / sn_embedding / batchnorm_2d /
ConditionalBatchNorm2d / SelfAttention / init_weights), but every forward runs libsgb200 kernels on NHWC bf16
activations.  Modules subclass nn.Conv2d / nn.Linear / nn.Embedding / nn.BatchNorm2d so that the reference's
``isinstance`` based toggles (src/utils/misc.py:192-267,345-364) keep matching.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn import init

from .. import autograd_ops as A

SN_EPS = 1e-6  # src/utils/ops.py:204,216,220,224


def _apply_spectral_norm(module, eps=SN_EPS):
    """Re-registers ``weight`` as ``weight_orig`` and draws u, v exactly like torch.nn.utils.spectral_norm
    (torch/nn/utils/spectral_norm.py:128-160): u ~ normalize(N(0,1)^h), v ~ normalize(N(0,1)^w), dim = 0."""
    weight = module._parameters.pop("weight")
    h = weight.shape[0]
    w = weight.numel() // h
    with torch.no_grad():
        u = F.normalize(weight.new_empty(h).normal_(0, 1), dim=0, eps=eps)
        v = F.normalize(weight.new_empty(w).normal_(0, 1), dim=0, eps=eps)
    module.register_parameter("weight_orig", weight)
    module.register_buffer("weight_u", u)
    module.register_buffer("weight_v", v)
    module._sn = A.SpectralNormState(module, eps)


def _w(module):
    return module.weight_orig if hasattr(module, "weight_orig") else module.weight


def _sn_divided(module):
    """W / sigma of a spectrally-normalised module whose weight is used as a tensor (image convs, embeddings, head layers):
    sigma from the library's power iteration (in train mode, as the reference's hook); where W needs a gradient, sigma is
    formed again as u . (W v) with u, v held constant, so that the gradient reaches ``weight_orig`` through ordinary autograd."""
    W = module.weight_orig
    sigma = module._sn.sigma(module.training)
    if torch.is_grad_enabled() and W.requires_grad:
        sigma = torch.dot(module.weight_u.detach().clone(), torch.mv(W.reshape(W.shape[0], -1), module.weight_v.detach().clone()))
    return W / sigma


class _ConvBase(nn.Conv2d):
    """Stride-1 convolution on the wgmma engine (3x3 / 1x1 as used by every BigGAN / ResNetGAN block)."""
    spectral = False

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True):
        super().__init__(in_channels, out_channels, kernel_size, stride=stride, padding=padding, dilation=dilation,
                         groups=groups, bias=bias)
        strided = self.stride == (2, 2) and self.kernel_size == (4, 4) and self.padding == (1, 1)     # DCGAN's down-sampling conv
        if (self.stride != (1, 1) and not strided) or self.dilation != (1, 1) or self.groups != 1 or self.padding[0] != self.padding[1]:
            raise NotImplementedError("sgb200 conv engine: stride-1 (or 4x4 / stride-2 / pad-1), dilation-1, groups-1 square-padded "
                                      "convolutions only")
        if self.spectral:
            _apply_spectral_norm(self)

    def forward(self, x, residual=None, relu=False, premasked=False, mask_input=False, res_up2=False):
        if self.in_channels == 3 and self.kernel_size == (3, 3) and self.padding == (1, 1):
            return self._forward_image(x, residual, relu, premasked)
        cfg = {"KH": self.kernel_size[0], "KW": self.kernel_size[1], "pad": self.padding[0], "relu": relu,
               "premasked": premasked, "mask_input": mask_input, "res_up2": res_up2, "stride": self.stride[0],
               "sn": getattr(self, "_sn", None), "do_power_iteration": self.training,
               "sn_cache": getattr(self, "_sn_cache", None), "sn_pass": getattr(self, "_sn_pass", None)}
        return A.ConvFn.call(x, _w(self), self.bias, residual, cfg)

    def _forward_image(self, x_col, residual, relu, premasked):
        """3 -> C convolution on an image: ``x_col`` is the [B, 32, H, W] patch tensor from ImageColFn and the layer runs
        as a K = 32 GEMM.  The [Cout, 3, 3, 3] weight (864..3456 numbers) is re-ordered to [Cout, (tap, c)] with tensor
        ops (spectral norm: _sn_divided)."""
        W = _sn_divided(self) if hasattr(self, "_sn") else self.weight
        Wp = W.permute(0, 2, 3, 1).reshape(W.shape[0], 27)
        cfg = {"KH": 1, "KW": 1, "pad": 0, "relu": relu, "premasked": premasked, "sn": None}
        return A.ConvFn.call(x_col, Wp, self.bias, residual, cfg)


class Conv2d(_ConvBase):
    spectral = False


class SNConv2d(_ConvBase):
    spectral = True


class _LinearBase(nn.Linear):
    """Linear layer as a 1x1 'convolution' over a [B, K, 1, 1] bf16 activation; returns [B, N, 1, 1].
    perm_S > 1 emits the output features in NHWC order (see sgb_weight_pack)."""
    spectral = False

    def __init__(self, in_features, out_features, bias=True):
        super().__init__(in_features, out_features, bias=bias)
        if self.spectral:
            _apply_spectral_norm(self)

    def forward(self, x, out_fp32=False, perm_S=1):
        if x.dim() == 2:
            x = A.ToBF16Fn.call(x) if x.dtype != torch.bfloat16 else x.view(x.shape[0], x.shape[1], 1, 1)
        bias = self.bias
        if bias is not None and perm_S > 1:
            bias = bias.view(-1, perm_S).t().reshape(-1)
        cfg = {"KH": 1, "KW": 1, "pad": 0, "relu": False, "out_fp32": out_fp32, "perm_S": perm_S,
               "sn": getattr(self, "_sn", None), "do_power_iteration": self.training,
               "sn_cache": getattr(self, "_sn_cache", None), "sn_pass": getattr(self, "_sn_pass", None)}
        return A.ConvFn.call(x, _w(self), bias, None, cfg)


class Linear(_LinearBase):
    spectral = False


class SNLinear(_LinearBase):
    spectral = True


class Embedding(nn.Embedding):
    pass


class SNEmbedding(nn.Embedding):
    """Spectrally-normalised embedding (projection discriminator, src/utils/ops.py:223-224).  The table is tiny
    ([num_classes, C]); sigma comes from the library's power-iteration kernel, the lookup itself is indexing."""

    def __init__(self, num_embeddings, embedding_dim):
        super().__init__(num_embeddings, embedding_dim)
        _apply_spectral_norm(self)

    def forward(self, label):
        return F.embedding(label, _sn_divided(self))


def conv2d(in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True):
    return Conv2d(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)


def snconv2d(in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True):
    return SNConv2d(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)


def linear(in_features, out_features, bias=True):
    return Linear(in_features, out_features, bias)


def snlinear(in_features, out_features, bias=True):
    return SNLinear(in_features, out_features, bias)


def embedding(num_embeddings, embedding_dim):
    return Embedding(num_embeddings, embedding_dim)


def sn_embedding(num_embeddings, embedding_dim):
    return SNEmbedding(num_embeddings, embedding_dim)


class ConvTranspose2d(nn.ConvTranspose2d):
    """nn.ConvTranspose2d(kernel 4, stride 2, padding 1) of the DCGAN generator on the stride-1 conv engine
    (autograd_ops.ConvTranspose4x4s2Fn)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=2, padding=0, dilation=1, groups=1, bias=True):
        super().__init__(in_channels, out_channels, kernel_size, stride=stride, padding=padding, dilation=dilation, groups=groups,
                         bias=bias)
        if self.kernel_size != (4, 4) or self.stride != (2, 2) or self.padding != (1, 1) or self.dilation != (1, 1) or \
                self.groups != 1 or self.output_padding != (0, 0):
            raise NotImplementedError("sgb200: transposed convolution with kernel 4 / stride 2 / padding 1 only (DCGAN)")

    def forward(self, x):
        return A.ConvTranspose4x4s2Fn.call(x, self.weight, self.bias)


def deconv2d(in_channels, out_channels, kernel_size, stride=2, padding=0, dilation=1, groups=1, bias=True):
    return ConvTranspose2d(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)


def sndeconv2d(*args, **kwargs):
    raise NotImplementedError("spectrally-normalised ConvTranspose2d (dim = 1 power iteration) is not on any BASELINE config")


class BatchNorm2d(nn.BatchNorm2d):
    """nn.BatchNorm2d whose forward is the fused stats -> (NCCL all-reduce) -> scale/shift [+ReLU] [+nearest x2] path.
    ``sync_group`` is set by models.model.prepare_parallel_training instead of converting to torch SyncBatchNorm."""
    sync_group = None
    # True: the inverse std of the reference's DataParallel-mode SynchronizedBatchNorm, bias_var.clamp(eps) ** -0.5
    # (src/sync_batchnorm/batchnorm.py:158-175), instead of torch's (var + eps) ** -0.5.  DataParallel replicas themselves
    # are not supported (DDP only); the switch exists so that statistics trained under that mode can be reproduced.
    dp_sync_semantics = False

    def forward(self, x, relu=False, up2=False, gain=None, bias=None):
        training = self.training or (self.running_mean is None)
        track = self.training and self.track_running_stats and self.running_mean is not None
        if track and self.num_batches_tracked is not None:
            self.num_batches_tracked.add_(1)
        if gain is not None:
            mode, g, b = 0, gain, bias
        elif self.affine:
            mode, g, b = 1, self.weight, self.bias
        else:
            mode, g, b = 2, None, None
        cfg = {"mode": mode, "relu": relu, "up2": up2, "use_batch_stats": training, "track": track,
               "momentum": self.momentum if self.momentum is not None else 0.1, "eps": self.eps,
               "group": self.sync_group if training else None, "clamp_eps": self.dp_sync_semantics}
        return A.BNActFn.call(x, g, b, self.running_mean, self.running_var, cfg)


def batchnorm_2d(in_features, eps=1e-4, momentum=0.1, affine=True):
    return BatchNorm2d(in_features, eps=eps, momentum=momentum, affine=affine, track_running_stats=True)


class ConditionalBatchNorm2d(nn.Module):
    """out = bn(x) * (1 + gain(y)) + bias(y)  (src/utils/ops.py:14-28); ``y`` is the [B, K, 1, 1] bf16 conditioning
    activation shared by all cBN layers of a generator pass.  ReLU and the nearest x2 upsample that follow in every
    generator block are fused into the same pass."""

    def __init__(self, in_features, out_features, MODULES):
        super().__init__()
        self.in_features = in_features
        self.bn = batchnorm_2d(out_features, eps=1e-4, momentum=0.1, affine=False)
        self.gain = MODULES.g_linear(in_features=in_features, out_features=out_features, bias=False)
        self.bias = MODULES.g_linear(in_features=in_features, out_features=out_features, bias=False)
        self.gain._cbn_affine = self.bias._cbn_affine = True        # snbatch keeps these packs contiguous (cbn_affine_all)

    def forward(self, x, y, relu=False, up2=False):
        pre_g, pre_b = getattr(self.gain, "_pre_out", None), getattr(self.bias, "_pre_out", None)
        if pre_g is not None and pre_b is not None and not torch.is_grad_enabled():
            # gradient-free pass of a generator whose cBN layers all see the same y: their affine maps were computed by ONE GEMM
            self.gain._pre_out = self.bias._pre_out = None
            return self.bn(x, relu=relu, up2=up2, gain=pre_g, bias=pre_b)
        gain = self.gain(y, out_fp32=True)
        bias = self.bias(y, out_fp32=True)
        return self.bn(x, relu=relu, up2=up2, gain=gain, bias=bias)


class SelfAttention(nn.Module):
    """Non-local block of SAGAN / BigGAN (src/utils/ops.py:31-103): same sub-module names and shapes."""

    def __init__(self, in_channels, is_generator, MODULES):
        super().__init__()
        self.in_channels = in_channels
        mk = MODULES.g_conv2d if is_generator else MODULES.d_conv2d
        self.conv1x1_theta = mk(in_channels=in_channels, out_channels=in_channels // 8, kernel_size=1, stride=1, padding=0,
                                bias=False)
        self.conv1x1_phi = mk(in_channels=in_channels, out_channels=in_channels // 8, kernel_size=1, stride=1, padding=0,
                              bias=False)
        self.conv1x1_g = mk(in_channels=in_channels, out_channels=in_channels // 2, kernel_size=1, stride=1, padding=0,
                            bias=False)
        self.conv1x1_attn = mk(in_channels=in_channels // 2, out_channels=in_channels, kernel_size=1, stride=1, padding=0,
                               bias=False)
        self.maxpool = nn.MaxPool2d(2, stride=2, padding=0)
        self.softmax = nn.Softmax(dim=-1)
        self.sigma = nn.Parameter(torch.zeros(1), requires_grad=True)

    def forward(self, x):
        mods = (self.conv1x1_theta, self.conv1x1_phi, self.conv1x1_g, self.conv1x1_attn)
        cfgs = tuple({"sn": getattr(m, "_sn", None), "do_power_iteration": m.training, "sn_cache": getattr(m, "_sn_cache", None), "sn_pass": getattr(m, "_sn_pass", None)}
                     for m in mods)
        return A.SelfAttentionFn.call(x, _w(mods[0]), _w(mods[1]), _w(mods[2]), _w(mods[3]), self.sigma, cfgs)


class LeCamEMA(object):
    """Exponential moving averages of the discriminator's mean logits / losses for the LeCam regulariser
    (src/utils/ops.py:106-132; host-side floats, five numbers)."""

    def __init__(self, init=7777, decay=0.9, start_iter=0):
        self.G_loss = self.D_loss_real = self.D_loss_fake = self.D_real = self.D_fake = init
        self.decay, self.start_itr = decay, start_iter

    def update(self, cur, mode, itr):
        decay = 0.0 if itr < self.start_itr else self.decay
        if mode not in ("G_loss", "D_loss_real", "D_loss_fake", "D_real", "D_fake"):
            raise KeyError(mode)
        setattr(self, mode, getattr(self, mode) * decay + cur * (1 - decay))


def init_weights(modules, initialize):
    """Same traversal and RNG consumption as src/utils/ops.py:135-162 (the reference initialises the spectral-norm
    modules through the ``weight`` alias of ``weight_orig``; here the parameter is addressed directly)."""
    for module in modules():
        if isinstance(module, (nn.Conv2d, nn.ConvTranspose2d, nn.Linear)):
            w = _w(module)
            if initialize == "ortho":
                init.orthogonal_(w)
            elif initialize == "N02":
                init.normal_(w, 0, 0.02)
            elif initialize in ["glorot", "xavier"]:
                init.xavier_uniform_(w)
            else:
                continue
            if module.bias is not None:
                module.bias.data.fill_(0.)
        elif isinstance(module, nn.Embedding):
            w = _w(module)
            if initialize == "ortho":
                init.orthogonal_(w)
            elif initialize == "N02":
                init.normal_(w, 0, 0.02)
            elif initialize in ["glorot", "xavier"]:
                init.xavier_uniform_(w)


def quantize_images(x):
    """src/utils/ops.py:251-255 (host path kept for API parity; the eval pipeline uses the fused device kernel)."""
    x = (x + 1) / 2
    x = (255.0 * x + 0.5).clamp(0.0, 255.0)
    return x.detach().cpu().numpy().astype(np.uint8)


# ----------------------------------------------------------------------------------------------------------------------
# Discriminator head.  After the sum-pool the features are a [B, C] fp32 matrix; the remaining arithmetic (one GEMV,
# one embedding row product per image) is a few kFLOP and is expressed directly on those tensors.  Spectral norm of the
# head layers still goes through the library's power-iteration kernel so u / v evolve exactly like every other layer.
# ----------------------------------------------------------------------------------------------------------------------
_HEAD_KEYS = ["embed", "proxy", "cls_output", "mi_embed", "mi_proxy", "mi_cls_output", "info_discrete_c_logits", "info_conti_mu",
              "info_conti_var"]


def _head_weight(module):
    return _sn_divided(module) if hasattr(module, "_sn") else module.weight


class _HeadTangent:
    """Tangent of the adversarial logit w.r.t. the pooled features (the head is linear in h): same effective weights,
    same embedding rows, no bias, no new power iteration."""

    @staticmethod
    def tangent(args, out, tan):
        h, w_eff, emb, mtd = args
        th = tan(h)
        if th is None:
            return None
        if mtd not in ("W/O", "PD"):
            raise NotImplementedError("gradient penalty with d_cond_mtd=%s" % mtd)
        t = torch.squeeze(F.linear(th, w_eff))
        if emb is not None:
            t = t + torch.sum(emb * th, 1)
        return t


def head_linear(module, h):
    return F.linear(h, _head_weight(module), module.bias)


def discriminator_head(D, h, label, adc_fake=False):
    """Everything after ``h = sum(relu(features), [2, 3])`` in the reference discriminators
    (src/models/big_resnet_deep_legacy.py:347-413; identical in big_resnet.py / resnet.py): adversarial logit,
    class conditioning (PD / AC / 2C / D2DCE / MD / MH), TAC / ADC extras, and the 12-key result dict."""
    mtd = D.d_cond_mtd
    if not (mtd in ("PD", "W/O") and D.aux_cls_type in ("W/O", "N/A", None) and D.linear1.out_features == 1 and h.is_cuda
            and h.dtype == torch.float32 and h.shape[1] % 8 == 0):
        return _head_tensor_ops(D, h, label, adc_fake)
    # hot-path heads (projection discriminator / unconditional): one library launch forward, two backward (A.DHeadFn)
    E = D.embedding if mtd == "PD" else None
    cfg = {"sn1": getattr(D.linear1, "_sn", None), "snE": getattr(E, "_sn", None) if E is not None else None,
           "training": D.linear1.training}
    adv = A.DHeadFn.call(h, _w(D.linear1), D.linear1.bias, _w(E) if E is not None else None, label, cfg)
    out = dict.fromkeys(_HEAD_KEYS)
    out.update({"h": h, "adv_output": adv, "label": label})
    return out


def _head_tensor_ops(D, h, label, adc_fake):
    """discriminator_head written as tensor arithmetic on h: every head that sgb_dhead_fwd / bwd do not cover."""
    out = dict.fromkeys(_HEAD_KEYS)
    mtd = D.d_cond_mtd
    w_eff = _head_weight(D.linear1)
    adv = torch.squeeze(F.linear(h, w_eff, D.linear1.bias))
    if D.aux_cls_type == "ADC":
        label = label * 2 + 1 if adc_fake else label * 2
    emb = None
    if mtd == "PD":
        emb = D.embedding(label)
        adv = adv + torch.sum(emb * h, 1)
    elif mtd == "AC":
        if D.normalize_d_embed:
            h = F.normalize(h, dim=1)
        out["cls_output"] = head_linear(D.linear2, h)
    elif mtd in ("2C", "D2DCE"):
        embed, proxy = head_linear(D.linear2, h), D.embedding(label)
        if D.normalize_d_embed:
            embed, proxy = F.normalize(embed, dim=1), F.normalize(proxy, dim=1)
        out["embed"], out["proxy"] = embed, proxy
    elif mtd == "MD":
        adv = adv[torch.arange(label.size(0), device=label.device), label]
    elif mtd not in ("W/O", "MH"):
        raise NotImplementedError(mtd)
    if D.aux_cls_type == "TAC":
        if mtd == "AC":
            out["mi_cls_output"] = head_linear(D.linear_mi, h)
        elif mtd in ("2C", "D2DCE"):
            mi_embed, mi_proxy = head_linear(D.linear_mi, h), D.embedding_mi(label)
            if D.normalize_d_embed:
                mi_embed, mi_proxy = F.normalize(mi_embed, dim=1), F.normalize(mi_proxy, dim=1)
            out["mi_embed"], out["mi_proxy"] = mi_embed, mi_proxy
    A.tape_record(_HeadTangent, (h, w_eff, emb, mtd), adv)
    out.update({"h": h, "adv_output": adv, "label": label})
    return out


def build_discriminator_head(D, MODULES, feat, d_cond_mtd, aux_cls_type, d_embed_dim, num_classes):
    """Registers the head layers in the reference's order (linear1, linear2 / embedding, linear_mi / embedding_mi;
    src/models/big_resnet.py:303-336, identical in resnet.py and big_resnet_deep_*.py)."""
    if d_cond_mtd == "MH":
        D.linear1 = MODULES.d_linear(in_features=feat, out_features=1 + num_classes, bias=True)
    elif d_cond_mtd == "MD":
        D.linear1 = MODULES.d_linear(in_features=feat, out_features=num_classes, bias=True)
    else:
        D.linear1 = MODULES.d_linear(in_features=feat, out_features=1, bias=True)
    D.linear1._head_layer = True                  # fp32 head path (ops.head_linear), not part of the batched SN / pack pass
    if aux_cls_type == "ADC":
        num_classes = num_classes * 2
    if d_cond_mtd == "AC":
        D.linear2 = MODULES.d_linear(in_features=feat, out_features=num_classes, bias=False)
    elif d_cond_mtd == "PD":
        D.embedding = MODULES.d_embedding(num_classes, feat)
    elif d_cond_mtd in ["2C", "D2DCE"]:
        D.linear2 = MODULES.d_linear(in_features=feat, out_features=d_embed_dim, bias=True)
        D.embedding = MODULES.d_embedding(num_classes, d_embed_dim)
    if aux_cls_type == "TAC":
        if d_cond_mtd == "AC":
            D.linear_mi = MODULES.d_linear(in_features=feat, out_features=num_classes, bias=False)
        elif d_cond_mtd in ["2C", "D2DCE"]:
            D.linear_mi = MODULES.d_linear(in_features=feat, out_features=d_embed_dim, bias=True)
            D.embedding_mi = MODULES.d_embedding(num_classes, d_embed_dim)
        else:
            raise NotImplementedError
    for name in ("linear2", "linear_mi"):
        if hasattr(D, name):
            getattr(D, name)._head_layer = True
