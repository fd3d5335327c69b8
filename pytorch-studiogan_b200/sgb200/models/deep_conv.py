"""DCGAN generator / discriminator (BASELINE config 1) on the sgb200 kernel set.

Drop-in for the reference ``src/models/deep_conv.py``: same constructor signatures, sub-module names / registration order
(state_dict keys, seeded initialisation), ``forward`` signatures and the 12-key discriminator dict.

  GenBlock  (ref :15-43)    ConvTranspose 4x4 / stride 2 / pad 1 -> BN (or cBN) -> ReLU
  DiscBlock (ref :129-153)  conv 3x3 -> [BN] -> ReLU -> conv 4x4 / stride 2 / pad 1 -> [BN] -> ReLU

Both stride-2 layers run on the stride-1 wgmma engine through exact identities (csrc/resample.cu): the transposed
convolution is a 4x4 same-size convolution of the zero-stuffed input, the strided convolution stores every other output of
a 4x4 same-size convolution (the engine's out_sub mode).  That spends 4x the minimal FLOPs on those layers -- DCGAN is the
reference's 0.8 GFLOP CPU-sized config; it is here for completeness of the model API, not for its roofline.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import autograd_ops as A
from ..snbatch import SNBatch
from ..utils import ops


class GenBlock(nn.Module):
    def __init__(self, in_channels, out_channels, g_cond_mtd, g_info_injection, affine_input_dim, MODULES):
        super().__init__()
        self.g_cond_mtd = g_cond_mtd
        self.g_info_injection = g_info_injection
        self.deconv0 = MODULES.g_deconv2d(in_channels=in_channels, out_channels=out_channels, kernel_size=4, stride=2, padding=1)
        if self.g_cond_mtd == "W/O" and self.g_info_injection in ["N/A", "concat"]:
            self.bn0 = MODULES.g_bn(in_features=out_channels)
            self.conditional = False
        elif self.g_cond_mtd == "cBN" or self.g_info_injection == "cBN":
            self.bn0 = MODULES.g_bn(affine_input_dim, out_channels, MODULES)
            self.conditional = True
        else:
            raise NotImplementedError
        self.activation = MODULES.g_act_fn

    def forward(self, x, affine):
        x = self.deconv0(x)
        return self.bn0(x, affine, relu=True) if self.conditional else self.bn0(x, relu=True)


class Generator(nn.Module):
    def __init__(self, z_dim, g_shared_dim, img_size, g_conv_dim, apply_attn, attn_g_loc, g_cond_mtd, num_classes, g_init, g_depth,
                 mixed_precision, MODULES, MODEL):
        super().__init__()
        self.in_dims = [512, 256, 128]
        self.out_dims = [256, 128, 64]
        self.z_dim = z_dim
        self.num_classes = num_classes
        self.g_cond_mtd = g_cond_mtd
        self.mixed_precision = mixed_precision
        self.MODEL = MODEL
        self.affine_input_dim = 0
        if getattr(MODEL, "info_type", "N/A") != "N/A":
            raise NotImplementedError("InfoGAN heads are outside the sgb200 hot-path scope (SURVEY.md section 8)")
        self.g_info_injection = getattr(MODEL, "g_info_injection", "N/A")
        if self.g_cond_mtd != "W/O" and self.g_cond_mtd == "cBN":
            self.affine_input_dim += self.num_classes

        self.linear0 = MODULES.g_linear(in_features=self.z_dim, out_features=self.in_dims[0] * 4 * 4, bias=True)

        blocks = []
        for index in range(len(self.in_dims)):
            blocks.append([GenBlock(in_channels=self.in_dims[index], out_channels=self.out_dims[index], g_cond_mtd=self.g_cond_mtd,
                                    g_info_injection=self.g_info_injection, affine_input_dim=self.affine_input_dim, MODULES=MODULES)])
            if index + 1 in attn_g_loc and apply_attn:
                blocks.append([ops.SelfAttention(self.out_dims[index], is_generator=True, MODULES=MODULES)])
        self.blocks = nn.ModuleList([nn.ModuleList(b) for b in blocks])

        self.conv4 = MODULES.g_conv2d(in_channels=self.out_dims[-1], out_channels=3, kernel_size=3, stride=1, padding=1)
        self.tanh = nn.Tanh()

        ops.init_weights(self.modules, g_init)
        self.linear0._perm_S = 16
        self._snb = SNBatch(self)

    def forward(self, z, label, shared_label=None, eval=False):
        self._snb.run()
        affines = None
        if self.g_cond_mtd != "W/O":
            affines = A.ToBF16Fn.call(F.one_hot(label, num_classes=self.num_classes).to(torch.float32))
        act = self.linear0(z, perm_S=16)                              # [B, 16 * 512, 1, 1], features already in (s, c) order
        B = act.shape[0]
        act = act.reshape(B, 4, 4, self.in_dims[0]).permute(0, 3, 1, 2)
        for blocklist in self.blocks:
            for block in blocklist:
                act = block(act) if isinstance(block, ops.SelfAttention) else block(act, affines)
        act = self.conv4(act)
        self._snb.clear()
        return A.ImageOutFn.call(act, 3)


class DiscBlock(nn.Module):
    def __init__(self, in_channels, out_channels, apply_d_sn, MODULES):
        super().__init__()
        self.apply_d_sn = apply_d_sn
        self.conv0 = MODULES.d_conv2d(in_channels=in_channels, out_channels=out_channels, kernel_size=3, stride=1, padding=1)
        self.conv1 = MODULES.d_conv2d(in_channels=out_channels, out_channels=out_channels, kernel_size=4, stride=2, padding=1)
        if not apply_d_sn:
            self.bn0 = MODULES.d_bn(in_features=out_channels)
            self.bn1 = MODULES.d_bn(in_features=out_channels)
        self.activation = MODULES.d_act_fn

    def forward(self, x):
        """``x``: NCHW fp32 image for the first block (in_channels 3), NHWC bf16 activation afterwards."""
        if self.conv0.in_channels == 3:
            x = A.ImageColFn.call(x)
        if self.apply_d_sn:
            x = self.conv0(x, relu=True)
            return self.conv1(x, relu=True)
        x = self.bn0(self.conv0(x), relu=True)
        return self.bn1(self.conv1(x), relu=True)


class Discriminator(nn.Module):
    def __init__(self, img_size, d_conv_dim, apply_d_sn, apply_attn, attn_d_loc, d_cond_mtd, aux_cls_type, d_embed_dim, normalize_d_embed,
                 num_classes, d_init, d_depth, mixed_precision, MODULES, MODEL):
        super().__init__()
        self.in_dims = [3] + [64, 128]
        self.out_dims = [64, 128, 256]
        self.apply_d_sn = apply_d_sn
        self.d_cond_mtd = d_cond_mtd
        self.aux_cls_type = aux_cls_type
        self.normalize_d_embed = normalize_d_embed
        self.num_classes = num_classes
        self.mixed_precision = mixed_precision
        self.MODEL = MODEL
        if getattr(MODEL, "info_type", "N/A") != "N/A":
            raise NotImplementedError("InfoGAN heads are outside the sgb200 hot-path scope (SURVEY.md section 8)")

        blocks = []
        for index in range(len(self.in_dims)):
            blocks.append([DiscBlock(in_channels=self.in_dims[index], out_channels=self.out_dims[index], apply_d_sn=self.apply_d_sn,
                                     MODULES=MODULES)])
            if index + 1 in attn_d_loc and apply_attn:
                blocks.append([ops.SelfAttention(self.out_dims[index], is_generator=False, MODULES=MODULES)])
        self.blocks = nn.ModuleList([nn.ModuleList(b) for b in blocks])

        self.activation = MODULES.d_act_fn
        self.conv1 = MODULES.d_conv2d(in_channels=256, out_channels=512, kernel_size=3, stride=1, padding=1)
        if not self.apply_d_sn:
            self.bn1 = MODULES.d_bn(in_features=512)
        ops.build_discriminator_head(self, MODULES, 512, d_cond_mtd, aux_cls_type, d_embed_dim, num_classes)
        if d_init:
            ops.init_weights(self.modules, d_init)
        self._snb = SNBatch(self)

    def forward(self, x, label, eval=False, adc_fake=False):
        self._snb.run()
        h = x
        for blocklist in self.blocks:
            for block in blocklist:
                h = block(h)
        h = self.conv1(h)
        relu_in_sum = True
        if not self.apply_d_sn:
            h = self.bn1(h, relu=True)
            relu_in_sum = False
        h = A.SumHWFn.call(h, relu_in_sum)                            # [relu +] sum over (H, W), fp32 [B, 512]
        self._snb.clear()
        return ops.discriminator_head(self, h, label, adc_fake)
