"""FID InceptionV3 feature extractor on the wgmma conv engine (reference ``src/metrics/inception_net.py``).

Same network as the reference's ``InceptionV3`` (torchvision ``inception_v3(num_classes=1008, aux_logits=False)`` with the
TF-compatible pooling variants FIDInceptionA/C/E_1/E_2, :110-249) in inference mode: BatchNorm (eps 1e-3) is folded into the
convolution weights/bias once at load time, every BasicConv2d becomes one conv launch with bias+ReLU in the epilogue, the
branches of a Mixed block write straight into channel slices of the block's output (no concatenation pass), and the four
stride-2 convolutions run on the stride-1 grid with an even-position store.  Input pre-processing (uint8 quantisation,
299x299 "legacy" bilinear resize, normalisation) is one fused device kernel that already emits the 3x3/stride-2 patches
of the first convolution (src/utils/ops.py:251-263, src/metrics/preparation.py:103-122) — the reference does it on the
host, image by image.

Weights: a state_dict in torchvision layout (the reference's ``pt_inception-2015-12-05-6726825d.pth`` has exactly these
keys).  That file cannot be downloaded here, so tests and benchmarks use seeded random weights; absolute FID/IS values
with the pretrained weights are "parity unpinned" (DESIGN.md).
"""
import torch

from .. import kernels as K

BN_EPS = 1e-3


def _fold(sd, name, dev):
    """(weight * gamma/sqrt(var+eps), beta - mean * gamma/sqrt(var+eps)) of a torchvision BasicConv2d."""
    w = sd[name + ".conv.weight"].to(dev, torch.float32)
    g, b = sd[name + ".bn.weight"].to(dev, torch.float32), sd[name + ".bn.bias"].to(dev, torch.float32)
    m, v = sd[name + ".bn.running_mean"].to(dev, torch.float32), sd[name + ".bn.running_var"].to(dev, torch.float32)
    s = g / torch.sqrt(v + BN_EPS)
    return (w * s[:, None, None, None]).contiguous(), (b - m * s).contiguous()


class _Conv:
    def __init__(self, sd, name, dev, pad=(0, 0), stride=1, same=None, image=False):
        w, b = _fold(sd, name, dev)
        self.Cout, self.Cin, self.KH, self.KW = w.shape
        self.pad, self.stride = pad, stride
        self.same = same if same is not None else (2 * pad[0] == self.KH - 1 and 2 * pad[1] == self.KW - 1)
        self.bias = b
        if image:       # first layer: consumes the 3x3 / stride-2 patch tensor -> K = 27 (padded to 32) GEMM
            wcol = w.permute(0, 2, 3, 1).reshape(self.Cout, 27).contiguous()
            self.wf, _ = K.weight_pack(wcol, None, self.Cout, 27, 1, True, False)
            self.KH = self.KW = 1
            self.pad, self.stride, self.same = (0, 0), 1, True
        else:
            self.wf, _ = K.weight_pack(w, None, self.Cout, self.Cin, self.KH * self.KW, True, False)

    def __call__(self, x, out=None):
        return K.conv_fprop(x, self.wf, self.Cout, self.KH, self.KW, self.pad[0], self.pad[1], bias=self.bias, relu=True, out=out,
                            same_size=self.same, stride=self.stride)


class InceptionV3(object):
    """forward(images) -> (pool features [B, 2048] fp32, logits [B, 1008] fp32)."""

    def __init__(self, state_dict, device):
        dev = self.device = torch.device(device)
        sd = state_dict
        c = lambda name, **kw: _Conv(sd, name, dev, **kw)  # noqa: E731
        self.stem = [c("Conv2d_1a_3x3", image=True), c("Conv2d_2a_3x3"), c("Conv2d_2b_3x3", pad=(1, 1)),
                     c("Conv2d_3b_1x1"), c("Conv2d_4a_3x3")]
        self.blocks = []
        for name in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
            self.blocks.append(("A", {
                "b1": c(name + ".branch1x1"), "b5_1": c(name + ".branch5x5_1"), "b5_2": c(name + ".branch5x5_2", pad=(2, 2)),
                "d1": c(name + ".branch3x3dbl_1"), "d2": c(name + ".branch3x3dbl_2", pad=(1, 1)),
                "d3": c(name + ".branch3x3dbl_3", pad=(1, 1)), "bp": c(name + ".branch_pool")}))
        self.blocks.append(("B", {
            "b3": c("Mixed_6a.branch3x3", stride=2), "d1": c("Mixed_6a.branch3x3dbl_1"),
            "d2": c("Mixed_6a.branch3x3dbl_2", pad=(1, 1)), "d3": c("Mixed_6a.branch3x3dbl_3", stride=2)}))
        for name in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
            self.blocks.append(("C", {
                "b1": c(name + ".branch1x1"),
                "s1": c(name + ".branch7x7_1"), "s2": c(name + ".branch7x7_2", pad=(0, 3)), "s3": c(name + ".branch7x7_3", pad=(3, 0)),
                "d1": c(name + ".branch7x7dbl_1"), "d2": c(name + ".branch7x7dbl_2", pad=(3, 0)),
                "d3": c(name + ".branch7x7dbl_3", pad=(0, 3)), "d4": c(name + ".branch7x7dbl_4", pad=(3, 0)),
                "d5": c(name + ".branch7x7dbl_5", pad=(0, 3)), "bp": c(name + ".branch_pool")}))
        self.blocks.append(("D", {
            "b3_1": c("Mixed_7a.branch3x3_1"), "b3_2": c("Mixed_7a.branch3x3_2", stride=2),
            "s1": c("Mixed_7a.branch7x7x3_1"), "s2": c("Mixed_7a.branch7x7x3_2", pad=(0, 3)),
            "s3": c("Mixed_7a.branch7x7x3_3", pad=(3, 0)), "s4": c("Mixed_7a.branch7x7x3_4", stride=2)}))
        for name, pool_mode in (("Mixed_7b", 0), ("Mixed_7c", 1)):
            self.blocks.append(("E", {
                "b1": c(name + ".branch1x1"), "b3_1": c(name + ".branch3x3_1"),
                "b3_2a": c(name + ".branch3x3_2a", pad=(0, 1)), "b3_2b": c(name + ".branch3x3_2b", pad=(1, 0)),
                "d1": c(name + ".branch3x3dbl_1"), "d2": c(name + ".branch3x3dbl_2", pad=(1, 1)),
                "d3a": c(name + ".branch3x3dbl_3a", pad=(0, 1)), "d3b": c(name + ".branch3x3dbl_3b", pad=(1, 0)),
                "bp": c(name + ".branch_pool"), "pool_mode": pool_mode}))
        fcw = sd["fc.weight"].to(dev, torch.float32).contiguous()
        self.fc_wf, _ = K.weight_pack(fcw, None, fcw.shape[0], fcw.shape[1], 1, True, False)
        self.fc_bias = sd["fc.bias"].to(dev, torch.float32).contiguous()
        self.fc_out = fcw.shape[0]

    @staticmethod
    def _cat(x, branches, H, W):
        """Allocate the block output and let each (conv, input) branch write its channel slice."""
        B = x.shape[0]
        total = sum(ch for ch, _ in branches)
        out = K.empty_nhwc(B, total, H, W, x.device)
        off = 0
        for ch, fn in branches:
            fn(out[:, off:off + ch])
            off += ch
        return out

    def _block(self, kind, L, x):
        B, C, H, W = x.shape
        if kind == "A":
            return self._cat(x, [
                (L["b1"].Cout, lambda o: L["b1"](x, o)),
                (L["b5_2"].Cout, lambda o: L["b5_2"](L["b5_1"](x), o)),
                (L["d3"].Cout, lambda o: L["d3"](L["d2"](L["d1"](x)), o)),
                (L["bp"].Cout, lambda o: L["bp"](K.pool3x3(x, 1, 1, 0), o))], H, W)
        if kind == "B":
            Ho = (H - 3) // 2 + 1
            return self._cat(x, [
                (L["b3"].Cout, lambda o: L["b3"](x, o)),
                (L["d3"].Cout, lambda o: L["d3"](L["d2"](L["d1"](x)), o)),
                (C, lambda o: K.pool3x3(x, 2, 0, 1, out=o))], Ho, Ho)
        if kind == "C":
            return self._cat(x, [
                (L["b1"].Cout, lambda o: L["b1"](x, o)),
                (L["s3"].Cout, lambda o: L["s3"](L["s2"](L["s1"](x)), o)),
                (L["d5"].Cout, lambda o: L["d5"](L["d4"](L["d3"](L["d2"](L["d1"](x)))), o)),
                (L["bp"].Cout, lambda o: L["bp"](K.pool3x3(x, 1, 1, 0), o))], H, W)
        if kind == "D":
            Ho = (H - 3) // 2 + 1
            return self._cat(x, [
                (L["b3_2"].Cout, lambda o: L["b3_2"](L["b3_1"](x), o)),
                (L["s4"].Cout, lambda o: L["s4"](L["s3"](L["s2"](L["s1"](x))), o)),
                (C, lambda o: K.pool3x3(x, 2, 0, 1, out=o))], Ho, Ho)
        if kind == "E":
            def b3(o):
                t = L["b3_1"](x)
                L["b3_2a"](t, o[:, :L["b3_2a"].Cout])
                L["b3_2b"](t, o[:, L["b3_2a"].Cout:])

            def dbl(o):
                t = L["d2"](L["d1"](x))
                L["d3a"](t, o[:, :L["d3a"].Cout])
                L["d3b"](t, o[:, L["d3a"].Cout:])
            return self._cat(x, [
                (L["b1"].Cout, lambda o: L["b1"](x, o)),
                (L["b3_2a"].Cout + L["b3_2b"].Cout, b3),
                (L["d3a"].Cout + L["d3b"].Cout, dbl),
                (L["bp"].Cout, lambda o: L["bp"](K.pool3x3(x, 1, 1, L["pool_mode"]), o))], H, W)
        raise ValueError(kind)

    @torch.no_grad()
    def forward_col(self, col):
        """``col``: [B, 32, 149, 149] patch tensor from kernels.quantize_resize_normalize."""
        s = self.stem
        x = s[2](s[1](s[0](col)))                 # 149 -> 147 -> 147
        x = K.pool3x3(x, 2, 0, 1)                 # 73
        x = s[4](s[3](x))                         # 73 -> 71
        x = K.pool3x3(x, 2, 0, 1)                 # 35
        for kind, layers in self.blocks:
            x = self._block(kind, layers, x)
        B, C, H, W = x.shape
        pool = K.sum_hw(x, False) / float(H * W)  # adaptive average pool -> [B, 2048] fp32
        feat = K.cast_f32_to_bf16(pool).view(B, C, 1, 1)
        logits = K.conv_fprop(feat, self.fc_wf, K.pad8(self.fc_out), 1, 1, 0, 0, bias=self.fc_bias, out_fp32=True)
        return pool, logits.reshape(B, -1)[:, :self.fc_out].contiguous()

    @torch.no_grad()
    def forward(self, images, quantize=True, resizer="legacy"):
        """``images``: NCHW fp32 in [-1, 1] (quantize=True, the generated-image path) or already 0..255 valued."""
        _, col = K.quantize_resize_normalize(images, 299, quantize=quantize, want_image=False, want_col=True, resizer=resizer)
        return self.forward_col(col)

    __call__ = forward


def seeded_state_dict(seed=0):
    """Random InceptionV3 weights in torchvision layout with O(1) activations (He-scaled convs, benign BN statistics):
    used wherever the pretrained FID weights (not downloadable here) would be loaded."""
    import torchvision
    torch.manual_seed(seed)
    net = torchvision.models.inception_v3(num_classes=1008, aux_logits=False, weights=None, init_weights=False)
    g = torch.Generator().manual_seed(seed)
    sd = net.state_dict()
    for k, v in sd.items():
        if k.endswith("conv.weight"):
            fan_in = v.shape[1] * v.shape[2] * v.shape[3]
            v.copy_(torch.randn(v.shape, generator=g) * (2.0 / fan_in) ** 0.5)
        elif k.endswith("bn.weight"):
            v.copy_(1.0 + 0.1 * torch.randn(v.shape, generator=g))
        elif k.endswith("bn.bias"):
            v.copy_(0.1 * torch.randn(v.shape, generator=g))
        elif k.endswith("running_mean"):
            v.copy_(0.1 * torch.randn(v.shape, generator=g))
        elif k.endswith("running_var"):
            v.copy_(1.0 + 0.2 * torch.rand(v.shape, generator=g))
        elif k == "fc.weight":
            v.copy_(torch.randn(v.shape, generator=g) * (1.0 / v.shape[1]) ** 0.5)
        elif k == "fc.bias":
            v.copy_(0.1 * torch.randn(v.shape, generator=g))
    return sd
