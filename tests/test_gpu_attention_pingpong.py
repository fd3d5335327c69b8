"""The attention softmax epilogues of conv_fprop_kernel (csrc/umma_conv.cu) on the ping-pong schedule, where each consumer
warpgroup owns whole 128-row tiles and takes a query row's max and sum from the four lanes of a quad of the accumulator
fragment.  The cases cover the edges that schedule meets, each for the statistics + apply passes (P = softmax(theta phi^T))
and the backward pass (dS = P * (do g^T - delta)) against float64:
* M = 192 / 320 keys: the last channel tile holds one 64-wide chunk (its other chunk is zero-filled and must not count);
* M = 64: a single 64-wide channel tile;
* query maps of 12 x 20 and 12 x 12: tiles with rows outside the map (ragged w and h), which store no statistics;
* B = 1 and B = 3 at the flagship's 64 x 64 map (M = 1024): 256 / 768 tiles over the persistent grid, so some CTAs leave one
  warpgroup a tile fewer than the other;
* rows with one dominant logit (in the first or in the partial last channel tile): the merge of the per-tile partials must
  rescale them to the row maximum.
Tolerances are those of test_gpu_conv_fused.test_attention_softmax_variants_at_flagship_shape_vs_float64."""
import ctypes

import pytest
import torch

from test_gpu_conv_fused import ACC_REL, _flags, _launched, _rows
from test_gpu_norm_shapes import _act, _cuda, _rounding_ratio

pytestmark = pytest.mark.gpu

# id: (B, query H, query W, key h, key w, dominant rows)
CASES = {
    "M=192 32x32 B=2":             (2, 32, 32, 12, 16, False),
    "M=320 ragged 12x20 B=2":      (2, 12, 20, 16, 20, False),
    "M=64 ragged 12x12 B=3":       (3, 12, 12, 8, 8, False),
    "M=1024 64x64 B=1":            (1, 64, 64, 32, 32, False),
    "M=1024 64x64 B=3":            (3, 64, 64, 32, 32, False),
    "M=192 dominant 32x32 B=2":    (2, 32, 32, 12, 16, True),
    "M=1024 dominant 64x64 B=1":   (1, 64, 64, 32, 32, True),
}


def _operands(dev, B, H, W, h, w, dominant):
    """theta [B, 64, H, W], phi [B, 64, h, w], g [B, 256, h, w], do [B, 256, H, W], bf16 NHWC.  dominant: every 5th query
    row is 4 phi[key] for a key in the first channel tile (even rows) or in the last one (odd rows), a logit ~4 |phi|^2 = 256
    against ~N(0, 32^2) for the other keys."""
    gen = torch.Generator(device=dev).manual_seed(43)
    theta = _act(gen, B, 64, H, W, dev)
    phi = _act(gen, B, 64, h, w, dev)
    g = _act(gen, B, 256, h, w, dev)
    do = _act(gen, B, 256, H, W, dev)
    if dominant:
        M = h * w
        tq = theta.permute(0, 2, 3, 1).reshape(B, H * W, 64)      # views of the NHWC storage
        kq = phi.permute(0, 2, 3, 1).reshape(B, M, 64)
        rows = torch.arange(0, H * W, 5, device=dev)
        keys = torch.where(rows % 2 == 0, rows % 128, M - 1 - rows % 64)
        tq[:, rows] = (4 * kq[:, keys].float()).to(torch.bfloat16)
    return theta, phi, g, do


@pytest.mark.parametrize("B,H,W,h,w,dominant", list(CASES.values()), ids=list(CASES))
def test_attention_softmax_pingpong_edges_vs_float64(B, H, W, h, w, dominant):
    from sgb200 import kernels as K
    dev = _cuda()
    M = h * w
    theta, phi, g, do = _operands(dev, B, H, W, h, w, dominant)

    def fwd():
        P, stats = K.conv_fprop(theta, phi, M, 1, 1, 0, 0, w_mode=1, sm_mode=1)
        K.conv_fprop(theta, phi, M, 1, 1, 0, 0, w_mode=1, sm_mode=2, sm_stats=stats, out=P)
        return P

    seen, _, P = _launched(fwd)
    assert seen == {("fprop", _flags("Full|SmStats")), ("fprop", _flags("Full|SmApply"))}, seen
    q, kk = _rows(theta), _rows(phi)
    logits, labs = q @ kk.transpose(1, 2), q.abs() @ kk.abs().transpose(1, 2)
    Pref = torch.softmax(logits, -1)
    atol = Pref * (2 * ACC_REL * labs.amax(-1, keepdim=True) + 2.0 ** -18) + 2.0 ** -126
    wp = _rounding_ratio(_rows(P), Pref, atol)
    if dominant:
        assert float(Pref.amax(-1).max()) > 0.999         # the construction did produce dominant rows

    Pk = _rows(P)
    dP = _rows(do) @ _rows(g).transpose(1, 2)
    delta = (Pk * dP).sum(-1).float().reshape(-1).contiguous()
    seen, _, dS = _launched(lambda: K.conv_fprop(do, g, M, 1, 1, 0, 0, w_mode=1, sm_mode=3, sm_delta=delta, sm_p=P))
    assert seen == {("fprop", _flags("Full|SmBwd"))}, seen
    dabs = _rows(do).abs() @ _rows(g).abs().transpose(1, 2)
    dref = Pk * (dP - delta.view(B, -1).double()[..., None])
    wd = _rounding_ratio(_rows(dS), dref, Pk * ACC_REL * dabs + 1e-30)
    print("B=%d %dx%d M=%d: P %.3g dS %.3g of one rounding" % (B, H, W, M, wp, wd))
    assert wp <= 1.0 and wd <= 1.0


def test_softmax_parts_is_one_per_channel_tile():
    """sgb_conv_softmax_parts (the sm_stats row length the caller allocates) = ceil(M / 128): one partial per channel tile."""
    from sgb200 import _lib as L
    lib = L.load()
    for M in (64, 128, 192, 320, 1024, 4096):
        d = L.ConvDesc()
        d.B, d.H, d.W, d.Cin, d.Cout, d.KH, d.KW, d.w_mode, d.sm_mode = 1, 64, 64, 64, M, 1, 1, 1, 1
        assert lib.sgb_conv_softmax_parts(ctypes.byref(d)) == (M + 127) // 128, M
