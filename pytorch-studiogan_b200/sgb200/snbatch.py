"""Batched spectral normalisation for a whole network: one power iteration + sigma + weight packs for EVERY conv / linear
layer in three kernel launches (``sgb_sn_batch``), run at the top of ``Generator.forward`` / ``Discriminator.forward``.

Semantics are those of the per-layer forward-pre-hooks of the reference (torch/nn/utils/spectral_norm.py:62-114): each
layer's iteration depends only on its own W, u, v, and every network forward performs exactly one iteration per layer,
so running them all before the first layer is arithmetically the same as running each right before its layer.

Implementation notes
* u / v buffers of all layers become views of two flat arenas (their values and state_dict keys are unchanged), so the
  copies the backward pass needs ("u, v at the time of this forward") are two clones instead of 2 x layers.
* packs of one forward live in one flat bf16 buffer per direction; each layer receives views.
* layers that are not spectrally normalised (e.g. SNGAN's generator) are packed by the same launch with sigma = 1.
"""
import numpy as np
import torch

from . import _lib as L
from . import kernels as K
from .utils import ops

LAYER_DTYPE = np.dtype([("W", "<u8"), ("u", "<u8"), ("v", "<u8"), ("ws", "<u8"), ("R", "<i4"), ("K", "<i4"),
                        ("Cout", "<i4"), ("Cin", "<i4"), ("taps", "<i4"), ("perm_S", "<i4"), ("Cout_p", "<i4"), ("Cin_p", "<i4"),
                        ("off_f", "<i8"), ("off_d", "<i8"), ("has_sn", "<i4"), ("tile_start", "<i4")])
assert LAYER_DTYPE.itemsize == 88
BWD_DTYPE = np.dtype([("W", "<u8"), ("dW", "<u8"), ("off_g", "<i8"), ("off_u", "<i8"), ("off_v", "<i8"), ("Cout", "<i4"),
                      ("Cin", "<i4"), ("taps", "<i4"), ("perm_S", "<i4"), ("Cin_p", "<i4"), ("has_sn", "<i4")])
assert BWD_DTYPE.itemsize == 64


class _Pass:
    """One network forward's spectral-norm state for the backward pass: sigma / u / v as they were at that forward, and a
    flat fp32 buffer into which every layer's weight-gradient launch accumulates (fprop-pack layout).  When the backward
    pass of the graph finishes, ONE batched launch pair applies the spectral-norm chain rule of all layers and adds the
    result to the flat gradient arena (instead of ~2 launches + a memset per layer)."""

    def __init__(self, owner, sigma, us, vs):
        self.owner, self.sigma, self.us, self.vs = owner, sigma, us, vs
        self.g_flat = None
        self.queued = False

    def usable(self):
        return self.us is not None and self.owner.bwd_table() is not None

    def g_slice(self, i):
        """fp32 [Cout_p][taps][Cin_p] accumulator of layer i (zero-initialised with the whole buffer on first use)."""
        o = self.owner
        if self.g_flat is None:
            self.g_flat = torch.zeros(o.total_f, device=o.device, dtype=torch.float32)
        of, _, nf, shf = o.slices[i][0], None, o.slices[i][2], o.slices[i][3]
        if not self.queued:
            self.queued = True
            torch.autograd.Variable._execution_engine.queue_callback(self.flush)
        return self.g_flat[of:of + nf].view(shf)

    def flush(self):
        o = self.owner
        self.queued = False
        if self.g_flat is None:
            return
        table = o.bwd_table()
        dots = torch.empty(len(o.mods), device=o.device, dtype=torch.float32)
        L.call("sgb_sn_backward_batch", L.ptr(table), len(o.mods), L.ptr(self.g_flat), L.ptr(self.sigma), L.ptr(self.us),
               L.ptr(self.vs), L.ptr(dots), 96, L.stream_ptr())
        self.g_flat = None


def _eligible(m):
    if isinstance(m, ops._ConvBase):
        return not (m.in_channels == 3 and m.kernel_size == (3, 3))      # image convs run the im2col path
    return isinstance(m, ops._LinearBase) and not getattr(m, "_head_layer", False)


class SNBatch:
    def __init__(self, net):
        self.net = net
        self.mods = None
        self.device = None

    def _build(self, device):
        mods = [m for m in self.net.modules() if _eligible(m)]
        mods.sort(key=lambda m: 0 if getattr(m, "_cbn_affine", False) else 1)     # (stable) cBN gain / bias packs first, contiguous
        nu = sum(ops._w(m).shape[0] for m in mods if hasattr(m, "_sn"))
        nv = sum(ops._w(m).numel() // ops._w(m).shape[0] for m in mods if hasattr(m, "_sn"))
        self.u_flat = torch.empty(max(nu, 1), device=device, dtype=torch.float32)
        self.v_flat = torch.empty(max(nv, 1), device=device, dtype=torch.float32)
        nws = sum(ops._w(m).shape[0] + ops._w(m).numel() // ops._w(m).shape[0] + 4 for m in mods if hasattr(m, "_sn"))
        self.ws_flat = torch.zeros(max(nws, 1), device=device, dtype=torch.float32)
        table = np.zeros(len(mods), dtype=LAYER_DTYPE)
        ou = ov = ows = 0
        off_f = off_d = 0
        self.slices = []
        mb1 = mb2 = 1
        tiles = 0
        for i, m in enumerate(mods):
            W = ops._w(m)
            Cout = W.shape[0]
            taps = W.shape[2] * W.shape[3] if W.dim() == 4 else 1
            Cin = W.numel() // (Cout * taps)
            R, Kd = Cout, Cin * taps
            Cout_p, Cin_p = K.pad8(Cout), K.pad8(Cin)
            e = table[i]
            e["W"] = W.data_ptr()
            e["R"], e["K"], e["Cout"], e["Cin"], e["taps"] = R, Kd, Cout, Cin, taps
            e["perm_S"] = getattr(m, "_perm_S", 1)
            e["Cout_p"], e["Cin_p"] = Cout_p, Cin_p
            nf = Cout_p * taps * Cin_p
            e["off_f"], e["off_d"] = off_f, off_d
            su = sv = None
            if hasattr(m, "_sn"):
                e["has_sn"] = 1
                with torch.no_grad():
                    self.u_flat[ou:ou + R].copy_(m.weight_u)
                    self.v_flat[ov:ov + Kd].copy_(m.weight_v)
                m.weight_u.data = self.u_flat[ou:ou + R]
                m.weight_v.data = self.v_flat[ov:ov + Kd]
                e["u"], e["v"] = m.weight_u.data_ptr(), m.weight_v.data_ptr()
                e["ws"] = self.ws_flat[ows:].data_ptr()
                su, sv = (ou, ou + R), (ov, ov + Kd)
                ou += R
                ov += Kd
                ows += R + Kd + 4
                mb1 = max(mb1, ((Kd + 255) // 256) * ((R + 63) // 64))
                mb2 = max(mb2, (R + 7) // 8)
            e["tile_start"] = tiles
            # work units of ~1024 weights: a 32 x 32 tile of a k-tap layer counts k, a 4096-element pseudo tile (k > 9) counts 4
            tiles += ((Cout + 31) // 32) * ((Cin + 31) // 32) * taps if taps <= 9 else 4 * ((Cout * Cin * taps + 4095) // 4096)
            self.slices.append((off_f, off_d, nf, (Cout_p, taps, Cin_p), (Cin_p, taps, Cout_p), su, sv))
            off_f += (nf + 63) // 64 * 64            # keep every pack 128-byte aligned (TMA base alignment)
            off_d += (nf + 63) // 64 * 64
        self.total_f, self.total_d = off_f, off_d
        self.table = torch.from_numpy(table.view(np.uint8).copy()).to(device)
        self.max_blocks = (min(mb1, 4096), min(mb2, 1024), tiles)     # (wtu grid, wv grid, total pack tiles)
        self.mods = mods
        self.device = device
        self.params = [ops._w(m) for m in mods]
        self.ptrs = [w.data_ptr() for w in self.params]
        self._bwd_table = self._bwd_key = None
        bt = np.zeros(len(mods), dtype=BWD_DTYPE)
        for i, (m, (of, od, nf, shf, shd, su, sv)) in enumerate(zip(mods, self.slices)):
            e = bt[i]
            e["W"], e["off_g"] = self.params[i].data_ptr(), of
            e["Cout"], e["Cin"], e["taps"], e["perm_S"], e["Cin_p"] = table[i]["Cout"], table[i]["Cin"], table[i]["taps"], table[i]["perm_S"], table[i]["Cin_p"]
            if su is not None:
                e["has_sn"], e["off_u"], e["off_v"] = 1, su[0], sv[0]
        self._bwd_host = bt
        # conditional-BN affine maps as ONE GEMM in gradient-free passes (cbn_affine_all): the leading packs form one [rows][K] matrix
        self.cbn = None
        n = sum(1 for m in mods if getattr(m, "_cbn_affine", False))
        if n >= 2:
            Kp = int(table[0]["Cin_p"])
            rows, ok, spans = 0, True, []
            for i in range(n):
                e = table[i]
                ok = ok and int(e["taps"]) == 1 and int(e["Cin_p"]) == Kp and int(e["perm_S"]) == 1 and \
                    self.slices[i][0] == self.slices[0][0] + rows * Kp
                spans.append((rows, int(e["Cout"])))
                rows += int(e["Cout_p"])
            if ok:
                self.cbn = (n, rows, Kp, self.slices[0][0], spans)
        self._pf = None

    def bwd_table(self):
        """Device table for sgb_sn_backward_batch, valid while every layer's ``.grad`` is its view of the flat gradient arena
        (utils/arena.GradArena.attach); None otherwise (the per-layer path is used then)."""
        from .autograd_ops import _direct_grad
        grads = [_direct_grad(w) for w in self.params]
        if any(g is None for g in grads):
            return None
        key = tuple(g.data_ptr() for g in grads)
        if key != self._bwd_key:
            bt = self._bwd_host.copy()
            for i, k in enumerate(key):
                bt[i]["dW"] = k
            self._bwd_table = torch.from_numpy(bt.view(np.uint8).copy()).to(self.device)
            self._bwd_key = key
        return self._bwd_table

    def run(self):
        """Power-iterate (layers in train mode, as the reference's hooks) and pack every layer; leaves per-layer views in
        ``module._sn_cache`` for the ops of this forward pass."""
        W0 = next(self.net.parameters())
        if self.mods is None or self.device != W0.device or any(w.data_ptr() != p for w, p in zip(self.params, self.ptrs)):
            self._build(W0.device)
        dev = self.device
        training = self.mods[0].training
        need_grad = torch.is_grad_enabled()
        sigma = torch.empty(len(self.mods), device=dev, dtype=torch.float32)
        pf = torch.zeros(self.total_f, device=dev, dtype=torch.bfloat16)
        pd = torch.zeros(self.total_d, device=dev, dtype=torch.bfloat16) if need_grad else None
        mb = self.max_blocks
        L.call("sgb_sn_batch", L.ptr(self.table), len(self.mods), L.ptr(sigma), L.ptr(pf), L.ptr(pd), ops.SN_EPS,
               1 if training else 0, mb[0], mb[1], mb[2], L.stream_ptr())
        us = self.u_flat.clone() if need_grad else None
        vs = self.v_flat.clone() if need_grad else None
        cur = _Pass(self, sigma, us, vs) if need_grad else None
        self._pf = pf
        for i, (m, (of, od, nf, shf, shd, su, sv)) in enumerate(zip(self.mods, self.slices)):
            m._sn_pass = (cur, i) if cur is not None else None
            wf = pf[of:of + nf].view(shf)
            wd = pd[od:od + nf].view(shd) if pd is not None else None
            has_sn = su is not None
            m._sn_cache = (wf, wd, sigma[i:i + 1] if has_sn else None,
                           us[su[0]:su[1]] if (has_sn and us is not None) else None,
                           vs[sv[0]:sv[1]] if (has_sn and vs is not None) else None)

    def cbn_affine_all(self, y):
        """Gradient-free passes of a generator whose conditional batch norms all take the same conditioning vector ``y``
        ([B, K, 1, 1] bf16): every gain(y) / bias(y) (src/utils/ops.py:24-28, 2 x 48 small GEMMs per BigGAN-Deep forward) as ONE
        GEMM against the contiguous packs; each layer then reads its column slice (``module._pre_out``)."""
        if self.cbn is None or self._pf is None or torch.is_grad_enabled():
            return False
        n, rows, Kp, of0, spans = self.cbn
        if y.shape[1] != Kp:
            return False
        w = self._pf[of0:of0 + rows * Kp].view(rows, 1, Kp)
        out = K.conv_fprop(y, w, rows, 1, 1, 0, 0, out_fp32=True)
        out2 = out.permute(0, 2, 3, 1).reshape(y.shape[0], rows)
        for m, (r0, c) in zip(self.mods[:n], spans):
            m._pre_out = out2[:, r0:r0 + c]
        return True

    def clear(self):
        self._pf = None
        if self.mods:
            for m in self.mods:
                m._sn_cache = None
                m._sn_pass = None
                if getattr(m, "_cbn_affine", False):
                    m._pre_out = None
