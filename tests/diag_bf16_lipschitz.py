"""Diagnostic (not a test, CPU only): the error bf16 STORAGE alone puts into the DRAGAN and max-gradient penalties.

The reference formulations (tests/lipschitz_oracle.py) run over the fp32 oracle discriminator with every convolution
input, weight and output and every batch-norm output (and their gradients, through both backward passes) rounded to bf16
(tests/diag_bf16_emulation.py), against the reference golden vectors.  Printed per golden: the penalty's relative error,
the first gradient g's relative L2, and dP/dtheta by lipschitz_oracle.split_grad_errors (worst / median per-parameter
relative L2 and smallest cosine over the parameters with a nonzero gradient; the analytically zero bias gradients against
the weight beside them).  Quoted in DESIGN.md section 4 and in tests/test_gpu_lipschitz.py:

    python tests/diag_bf16_lipschitz.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "pytorch-studiogan_b200")):
    sys.path.insert(0, p)
import diag_bf16_emulation as E  # noqa: E402
import lipschitz_oracle as LO  # noqa: E402
from oracle import studiogan_oracle as O  # noqa: E402
from test_resfamily_cpu import load_sd  # noqa: E402


if __name__ == "__main__":
    O.conv, O.batch_norm = E.conv, E.bn
    for tag in ("dra_resnet32_bn_c16", "maxgp_resnet32_bn_c16"):
        g = np.load(os.path.join(ROOT, "tests", "golden", tag + ".npz"))
        sd = load_sd(g, "D0/", grad=True)
        yr = torch.from_numpy(g["y_real"])
        real, fake, alpha = (torch.from_numpy(g[k]) for k in ("real", "fake", "alpha"))
        disc = lambda x: O.res_discriminator(sd, x, yr, 32, 16, cond="W/O")[0]   # noqa: E731
        x = torch.from_numpy(g["x_hat"]).requires_grad_(True)
        (gr,) = torch.autograd.grad(disc(x).sum(), x)
        for v in sd.values():
            v.grad = None
        sd = load_sd(g, "D0/", grad=True)
        if tag.startswith("dra"):
            pen = LO.dra_penalty(disc, real, torch.from_numpy(g["noise"]), alpha)
        else:
            pen = LO.maxgrad_penalty(disc, real, fake, alpha)
        pen.backward()
        e_pen = abs(float(pen.detach()) - float(g["penalty"])) / abs(float(g["penalty"]))
        e_g = float((gr - torch.from_numpy(g["g"])).norm() / torch.from_numpy(g["g"]).norm())
        got = {k[6:]: (sd[k[6:]].grad if sd[k[6:]].grad is not None else torch.zeros(g[k].shape)) for k in g.files
               if k.startswith("Dgrad/")}
        worst, median, cos, ratio = LO.split_grad_errors(got, {n: torch.from_numpy(g["Dgrad/" + n]) for n in got})
        print("%-22s penalty err %.4f  g err %.3f  dP/dtheta worst %.3f median %.3f cosine %.4f, zero-gradient biases %.3g" % (
            tag, e_pen, e_g, worst[0], median, cos, ratio))
