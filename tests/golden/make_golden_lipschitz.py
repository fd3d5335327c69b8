"""Generates the DRAGAN and max-gradient penalty goldens under tests/golden/ by running the UNMODIFIED reference (a
PyTorch-StudioGAN checkout; SGB_REFERENCE = its src/ directory) on seeded CPU inputs, with the stubs and helpers of
make_golden.py:

    SGB_REFERENCE=<checkout>/src PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_lipschitz.py [dra] [maxgp]

Writes dra_resnet32_bn_c16.npz and maxgp_resnet32_bn_c16.npz (both when no name is given); no other fixture is touched.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, MODEL, modules, rlosses, rres, sd_np, torch  # noqa: E402


def _lipschitz_setup(B, img_size=32, conv_dim=16, classes=5):
    """The WGAN-style resnet discriminator of golden_gp("gp_resnet32_bn_c16"): batch norm, no spectral norm, no
    conditioning; seeded real / fake / labels."""
    torch.manual_seed(777)
    M = modules(g_sn=True, d_sn=False, cbn=True)
    D = rres.Discriminator(img_size=img_size, d_conv_dim=conv_dim, apply_d_sn=False, apply_attn=False, attn_d_loc=[1],
                           d_cond_mtd="W/O", aux_cls_type="W/O", d_embed_dim="N/A", normalize_d_embed=False, num_classes=classes,
                           d_init="ortho", d_depth="N/A", mixed_precision=False, MODULES=M, MODEL=MODEL)
    D.train()
    real = torch.rand(B, 3, img_size, img_size) * 2 - 1
    fake = torch.tanh(torch.randn(B, 3, img_size, img_size))
    y_real = torch.randint(0, classes, (B,))
    return D, real, fake, y_real


def _lipschitz_save(tag, D, D0, x_hat, y_real, pen, extra):
    """First gradient g on a copy of the initial discriminator (every forward moves the running statistics), then the
    penalty's own dP/dtheta (already in D's .grad) and the D1 buffers."""
    import copy
    D2 = copy.deepcopy(D0)
    x = x_hat.detach().clone().requires_grad_(True)
    adv = D2(x, y_real, eval=False)["adv_output"]
    g = rlosses.cal_deriv(inputs=x, outputs=adv, device="cpu")
    out = {}
    out.update(sd_np(D0, "D0/"))
    out.update(extra)
    out.update({"x_hat": x_hat.detach().numpy(), "adv_hat": adv.detach().numpy(), "g": g.detach().numpy(), "y_real": y_real.numpy(),
                "sumsq": (g.flatten(1).norm(dim=1) ** 2).detach().numpy(), "penalty": pen.detach().numpy()})
    for k, p in D.named_parameters():
        out["Dgrad/" + k] = (p.grad.detach().numpy().copy() if p.grad is not None else np.zeros(tuple(p.shape), np.float32))
    out.update(sd_np(D, "D1/", True))
    np.savez_compressed(os.path.join(HERE, tag + ".npz"), **out)
    print(tag, "keys", len(out), "penalty", float(pen.detach()), "||g||^2 per sample", out["sumsq"].tolist())
    return out


def golden_dra(tag="dra_resnet32_bn_c16", B=8):
    """losses.cal_dra_penalty (src/utils/losses.py:319-335) on the WGAN-style discriminator.  Its two host draws (alpha
    [B,1,1,1], then the noise shaped like the batch) are captured by re-seeding torch's host RNG before the call."""
    import copy
    D, real, fake, y_real = _lipschitz_setup(B)
    D0 = copy.deepcopy(D)
    torch.manual_seed(101)
    alpha = torch.rand(B, 1, 1, 1)
    noise = torch.rand(real.size())
    sigma = real.std()
    x_hat = real + (alpha * (0.5 * sigma * noise))
    torch.manual_seed(101)
    pen = rlosses.cal_dra_penalty(real_images=real, real_labels=y_real, discriminator=D, device="cpu")
    pen.backward()
    _lipschitz_save(tag, D, D0, x_hat, y_real, pen, {"real": real.numpy(), "fake": fake.numpy(), "alpha": alpha.numpy(),
                                                     "noise": noise.numpy(), "sigma": sigma.numpy()})


def golden_maxgp(tag="maxgp_resnet32_bn_c16", B=8, gap=1.25):
    """losses.cal_maxgrad_penalty (src/utils/losses.py:337-353) on the WGAN-style discriminator, alpha [B,1] captured by
    re-seeding.  The seed is the first one whose largest ||g_b||^2 exceeds the runner-up by ``gap``: bf16 rounding of g
    on the device (a few percent) then cannot move the arg-max."""
    import copy
    D, real, fake, y_real = _lipschitz_setup(B)
    D0 = copy.deepcopy(D)
    for seed in range(200, 300):
        torch.manual_seed(seed)
        alpha = torch.rand(B, 1)
        a4 = alpha.view(B, 1, 1, 1)
        x = (a4 * real + (1 - a4) * fake).requires_grad_(True)
        g = rlosses.cal_deriv(inputs=x, outputs=copy.deepcopy(D0)(x, y_real, eval=False)["adv_output"], device="cpu")
        top = (g.flatten(1).norm(dim=1) ** 2).detach().sort(descending=True).values
        if float(top[0]) >= gap * float(top[1]):
            break
    assert float(top[0]) >= gap * float(top[1]), (seed, top[:2])
    torch.manual_seed(seed)
    pen = rlosses.cal_maxgrad_penalty(real_images=real, real_labels=y_real, fake_images=fake, discriminator=D, device="cpu")
    pen.backward()
    _lipschitz_save(tag, D, D0, (a4 * real + (1 - a4) * fake), y_real, pen, {"real": real.numpy(), "fake": fake.numpy(),
                                                                              "alpha": alpha.numpy()})


GOLDENS = {"dra": golden_dra, "maxgp": golden_maxgp}

if __name__ == "__main__":
    for name in sys.argv[1:] or list(GOLDENS):
        GOLDENS[name]()
