"""DRAGAN (WGAN-DRA), max-gradient (LGAN) and weight-clipping (WGAN-WC) training on the CPU: the reference formulations
pinned to the reference's own numbers, the three reference yaml files, the worker's accepted / refused flags, and the
reverse-over-forward identity for both penalties' seeds (utils/gp.py) in float64."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lipschitz_oracle as LO
from oracle import studiogan_oracle as O
from sgb200 import config as C
from test_resfamily_cpu import load_sd

GOLDENS = ["dra_resnet32_bn_c16", "maxgp_resnet32_bn_c16"]


@pytest.mark.parametrize("tag", GOLDENS)
def test_oracle_penalty_matches_reference(golden_dir, tag):
    """The reference formulations over O.res_discriminator (the WGAN-style batch-norm discriminator, conv_dim 16, B = 8)
    reproduce cal_dra_penalty / cal_maxgrad_penalty (src/utils/losses.py:319-353): x_hat bit exact, g, the penalty and
    dP/dtheta from the double backward, and the running statistics afterwards."""
    g = np.load(os.path.join(golden_dir, tag + ".npz"))
    sdD = load_sd(g, "D0/", grad=True)
    real, fake, yr = (torch.from_numpy(g[k]) for k in ("real", "fake", "y_real"))
    alpha = torch.from_numpy(g["alpha"])

    def disc(x):
        return O.res_discriminator(sdD, x, yr, 32, 16, cond="W/O")[0]
    if tag.startswith("dra"):
        noise = torch.from_numpy(g["noise"])
        assert float(real.std()) == float(g["sigma"])
        assert np.array_equal(LO.dra_interpolate(real, noise, alpha).numpy(), g["x_hat"])
        pen = LO.dra_penalty(disc, real, noise, alpha)
    else:
        a4 = alpha.view(-1, 1, 1, 1)
        assert np.array_equal((a4 * real + (1 - a4) * fake).numpy(), g["x_hat"])
        top = np.sort(g["sumsq"])[::-1]
        assert top[0] >= 1.25 * top[1]                # the arg-max cannot move under bf16 rounding of g
        pen = LO.maxgrad_penalty(disc, real, fake, alpha)
    np.testing.assert_allclose(pen.item(), g["penalty"], rtol=2e-4)
    x = torch.from_numpy(g["x_hat"]).requires_grad_(True)
    sd2 = load_sd(g, "D0/")
    (gr,) = torch.autograd.grad(O.res_discriminator(sd2, x, yr, 32, 16, cond="W/O")[0].sum(), x)
    assert float((gr - torch.from_numpy(g["g"])).norm() / torch.from_numpy(g["g"]).norm()) < 1e-4
    pen.backward()
    gmax = max(np.abs(g[k]).max() for k in g.files if k.startswith("Dgrad/"))
    for k in g.files:
        if k.startswith("Dgrad/"):
            got = sdD[k[6:]].grad
            got = got.numpy() if got is not None else np.zeros_like(g[k])
            assert np.abs(got - g[k]).max() <= 1e-2 * (1e-3 * gmax + np.abs(g[k]).max()), k
    for k in g.files:
        if k.startswith("D1/") and "running_" in k:
            np.testing.assert_allclose(sdD[k[3:]].detach().numpy(), g[k], rtol=2e-4, atol=1e-5, err_msg=k)


def test_reference_lipschitz_yaml_configs_load(golden_dir):
    """The reference's WGAN-DRA, LGAN and WGAN-WC yaml files (copies under tests/golden/reference_configs) load unchanged."""
    ref_cfgs = os.path.join(golden_dir, "reference_configs", "CIFAR10")
    want = {"WGAN-DRA.yaml": ("apply_dra", "dra_lambda", 10.0), "LGAN.yaml": ("apply_maxgp", "maxgp_lambda", 10.0),
            "WGAN-WC.yaml": ("apply_wc", "wc_bound", 0.01)}
    for name, (flag, key, value) in want.items():
        cfg = C.Configurations(os.path.join(ref_cfgs, name))
        assert getattr(cfg.LOSS, flag) is True and getattr(cfg.LOSS, key) == value
        assert cfg.MODEL.backbone == "resnet" and callable(cfg.LOSS.d_loss)


def _worker(cfgs):
    from sgb200.worker import WORKER
    return WORKER(cfgs=cfgs, run_name="t", Gen=None, Gen_mapping=None, Gen_synthesis=None, Dis=None, Gen_ema=None,
                  Gen_ema_mapping=None, Gen_ema_synthesis=None, ema=None, eval_model=None, train_dataloader=None,
                  eval_dataloader=None, global_rank=0, local_rank="cpu", mu=None, sigma=None, real_feats=None, logger=None)


def test_worker_accepts_lipschitz_flags_and_refuses_the_rest(golden_dir):
    ref_cfgs = os.path.join(golden_dir, "reference_configs", "CIFAR10")
    for name in ("WGAN-DRA.yaml", "LGAN.yaml", "WGAN-WC.yaml"):
        _worker(C.Configurations(os.path.join(ref_cfgs, name)))
    for flag in ("apply_lo", "apply_topk", "apply_r1_reg", "apply_fm", "apply_inv_reg"):
        cfgs = C.Configurations(None)
        setattr(cfgs.LOSS, flag, True)
        with pytest.raises(NotImplementedError, match=flag):
            _worker(cfgs)
    cfgs = C.Configurations(None)
    cfgs.LOSS.adv_loss = "MH"
    with pytest.raises(NotImplementedError):
        _worker(cfgs)


def test_worker_weight_clipping_on_the_torch_optimiser_path():
    """Without the arena optimiser (CPU parameters) the clip is torch's own clamp_ on every discriminator parameter."""
    cfgs = C.Configurations(None)
    cfgs.LOSS.apply_wc, cfgs.LOSS.wc_bound = True, 0.01
    D = torch.nn.Sequential(torch.nn.Conv2d(3, 4, 3), torch.nn.BatchNorm2d(4))
    cfgs.OPTIMIZATION.d_optimizer = torch.optim.Adam(D.parameters())
    w = _worker(cfgs)
    w.Dis = D
    ref = [p.detach().clamp(-0.01, 0.01) for p in D.parameters()]
    w._clip_discriminator_weights()
    for p, r in zip(D.parameters(), ref):
        assert torch.equal(p.detach(), r)
    assert any(float(p.detach().abs().max()) == np.float32(0.01) for p in D.parameters())


# ------------------------------------------------------------------------------------ reverse-over-forward identity
EPS = 1e-4


def _tiny_disc(seed):
    """conv -> BN -> ReLU -> conv -> ReLU -> spatial sum -> linear, float64: (params, forward, tangent forward)."""
    g = torch.Generator().manual_seed(seed)
    dd = torch.float64
    w1 = (torch.randn(6, 3, 3, 3, dtype=dd, generator=g) * 0.3).requires_grad_(True)
    w2 = (torch.randn(4, 6, 3, 3, dtype=dd, generator=g) * 0.3).requires_grad_(True)
    g1 = (torch.rand(6, dtype=dd, generator=g) + 0.5).requires_grad_(True)
    b1 = torch.zeros(6, dtype=dd, requires_grad=True)
    wl = torch.randn(1, 4, dtype=dd, generator=g, requires_grad=True)
    params = (w1, w2, g1, wl)

    def disc(img):
        h = F.relu(F.batch_norm(F.conv2d(img, w1, padding=1), None, None, g1, b1, True, 0.1, EPS))
        return F.linear(F.relu(F.conv2d(h, w2, padding=1)).sum((2, 3)), wl).squeeze(1)

    def tangent(x_hat, v):
        """Output of the tangent pass along v, as utils/gp.py replays the tape: linear maps on the tangent, the primal's ReLU
        masks, and the batch-norm tangent with the batch statistics' terms."""
        h, th = F.conv2d(x_hat, w1, padding=1), F.conv2d(v, w1, padding=1)
        y = F.relu(F.batch_norm(h, None, None, g1, b1, True, 0.1, EPS))
        ty = O.bn_tangent(h, th, g1, EPS) * (y > 0)
        h2, th2 = F.conv2d(y, w2, padding=1), F.conv2d(ty, w2, padding=1)
        return F.linear((th2 * (h2 > 0)).sum((2, 3)), wl).squeeze(1)
    return params, disc, tangent


def _reverse_over_forward(params, disc, tangent, x_hat, seed_fn):
    x = x_hat.detach().requires_grad_(True)
    (gr,) = torch.autograd.grad(disc(x).sum(), x)
    pen, v = seed_fn(gr)
    return pen, torch.autograd.grad(tangent(x.detach(), v).sum(), params)


def _max_seed(gr):
    """The sgb_gp_seed_max formula: 2 g_b / n_ties on the arg-max sample(s)."""
    s = gr.flatten(1).pow(2).sum(1)
    tie = (s == s.max()).to(gr.dtype)
    return s.max(), (2.0 * tie / tie.sum()).view(-1, 1, 1, 1) * gr


def _unit_norm_seed(gr):
    """The sgb_gp_seed formula: 2 (||g_b|| - 1) / (B ||g_b||) g_b."""
    n = gr.flatten(1).norm(dim=1)
    return ((n - 1) ** 2).mean(), (2 * (n - 1) / (len(n) * n)).view(-1, 1, 1, 1) * gr


@pytest.mark.parametrize("tie", [False, True])
def test_maxgrad_seed_reverse_over_forward_equals_double_backward(tie):
    """dP/dtheta of the max-gradient penalty from the seed 2 g_b / n_ties through a tangent pass equals the reference's
    double backward (torch's max() backward splits the gradient over ties), with one arg-max and with a two-way tie."""
    params, disc, tangent = _tiny_disc(0)
    dd = torch.float64
    gen = torch.Generator().manual_seed(1)
    real, fake = torch.randn(5, 3, 6, 6, dtype=dd, generator=gen), torch.randn(5, 3, 6, 6, dtype=dd, generator=gen)
    alpha = torch.rand(5, 1, dtype=dd, generator=gen)
    if tie:      # two identical samples: identical input gradients under batch norm's symmetric statistics
        a4 = alpha.view(5, 1, 1, 1)
        x0 = a4 * real + (1 - a4) * fake
        (gr,) = torch.autograd.grad(disc(x0.requires_grad_(True)).sum(), x0)
        k = int(gr.flatten(1).norm(dim=1).argmax())
        j = (k + 1) % 5
        real[j], fake[j], alpha[j] = real[k], fake[k], alpha[k]
    ref_pen = LO.maxgrad_penalty(disc, real, fake, alpha)
    ref = torch.autograd.grad(ref_pen, params)
    a4 = alpha.view(5, 1, 1, 1)
    pen, got = _reverse_over_forward(params, disc, tangent, a4 * real + (1 - a4) * fake, _max_seed)
    x = (a4 * real + (1 - a4) * fake).requires_grad_(True)
    (gr,) = torch.autograd.grad(disc(x).sum(), x)
    s = gr.flatten(1).pow(2).sum(1)
    assert int((s == s.max()).sum()) == (2 if tie else 1)
    assert abs(float(pen) - float(ref_pen.detach())) < 1e-10 * float(ref_pen.detach())
    for r_, g_ in zip(ref, got):
        assert float((r_ - g_).abs().max()) < 1e-8 * (1 + float(r_.abs().max()))


def test_dra_seed_reverse_over_forward_equals_double_backward():
    """The same identity for the DRAGAN penalty at its perturbed real batch (x_hat does not depend on theta)."""
    params, disc, tangent = _tiny_disc(2)
    dd = torch.float64
    gen = torch.Generator().manual_seed(3)
    real = torch.randn(4, 3, 6, 6, dtype=dd, generator=gen)
    noise, alpha = torch.rand(4, 3, 6, 6, dtype=dd, generator=gen), torch.rand(4, 1, 1, 1, dtype=dd, generator=gen)
    ref_pen = LO.dra_penalty(disc, real, noise, alpha)
    ref = torch.autograd.grad(ref_pen, params)
    pen, got = _reverse_over_forward(params, disc, tangent, LO.dra_interpolate(real, noise, alpha), _unit_norm_seed)
    assert abs(float(pen) - float(ref_pen.detach())) < 1e-10 * float(ref_pen.detach())
    for r_, g_ in zip(ref, got):
        assert float((r_ - g_).abs().max()) < 1e-8 * (1 + float(r_.abs().max()))
