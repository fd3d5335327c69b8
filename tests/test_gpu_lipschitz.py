"""DRAGAN (WGAN-DRA), max-gradient (LGAN) and weight-clipping (WGAN-WC) training through the CUDA path (pytest -m gpu):
the four new kernels, both penalties against the reference's own numbers and against float64 at the configs' own shape,
and WORKER steps with each flag.

Tolerances of the penalties (the golden comparison follows test_gpu_parity.test_grad_penalty_vs_reference_golden; the
bounds come from tests/diag_bf16_lipschitz.py, the fp32 oracle with bf16 storage at every layer boundary, whose figures on
the two goldens are
    dra_resnet32_bn_c16    penalty 0.0011  g 0.162  dP/dtheta worst 0.191 median 0.105 cosine 0.983
    maxgp_resnet32_bn_c16  penalty 0.0034  g 0.164  dP/dtheta worst 0.254 median 0.185 cosine 0.967):
* first gradient g: relative L2 <= 0.25, as for the batch-norm WGAN-GP golden;
* penalty value: 5e-2 relative;
* dP/dtheta (lipschitz_oracle.split_grad_errors): worst per-parameter relative L2 <= 0.35, cosine >= 0.93, median <= 0.15
  for DRAGAN.  The max-gradient penalty's seed lives on one sample, so nothing averages its rounding over the batch: the
  emulation's median is 0.185 already, and the bound is 0.25.  Biases with an analytically zero gradient (the head bias,
  those a later batch norm removes; round-off in the reference) carry only rounding noise of the tangent pass: <= 2e-2 of
  the gradient of the weight beside them, the rule of test_gpu_resfamily_shapes.py.
"""
import copy
import os

import numpy as np
import pytest
import torch

import lipschitz_oracle as LO
from oracle import studiogan_oracle as O
from test_gpu_parity import _cuda, l2_err, rel_err

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_CFGS = os.path.join(ROOT, "tests", "golden", "reference_configs", "CIFAR10")
BOUND = {"dra": dict(penalty=5e-2, worst=0.35, median=0.15, cos=0.93),
         "maxgp": dict(penalty=5e-2, worst=0.35, median=0.25, cos=0.93)}


# ------------------------------------------------------------------------------------------------ kernels
def test_dra_std_and_perturb_kernels(golden_dir):
    """sgb_dra_std: the golden sigma (torch's fp32 std of the batch) to within one ulp, and 1e-6 relative of the float64
    std on a 64-image 128x128 batch; sgb_dra_perturb fed the golden sigma: the golden x_hat bit for bit."""
    from sgb200 import kernels as K
    dev = _cuda()
    g = np.load(os.path.join(golden_dir, "dra_resnet32_bn_c16.npz"))
    real = torch.from_numpy(g["real"]).to(dev)
    s, ref = np.float32(K.dra_std(real).item()), np.float32(g["sigma"])
    assert s in (np.nextafter(ref, np.float32(-np.inf)), ref, np.nextafter(ref, np.float32(np.inf))), (s, ref)
    big = torch.rand((64, 3, 128, 128), generator=torch.Generator(device=dev).manual_seed(5), device=dev) * 1.7 - 0.4
    s64 = float(big.double().std())
    assert abs(K.dra_std(big).item() - s64) <= 1e-6 * s64
    sigma = torch.from_numpy(g["sigma"]).reshape(1).to(dev)
    alpha, noise = torch.from_numpy(g["alpha"]).reshape(-1).to(dev), torch.from_numpy(g["noise"]).to(dev)
    x_hat = K.dra_perturb(real, sigma, alpha, noise)
    assert np.array_equal(x_hat.cpu().numpy(), g["x_hat"])


@pytest.mark.parametrize("tie", [False, True])
def test_gp_seed_max_matches_autograd_of_max(tie):
    """P and dP/dg of max_b ||g_b||^2 against torch autograd in float64; with an exact two-way tie the gradient is split
    evenly between the tied samples, as torch's max() backward does."""
    from sgb200 import kernels as K
    dev = _cuda()
    gr = torch.randn(6, 3, 8, 8, generator=torch.Generator().manual_seed(4))
    gr[1] *= 1.5
    if tie:
        gr[4] = gr[1]
    gd = gr.to(dev)
    ss = K.gp_sumsq(gd)
    pen, v = K.gp_seed_max(gd, ss)
    g64 = gr.double().requires_grad_(True)
    P = torch.max(g64.flatten(1).norm(dim=1) ** 2)
    (dg,) = torch.autograd.grad(P, g64)
    assert abs(pen.item() - float(P)) <= 1e-6 * float(P)
    np.testing.assert_allclose(v.cpu().double().numpy(), dg.numpy(), rtol=1e-5, atol=1e-7)
    nonzero = [b for b in range(6) if float(v[b].abs().max()) > 0]
    assert nonzero == ([1, 4] if tie else [1]), nonzero
    if tie:
        assert ss[1].item() == ss[4].item()


def test_clamp_kernel_bit_exact_against_torch_clamp():
    """sgb_clamp == torch.clamp(-c, c) bit for bit on a ragged length, with values at +-c, +-0, +-inf and NaN."""
    from sgb200 import kernels as K
    dev = _cuda()
    c = 0.01
    x = torch.randn(1000003, generator=torch.Generator().manual_seed(6)) * 0.02
    cf = float(np.float32(c))
    f32 = np.float32
    special = [cf, -cf, 0.0, -0.0, float("inf"), -float("inf"), float("nan"), float(np.nextafter(f32(c), f32(1))),
               float(np.nextafter(f32(-c), f32(-1))), float(np.nextafter(f32(c), f32(0))), 1e30, -1e-30]
    x[:len(special)] = torch.tensor(special)
    x[-len(special):] = torch.tensor(special)
    xd = x.to(dev)
    ref = xd.clamp(-c, c)
    K.clamp_(xd, c)
    assert torch.equal(xd.view(torch.int32), ref.view(torch.int32))


# ------------------------------------------------------------------------------------------------ penalties vs goldens
def _golden_disc(g, dev):
    from sgb200 import config as C
    from sgb200.models import resnet
    M = C.make_modules(True, False, "cBN", "resnet")
    MODEL = C._Section(info_type="N/A", g_info_injection="N/A")
    D = resnet.Discriminator(img_size=32, d_conv_dim=16, apply_d_sn=False, apply_attn=False, attn_d_loc=[1], d_cond_mtd="W/O",
                             aux_cls_type="W/O", d_embed_dim="N/A", normalize_d_embed=False, num_classes=5, d_init="ortho",
                             d_depth="N/A", mixed_precision=False, MODULES=M, MODEL=MODEL)
    D.load_state_dict({k[3:]: torch.from_numpy(g[k].copy()) for k in g.files if k.startswith("D0/")}, strict=True)
    return D.to(dev).train()


@pytest.mark.parametrize("kind", ["dra", "maxgp"])
def test_penalty_vs_reference_golden(golden_dir, kind):
    """losses.cal_dra_penalty / cal_maxgrad_penalty through the CUDA path (primal, input-gradient and tangent passes)
    against the reference's double backward with the same host draws, on the WGAN-style batch-norm discriminator
    (conv_dim 16, B = 8).  For max-GP the arg-max sample is checked first.  Bounds: BOUND (module docstring)."""
    from sgb200 import kernels as K
    from sgb200.utils import gp as gp_mod
    from sgb200.utils import losses
    dev = _cuda()
    g = np.load(os.path.join(golden_dir, kind + "_resnet32_bn_c16.npz"))
    D = _golden_disc(g, dev)
    real, fake, yr = (torch.from_numpy(g[k]).to(dev) for k in ("real", "fake", "y_real"))
    alpha = torch.from_numpy(g["alpha"])
    D2 = copy.deepcopy(D)
    x_hat = torch.from_numpy(g["x_hat"]).to(dev).requires_grad_(True)
    adv = D2(x_hat, yr)["adv_output"]
    assert l2_err(adv, torch.from_numpy(g["adv_hat"])) < 4e-2
    g1 = gp_mod.cal_deriv(x_hat, adv)
    e_g = l2_err(g1, torch.from_numpy(g["g"]))
    assert e_g < 0.25, e_g
    ss = K.gp_sumsq(g1).cpu().numpy()
    if kind == "maxgp":
        assert int(np.argmax(ss)) == int(np.argmax(g["sumsq"])), (ss, g["sumsq"])
        pen = losses.cal_maxgrad_penalty(real_images=real, real_labels=yr, fake_images=fake, discriminator=D, device=dev,
                                         alpha=alpha)
    else:
        pen = losses.cal_dra_penalty(real_images=real, real_labels=yr, discriminator=D, device=dev, alpha=alpha,
                                     noise=torch.from_numpy(g["noise"]))
    pen.backward()
    got = {n: (p.grad if p.grad is not None else torch.zeros_like(p)).cpu() for n, p in D.named_parameters()}
    worst, median, cos, zero_ratio = LO.split_grad_errors(got, {n: torch.from_numpy(g["Dgrad/" + n]) for n in got})
    e_pen = abs(float(pen.detach()) - float(g["penalty"])) / abs(float(g["penalty"]))
    print("%s golden: g err %.3f, ||g_b||^2 err %.2e, penalty err %.2e; grads worst %.3f (%s) median %.3f min cosine %.4f; "
          "zero-gradient biases %.3g of their weight" % (kind, e_g, float(np.abs(ss / g["sumsq"] - 1).max()), e_pen, worst[0],
                                                        worst[1], median, cos, zero_ratio))
    b = BOUND[kind]
    assert e_pen <= b["penalty"], (float(pen.detach()), float(g["penalty"]))
    assert worst[0] <= b["worst"] and median <= b["median"] and cos >= b["cos"], (worst, median, cos)
    assert zero_ratio <= 2e-2
    for n, buf in D.named_buffers():
        if "running_" in n:
            assert rel_err(buf, torch.from_numpy(g["D1/" + n])) < 1e-2, n


# ------------------------------------------------------------------------------------------------ the configs' own shape
def _config_disc(B=64, img=32, conv_dim=64):
    """The resnet discriminator the three CIFAR10 configs build (d_conv_dim 64, batch norm, no SN), made on the CPU with
    seeded biases and batch-norm affine parameters (the initialisation zeroes them), plus seeded real / fake batches."""
    from sgb200 import config as C
    from sgb200.models import resnet
    from sgb200.utils import ops
    M = C.make_modules(False, False, "W/O", "resnet")
    MODEL = C._Section(info_type="N/A", g_info_injection="N/A")
    torch.manual_seed(0)
    D = resnet.Discriminator(img_size=img, d_conv_dim=conv_dim, apply_d_sn=False, apply_attn=False, attn_d_loc=["N/A"],
                             d_cond_mtd="W/O", aux_cls_type="W/O", d_embed_dim="N/A", normalize_d_embed=False, num_classes=10,
                             d_init="ortho", d_depth="N/A", mixed_precision=False, MODULES=M, MODEL=MODEL)
    gen = torch.Generator().manual_seed(2)
    with torch.no_grad():
        for m in D.modules():
            if isinstance(m, (torch.nn.Conv2d, torch.nn.Linear)) and m.bias is not None:
                m.bias.copy_(0.3 * torch.randn(m.bias.shape, generator=gen))
            if isinstance(m, ops.BatchNorm2d) and m.affine:
                m.weight.copy_(0.5 + torch.rand(m.weight.shape, generator=gen))
                m.bias.copy_(0.3 * torch.randn(m.bias.shape, generator=gen))
    gen = torch.Generator().manual_seed(91)
    real = torch.rand((B, 3, img, img), generator=gen) * 2 - 1
    fake = torch.tanh(torch.randn((B, 3, img, img), generator=gen))
    return D, real, fake


@pytest.mark.parametrize("kind", ["dra", "maxgp"])
def test_penalty_at_config_shape_vs_float64_double_backward(kind):
    """Both penalties through the 32x32 resnet discriminator at d_conv_dim 64 and B = 64 (the WGAN-DRA / LGAN configs'
    defaults) against the reference formulation over O.res_discriminator in float64 on the product's state dict.
    Gradients compared as for the goldens.  For max-GP the float64 top two ||g_b||^2 must differ by 5 % (alpha seed 117:
    8.8 %; the product's per-sample ||g_b||^2 measured up to 4 % off float64 on an H100) and the product must pick the
    same sample."""
    from sgb200 import kernels as K
    from sgb200.utils import gp as gp_mod
    from sgb200.utils import losses
    dev = _cuda()
    D, real, fake = _config_disc()
    B = real.shape[0]
    D = D.to(dev).train()
    labels = torch.zeros(B, dtype=torch.long, device=dev)
    names = [n for n, _ in D.named_parameters()]
    sd = {k: v.detach().double().clone().requires_grad_(k in names) for k, v in D.state_dict().items()}
    disc64 = lambda x: O.res_discriminator(sd, x, labels, 32, 64, cond="W/O")[0]   # noqa: E731
    real_d, fake_d = real.to(dev), fake.to(dev)
    if kind == "dra":
        gen = torch.Generator().manual_seed(93)
        alpha, noise = torch.rand((B, 1, 1, 1), generator=gen), torch.rand(real.shape, generator=gen)
        pen = losses.cal_dra_penalty(real_images=real_d, real_labels=labels, discriminator=D, device=dev, alpha=alpha, noise=noise)
        pen_ref = LO.dra_penalty(disc64, real_d.double(), noise.double().to(dev), alpha.double().to(dev))
    else:
        alpha = torch.rand((B, 1), generator=torch.Generator().manual_seed(117))
        a4 = alpha.view(B, 1, 1, 1).double().to(dev)
        x64 = (a4 * real_d.double() + (1 - a4) * fake_d.double()).requires_grad_(True)
        (g64,) = torch.autograd.grad(disc64(x64).sum(), x64)
        s64 = g64.flatten(1).pow(2).sum(1)
        top = s64.sort(descending=True).values
        assert float(top[0]) >= 1.05 * float(top[1]), top[:2]
        x_hat = K.gp_interpolate(real_d, fake_d, alpha.reshape(B).to(dev)).requires_grad_(True)
        g1 = gp_mod.cal_deriv(x_hat, copy.deepcopy(D)(x_hat, labels)["adv_output"])
        ss = K.gp_sumsq(g1)
        print("max-GP float64 top-two ratio %.4f, product ||g_b||^2 worst relative error %.2e" % (
            float(top[0] / top[1]), float((ss.double() / s64 - 1).abs().max())))
        assert int(ss.argmax()) == int(s64.argmax())
        for v in sd.values():
            v.grad = None
        pen = losses.cal_maxgrad_penalty(real_images=real_d, real_labels=labels, fake_images=fake_d, discriminator=D,
                                         device=dev, alpha=alpha)
        pen_ref = LO.maxgrad_penalty(disc64, real_d.double(), fake_d.double(), alpha.double().to(dev))
    pen.backward()
    pen_ref.backward()
    got = {n: (p.grad if p.grad is not None else torch.zeros_like(p)) for n, p in D.named_parameters()}
    worst, median, cos, zero_ratio = LO.split_grad_errors(got, {n: sd[n].grad for n in names})
    e_pen = abs(float(pen.detach()) - float(pen_ref.detach())) / abs(float(pen_ref.detach()))
    print("%s B=%d c64: penalty %.6g (float64 %.6g) err %.2e; grads worst %.3f (%s) median %.3f min cosine %.4f; zero-gradient "
          "biases %.3g of their weight" % (kind, B, float(pen.detach()), float(pen_ref.detach()), e_pen, worst[0], worst[1],
                                           median, cos, zero_ratio))
    b = BOUND[kind]
    assert e_pen <= b["penalty"] and worst[0] <= b["worst"] and median <= b["median"] and cos >= b["cos"]
    assert zero_ratio <= 2e-2


# ------------------------------------------------------------------------------------------------ worker
def _worker(yaml_name, cuda_graphs=False, d_updates=2):
    """WORKER from one of the reference yaml files, with 16-channel networks and B = 16 for speed."""
    from sgb200 import config as C
    from sgb200.models import model as M
    from sgb200.worker import WORKER
    dev = _cuda()
    cfgs = C.Configurations(os.path.join(REF_CFGS, yaml_name))
    cfgs.MODEL.z_dim, cfgs.MODEL.g_conv_dim, cfgs.MODEL.d_conv_dim, cfgs.MODEL.apply_g_ema = 32, 16, 16, False
    o = cfgs.OPTIMIZATION
    o.batch_size, o.d_updates_per_step, o.g_updates_per_step, o.acml_steps = 16, d_updates, 1, 1
    cfgs.RUN.cuda_graphs = cuda_graphs
    torch.manual_seed(0)
    Gen, _, _, Dis, Gen_ema, _, _, ema = M.load_generator_discriminator(cfgs.DATA, o, cfgs.MODEL, cfgs.STYLEGAN, cfgs.MODULES,
                                                                        cfgs.RUN, dev, None)
    cfgs.define_optimizer(Gen, Dis)

    class Loader:
        def __init__(self):
            self.i = 0

        def __iter__(self):
            return self

        def __next__(self):
            self.i += 1
            g = torch.Generator().manual_seed(self.i)
            n = 16 * d_updates
            return (torch.rand(n, 3, 32, 32, generator=g) * 2 - 1).pin_memory(), torch.randint(0, 10, (n,), generator=g).pin_memory()
    w = WORKER(cfgs=cfgs, run_name="t", Gen=Gen, Gen_mapping=None, Gen_synthesis=None, Dis=Dis, Gen_ema=Gen_ema, Gen_ema_mapping=None,
               Gen_ema_synthesis=None, ema=ema, eval_model=None, train_dataloader=Loader(), eval_dataloader=None, global_rank=0,
               local_rank=dev, mu=None, sigma=None, real_feats=None, logger=None)
    return w, cfgs, Gen, Dis


@pytest.mark.parametrize("yaml_name", ["WGAN-DRA.yaml", "LGAN.yaml"])
def test_worker_penalty_step_runs(yaml_name):
    """WORKER.train_discriminator / train_generator with LOSS.apply_dra (src/worker.py:378-384) or apply_maxgp (:386-392),
    from the reference's yaml: the penalty's three discriminator passes run inside the D phase, losses stay finite and
    both networks move; no CUDA graph (the penalties draw on the host RNG)."""
    w, cfgs, Gen, Dis = _worker(yaml_name, cuda_graphs=True)
    assert not w._graphs_enabled()
    d0 = [p.detach().clone() for p in Dis.parameters()]
    g0 = [p.detach().clone() for p in Gen.parameters()]
    for step in range(2):
        _, d_loss = w.train_discriminator(step)
        g_loss = w.train_generator(step)
        assert torch.isfinite(d_loss).all() and torch.isfinite(g_loss).all()
    assert all(torch.isfinite(p).all() for p in list(Dis.parameters()) + list(Gen.parameters()))
    assert any(float((p.detach() - q).abs().max()) > 0 for p, q in zip(Dis.parameters(), d0))
    assert any(float((p.detach() - q).abs().max()) > 0 for p, q in zip(Gen.parameters(), g0))


def _check_clipped(Dis, opt, c):
    params = list(Dis.parameters())
    assert all(float(p.detach().abs().max()) <= c for p in params)
    assert any(bool((p.detach().abs() == c).any()) for p in params)
    used = torch.zeros(opt.arena.flat.numel(), dtype=torch.bool, device=opt.arena.flat.device)
    for o, p in opt._offsets():
        used[o:o + p.numel()] = True
    pad = opt.arena.flat[~used]
    assert pad.numel() == 0 or float(pad.abs().max()) == 0.0


@pytest.mark.parametrize("cuda_graphs", [False, True])
def test_worker_weight_clipping(cuda_graphs):
    """LOSS.apply_wc (src/worker.py:490-492, WGAN-WC yaml, bound 0.01): after every train_discriminator each discriminator
    parameter lies in [-c, c], some sit exactly at +-c, the arena's padding stays zero.  With RUN.cuda_graphs the D phase,
    clip included, is captured and the bound holds after its replays."""
    w, cfgs, Gen, Dis = _worker("WGAN-WC.yaml", cuda_graphs=cuda_graphs)
    c = np.float32(cfgs.LOSS.wc_bound)
    assert w._graphs_enabled() == cuda_graphs
    for step in range(5):
        _, d_loss = w.train_discriminator(step)
        g_loss = w.train_generator(step)
        torch.cuda.synchronize()
        assert torch.isfinite(d_loss).all() and torch.isfinite(g_loss).all()
        _check_clipped(Dis, cfgs.OPTIMIZATION.d_optimizer, c)
    if cuda_graphs:
        assert w._d_graph.graph is not None and not w._d_graph.failed
        assert cfgs.OPTIMIZATION.d_optimizer.step_count == 10
