"""Generates the golden vectors under tests/golden/ by running the UNMODIFIED reference (a PyTorch-StudioGAN checkout;
SGB_REFERENCE = its src/ directory) on seeded CPU inputs:

    SGB_REFERENCE=<checkout>/src PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden.py

The tests must not depend on a reference checkout, so the resulting .npz files are committed next to this
script.  Missing plotting / IO packages of the reference are stubbed (they are not on the hot path), see SURVEY.md A.1.
"""
import os
import sys
import types
from unittest.mock import MagicMock

import numpy as np

os.environ.setdefault("PYTHONDONTWRITEBYTECODE", "1")
sys.dont_write_bytecode = True
for name in ["matplotlib", "matplotlib.pyplot", "seaborn", "h5py", "kornia", "kornia.filters", "kornia.geometry",
             "kornia.geometry.transform", "timm", "timm.models", "timm.models.layers"]:
    sys.modules[name] = MagicMock()
REF = os.environ.get("SGB_REFERENCE")
if not REF or not os.path.isdir(REF):
    sys.exit("set SGB_REFERENCE to the src/ directory of a PyTorch-StudioGAN checkout")
sys.path.insert(0, REF)

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

import utils.ops as rops  # noqa: E402  (reference)
import utils.losses as rlosses  # noqa: E402
import utils.ema as rema  # noqa: E402
import models.big_resnet_deep_legacy as rdeep  # noqa: E402
import models.big_resnet_deep_studiogan as rdeep_sg  # noqa: E402
import models.big_resnet as rbig  # noqa: E402
import models.resnet as rres  # noqa: E402
import models.deep_conv as rdc  # noqa: E402
import scipy.linalg  # noqa: E402
import metrics.fid as rfid  # noqa: E402
import metrics.ins as rins  # noqa: E402
import metrics.prdc as rprdc  # noqa: E402
import utils.resize as rresize  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def modules(g_sn=True, d_sn=True, cbn=True):
    m = types.SimpleNamespace()
    m.g_conv2d = rops.snconv2d if g_sn else rops.conv2d
    m.g_deconv2d = rops.sndeconv2d if g_sn else rops.deconv2d
    m.g_linear = rops.snlinear if g_sn else rops.linear
    m.g_embedding = rops.sn_embedding if g_sn else rops.embedding
    m.d_conv2d = rops.snconv2d if d_sn else rops.conv2d
    m.d_linear = rops.snlinear if d_sn else rops.linear
    m.d_embedding = rops.sn_embedding if d_sn else rops.embedding
    m.g_bn = rops.ConditionalBatchNorm2d if cbn else rops.batchnorm_2d
    if not d_sn:
        m.d_bn = rops.batchnorm_2d
    m.g_act_fn = nn.ReLU(inplace=True)
    m.d_act_fn = nn.ReLU(inplace=True)
    return m


MODEL = types.SimpleNamespace(info_type="N/A", g_info_injection="N/A")


def sd_np(module, prefix, buffers_only=False):
    """state_dict as numpy; ``buffers_only`` keeps u / v / running statistics only (parameters are unchanged between the
    G0/D0 and G1/D1 snapshots, so storing them twice would only bloat the fixtures)."""
    params = {k for k, _ in module.named_parameters()}
    return {prefix + k: v.detach().cpu().numpy().copy() for k, v in module.state_dict().items()
            if not (buffers_only and k in params)}


def golden_deep(tag, img_size, conv_dim, depth, attn, z_dim=16, shared=16, classes=5, B=3, rdeep=rdeep):
    torch.manual_seed(1234)
    M = modules()
    G = rdeep.Generator(z_dim=z_dim, g_shared_dim=shared, img_size=img_size, g_conv_dim=conv_dim, apply_attn=attn,
                        attn_g_loc=[2], g_cond_mtd="cBN", num_classes=classes, g_init="ortho", g_depth=depth,
                        mixed_precision=False, MODULES=M, MODEL=MODEL)
    D = rdeep.Discriminator(img_size=img_size, d_conv_dim=conv_dim, apply_d_sn=True, apply_attn=attn, attn_d_loc=[1],
                            d_cond_mtd="PD", aux_cls_type="W/O", d_embed_dim="N/A", normalize_d_embed=False,
                            num_classes=classes, d_init="ortho", d_depth=depth, mixed_precision=False, MODULES=M, MODEL=MODEL)
    G.train()
    D.train()
    # make the attention gate non-trivial (its init value 0 would hide the whole branch)
    with torch.no_grad():
        for mod in list(G.modules()) + list(D.modules()):
            if isinstance(mod, rops.SelfAttention):
                mod.sigma.fill_(0.37)
    out = {}
    out.update(sd_np(G, "G0/"))
    out.update(sd_np(D, "D0/"))
    z = torch.randn(B, z_dim)
    y_fake = torch.randint(0, classes, (B,))
    real = torch.rand(B, 3, img_size, img_size) * 2 - 1
    y_real = torch.randint(0, classes, (B,))
    out.update({"z": z.numpy(), "y_fake": y_fake.numpy(), "real": real.numpy(), "y_real": y_real.numpy()})

    # ---- discriminator phase (src/worker.py:213-497): G forward without graph, D(real), D(fake), hinge, backward
    for p in G.parameters():
        p.requires_grad_(False)
    fake = G(z, y_fake)
    real_d = D(real, y_real)
    fake_d = D(fake.detach(), y_fake)
    d_loss = rlosses.d_hinge(real_d["adv_output"], fake_d["adv_output"], False)
    d_loss.backward()
    out.update({"fake": fake.detach().numpy(), "adv_real": real_d["adv_output"].detach().numpy(),
                "adv_fake": fake_d["adv_output"].detach().numpy(), "h_real": real_d["h"].detach().numpy(),
                "d_loss": d_loss.detach().numpy()})
    for k, p in D.named_parameters():
        out["Dgrad/" + k] = p.grad.detach().numpy().copy()
    out.update(sd_np(G, "G1/", True))   # buffers after one forward (u, v, running stats)
    out.update(sd_np(D, "D1/", True))   # buffers after two forwards

    # ---- generator phase (src/worker.py:502-681): G forward with graph, D forward with frozen params, hinge, backward
    D.zero_grad()
    for p in G.parameters():
        p.requires_grad_(True)
    for p in D.parameters():
        p.requires_grad_(False)
    fake2 = G(z, y_fake)
    g_loss = rlosses.g_hinge(D(fake2, y_fake)["adv_output"], False)
    g_loss.backward()
    out.update({"fake2": fake2.detach().numpy(), "g_loss": g_loss.detach().numpy()})
    for k, p in G.named_parameters():
        out["Ggrad/" + k] = p.grad.detach().numpy().copy()
    np.savez_compressed(os.path.join(HERE, tag + ".npz"), **out)
    print(tag, "keys", len(out), "d_loss", float(d_loss), "g_loss", float(g_loss))


def grad_digest(out, prefix, named_params, full_below=16384, nproj=8):
    """Gradient record that stays small for MB-sized models: every tensor's norm and ``nproj`` seeded +-1 projections
    (an error e moves a projection by ~||e||), the full gradient for tensors below ``full_below`` elements."""
    for i, (k, p) in enumerate(named_params):
        g = p.grad.detach().double().flatten()
        out[prefix + "norm/" + k] = np.array(float(g.norm()))
        r = torch.randint(0, 2, (nproj, g.numel()), generator=torch.Generator().manual_seed(1000 + i)).double() * 2 - 1
        out[prefix + "proj/" + k] = (r @ g).numpy()
        if g.numel() <= full_below:
            out[prefix + "full/" + k] = p.grad.detach().numpy().copy()


def golden_deep_bench_shape(tag="deep256_c16_attn_d2", img_size=256, conv_dim=16, depth=2, B=16, z_dim=16, shared=16, classes=5):
    """BigGAN-Deep at BASELINE config 4's resolution and topology (256x256, g_depth = d_depth = 2, attention at 64x64 ->
    N = 4096 queries x M = 1024 keys, attn_g_loc [4] / attn_d_loc [2]) with conv_dim 16 so that the CPU reference runs in
    seconds.  No weights are stored: the reference modules are built under torch.manual_seed(1234) and the product modules
    reproduce that initialisation bit for bit (tests/test_host_cpu.py checks this); inputs are regenerated from seeds too.
    Stored: labels / z, sub-sampled images, logits, losses, buffer states and gradient digests (grad_digest)."""
    torch.manual_seed(1234)
    M = modules()
    G = rdeep.Generator(z_dim=z_dim, g_shared_dim=shared, img_size=img_size, g_conv_dim=conv_dim, apply_attn=True,
                        attn_g_loc=[4], g_cond_mtd="cBN", num_classes=classes, g_init="ortho", g_depth=depth,
                        mixed_precision=False, MODULES=M, MODEL=MODEL)
    D = rdeep.Discriminator(img_size=img_size, d_conv_dim=conv_dim, apply_d_sn=True, apply_attn=True, attn_d_loc=[2],
                            d_cond_mtd="PD", aux_cls_type="W/O", d_embed_dim="N/A", normalize_d_embed=False,
                            num_classes=classes, d_init="ortho", d_depth=depth, mixed_precision=False, MODULES=M, MODEL=MODEL)
    G.train(); D.train()
    with torch.no_grad():
        for mod in list(G.modules()) + list(D.modules()):
            if isinstance(mod, rops.SelfAttention):
                mod.sigma.fill_(0.37)
    out = {"param_l1_G": np.array(sum(float(p.detach().double().abs().sum()) for p in G.parameters())),
           "param_l1_D": np.array(sum(float(p.detach().double().abs().sum()) for p in D.parameters()))}
    gi = torch.Generator().manual_seed(77)
    z = torch.randn(B, z_dim, generator=gi)
    y_fake = torch.randint(0, classes, (B,), generator=gi)
    real = torch.rand(B, 3, img_size, img_size, generator=gi) * 2 - 1
    y_real = torch.randint(0, classes, (B,), generator=gi)
    out.update({"z": z.numpy(), "y_fake": y_fake.numpy(), "y_real": y_real.numpy(), "real_sum": np.array(float(real.double().sum()))})
    for p in G.parameters():
        p.requires_grad_(False)
    fake = G(z, y_fake)
    real_d = D(real, y_real)
    fake_d = D(fake.detach(), y_fake)
    # Wasserstein losses: every sample of both branches carries gradient (the seeded-init logits sit outside the hinge margins)
    d_loss = rlosses.d_wasserstein(real_d["adv_output"], fake_d["adv_output"], False)
    d_loss.backward()
    out.update({"fake_sub8": fake.detach()[:, :, ::8, ::8].numpy().copy(), "fake_mean_abs": np.array(float(fake.detach().abs().mean())),
                "adv_real": real_d["adv_output"].detach().numpy(), "adv_fake": fake_d["adv_output"].detach().numpy(),
                "h_real": real_d["h"].detach().numpy(), "d_loss": d_loss.detach().numpy()})
    grad_digest(out, "Dgrad/", list(D.named_parameters()))
    out.update(sd_np(G, "G1/", True))
    out.update(sd_np(D, "D1/", True))
    D.zero_grad()
    for p in G.parameters():
        p.requires_grad_(True)
    for p in D.parameters():
        p.requires_grad_(False)
    fake2 = G(z, y_fake)
    g_loss = rlosses.g_wasserstein(D(fake2, y_fake)["adv_output"], False)
    g_loss.backward()
    out.update({"fake2_sub8": fake2.detach()[:, :, ::8, ::8].numpy().copy(), "g_loss": g_loss.detach().numpy()})
    grad_digest(out, "Ggrad/", list(G.named_parameters()))
    np.savez_compressed(os.path.join(HERE, tag + ".npz"), **out)
    print(tag, "keys", len(out), "d_loss", float(d_loss), "g_loss", float(g_loss), "params",
          sum(p.numel() for p in G.parameters()), sum(p.numel() for p in D.parameters()))


def golden_resfamily(tag, family, conv_dim, attn, g_sn, d_sn, g_cond, d_cond, adv, z_dim=20, shared=16, classes=5, B=8, img_size=32):
    """BigGAN (big_resnet) / ResNetGAN (resnet): D phase + G phase exactly as golden_deep."""
    torch.manual_seed(4321)
    M = modules(g_sn=g_sn, d_sn=d_sn, cbn=(g_cond == "cBN" or family == "big_resnet"))
    mod = rbig if family == "big_resnet" else rres
    G = mod.Generator(z_dim=z_dim, g_shared_dim=shared, img_size=img_size, g_conv_dim=conv_dim, apply_attn=attn, attn_g_loc=[2],
                      g_cond_mtd=g_cond, num_classes=classes, g_init="ortho", g_depth="N/A", mixed_precision=False, MODULES=M, MODEL=MODEL)
    D = mod.Discriminator(img_size=img_size, d_conv_dim=conv_dim, apply_d_sn=d_sn, apply_attn=attn, attn_d_loc=[1], d_cond_mtd=d_cond,
                          aux_cls_type="W/O", d_embed_dim="N/A", normalize_d_embed=False, num_classes=classes, d_init="ortho",
                          d_depth="N/A", mixed_precision=False, MODULES=M, MODEL=MODEL)
    G.train(); D.train()
    with torch.no_grad():
        for m_ in list(G.modules()) + list(D.modules()):
            if isinstance(m_, rops.SelfAttention):
                m_.sigma.fill_(0.37)
    d_loss_fn = {"hinge": rlosses.d_hinge, "wasserstein": rlosses.d_wasserstein}[adv]
    g_loss_fn = {"hinge": rlosses.g_hinge, "wasserstein": rlosses.g_wasserstein}[adv]
    out = {}
    out.update(sd_np(G, "G0/")); out.update(sd_np(D, "D0/"))
    z = torch.randn(B, z_dim); y_fake = torch.randint(0, classes, (B,))
    real = torch.rand(B, 3, img_size, img_size) * 2 - 1; y_real = torch.randint(0, classes, (B,))
    out.update({"z": z.numpy(), "y_fake": y_fake.numpy(), "real": real.numpy(), "y_real": y_real.numpy()})
    for p in G.parameters():
        p.requires_grad_(False)
    fake = G(z, y_fake)
    real_d = D(real, y_real); fake_d = D(fake.detach(), y_fake)
    d_loss = d_loss_fn(real_d["adv_output"], fake_d["adv_output"], False)
    d_loss.backward()
    out.update({"fake": fake.detach().numpy(), "adv_real": real_d["adv_output"].detach().numpy(),
                "adv_fake": fake_d["adv_output"].detach().numpy(), "h_real": real_d["h"].detach().numpy(), "d_loss": d_loss.detach().numpy()})
    for k, p in D.named_parameters():
        out["Dgrad/" + k] = p.grad.detach().numpy().copy()
    out.update(sd_np(G, "G1/", True)); out.update(sd_np(D, "D1/", True))
    D.zero_grad()
    for p in G.parameters():
        p.requires_grad_(True)
    for p in D.parameters():
        p.requires_grad_(False)
    fake2 = G(z, y_fake)
    g_loss = g_loss_fn(D(fake2, y_fake)["adv_output"], False)
    g_loss.backward()
    out.update({"fake2": fake2.detach().numpy(), "g_loss": g_loss.detach().numpy()})
    for k, p in G.named_parameters():
        out["Ggrad/" + k] = p.grad.detach().numpy().copy()
    np.savez_compressed(os.path.join(HERE, tag + ".npz"), **out)
    print(tag, "keys", len(out), "d_loss", float(d_loss), "g_loss", float(g_loss))


def golden_gp(tag, family, conv_dim, d_sn, d_cond, classes=5, B=8, img_size=32, depth=1):
    """losses.cal_grad_penalty (src/utils/losses.py:301-316) of the reference discriminators: penalty value, the first
    gradient g = d(sum adv)/d(x_hat), and dP/dtheta from the reference's double backward.  alpha is captured by re-seeding
    torch's host RNG right before the call."""
    import copy
    torch.manual_seed(777)
    M = modules(g_sn=True, d_sn=d_sn, cbn=True)
    mod = {"big_resnet": rbig, "resnet": rres, "deep": rdeep}[family]
    D = mod.Discriminator(img_size=img_size, d_conv_dim=conv_dim, apply_d_sn=d_sn, apply_attn=False, attn_d_loc=[1], d_cond_mtd=d_cond,
                          aux_cls_type="W/O", d_embed_dim="N/A", normalize_d_embed=False, num_classes=classes, d_init="ortho",
                          d_depth=depth if family == "deep" else "N/A", mixed_precision=False, MODULES=M, MODEL=MODEL)
    D.train()
    out = {}
    out.update(sd_np(D, "D0/"))
    real = torch.rand(B, 3, img_size, img_size) * 2 - 1
    fake = torch.tanh(torch.randn(B, 3, img_size, img_size))
    y_real = torch.randint(0, classes, (B,))
    torch.manual_seed(99)
    alpha = torch.rand(B, 1)
    # first gradient on a copy (every forward moves u / running statistics)
    D2 = copy.deepcopy(D)
    a4 = alpha.view(B, 1, 1, 1)
    x_hat = (a4 * real + (1 - a4) * fake).requires_grad_(True)
    adv2 = D2(x_hat, y_real, eval=False)["adv_output"]
    g = rlosses.cal_deriv(inputs=x_hat, outputs=adv2, device="cpu")
    out.update({"x_hat": x_hat.detach().numpy(), "adv_hat": adv2.detach().numpy(), "g": g.detach().numpy()})
    torch.manual_seed(99)
    gp = rlosses.cal_grad_penalty(real_images=real, real_labels=y_real, fake_images=fake, discriminator=D, device="cpu")
    gp.backward()
    out.update({"real": real.numpy(), "fake": fake.numpy(), "y_real": y_real.numpy(), "alpha": alpha.numpy(), "gp": gp.detach().numpy()})
    for k, p in D.named_parameters():
        out["Dgrad/" + k] = (p.grad.detach().numpy().copy() if p.grad is not None else np.zeros(tuple(p.shape), np.float32))
    out.update(sd_np(D, "D1/", True))
    np.savez_compressed(os.path.join(HERE, tag + ".npz"), **out)
    print(tag, "keys", len(out), "gp", float(gp), "|g| per sample", g.flatten(1).norm(dim=1)[:4].tolist())


def golden_inception():
    """The reference's LoadEvalModel("InceptionV3_tf", "legacy").get_outputs (src/metrics/preparation.py:103-122 ->
    src/metrics/inception_net.py:81-107, FID blocks :135-249) on the seeded weights of
    sgb200.metrics.inception_net.seeded_state_dict(0): the pretrained file cannot be downloaded here, so the weight
    download inside fid_inception_v3 (:130) is replaced by that state dict -- topology and arithmetic are the reference's."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "pytorch-studiogan_b200"))
    from sgb200.metrics.inception_net import seeded_state_dict
    import metrics.inception_net as rinc
    import metrics.preparation as rprep
    rinc.load_state_dict_from_url = lambda *a, **k: seeded_state_dict(0)
    ev = rprep.LoadEvalModel("InceptionV3_tf", "legacy", 1, False, "cpu")
    ev.eval()
    torch.manual_seed(11)
    x = torch.tanh(torch.randn(2, 3, 32, 32) * 1.2)
    with torch.no_grad():
        pool, logits = ev.get_outputs(x, quantize=True)
    np.savez_compressed(os.path.join(HERE, "inception_seed0.npz"), x=x.numpy(), pool=pool.numpy(), logits=logits.numpy())
    print("inception_seed0 pool", tuple(pool.shape), float(pool.abs().mean()), "logits", tuple(logits.shape))


def golden_cond_losses():
    """Reference conditioning losses (src/utils/losses.py:38-165) on seeded embeddings: values and input gradients."""
    torch.manual_seed(2024)
    B, d, classes = 12, 16, 4
    out = {}
    label = torch.randint(0, classes, (B,))
    logits = torch.randn(B, classes, requires_grad=True)
    ce = rlosses.CrossEntropyLoss()(cls_output=logits, label=label)
    ce.backward()
    out.update({"label": label.numpy(), "logits": logits.detach().numpy(), "ce": ce.detach().numpy(), "ce_dlogits": logits.grad.numpy()})
    for name, cls, kw in (("c2", rlosses.ConditionalContrastiveLoss, dict(temperature=0.5)),
                          ("d2dce", rlosses.Data2DataCrossEntropyLoss, dict(temperature=0.5, m_p=0.98))):
        embed = torch.randn(B, d, requires_grad=True)
        proxy = torch.randn(B, d, requires_grad=True)
        loss = cls(num_classes=classes, master_rank="cpu", DDP=False, **kw)(embed=embed, proxy=proxy, label=label)
        loss.backward()
        out.update({name + "_embed": embed.detach().numpy(), name + "_proxy": proxy.detach().numpy(), name: loss.detach().numpy(),
                    name + "_dembed": embed.grad.numpy(), name + "_dproxy": proxy.grad.numpy()})
    np.savez_compressed(os.path.join(HERE, "cond_losses.npz"), **out)
    print("cond_losses", {k: float(out[k]) for k in ("ce", "c2", "d2dce")})


def golden_dcgan(tag="dcgan32", B=8, z_dim=16):
    """BASELINE config 1 (src/configs/CIFAR10/DCGAN.yaml): DCGAN, unconditional, vanilla loss, BatchNorm in G and D --
    one D phase + one G phase exactly as golden_resfamily.  The 6.4 M weights are NOT stored: both sides regenerate them
    from a seed (oracle.seeded_state); the fixture holds inputs, outputs, losses, per-parameter gradient norms and the full
    gradients / updated statistics of the 1-D parameters."""
    import json
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import studiogan_oracle as O
    M = modules(g_sn=False, d_sn=False, cbn=False)
    G = rdc.Generator(z_dim=z_dim, g_shared_dim="N/A", img_size=32, g_conv_dim="N/A", apply_attn=False, attn_g_loc=[], g_cond_mtd="W/O",
                      num_classes=10, g_init="ortho", g_depth="N/A", mixed_precision=False, MODULES=M, MODEL=MODEL)
    D = rdc.Discriminator(img_size=32, d_conv_dim="N/A", apply_d_sn=False, apply_attn=False, attn_d_loc=[], d_cond_mtd="W/O",
                          aux_cls_type="W/O", d_embed_dim="N/A", normalize_d_embed=False, num_classes=10, d_init="ortho",
                          d_depth="N/A", mixed_precision=False, MODULES=M, MODEL=MODEL)
    ks_g = [(k, list(v.shape)) for k, v in G.state_dict().items()]
    ks_d = [(k, list(v.shape)) for k, v in D.state_dict().items()]
    G.load_state_dict(O.seeded_state(ks_g, 101), strict=True)
    D.load_state_dict(O.seeded_state(ks_d, 202), strict=True)
    G.train(); D.train()
    torch.manual_seed(31)
    out = {"keys_g": np.array(json.dumps(ks_g)), "keys_d": np.array(json.dumps(ks_d))}
    z = torch.randn(B, z_dim); y = torch.randint(0, 10, (B,))
    real = torch.rand(B, 3, 32, 32) * 2 - 1
    out.update({"z": z.numpy(), "y": y.numpy(), "real": real.numpy()})
    for p in G.parameters():
        p.requires_grad_(False)
    fake = G(z, y)
    rd, fd = D(real, y), D(fake.detach(), y)
    d_loss = rlosses.d_vanilla(rd["adv_output"], fd["adv_output"], False)
    d_loss.backward()
    out.update({"fake": fake.detach().numpy(), "adv_real": rd["adv_output"].detach().numpy(), "adv_fake": fd["adv_output"].detach().numpy(),
                "d_loss": d_loss.detach().numpy()})
    for k, p in D.named_parameters():
        out["Dgnorm/" + k] = p.grad.norm().numpy()
        if p.dim() == 1:
            out["Dgrad/" + k] = p.grad.detach().numpy().copy()
    for k, v in list(G.state_dict().items()) + list(D.state_dict().items()):
        pass
    out.update({"G1/" + k: v.numpy().copy() for k, v in G.state_dict().items() if "running_" in k})
    out.update({"D1/" + k: v.numpy().copy() for k, v in D.state_dict().items() if "running_" in k})
    D.zero_grad()
    for p in G.parameters():
        p.requires_grad_(True)
    for p in D.parameters():
        p.requires_grad_(False)
    fake2 = G(z, y)
    fake2.retain_grad()
    g_loss = rlosses.g_vanilla(D(fake2, y)["adv_output"], False)
    g_loss.backward()
    out.update({"fake2": fake2.detach().numpy(), "g_loss": g_loss.detach().numpy(), "dfake2": fake2.grad.numpy().copy()})
    for k, p in G.named_parameters():
        out["Ggnorm/" + k] = p.grad.norm().numpy()
        if p.dim() == 1:
            out["Ggrad/" + k] = p.grad.detach().numpy().copy()
    np.savez_compressed(os.path.join(HERE, tag + ".npz"), **out)
    print(tag, "keys", len(out), "d_loss", float(d_loss), "g_loss", float(g_loss))


def golden_sampler():
    """utils.sample.sample_zy of the reference (src/utils/sample.py:69-90) on the CPU generator: labels are drawn BEFORE
    the latents; gaussian / uniform priors, the eps-ball branch, truncation (scipy truncnorm on numpy's global RNG) and the
    visualisation label samplers."""
    import utils.sample as rsample
    out = {}
    for name, kw in (("gauss", dict(z_prior="gaussian", truncation_factor=-1.0, y_sampler="totally_random", radius="N/A")),
                     ("uniform", dict(z_prior="uniform", truncation_factor=-1.0, y_sampler="totally_random", radius="N/A")),
                     ("eps", dict(z_prior="gaussian", truncation_factor=-1.0, y_sampler="totally_random", radius=0.5)),
                     ("trunc", dict(z_prior="gaussian", truncation_factor=0.7, y_sampler="totally_random", radius="N/A")),
                     ("some", dict(z_prior="gaussian", truncation_factor=-1.0, y_sampler="acending_some", radius="N/A")),
                     ("all", dict(z_prior="gaussian", truncation_factor=-1.0, y_sampler="acending_all", radius="N/A")),
                     ("fixed", dict(z_prior="gaussian", truncation_factor=-1.0, y_sampler=3, radius="N/A"))):
        torch.manual_seed(2718)
        np.random.seed(31)
        zs, y, zs_eps = rsample.sample_zy(batch_size=16, z_dim=12, num_classes=7, device="cpu", **kw)
        out[name + "_z"], out[name + "_y"] = zs.numpy(), y.numpy()
        if zs_eps is not None:
            out[name + "_zeps"] = zs_eps.numpy()
    np.savez_compressed(os.path.join(HERE, "sampler.npz"), **out)
    print("sampler", {k: v.shape for k, v in out.items()})


def golden_augment():
    """Reference DiffAugment (src/utils/diffaug.py) and CR augmentation (src/utils/cr.py) on seeded CPU inputs: outputs and,
    for DiffAugment, the input gradient of a seeded cotangent.  The seeds are re-applied right before each call so that the
    product's parameter draw (same RNG order) can be checked together with the arithmetic."""
    import utils.diffaug as rdiff
    import utils.cr as rcr
    out = {}
    g = torch.Generator().manual_seed(606)
    for tag, (B, H, W) in (("a", (5, 16, 16)), ("b", (3, 12, 20))):
        x = torch.randn(B, 3, H, W, generator=g)
        ct = torch.randn(B, 3, H, W, generator=g)
        out["x_" + tag], out["ct_" + tag] = x.numpy(), ct.numpy()
        for pname, policy in (("full", "color,translation,cutout"), ("color", "color"), ("geo", "translation,cutout")):
            xr = x.clone().requires_grad_(True)
            torch.manual_seed(4242)
            y = rdiff.apply_diffaug(xr, policy=policy)
            y.backward(ct)
            out["diffaug_%s_%s" % (pname, tag)] = y.detach().numpy()
            out["diffaug_%s_%s_dx" % (pname, tag)] = xr.grad.numpy().copy()
        torch.manual_seed(777)
        out["cr_" + tag] = rcr.apply_cr_aug(x).numpy()
    np.savez_compressed(os.path.join(HERE, "augment.npz"), **out)
    print("augment", {k: v.shape for k, v in out.items() if k.startswith("diffaug_full")})


def golden_metrics():
    rng = np.random.RandomState(0)
    out = {}
    # quantisation + legacy resize (src/utils/ops.py:251-263, src/utils/resize.py:50-94)
    x = torch.from_numpy(rng.uniform(-1.1, 1.1, size=(2, 3, 8, 8)).astype(np.float32))
    q = rops.quantize_images(x)
    out["q_in"], out["q_out"] = x.numpy(), q
    resizer = rresize.build_resizer("legacy", "InceptionV3_tf", 19)
    rs = np.stack([resizer(img) for img in q.transpose(0, 2, 3, 1)], 0)
    out["resize_legacy_19"] = rs
    # "friendly" = PIL bilinear on float32 channels: up-scaling (8 -> 19) and anti-aliased down-scaling (20 -> 13)
    fr = rresize.build_resizer("friendly", "InceptionV3_tf", 19)
    out["resize_friendly_19"] = np.stack([fr(img) for img in q.transpose(0, 2, 3, 1)], 0)
    x20 = torch.from_numpy(np.random.RandomState(5).uniform(-1.1, 1.1, size=(2, 3, 20, 20)).astype(np.float32))   # own stream: the draws below keep their values
    q20 = rops.quantize_images(x20)
    out["q20_in"] = x20.numpy()
    fr13 = rresize.build_resizer("friendly", "InceptionV3_tf", 13)
    out["resize_friendly_20to13"] = np.stack([fr13(img) for img in q20.transpose(0, 2, 3, 1)], 0)
    # FID / moments
    real = rng.randn(300, 24).astype(np.float64)
    fake = (rng.randn(280, 24) * 1.1 + 0.05).astype(np.float32)
    rfid.linalg = types.SimpleNamespace(sqrtm=lambda m, disp=True: (scipy.linalg.sqrtm(m), None) if disp is False
                                        else scipy.linalg.sqrtm(m))
    mu1, s1 = np.mean(fake, axis=0), np.cov(fake, rowvar=False)
    mu2, s2 = np.mean(real, axis=0), np.cov(real, rowvar=False)
    out["feat_real"], out["feat_fake"] = real, fake
    out["fid"] = np.array(rfid.frechet_inception_distance(mu1, s1, mu2, s2))
    # IS
    logits = rng.randn(200, 11).astype(np.float32)
    probs = torch.softmax(torch.from_numpy(logits), 1)
    m, s = rins.calculate_kl_div(probs, splits=1)
    m4, s4 = rins.calculate_kl_div(probs, splits=4)
    out["probs"] = probs.numpy()
    out["is_1"] = np.array([float(m), float(s)])
    out["is_4"] = np.array([float(m4), float(s4)])
    # PRDC
    pr = rprdc.compute_prdc(real_features=real[:200], fake_features=fake[:180].astype(np.float64), nearest_k=5)
    out["prdc"] = np.array([pr["precision"], pr["recall"], pr["density"], pr["coverage"]])
    # EMA (src/utils/ema.py:27-40)
    torch.manual_seed(3)
    src = nn.Sequential(nn.Conv2d(3, 4, 3), nn.BatchNorm2d(4))
    tgt = nn.Sequential(nn.Conv2d(3, 4, 3), nn.BatchNorm2d(4))
    out.update({"ema_src/" + k: v.numpy().copy() for k, v in src.state_dict().items()})
    out.update({"ema_tgt0/" + k: v.numpy().copy() for k, v in tgt.state_dict().items()})
    e = rema.Ema(src, tgt, decay=0.9, start_iter=2)
    out.update({"ema_init/" + k: v.numpy().copy() for k, v in tgt.state_dict().items()})
    with torch.no_grad():
        for p in src.parameters():
            p.add_(0.5)
        src[1].running_mean.add_(0.25)
    out.update({"ema_src2/" + k: v.numpy().copy() for k, v in src.state_dict().items()})
    e.update(5)
    out.update({"ema_after/" + k: v.numpy().copy() for k, v in tgt.state_dict().items()})
    # losses
    a, b = torch.from_numpy(rng.randn(16).astype(np.float32)), torch.from_numpy(rng.randn(16).astype(np.float32))
    out["loss_in_real"], out["loss_in_fake"] = a.numpy(), b.numpy()
    out["losses"] = np.array([float(rlosses.d_hinge(a, b, False)), float(rlosses.g_hinge(b, False)),
                              float(rlosses.d_wasserstein(a, b, False)), float(rlosses.g_wasserstein(b, False)),
                              float(rlosses.d_vanilla(a, b, False)), float(rlosses.g_vanilla(b, False))])
    np.savez_compressed(os.path.join(HERE, "metrics.npz"), **out)
    print("metrics", {k: out[k] for k in ["fid", "is_1", "prdc", "losses"]})


if __name__ == "__main__":
    golden_deep("deep32_c8", 32, 8, 1, attn=False)
    golden_deep("deep32_c16_attn_d2", 32, 16, 2, attn=True, B=2)
    golden_deep("deepsg32_c8", 32, 8, 1, attn=False, B=8, rdeep=rdeep_sg)  # StudioGAN flavour of BigGAN-Deep
    golden_deep("deep32_c8_b16", 32, 8, 1, attn=False, B=16)      # well-conditioned BatchNorm statistics for gradient parity
    golden_resfamily("biggan32_c32_attn", "big_resnet", 32, True, True, True, "cBN", "PD", "hinge", B=4)
    golden_resfamily("sngan32_c16", "resnet", 16, False, False, True, "W/O", "W/O", "hinge", z_dim=32)
    golden_resfamily("resnet32_cbn_c16", "resnet", 16, False, False, True, "cBN", "PD", "hinge", z_dim=32)
    golden_resfamily("wgan32_bn_c16", "resnet", 16, False, False, False, "W/O", "W/O", "wasserstein", z_dim=32)
    golden_metrics()
    golden_dcgan()
    golden_cond_losses()
    golden_inception()
    golden_gp("gp_resnet32_bn_c16", "resnet", 16, False, "W/O")           # the WGAN-GP config's discriminator (BatchNorm, no SN)
    golden_gp("gp_resnet32_sn_c16_pd", "resnet", 16, True, "PD")
    golden_gp("gp_deep32_sn_c8_pd", "deep", 8, True, "PD")
    golden_deep_bench_shape()
    golden_sampler()
    golden_augment()
