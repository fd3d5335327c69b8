"""GPU tests of the evaluation path (SURVEY.md 8a rows a18-a24): device pre-processing, Inception conv pipeline on the
wgmma conv engine, and IS / FID / PRDC computed from its features, against the oracle and the reference goldens."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import studiogan_oracle as O  # noqa: E402


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def l2_err(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return float((got - ref).norm() / (ref.norm() + 1e-30))


def test_quantize_is_bit_exact_and_resize_matches_legacy(golden_dir):
    from sgb200 import kernels as K
    dev = _cuda()
    g = np.load(os.path.join(golden_dir, "metrics.npz"))
    x = torch.from_numpy(g["q_in"]).to(dev)
    assert np.array_equal(K.quantize_u8(x).cpu().numpy(), g["q_out"])                     # integer path: bit exact
    torch.manual_seed(0)
    img = torch.rand(3, 3, 40, 56) * 2.4 - 1.2
    ref = O.eval_preprocess(img, 299, True)
    got, col = K.quantize_resize_normalize(img.to(dev), 299, quantize=True, want_image=True, want_col=True)
    assert float((got.cpu() - ref).abs().max()) < 5e-5                                    # fp32 bilinear weights
    # the patch tensor is the stride-2 valid 3x3 unfold of the same image (bf16)
    unf = F.unfold(ref, kernel_size=3, stride=2).view(3, 3, 9, 149, 149).permute(0, 3, 4, 2, 1).reshape(3, 149, 149, 27)
    colc = col.permute(0, 2, 3, 1).float().cpu()
    assert float((colc[..., :27] - unf.bfloat16().float()).abs().max()) < 1e-2 and float(colc[..., 27:].abs().max()) == 0.0


@pytest.mark.parametrize("S_in", [32, 128, 256, 512])
def test_friendly_resizer_matches_pil_f_mode_bilinear(golden_dir, S_in):
    """post_resizer "friendly" (src/utils/resize.py:50-53,72-82): the device kernel against Pillow itself at the
    evaluation size 299 (up-scaling from 32 / 128 / 256, anti-aliased down-scaling from 512) and against the reference's
    golden at small sizes.  Same arithmetic (float64 taps and sums, float32 after each pass): agreement to float32
    round-off of the 0..255 values (2e-5 absolute on the 255-scale, i.e. 1.6e-7 after normalisation x 2/255)."""
    from PIL import Image
    from sgb200 import kernels as K
    dev = _cuda()
    rs = np.random.RandomState(S_in)
    u8 = rs.randint(0, 256, size=(2, 3, S_in, S_in)).astype(np.float32)
    got, _ = K.quantize_resize_normalize(torch.from_numpy(u8).to(dev), 299, quantize=False, want_image=True, want_col=False,
                                         resizer="friendly")
    ref = np.stack([[np.asarray(Image.fromarray(u8[b, c], mode="F").resize((299, 299), resample=Image.BILINEAR)) for c in range(3)]
                    for b in range(2)])
    ref = (torch.from_numpy(ref) / 255.0 - 0.5) / 0.5
    assert float((got.cpu() - ref).abs().max()) < 4e-7
    if S_in == 32:
        g = np.load(os.path.join(golden_dir, "metrics.npz"))
        for key_in, key_out, S in (("q_in", "resize_friendly_19", 19), ("q20_in", "resize_friendly_20to13", 13)):
            x = torch.from_numpy(g[key_in]).to(dev)
            got, _ = K.quantize_resize_normalize(x, S, quantize=True, want_image=True, want_col=False, resizer="friendly")
            ref = (torch.from_numpy(g[key_out].transpose(0, 3, 1, 2)) / 255.0 - 0.5) / 0.5
            assert float((got.cpu() - ref).abs().max()) < 4e-7


@pytest.mark.parametrize("stride,pad,mode", [(2, 0, 1), (1, 1, 0), (1, 1, 1)])
def test_pool3x3_modes(stride, pad, mode):
    from sgb200 import kernels as K
    dev = _cuda()
    x = torch.randn(2, 16, 17, 17).bfloat16().float()
    xd = x.to(dev).bfloat16().permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    ref = F.max_pool2d(x, 3, stride, pad) if mode == 1 else F.avg_pool2d(x, 3, stride, pad, count_include_pad=False)
    got = K.pool3x3(xd, stride, pad, mode)
    assert got.shape == ref.shape and float((got.float().cpu() - ref).abs().max()) < 2e-2


@pytest.mark.parametrize("Cin,Cout,KH,KW,ph,pw,stride,same,H", [(32, 32, 3, 3, 0, 0, 1, False, 21), (64, 96, 3, 3, 0, 0, 2, False, 35),
                                                                 (128, 128, 1, 7, 0, 3, 1, True, 17), (48, 64, 5, 5, 2, 2, 1, True, 35),
                                                                 (80, 192, 3, 3, 0, 0, 1, False, 73)])
def test_inception_conv_shapes(Cin, Cout, KH, KW, ph, pw, stride, same, H):
    from sgb200 import kernels as K
    dev = _cuda()
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(2, Cin, H, H, generator=g)).bfloat16().float()
    w = (torch.randn(Cout, Cin, KH, KW, generator=g) * (2.0 / (Cin * KH * KW)) ** 0.5).bfloat16().float()
    b = torch.randn(Cout, generator=g)
    ref = F.relu(F.conv2d(x, w, b, stride=stride, padding=(ph, pw)))
    xd = x.to(dev).bfloat16().permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    wf, _ = K.weight_pack(w.to(dev), None, Cout, Cin, KH * KW, True, False)
    got = K.conv_fprop(xd, wf, Cout, KH, KW, ph, pw, bias=b.to(dev), relu=True, same_size=same, stride=stride)
    assert got.shape == ref.shape
    assert float((got.float().cpu() - ref).abs().max()) < 1e-2 * (1 + float(ref.abs().max()))


def test_inception_features_vs_reference_golden(golden_dir):
    """Product InceptionV3 (bf16 conv pipeline, folded BN) vs the reference's LoadEvalModel.get_outputs on the same seeded
    weights and inputs.  Tolerance: relative L2 <= 3e-2 on the 2048-d pool features and on the 1008 logits."""
    from sgb200.metrics.preparation import LoadEvalModel
    dev = _cuda()
    g = np.load(os.path.join(golden_dir, "inception_seed0.npz"))
    ev = LoadEvalModel("InceptionV3_tf", "legacy", 1, False, dev)
    pool, logits = ev.get_outputs(torch.from_numpy(g["x"]).to(dev), quantize=True)
    assert pool.shape == (2, 2048) and logits.shape == (2, 1008)
    assert l2_err(pool, torch.from_numpy(g["pool"])) < 3e-2
    assert l2_err(logits, torch.from_numpy(g["logits"])) < 3e-2


def test_fid_is_prdc_from_cuda_features_vs_oracle_features():
    """FID / IS / PRDC of structured images: CUDA Inception features vs the fp32 oracle features (same seeded weights).
    Stated tolerance (north_star): FID and IS within +-0.5 %; PRDC within 0.03 absolute at this tiny N.
    Conditioning: FID-50k has N / d = 50000 / 2048 ~ 24 samples per feature dimension; with the N = 384 images a CPU
    oracle can afford, the full 2048-d covariance would be rank deficient and tr sqrt(S1 S2) infinitely sensitive, so
    the +-0.5 % bar is checked on a 16-d feature subset (every 128th dimension: N / d = 24, same pipeline), and the
    full-dimension value is held to 3 %."""
    from sgb200.metrics import fid, ins, prdc
    from sgb200.metrics.inception_net import InceptionV3, seeded_state_dict
    dev = _cuda()
    sd = seeded_state_dict(0)
    net = InceptionV3(sd, dev)
    onet = O.fid_inception(sd)
    g = torch.Generator().manual_seed(5)

    def images(n, gain, shift, res):
        base = F.interpolate(torch.randn(n, 3, res, res, generator=g), size=(48, 48), mode="bilinear", align_corners=False)
        return torch.tanh(base * gain + shift)
    real, fake = images(384, 1.5, 0.0, 8), images(384, 0.6, 0.5, 4)      # clearly different distributions
    feats, probs = {}, {}
    for name, imgs in (("real", real), ("fake", fake)):
        ps, ls, pos, los = [], [], [], []
        for i in range(0, imgs.shape[0], 96):
            p, l = net.forward(imgs[i:i + 96].to(dev), quantize=True)
            po, lo = O.fid_inception_forward(onet, O.eval_preprocess(imgs[i:i + 96], 299, True))
            ps.append(p.cpu()); ls.append(l.cpu()); pos.append(po); los.append(lo)
        feats[name] = (torch.cat(ps).double(), torch.cat(pos).double())
        probs[name] = (torch.softmax(torch.cat(ls), 1), torch.softmax(torch.cat(los), 1))
    out = []
    for k in (0, 1):
        full = fid.frechet_distance_device(*fid.calculate_moments(feats["fake"][k]), *fid.calculate_moments(feats["real"][k]))
        sub = fid.frechet_distance_device(*fid.calculate_moments(feats["fake"][k][:, ::128]),
                                          *fid.calculate_moments(feats["real"][k][:, ::128]))
        out.append((full, sub, float(ins.calculate_kl_div(probs["fake"][k], 1)[0]),
                    prdc.compute_prdc(feats["real"][k][:192], feats["real"][k][192:], 5)))
    (fid_c, sub_c, is_c, pr_c), (fid_o, sub_o, is_o, pr_o) = out
    print("FID cuda/oracle", fid_c, fid_o, "16-d", sub_c, sub_o, "IS", is_c, is_o, "PRDC", pr_c, pr_o)
    assert abs(sub_c - sub_o) <= 5e-3 * abs(sub_o)
    assert abs(fid_c - fid_o) <= 3e-2 * abs(fid_o)
    assert abs(is_c - is_o) <= 5e-3 * abs(is_o)
    for key in pr_o:
        assert abs(pr_c[key] - pr_o[key]) <= 0.03, key


def test_worker_evaluate_runs_end_to_end():
    """WORKER.evaluate on a small BigGAN-Deep: generator (EMA off) -> device pre-processing -> Inception -> IS/FID/PRDC."""
    from sgb200 import config as C
    from sgb200.metrics import fid
    from sgb200.metrics.preparation import LoadEvalModel
    from sgb200.models import model as M
    from sgb200.worker import WORKER
    dev = _cuda()
    cfgs = C.Configurations(None)
    cfgs.DATA.img_size, cfgs.DATA.num_classes = 32, 10
    m = cfgs.MODEL
    m.backbone, m.g_cond_mtd, m.d_cond_mtd, m.apply_g_sn, m.apply_d_sn = "big_resnet_deep_legacy", "cBN", "PD", True, True
    m.z_dim, m.g_shared_dim, m.g_conv_dim, m.d_conv_dim, m.g_depth, m.d_depth = 32, 32, 16, 16, 1, 1
    cfgs.LOSS.adv_loss = "hinge"
    cfgs.OPTIMIZATION.batch_size = 32
    cfgs.define_modules()
    cfgs.define_losses()
    torch.manual_seed(0)
    Gen, _, _, Dis, _, _, _, _ = M.load_generator_discriminator(cfgs.DATA, cfgs.OPTIMIZATION, cfgs.MODEL, cfgs.STYLEGAN, cfgs.MODULES,
                                                                 cfgs.RUN, dev, None)
    ev = LoadEvalModel("InceptionV3_tf", "legacy", 1, False, dev)
    real = torch.rand(96, 3, 32, 32) * 2 - 1
    rf, _ = ev.get_outputs(real.to(dev), quantize=True)
    mu, sigma = fid.calculate_moments(rf)
    w = WORKER(cfgs=cfgs, run_name="t", Gen=Gen, Gen_mapping=None, Gen_synthesis=None, Dis=Dis, Gen_ema=None, Gen_ema_mapping=None,
               Gen_ema_synthesis=None, ema=None, eval_model=ev, train_dataloader=None, eval_dataloader=None, global_rank=0,
               local_rank=dev, mu=mu, sigma=sigma, real_feats=rf, logger=None, num_eval=96)
    best = w.evaluate(step=0, metrics=["is", "fid", "prdc"], writing=False, training=True)
    r = w.last_metrics
    assert best is True and np.isfinite(r["FID"]) and r["FID"] > 0 and np.isfinite(r["IS"]) and 0.0 <= r["Coverage"] <= 1.0
    assert Gen.training and Dis.training                       # make_GAN_trainable restored the modes


def test_feature_moments_kernel_matches_numpy_cov():
    """sgb_feat_moments_accumulate / finalize (fp64) against np.mean / np.cov(rowvar=False) (src/metrics/fid.py:65-98) on
    features folded in over uneven batches; D = 200 exercises ragged 64-wide blocks, D = 2048 the evaluation size."""
    from sgb200.metrics import fid
    dev = _cuda()
    rs = np.random.RandomState(3)
    for D, sizes in ((200, (37, 64, 1, 130)), (2048, (256, 100))):
        f = (rs.randn(sum(sizes), D) * (1 + rs.rand(D)) + rs.randn(D)).astype(np.float32)
        acc = fid.MomentsAccumulator(D, dev)
        s = 0
        for n in sizes:
            acc.update(torch.from_numpy(f[s:s + n]).to(dev))
            s += n
        mu, sigma = acc.finalize()
        f64 = f.astype(np.float64)
        np.testing.assert_allclose(mu.cpu().numpy(), f64.mean(0), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(sigma.cpu().numpy(), np.cov(f64, rowvar=False), rtol=1e-9, atol=1e-10)
        mu2, sigma2 = fid.calculate_moments(torch.from_numpy(f).to(dev))           # 4096-row blocks: another summation order
        np.testing.assert_allclose(mu2.cpu().numpy(), mu.cpu().numpy(), rtol=1e-13, atol=1e-13)
        np.testing.assert_allclose(sigma2.cpu().numpy(), sigma.cpu().numpy(), rtol=1e-10, atol=1e-11)


def test_prdc_tile_kernels_match_reference_golden_and_host_path(golden_dir):
    """csrc/metrics.cu PRDC kernels (radii + cross reductions, fp64 distance tiles never stored) against the reference's
    compute_prdc golden (tests/golden/metrics.npz: sklearn pairwise_distances + argpartition) -- the four values are
    ratios of integer counts and must agree exactly -- and against the host tensor path on a larger ragged problem."""
    from sgb200.metrics import prdc
    dev = _cuda()
    g = np.load(os.path.join(golden_dir, "metrics.npz"))
    real, fake = torch.from_numpy(g["feat_real"][:200]), torch.from_numpy(g["feat_fake"][:180].astype(np.float64))
    got = prdc.compute_prdc(real.to(dev), fake.to(dev), 5)
    np.testing.assert_allclose([got["precision"], got["recall"], got["density"], got["coverage"]], g["prdc"], rtol=1e-12, atol=0)
    rs = np.random.RandomState(4)
    real = torch.from_numpy(rs.randn(333, 70))
    fake = torch.from_numpy(rs.randn(401, 70) * 1.05 + 0.1)
    ref = prdc.compute_prdc(real, fake, 3)
    got = prdc.compute_prdc(real.to(dev), fake.to(dev), 3)
    for k in ref:
        assert abs(ref[k] - got[k]) < 1e-12, (k, ref[k], got[k])
    # the radii themselves
    from sgb200 import _lib as L
    x = real.to(dev).contiguous()
    rn, rad = torch.empty(333, dtype=torch.float64, device=dev), torch.empty(333, dtype=torch.float64, device=dev)
    L.call("sgb_prdc_radii", L.ptr(x), 333, 70, 3, L.ptr(rn), L.ptr(rad), L.stream_ptr())
    np.testing.assert_allclose(rad.cpu().numpy(), prdc.kth_nn_distances(real, 3).numpy(), rtol=1e-9, atol=1e-9)


def test_device_basket_loader_is_bit_identical_to_the_cpu_transform_chain(tmp_path):
    """Data path: uint8 baskets through pinned staging, side-stream H2D and sgb_u8_to_img (flip + ToTensor + Normalize) equal
    the per-sample CPU chain of src/data_util.py:86-99 exactly, for several consecutive baskets (double buffering)."""
    from sgb200 import data_util
    dev = _cuda()
    rs = np.random.RandomState(1)
    imgs = rs.randint(0, 256, size=(64, 16, 12, 3)).astype(np.uint8)
    labels = rs.randint(0, 7, size=64)
    path = str(tmp_path / "toy.npz")
    np.savez(path, imgs=imgs, labels=labels)
    ds = data_util.Dataset_("toy", None, True, hdf5_path=path, random_flip=True)
    loader = data_util.DeviceBasketLoader(ds, basket=24, device=dev, shuffle=True, seed=5)
    order = np.random.RandomState(5).permutation(64)
    gen = torch.Generator().manual_seed(5)
    pos = 0
    for it in range(5):
        if pos + 24 > 64:
            order, pos = None, 0
        x, y = next(loader)
        if order is None:
            break                                   # the reshuffle draws from the loader's own stream; first epoch is enough here
        idx = order[pos:pos + 24]
        pos += 24
        flip = torch.rand(24, generator=gen) < 0.5
        ref = (torch.from_numpy(imgs[idx]).permute(0, 3, 1, 2).float().div(255) - 0.5) / 0.5
        ref = torch.where(flip[:, None, None, None], ref.flip(3), ref)
        assert x.shape == (24, 3, 16, 12) and x.dtype == torch.float32
        assert torch.equal(x.cpu(), ref) and y.cpu().tolist() == labels[idx].tolist()


def test_folder_evaluator_matches_feature_level_metrics(tmp_path):
    """sgb200.evaluate (src/evaluate.py:112-288, folder mode): two PNG folders -> IS / FID / PRDC.  Checked against the same
    metrics computed from features extracted directly from the in-memory uint8 arrays (PNG is lossless, so the folder path
    must reproduce them exactly), plus the pre-computed ``dset1_moments`` / ``dset1_feats`` entry points."""
    from PIL import Image
    from sgb200 import evaluate as E
    from sgb200.metrics import fid, prdc
    from sgb200.metrics.preparation import LoadEvalModel
    dev = _cuda()
    rs = np.random.RandomState(7)
    sets = {}
    for name, n, shift in (("a", 24, 0), ("b", 20, 40)):
        arr = np.clip(rs.randint(0, 216, size=(n, 32, 32, 3)) + shift, 0, 255).astype(np.uint8)
        os.makedirs(tmp_path / name / "cls0")
        os.makedirs(tmp_path / name / "cls1")
        for i in range(n):
            Image.fromarray(arr[i]).save(str(tmp_path / name / ("cls%d" % (i % 2)) / ("%03d.png" % i)))
        # ImageFolder order: all of cls0 (even i) then all of cls1 (odd i)
        sets[name] = np.concatenate([arr[0::2], arr[1::2]], 0)
    res = E.evaluate(str(tmp_path / "a"), str(tmp_path / "b"), batch_size=16, device=dev)
    assert res["dset1_size"] == 24 and res["dset2_size"] == 20
    ev = LoadEvalModel("InceptionV3_tf", "legacy", 1, False, dev)
    feats = {}
    for name, arr in sets.items():
        f, _ = ev.get_outputs(torch.from_numpy(arr).permute(0, 3, 1, 2).float().to(dev), quantize=False)
        feats[name] = f
    m1, s1 = fid.calculate_moments(feats["a"])
    m2, s2 = fid.calculate_moments(feats["b"])
    ref_fid = fid.frechet_distance_device(m1, s1, m2, s2)
    assert abs(res["FID"] - ref_fid) <= 1e-6 * max(1.0, abs(ref_fid))
    ref_pr = prdc.compute_prdc(feats["a"].double(), feats["b"].double(), 5)
    assert abs(res["Improved_Precision"] - ref_pr["precision"]) < 1e-12 and abs(res["Coverage"] - ref_pr["coverage"]) < 1e-12
    # pre-computed statistics of dset1 instead of the folder
    np.savez(str(tmp_path / "m.npz"), mu=m1.cpu().numpy(), sigma=s1.cpu().numpy())
    np.savez(str(tmp_path / "f.npz"), real_feats=feats["a"].double().cpu().numpy())
    res2 = E.evaluate(None, str(tmp_path / "b"), dset1_moments=str(tmp_path / "m.npz"), dset1_feats=str(tmp_path / "f.npz"),
                      batch_size=16, device=dev)
    assert abs(res2["FID"] - res["FID"]) <= 1e-6 * max(1.0, abs(res["FID"])) and res2["Density"] == res["Density"]
