"""Step runtime with the reference's API (``src/worker.py``): ``WORKER.train_discriminator(step)`` ->
(real_cond_loss, dis_acml_loss), ``WORKER.train_generator(step)`` -> gen_acml_loss, in the reference's order of
operations (D phase :213-497, G phase :502-681): toggle_grad, BN tracking toggles, ``d_updates_per_step`` x ``acml_steps``
loops, labels-then-z sampling, two separate discriminator passes for real and fake, loss / acml_steps, optimiser step,
EMA update after the generator step.  Mixed precision / GradScaler do not exist here: the kernels compute in bf16 with
fp32 accumulation and fp32 master weights, which needs no loss scaling.
"""
import torch

from . import _lib
from . import kernels as K
from .models import model as model_lib
from .utils import losses, misc, sample
from .utils.optim import ArenaAdam


class _GraphedPhase:
    """One training phase (all of train_discriminator's or train_generator's device work) captured into a CUDA graph
    after ``warmup`` eager calls and replayed afterwards: at small per-GPU batches (8-GPU strong scaling: 32 images per
    rank) the phase is ~1.8k library launches and the host cannot issue them as fast as the GPU retires them.  Inputs
    live in static device buffers filled before each replay; z / labels come from the device RNG inside the graph; the
    Adam step counters live on the device (ArenaAdam.step_t).  Any capture failure falls back to eager execution."""

    POOL = None                                   # one memory pool for every captured phase: they never replay concurrently

    def __init__(self, fn, warmup=2):
        self.fn, self.warmup = fn, warmup
        self.calls = 0
        self.graph = self.out = None
        self.failed = False
        self.launches = 0                         # library launches recorded in the graph (re-issued by every replay)

    def _result(self):
        """The phase's result copied out of the graph pool: the pool is shared between the phases, so the next replay of the
        OTHER phase may reuse the memory the captured result lives in."""
        return self.out.clone() if torch.is_tensor(self.out) else self.out

    def __call__(self):
        if self.graph is not None:
            self.graph.replay()
            _lib.LAUNCHES[0] += self.launches
            return self._result()
        self.calls += 1
        if self.failed or self.calls <= self.warmup:
            return self.fn()
        try:
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            g = torch.cuda.CUDAGraph()
            n0 = _lib.LAUNCHES[0]
            if _GraphedPhase.POOL is None:
                _GraphedPhase.POOL = torch.cuda.graph_pool_handle()
            with torch.cuda.graph(g, pool=_GraphedPhase.POOL):     # D-phase and G-phase graphs share their activation memory
                out = self.fn()
            self.launches = _lib.LAUNCHES[0] - n0
            self.graph, self.out = g, out
            g.replay()
            return self._result()
        except Exception as ex:  # noqa: BLE001 - keep training alive, eagerly
            self.failed = True
            self.graph = None
            import warnings
            warnings.warn("sgb200: CUDA-graph capture failed (%r); continuing without graphs" % (ex,))
            torch.cuda.synchronize()
            return self.fn()


class WORKER(object):
    def __init__(self, cfgs, run_name, Gen, Gen_mapping, Gen_synthesis, Dis, Gen_ema, Gen_ema_mapping, Gen_ema_synthesis, ema,
                 eval_model, train_dataloader, eval_dataloader, global_rank, local_rank, mu, sigma, real_feats, logger,
                 aa_p=None, best_step=0, best_fid=None, best_ckpt_path=None, lecam_emas=None, num_eval=None, loss_list_dict=None,
                 metric_dict_during_train=None):
        self.cfgs = cfgs
        self.run_name = run_name
        self.Gen, self.Dis, self.Gen_ema, self.ema = Gen, Dis, Gen_ema, ema
        self.eval_model = eval_model
        self.train_dataloader = train_dataloader
        self.eval_dataloader = eval_dataloader
        self.global_rank, self.local_rank = global_rank, local_rank
        self.mu, self.sigma, self.real_feats = mu, sigma, real_feats
        self.logger = logger
        self.best_step, self.best_fid, self.best_ckpt_path = best_step, best_fid, best_ckpt_path
        self.num_eval = num_eval
        self.last_metrics = None
        self.DATA, self.MODEL, self.LOSS, self.OPTIMIZATION, self.RUN = cfgs.DATA, cfgs.MODEL, cfgs.LOSS, cfgs.OPTIMIZATION, cfgs.RUN
        self.DDP = self.RUN.distributed_data_parallel
        self.train_iter = iter(train_dataloader) if train_dataloader is not None else None
        self.is_stylegan = False
        if self.LOSS.adv_loss == "MH":
            raise NotImplementedError("the multi-hinge loss is queued behind the hot path (SURVEY 8f-3)")
        # class-conditioning loss of the classifier-based GANs (src/worker.py:136-157)
        self.adc_fake = self.MODEL.aux_cls_type == "ADC"
        n_cls = self.DATA.num_classes * (2 if self.adc_fake else 1)
        self.cond_loss = losses.make_cond_loss(self.MODEL.d_cond_mtd, n_cls, self.LOSS, self.DDP)
        self.cond_loss_mi = None
        if self.MODEL.aux_cls_type == "TAC":
            import copy
            self.cond_loss_mi = copy.deepcopy(self.cond_loss)
        if self.MODEL.aux_cls_type not in ("W/O", "N/A", "TAC", "ADC"):
            raise NotImplementedError("aux_cls_type %s" % self.MODEL.aux_cls_type)
        for flag in ("apply_lo", "apply_topk", "apply_r1_reg", "apply_fm", "apply_inv_reg"):
            if getattr(self.LOSS, flag, False):
                raise NotImplementedError("LOSS.%s is outside the sgb200 hot-path scope" % flag)
        # a YAML that asks for an augmentation this path does not implement must not silently train a different recipe
        # (Configurations.define_augments raises for ADA / APA / SimCLR types; DiffAugment and the CR augmentation are built)
        self.AUG = getattr(cfgs, "AUG", None)
        if self.AUG is None or not hasattr(self.AUG, "series_augment"):
            from .utils import misc as _misc
            import types as _types
            self.AUG = _types.SimpleNamespace(series_augment=_misc.identity, parallel_augment=_misc.identity, apply_diffaug=False)
        self.l2_loss = torch.nn.MSELoss()
        # LeCam regulariser state (src/worker.py:119-122; the five EMA numbers travel in checkpoints as ``lecam_emas``)
        from .utils import ops as _ops
        self.lecam_ema = _ops.LeCamEMA()
        if lecam_emas is not None:
            self.lecam_ema.__dict__ = lecam_emas
        if self.LOSS.apply_lecam:
            self.lecam_ema.decay, self.lecam_ema.start_itr = self.LOSS.lecam_ema_decay, self.LOSS.lecam_ema_start_iter
        self._current_step = 0

    # ------------------------------------------------------------------------------------------------ data
    def sample_data_basket_raw(self):
        try:
            return next(self.train_iter)
        except StopIteration:
            self.train_iter = iter(self.train_dataloader)
            return next(self.train_iter)

    def sample_data_basket(self):
        """One loader item carries batch_size * acml_steps * d_updates_per_step samples (src/worker.py:194-208)."""
        try:
            real_image_basket, real_label_basket = next(self.train_iter)
        except StopIteration:
            self.train_iter = iter(self.train_dataloader)
            real_image_basket, real_label_basket = next(self.train_iter)
        bs = self.OPTIMIZATION.batch_size
        return torch.split(real_image_basket, bs), torch.split(real_label_basket, bs)

    def _generate(self, is_train=True):
        return sample.generate_images(z_prior=self.MODEL.z_prior, truncation_factor=-1.0, batch_size=self.OPTIMIZATION.batch_size,
                                      z_dim=self.MODEL.z_dim, num_classes=self.DATA.num_classes, y_sampler="totally_random",
                                      radius=self.LOSS.radius if self.LOSS.apply_zcr else "N/A", generator=self.Gen, discriminator=self.Dis, is_train=is_train, LOSS=self.LOSS,
                                      RUN=self.RUN, MODEL=self.MODEL, device=self.local_rank)

    # ------------------------------------------------------------------------------------------------ D phase
    def _graphs_enabled(self):
        plain = not (self.LOSS.apply_cr or self.LOSS.apply_bcr or self.LOSS.apply_zcr or self.LOSS.apply_lecam or
                     getattr(self.AUG, "apply_diffaug", False))      # host-side RNG / EMA state: not capturable
        penalties = self.LOSS.apply_gp or self.LOSS.apply_dra or self.LOSS.apply_maxgp      # alpha / noise: host RNG draws
        return bool(getattr(self.RUN, "cuda_graphs", False)) and not penalties and self.cond_loss is None and plain

    def train_discriminator(self, current_step):
        self._current_step = current_step
        real_image_basket, real_label_basket = self.sample_data_basket_raw()
        if self._graphs_enabled():
            # static input buffers: the graph reads the same addresses every replay
            if getattr(self, "_static_imgs", None) is None or self._static_imgs.shape != real_image_basket.shape:
                self._static_imgs = torch.empty(real_image_basket.shape, device=self.local_rank, dtype=real_image_basket.dtype)
                self._static_labels = torch.empty(real_label_basket.shape, device=self.local_rank, dtype=real_label_basket.dtype)
                self._d_graph = _GraphedPhase(self._d_phase_static)
            self._static_imgs.copy_(real_image_basket, non_blocking=True)
            self._static_labels.copy_(real_label_basket, non_blocking=True)
            return "N/A", self._d_graph()
        dis_acml_loss = self._d_phase(real_image_basket, real_label_basket)
        return self._real_cond_loss, dis_acml_loss

    def _consistency_terms(self, real_images, real_labels, fake_images, fake_labels, fake_images_eps, real_dict, fake_dict):
        """CR (src/worker.py:326-336), bCR (:339-354) and zCR (:357-366) terms of the discriminator loss: squared distance
        between the discriminator's outputs on an image and on its augmented / latent-perturbed copy."""
        if not (self.LOSS.apply_cr or self.LOSS.apply_bcr or self.LOSS.apply_zcr):
            return 0.0
        mtd = self.MODEL.d_cond_mtd

        def pair_loss(a, b):
            loss = self.l2_loss(a["adv_output"], b["adv_output"])
            if mtd == "AC":
                loss = loss + self.l2_loss(a["cls_output"], b["cls_output"])
            elif mtd in ("2C", "D2DCE"):
                loss = loss + self.l2_loss(a["embed"], b["embed"])
            return loss
        total = 0.0
        if self.LOSS.apply_cr:
            real_prl = self.Dis(self.AUG.parallel_augment(real_images), real_labels)
            total = total + self.LOSS.cr_lambda * pair_loss(real_dict, real_prl)
        if self.LOSS.apply_bcr:
            real_prl = self.Dis(self.AUG.parallel_augment(real_images), real_labels)
            fake_prl = self.Dis(self.AUG.parallel_augment(fake_images), fake_labels, adc_fake=self.adc_fake)
            total = total + self.LOSS.real_lambda * pair_loss(real_dict, real_prl) + self.LOSS.fake_lambda * pair_loss(fake_dict, fake_prl)
        if self.LOSS.apply_zcr:
            fake_eps = self.Dis(fake_images_eps, fake_labels, adc_fake=self.adc_fake)
            total = total + self.LOSS.d_lambda * pair_loss(fake_dict, fake_eps)
        return total

    def _d_phase_static(self):
        return self._d_phase(self._static_imgs, self._static_labels)

    def _d_phase(self, real_images_all, real_labels_all):
        bs = self.OPTIMIZATION.batch_size
        real_image_basket, real_label_basket = torch.split(real_images_all, bs), torch.split(real_labels_all, bs)
        misc.make_GAN_trainable(self.Gen, self.Gen_ema, self.Dis)
        misc.toggle_grad(self.Gen, False)
        misc.toggle_grad(self.Dis, True, self.RUN.freezeD)
        # the generator uses batch statistics here but must not move its running statistics (src/worker.py:225)
        self.Gen.apply(misc.untrack_bn_statistics)
        batch_counter = 0
        dis_acml_loss = None
        self._real_cond_loss = "N/A"
        for _ in range(self.OPTIMIZATION.d_updates_per_step):
            self.OPTIMIZATION.d_optimizer.zero_grad()
            for _ in range(self.OPTIMIZATION.acml_steps):
                real_images = real_image_basket[batch_counter].to(self.local_rank, non_blocking=True)
                real_labels = real_label_basket[batch_counter].to(self.local_rank, non_blocking=True)
                fake_images, fake_labels, fake_images_eps, _, _, _, _ = self._generate(True)
                # differentiable augmentation of everything the discriminator sees (src/worker.py:276-285)
                real_dict = self.Dis(self.AUG.series_augment(real_images), real_labels)
                fake_dict = self.Dis(self.AUG.series_augment(fake_images), fake_labels, adc_fake=self.adc_fake)
                dis_acml_loss = self.LOSS.d_loss(real_dict["adv_output"], fake_dict["adv_output"], DDP=self.DDP)
                if self.cond_loss is not None:          # src/worker.py:306-319
                    real_cond_loss = self.cond_loss(**real_dict)
                    dis_acml_loss = dis_acml_loss + self.LOSS.cond_lambda * real_cond_loss
                    if self.cond_loss_mi is not None:
                        dis_acml_loss = dis_acml_loss + self.LOSS.tac_dis_lambda * self.cond_loss_mi(**fake_dict)
                    elif self.adc_fake:
                        dis_acml_loss = dis_acml_loss + self.LOSS.cond_lambda * self.cond_loss(**fake_dict)
                    self._real_cond_loss = real_cond_loss.detach()
                dis_acml_loss = dis_acml_loss + self._consistency_terms(real_images, real_labels, fake_images, fake_labels,
                                                                        fake_images_eps, real_dict, fake_dict)
                if self.LOSS.apply_lecam:                # src/worker.py:394-407
                    self.lecam_ema.update(torch.mean(real_dict["adv_output"]).item(), "D_real", self._current_step)
                    self.lecam_ema.update(torch.mean(fake_dict["adv_output"]).item(), "D_fake", self._current_step)
                    if self._current_step > self.LOSS.lecam_ema_start_iter:
                        dis_acml_loss = dis_acml_loss + self.LOSS.lecam_lambda * losses.lecam_reg(
                            real_dict["adv_output"], fake_dict["adv_output"], self.lecam_ema)
                # src/worker.py:369-392, in this order: each penalty draws its alpha (and DRAGAN its noise) from the host RNG
                if self.LOSS.apply_gp:
                    dis_acml_loss = dis_acml_loss + self.LOSS.gp_lambda * losses.cal_grad_penalty(
                        real_images=real_images, real_labels=real_labels, fake_images=fake_images, discriminator=self.Dis,
                        device=self.local_rank)
                if self.LOSS.apply_dra:
                    dis_acml_loss = dis_acml_loss + self.LOSS.dra_lambda * losses.cal_dra_penalty(
                        real_images=real_images, real_labels=real_labels, discriminator=self.Dis, device=self.local_rank)
                if self.LOSS.apply_maxgp:
                    dis_acml_loss = dis_acml_loss + self.LOSS.maxgp_lambda * losses.cal_maxgrad_penalty(
                        real_images=real_images, real_labels=real_labels, fake_images=fake_images, discriminator=self.Dis,
                        device=self.local_rank)
                dis_acml_loss = dis_acml_loss / self.OPTIMIZATION.acml_steps
                dis_acml_loss.backward()
                batch_counter += 1
            model_lib.allreduce_gradients(self.Dis, self.OPTIMIZATION.d_optimizer)
            self.OPTIMIZATION.d_optimizer.step()
            if self.LOSS.apply_wc:
                self._clip_discriminator_weights()
        return dis_acml_loss.detach()

    @torch.no_grad()
    def _clip_discriminator_weights(self):
        """WGAN weight clipping after every discriminator update (src/worker.py:490-492): every D parameter into
        [-wc_bound, wc_bound], frozen ones included.  With the arena optimiser that is one launch over the flat arena."""
        c = float(self.LOSS.wc_bound)
        if isinstance(self.OPTIMIZATION.d_optimizer, ArenaAdam):
            K.clamp_(self.OPTIMIZATION.d_optimizer.arena.flat, c)
        else:
            for p in self.Dis.parameters():
                p.data.clamp_(-c, c)

    # ------------------------------------------------------------------------------------------------ G phase
    def train_generator(self, current_step):
        if self._graphs_enabled():
            if getattr(self, "_g_graph", None) is None:
                self._g_graph = _GraphedPhase(self._g_phase)
            gen_acml_loss = self._g_graph()
            if self.MODEL.apply_g_ema:           # decay depends on the step number: stays outside the graph (5 launches)
                self.ema.update(current_step)
            return gen_acml_loss
        return self._g_phase(current_step)

    def _g_phase(self, ema_step=None):
        """``ema_step`` None: graph capture / replay (the EMA update follows outside, needs g_updates_per_step == 1)."""
        if ema_step is None and self.OPTIMIZATION.g_updates_per_step != 1 and self.MODEL.apply_g_ema:
            raise NotImplementedError("CUDA graphs with g_updates_per_step > 1 and EMA")
        misc.make_GAN_trainable(self.Gen, self.Gen_ema, self.Dis)
        misc.toggle_grad(self.Dis, False)
        misc.toggle_grad(self.Gen, True)
        self.Gen.apply(misc.track_bn_statistics)
        gen_acml_loss = None
        for _ in range(self.OPTIMIZATION.g_updates_per_step):
            self.OPTIMIZATION.g_optimizer.zero_grad()
            for _ in range(self.OPTIMIZATION.acml_steps):
                fake_images, fake_labels, fake_images_eps, _, _, _, _ = self._generate(True)
                fake_dict = self.Dis(self.AUG.series_augment(fake_images), fake_labels)      # src/worker.py:549-552
                gen_acml_loss = self.LOSS.g_loss(fake_dict["adv_output"], DDP=self.DDP)
                if self.LOSS.apply_zcr:                  # src/worker.py:603-605: push G(z) and G(z + eps) apart
                    gen_acml_loss = gen_acml_loss - self.LOSS.g_lambda * self.l2_loss(fake_images, fake_images_eps)
                if self.cond_loss is not None:          # src/worker.py:574-585
                    gen_acml_loss = gen_acml_loss + self.LOSS.cond_lambda * self.cond_loss(**fake_dict)
                    if self.cond_loss_mi is not None:
                        gen_acml_loss = gen_acml_loss - self.LOSS.tac_gen_lambda * self.cond_loss_mi(**fake_dict)
                    elif self.adc_fake:
                        adc_fake_dict = self.Dis(fake_images, fake_labels, adc_fake=True)
                        gen_acml_loss = gen_acml_loss - self.LOSS.cond_lambda * self.cond_loss(**adc_fake_dict)
                gen_acml_loss = gen_acml_loss / self.OPTIMIZATION.acml_steps
                gen_acml_loss.backward()
            model_lib.allreduce_gradients(self.Gen, self.OPTIMIZATION.g_optimizer)
            self.OPTIMIZATION.g_optimizer.step()
            if ema_step is not None and self.MODEL.apply_g_ema:
                self.ema.update(ema_step)
        return gen_acml_loss.detach()


# ------------------------------------------------------------------------------------------------------ evaluation
def _evaluate(self, step, metrics, writing=True, training=False):
    """WORKER.evaluate (reference src/worker.py:805-935): generated images -> device pre-processing -> Inception
    features -> IS / FID / PRDC, with the reference's mode choreography (make_GAN_untrainable keeps the spectral-norm
    power iteration running, BN uses running statistics) and best-FID bookkeeping.  Results are also kept in
    ``self.last_metrics``.  wandb / npy dumps are outside the hot-path scope."""
    from .metrics import features, fid, ins, prdc
    is_best, num_splits, nearest_k = False, 1, 5
    is_acc = "ImageNet" in self.DATA.name and "Tiny" not in self.DATA.name
    num_eval = self.num_eval if isinstance(self.num_eval, int) else self.num_eval[getattr(self.RUN, "ref_dataset", "train")]
    metric_dict = {}
    with torch.no_grad():
        misc.make_GAN_untrainable(self.Gen, self.Gen_ema, self.Dis)
        generator = self.Gen_ema if (self.MODEL.apply_g_ema and self.Gen_ema is not None) else self.Gen
        # GeneratorController.prepare_generator (src/utils/misc.py:77-106), in place like the reference: the standing
        # statistics are accumulated ONCE per run (std_stat_counter, src/worker.py:809-810), the generator is then put in
        # eval mode with conv / linear / embedding back in train mode (the spectral-norm iteration keeps running).
        if getattr(self.RUN, "standing_statistics", False):
            self.std_stat_counter = getattr(self, "std_stat_counter", 0) + 1
            if self.std_stat_counter <= 1:
                misc.apply_standing_statistics(generator=generator, standing_max_batch=self.RUN.standing_max_batch,
                                               standing_step=self.RUN.standing_step, DATA=self.DATA, MODEL=self.MODEL, LOSS=self.LOSS,
                                               OPTIMIZATION=self.OPTIMIZATION, RUN=self.RUN, device=self.local_rank,
                                               global_rank=self.global_rank, logger=self.logger)
            generator.eval()
            generator.apply(misc.set_deterministic_op_trainable)
        elif getattr(self.RUN, "batch_statistics", False):
            generator.apply(misc.set_bn_trainable)
            generator.apply(misc.untrack_bn_statistics)
        # FID statistics are accumulated on the fly ([sum f, sum f f^T], fp64) and, under DDP, all-reduced (33.5 MB) --
        # the gathered [N, 2048] feature matrix is only needed by PRDC
        moments = fid.MomentsAccumulator(2048, self.local_rank) if "fid" in metrics else None
        fake_feats, fake_probs, fake_labels = features.generate_images_and_stack_features(
            generator=generator, discriminator=self.Dis, eval_model=self.eval_model, num_generate=num_eval,
            y_sampler="totally_random", batch_size=self.OPTIMIZATION.batch_size, z_prior=self.MODEL.z_prior,
            truncation_factor=self.RUN.truncation_factor, z_dim=self.MODEL.z_dim, num_classes=self.DATA.num_classes, LOSS=self.LOSS,
            RUN=self.RUN, MODEL=self.MODEL, quantize=True, world_size=getattr(self.OPTIMIZATION, "world_size", 1), DDP=self.DDP,
            device=self.local_rank, logger=self.logger, moments=moments)
        if "is" in metrics:
            features._tick(None, self.local_rank)
            kl_score, kl_std, top1, top5 = ins.eval_features(probs=fake_probs, labels=fake_labels, data_loader=self.eval_dataloader,
                                                             num_features=num_eval, split=num_splits, is_acc=is_acc)
            metric_dict.update({"IS": float(kl_score), "Top1_acc": top1, "Top5_acc": top5})
            features._tick("inception score", self.local_rank)
        if "fid" in metrics:
            if self.DDP:
                moments.all_reduce(getattr(self.Gen, "sgb_group", None))
                features._tick("moments all-reduce", self.local_rank)
            m1, c1 = moments.finalize()
            fid_score = fid.frechet_distance_device(m1, c1, torch.as_tensor(self.mu, device=m1.device),
                                                    torch.as_tensor(self.sigma, device=m1.device))
            if self.best_fid is None or fid_score <= self.best_fid:
                self.best_fid, self.best_step, is_best = fid_score, step, True
            metric_dict.update({"FID": fid_score})
            features._tick("moments finalize + Frechet distance", self.local_rank)
        if "prdc" in metrics:
            pr = prdc.compute_prdc(real_features=torch.as_tensor(self.real_feats, dtype=torch.float64, device=fake_feats.device),
                                   fake_features=fake_feats[:num_eval].to(torch.float64), nearest_k=nearest_k)
            metric_dict.update({"Improved_Precision": pr["precision"], "Improved_Recall": pr["recall"], "Density": pr["density"],
                                "Coverage": pr["coverage"]})
    self.last_metrics = metric_dict
    if self.global_rank == 0 and self.logger is not None:
        self.logger.info("evaluation (step {}): {}".format(step, metric_dict))
    misc.make_GAN_trainable(self.Gen, self.Gen_ema, self.Dis)
    return is_best


WORKER.evaluate = _evaluate
