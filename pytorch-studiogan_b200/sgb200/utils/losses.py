"""Adversarial losses with the reference's names and signatures (src/utils/losses.py:197-239): scalar reductions over the
[B] logit vector coming out of the discriminator head, plus GatherLayer (:19-37) and the WGAN-GP penalty entry point."""
import torch
import torch.distributed as dist
import torch.nn.functional as F


class GatherLayer(torch.autograd.Function):
    """all_gather with a gradient (src/utils/losses.py:19-37): each rank receives the gradient of its own shard."""

    @staticmethod
    def forward(ctx, input):
        ctx.save_for_backward(input)
        out = [torch.zeros_like(input) for _ in range(dist.get_world_size())]
        dist.all_gather(out, input)
        return tuple(out)

    @staticmethod
    def backward(ctx, *grads):
        (input,) = ctx.saved_tensors
        g = torch.zeros_like(input)
        g[:] = grads[dist.get_rank()]
        return g


def d_vanilla(d_logit_real, d_logit_fake, DDP=False):
    return torch.mean(F.softplus(-d_logit_real)) + torch.mean(F.softplus(d_logit_fake))


def g_vanilla(d_logit_fake, DDP=False):
    return torch.mean(F.softplus(-d_logit_fake))


def d_logistic(d_logit_real, d_logit_fake, DDP=False):
    return (F.softplus(-d_logit_real) + F.softplus(d_logit_fake)).mean()


def g_logistic(d_logit_fake, DDP=False):
    return F.softplus(-d_logit_fake).mean()


def d_ls(d_logit_real, d_logit_fake, DDP=False):
    return (0.5 * (d_logit_real - 1.0) ** 2 + 0.5 * d_logit_fake ** 2).mean()


def g_ls(d_logit_fake, DDP=False):
    return (0.5 * (d_logit_fake - 1.0) ** 2).mean()


def d_hinge(d_logit_real, d_logit_fake, DDP=False):
    return torch.mean(F.relu(1. - d_logit_real)) + torch.mean(F.relu(1. + d_logit_fake))


def g_hinge(d_logit_fake, DDP=False):
    return -torch.mean(d_logit_fake)


def d_wasserstein(d_logit_real, d_logit_fake, DDP=False):
    return torch.mean(d_logit_fake - d_logit_real)


def g_wasserstein(d_logit_fake, DDP=False):
    return -torch.mean(d_logit_fake)


def cal_deriv(inputs, outputs, device=None):
    from . import gp
    return gp.cal_deriv(inputs, outputs, device)


def cal_grad_penalty(real_images, real_labels, fake_images, discriminator, device=None, alpha=None):
    """src/utils/losses.py:301-316; see utils/gp.py for how the second-order term is evaluated."""
    from . import gp
    return gp.cal_grad_penalty(real_images, real_labels, fake_images, discriminator, device, alpha)


def cal_dra_penalty(real_images, real_labels, discriminator, device=None, alpha=None, noise=None):
    """src/utils/losses.py:319-335 (DRAGAN); see utils/gp.py."""
    from . import gp
    return gp.cal_dra_penalty(real_images, real_labels, discriminator, device, alpha, noise)


def cal_maxgrad_penalty(real_images, real_labels, fake_images, discriminator, device=None, alpha=None):
    """src/utils/losses.py:337-353 (LGAN max-gradient penalty); see utils/gp.py."""
    from . import gp
    return gp.cal_maxgrad_penalty(real_images, real_labels, fake_images, discriminator, device, alpha)


# ----------------------------------------------------------------------------------------------------------------------
# Class-conditioning losses of the classifier-based GANs (ACGAN "AC", ContraGAN "2C", ReACGAN "D2DCE"):
# reference src/utils/losses.py:38-165.  They act on the discriminator head's [B, .] fp32 outputs; the label masks are
# built on the device (label == label^T) instead of the reference's per-class numpy loops -- same values.
# ----------------------------------------------------------------------------------------------------------------------
def _gather_ddp(*tensors):
    return tuple(torch.cat(GatherLayer.apply(t), dim=0) for t in tensors)


def _off_diagonal(M):
    """[h, h] -> [h, h-1] without the diagonal (reference ``_remove_diag`` / ``remove_diag``)."""
    h = M.shape[0]
    keep = ~torch.eye(h, dtype=torch.bool, device=M.device)
    return M[keep].view(h, h - 1)


def _cosine_matrix(x, y):
    return F.cosine_similarity(x.unsqueeze(1), y.unsqueeze(0), dim=-1)


class CrossEntropyLoss(torch.nn.Module):
    """ACGAN classification loss (src/utils/losses.py:38-44)."""

    def forward(self, cls_output, label, **_):
        return F.cross_entropy(cls_output, label).mean()


class ConditionalContrastiveLoss(torch.nn.Module):
    """ContraGAN's 2C loss (src/utils/losses.py:47-98)."""

    def __init__(self, num_classes, temperature, master_rank=None, DDP=False):
        super().__init__()
        self.num_classes, self.temperature, self.master_rank, self.DDP = num_classes, temperature, master_rank, DDP

    def forward(self, embed, proxy, label, **_):
        if self.DDP:
            embed, proxy, label = _gather_ddp(embed, proxy, label)
        sim_matrix = torch.exp(_off_diagonal(_cosine_matrix(embed, embed)) / self.temperature)
        same_class = (label.unsqueeze(1) == label.unsqueeze(0)).to(torch.long)       # == mask_multi[label] of the reference
        sim_pos_only = _off_diagonal(same_class) * sim_matrix
        emb2proxy = torch.exp(F.cosine_similarity(embed, proxy, dim=-1) / self.temperature)
        numerator = emb2proxy + sim_pos_only.sum(dim=1)
        denominator = torch.cat([emb2proxy.unsqueeze(1), sim_matrix], dim=1).sum(dim=1)
        return -torch.log(numerator / denominator).mean()


class Data2DataCrossEntropyLoss(torch.nn.Module):
    """ReACGAN's D2D-CE loss (src/utils/losses.py:101-165)."""

    def __init__(self, num_classes, temperature, m_p, master_rank=None, DDP=False):
        super().__init__()
        self.num_classes, self.temperature, self.m_p, self.master_rank, self.DDP = num_classes, temperature, m_p, master_rank, DDP

    def forward(self, embed, proxy, label, **_):
        if self.DDP:
            embed, proxy, label = _gather_ddp(embed, proxy, label)
        sim_matrix = _off_diagonal((_cosine_matrix(embed, embed) + self.m_p - 1) / self.temperature)
        sim_max, _ = torch.max(sim_matrix, dim=1, keepdim=True)
        sim_matrix = F.relu(sim_matrix) - sim_max.detach()                            # numerical stability, as the reference
        smp2proxy = F.cosine_similarity(embed, proxy, dim=-1)
        other_class = (label.unsqueeze(1) != label.unsqueeze(0)).to(torch.long)      # false-negative removal mask
        improved_sim_matrix = _off_diagonal(other_class) * torch.exp(sim_matrix)
        pos_attr = F.relu((self.m_p - smp2proxy) / self.temperature)
        neg_repul = torch.log(torch.exp(-pos_attr) + improved_sim_matrix.sum(dim=1))
        return (pos_attr + neg_repul).mean()


def make_cond_loss(d_cond_mtd, num_classes, LOSS, DDP):
    """The conditioning loss WORKER installs for ``MODEL.d_cond_mtd`` (src/worker.py:140-154)."""
    if d_cond_mtd == "AC":
        return CrossEntropyLoss()
    if d_cond_mtd == "2C":
        return ConditionalContrastiveLoss(num_classes=num_classes, temperature=LOSS.temperature, DDP=DDP)
    if d_cond_mtd == "D2DCE":
        return Data2DataCrossEntropyLoss(num_classes=num_classes, temperature=LOSS.temperature, m_p=LOSS.m_p, DDP=DDP)
    return None


def lecam_reg(d_logit_real, d_logit_fake, ema):
    """LeCam regulariser (src/utils/losses.py:262-265): mean relu(D(real) - ema.D_fake)^2 + mean relu(ema.D_real - D(fake))^2."""
    return torch.mean(F.relu(d_logit_real - ema.D_fake).pow(2)) + torch.mean(F.relu(ema.D_real - d_logit_fake).pow(2))
