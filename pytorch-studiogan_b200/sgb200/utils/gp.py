"""WGAN-GP gradient penalty (reference: src/utils/losses.py:268-275 ``cal_deriv`` and :301-316 ``cal_grad_penalty``).

    x_hat = alpha * real + (1 - alpha) * fake,  alpha ~ U[0,1) per sample (host RNG, as the reference)
    g     = d(sum_b D(x_hat)_b) / d(x_hat)
    P     = mean_b (||g_b||_2 - 1)^2

The reference obtains dP/dtheta by differentiating through its first backward pass (``create_graph=True``).  Here the same
quantity is evaluated as *reverse over forward*: with v = dP/dg (a constant once g is known),

    dP/dtheta = d/dtheta <v, g(theta)>,   and   <v, g(theta)> = d/d(eps) sum_b D(x_hat + eps v; theta)_b |_{eps=0},

i.e. the output of a tangent (JVP) pass of the discriminator along v.  Three passes over the discriminator:
  1. primal forward on x_hat, every op recorded on the tangent tape (autograd_ops.TAPE);
  2. an ordinary backward to x_hat only (no weight gradients) -> g -> per-sample norms, P and the seed v (library kernels);
  3. the tape replayed on v: convolutions / pools are linear so their tangent is the same kernel on the tangent tensor,
     ReLU passes the tangent where the primal was positive, training-mode batch norm uses its own tangent kernel whose
     backward is torch's batchnorm_double_backward.
The returned tensor has P's value and the gradient of the pass-3 scalar, so ``(loss + lambda * gp).backward()`` deposits
exactly dP/dtheta (through the tangent graph and, for batch-norm discriminators, the primal graph it shares).

The same three passes serve the other penalties of this family; each brings its own x_hat and its own (P, v) step:
  * DRAGAN (src/utils/losses.py:319-335): x_hat = real + alpha_b * 0.5 * std(real) * u, P and v as above;
  * max-gradient / LGAN (:337-353): x_hat as above, P = max_b ||g_b||^2, v = 2 g_b / n_ties on the arg-max sample(s)."""
import torch

from .. import autograd_ops as A
from .. import kernels as K


def replay(tape, seeds):
    """Push tangents through a recorded tape.  ``seeds``: {id(primal tensor): tangent}.  Returns ``tan(t)``."""
    tmap = dict(seeds)

    def tan(t):
        return tmap.get(id(t)) if t is not None else None

    for rule, args, out in tape:
        touts = rule.tangent(args, out, tan)
        outs = out if isinstance(out, tuple) else (out,)
        touts = touts if isinstance(touts, tuple) else (touts,)
        for o, t in zip(outs, touts):
            if t is not None:
                tmap[id(o)] = t
    return tan


def cal_deriv(inputs, outputs, device=None):
    """d(sum outputs)/d(inputs) without a second-order graph (first pass of the penalty)."""
    A.SKIP_PARAM_GRADS = True
    try:
        (g,) = torch.autograd.grad(outputs=outputs, inputs=inputs, grad_outputs=torch.ones_like(outputs), retain_graph=True)
    finally:
        A.SKIP_PARAM_GRADS = False
    return g


def _penalty_passes(x_hat, real_labels, discriminator, penalty_and_seed):
    """Passes 1-3 on an input x_hat built by the caller; ``penalty_and_seed(g) -> (P, dP/dg)`` is the penalty's own step."""
    if A.TAPE is not None:
        raise RuntimeError("nested gradient-penalty passes are not supported")
    x_hat.requires_grad_(True)
    A.TAPE = tape = []
    try:
        out = discriminator(x_hat, real_labels, eval=False)
    finally:
        A.TAPE = None
    adv = out["adv_output"]
    g = cal_deriv(x_hat, adv)
    penalty, v = penalty_and_seed(g)
    t_adv = replay(tape, {id(x_hat): v})(adv)
    if t_adv is None:
        raise RuntimeError("gradient penalty: the tangent did not reach the discriminator output")
    surrogate = t_adv.sum()
    return penalty.detach() + (surrogate - surrogate.detach())


def _unit_norm_seed(g):
    """P = mean_b (||g_b|| - 1)^2 and its seed (WGAN-GP and DRAGAN)."""
    sumsq = K.gp_sumsq(g)
    return ((torch.sqrt(sumsq) - 1.0) ** 2).mean(), K.gp_seed(g, sumsq)


def _max_norm_seed(g):
    """P = max_b ||g_b||^2 and its seed (ties split evenly, as torch's max backward)."""
    return K.gp_seed_max(g, K.gp_sumsq(g))


def _interpolate(real_images, fake_images, alpha):
    batch_size = real_images.shape[0]
    alpha = alpha.reshape(batch_size).to(device=real_images.device, dtype=torch.float32)
    return K.gp_interpolate(real_images.detach().float(), fake_images.detach().float().to(real_images.device), alpha)


def cal_grad_penalty(real_images, real_labels, fake_images, discriminator, device=None, alpha=None):
    if alpha is None:
        alpha = torch.rand(real_images.shape[0], 1)                    # host RNG (src/utils/losses.py:303)
    x_hat = _interpolate(real_images, fake_images, alpha)
    return _penalty_passes(x_hat, real_labels, discriminator, _unit_norm_seed)


def cal_dra_penalty(real_images, real_labels, discriminator, device=None, alpha=None, noise=None):
    """DRAGAN (src/utils/losses.py:319-335): x_hat = real + alpha_b * 0.5 * std(real) * u, u ~ U[0,1) per element,
    P = mean_b (||g_b|| - 1)^2.  std is taken over this rank's batch, as in the reference."""
    batch_size = real_images.shape[0]
    if alpha is None:
        alpha = torch.rand(batch_size, 1, 1, 1)                         # host RNG, in the reference's order (:321, :325)
    if noise is None:
        noise = torch.rand(real_images.size())
    real = real_images.detach().float().contiguous()
    alpha = alpha.reshape(batch_size).to(device=real.device, dtype=torch.float32)
    noise = noise.to(device=real.device, dtype=torch.float32)
    x_hat = K.dra_perturb(real, K.dra_std(real), alpha, noise)
    return _penalty_passes(x_hat, real_labels, discriminator, _unit_norm_seed)


def cal_maxgrad_penalty(real_images, real_labels, fake_images, discriminator, device=None, alpha=None):
    """Max-gradient penalty of LGAN (src/utils/losses.py:337-353): x_hat as for WGAN-GP, P = max_b ||g_b||^2 over this
    rank's batch."""
    if alpha is None:
        alpha = torch.rand(real_images.shape[0], 1)                    # host RNG (src/utils/losses.py:339)
    x_hat = _interpolate(real_images, fake_images, alpha)
    return _penalty_passes(x_hat, real_labels, discriminator, _max_norm_seed)
