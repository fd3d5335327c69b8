"""Reference formulations of the DRAGAN and max-gradient penalties for the tests, written like O.grad_penalty
(oracle/studiogan_oracle.py): the reference's expressions with its host draws passed in, and dP/dtheta by the create_graph
double backward.  ``disc_fn(x) -> [B]`` logits."""
import torch


def _input_gradient(disc_fn, interp):
    out = disc_fn(interp)
    grads = torch.autograd.grad(outputs=out, inputs=interp, grad_outputs=torch.ones_like(out), create_graph=True,
                                retain_graph=True, only_inputs=True)[0]
    return grads.view(len(grads), -1)


def dra_interpolate(real, noise, alpha):
    """x_hat of cal_dra_penalty (src/utils/losses.py:319-335); alpha [B,1,1,1], noise shaped like real."""
    return real + (alpha.view(-1, 1, 1, 1) * (0.5 * real.std() * noise))


def dra_penalty(disc_fn, real, noise, alpha):
    """cal_dra_penalty (src/utils/losses.py:319-335): mean_b (||g_b|| - 1)^2 at x_hat = real + alpha * 0.5 std(real) u."""
    interp = dra_interpolate(real, noise, alpha).detach().requires_grad_(True)
    grads = _input_gradient(disc_fn, interp)
    return ((grads.norm(2, dim=1) - 1) ** 2).mean() + interp[:, 0, 0, 0].mean() * 0


def maxgrad_penalty(disc_fn, real, fake, alpha):
    """cal_maxgrad_penalty (src/utils/losses.py:337-353): max_b ||g_b||^2 at x_hat = alpha real + (1 - alpha) fake."""
    B, c, h, w = real.shape
    a = alpha.expand(B, real.nelement() // B).contiguous().view(B, c, h, w)
    interp = (a * real + (1 - a) * fake).detach().requires_grad_(True)
    grads = _input_gradient(disc_fn, interp)
    return torch.max(grads.norm(2, dim=1) ** 2) + interp[:, 0, 0, 0].mean() * 0


def split_grad_errors(got, ref):
    """Per-parameter comparison of dP/dtheta (name -> tensor) against a reference.  Parameters whose reference gradient is
    zero up to round-off (<= 1e-5 of the largest: the head bias and every bias a later batch norm removes; they do not
    change the penalty) are held to the weight beside them; the others by relative L2 and cosine.
    Returns (worst (error, name), median error, smallest cosine, largest |grad(zero bias)| / |grad(its weight)|)."""
    ref = {n: (r.double() if r is not None else None) for n, r in ref.items()}
    top = max(float(r.norm()) for r in ref.values() if r is not None)
    zero = [n for n, r in ref.items() if r is None or float(r.norm()) <= 1e-5 * top]
    assert all(n.endswith("bias") for n in zero), zero
    errs, coss = {}, {}
    for n, r in ref.items():
        if n not in zero:
            a = got[n].double()
            errs[n] = float((a - r).norm() / r.norm())
            coss[n] = float((a * r).sum() / (a.norm() * r.norm() + 1e-30))
    ratio = max([float(got[n].double().norm() / got[n[:-4] + "weight"].double().norm()) for n in zero] or [0.0])
    worst = max(errs, key=errs.get)
    return (errs[worst], worst), float(torch.tensor(list(errs.values())).median()), min(coss.values()), ratio
