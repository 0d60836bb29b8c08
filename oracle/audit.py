"""float64 references for auditing one training step layer by layer.  TEST INFRASTRUCTURE (see oracle/__init__.py).

The convolution itself is `spconv_cpu.native_conv` run in float64 (its input and weight gradients from autograd); this
module adds only BatchNorm1d + ReLU from given statistics, forward and backward, and the bound a bf16-rounded result
is held to."""
from __future__ import annotations

import torch

from .spconv_cpu import native_conv

BF16_REL = 2.0 ** -8        # |bf16_rn(r) - r| <= half a bf16 ulp < 2^-8 |r| (8 significant bits); a kernel rounds its fp32
                            # value, which may sit a few fp32 ulps from r: only a tie within 2^-16 of the bound could cross it
ABS_REL = 1e-6              # ... plus an absolute part relative to the largest element (values next to zero)


def conv(inp, w, nbr, n_out):
    """out[o] = sum_k inp[nbr[k, o]] @ w[:, k, :].T in float64 (w [C_out, K, C_in]; nbr [K, >= n_out], -1 = no pair)."""
    return native_conv(inp.double(), w.double(), nbr[:, :n_out].long(), n_out, False)


def conv_grads(inp, w, nbr, n_out, dout, need_din=True):
    """(din or None, dw) of conv() for the output gradient dout [n_out, C_out], float64, by autograd."""
    x = inp.detach().double().requires_grad_(need_din)
    wd = w.detach().double().requires_grad_(True)
    out = conv(x, wd, nbr, n_out)
    grads = torch.autograd.grad(out, [x, wd] if need_din else [wd], dout.double())
    return (grads[0], grads[1]) if need_din else (None, grads[0])


def batch_stats(x, eps):
    """(mean, invstd, biased var, unbiased var) per channel of x [n, c], float64."""
    x = x.double()
    mean = x.mean(0)
    var = (x - mean).pow(2).mean(0)
    n = x.shape[0]
    return mean, 1.0 / torch.sqrt(var + eps), var, var * n / max(n - 1, 1)


def running_update(running_mean, running_var, mean, var_unbiased, momentum):
    """torch.nn.BatchNorm1d's update of the running buffers, float64."""
    rm = (1.0 - momentum) * running_mean.double() + momentum * mean.double()
    rv = (1.0 - momentum) * running_var.double() + momentum * var_unbiased.double()
    return rm, rv


def bn_relu_fwd(x, mean, invstd, gamma, beta):
    """relu((x - mean) * invstd * gamma + beta), float64."""
    x = x.double()
    return torch.relu((x - mean.double()) * invstd.double() * gamma.double() + beta.double())


def bn_relu_bwd(dy, x, mean, invstd, gamma, beta, training=True, active=None):
    """Backward of bn_relu_fwd with the statistics held fixed in eval mode and taken from the batch in training mode
    (torch.nn.BatchNorm1d): -> (dx, dgamma, dbeta), float64.  active [n, c] bool: where the ReLU passes the gradient
    (default: relu_mask; a caller may pass the mask the kernel itself decided)."""
    if active is None:
        active = relu_mask(x, mean, invstd, gamma, beta)
    x, dy = x.double(), dy.double()
    mean, invstd, gamma = mean.double(), invstd.double(), gamma.double()
    xhat = (x - mean) * invstd
    g = torch.where(active, dy, torch.zeros_like(dy))
    dbeta = g.sum(0)
    dgamma = (g * xhat).sum(0)
    if training:
        n = x.shape[0]
        dx = gamma * invstd * (g - dbeta / n - xhat * dgamma / n)
    else:
        dx = gamma * invstd * g
    return dx, dgamma, dbeta


def relu_mask(x, mean, invstd, gamma, beta):
    """The float64 pre-activation of bn_relu_fwd is positive."""
    x = x.double()
    return (x - mean.double()) * invstd.double() * gamma.double() + beta.double() > 0


def bound_excess(got, ref, rel=BF16_REL, abs_rel=ABS_REL):
    """max over elements of |got - ref| / (rel |ref| + abs_rel max|ref|): <= 1 means every element is within the bound
    (rel = 2^-8: a bf16 rounding of the float64 value; rel = 0: a plain absolute bound)."""
    got, ref = got.double(), ref.double()
    if ref.numel() == 0:
        return 0.0
    lim = rel * ref.abs() + abs_rel * float(ref.abs().max())
    return float(((got - ref).abs() / lim.clamp_min(1e-300)).max())
