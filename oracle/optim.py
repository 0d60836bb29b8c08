"""The adam_onecycle / adam_cosin parameter update restated in numpy float64 (what vc_optim_step computes), and the
OneCycle schedule that drives it.

One step, for tensors p with gradients g (None: the tensor received no gradient), Adam state m, v and step count t:

    total_norm = sqrt(sum over every g of sum g^2)                              (clip_grad_norm_, train_utils.py:50)
    clip_coef  = min(1, max_norm / (total_norm + 1e-6))                          (1 without max_norm)
    skip the step (nothing changes, `skipped` += 1) when total_norm is not finite or a guard word is non-zero
    t += 1;  gh = clip_coef * g
    p <- p * (1 - wd * lr)                       every tensor, with or without gradient   (fastai_optim.py:135-147)
    m <- m + (1 - beta1) * (gh - m);  v <- beta2 * v + (1 - beta2) * gh^2                   (torch.optim.Adam)
    p <- p - lr / (1 - beta1^t) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps)
beta1 is the momentum of THIS step (OneCycle changes it every step; torch raises the current value to the power t).
Tensors of `norm_only` gradients count in total_norm and are not updated (parameters clip_grad_norm_ sees and the
optimizer does not own).
"""
from __future__ import annotations

import numpy as np


def annealing_cos(start, end, pct):
    return end + (start - end) / 2 * (np.cos(np.pi * pct) + 1)


def one_cycle(step, total_step, lr_max, moms, div_factor, pct_start):
    """-> (lr, mom) of iteration `step`: cosine from lr_max / div_factor up to lr_max over the first int(total_step *
    pct_start) iterations, then down to lr_max / div_factor / 1e4; the momentum moms[0] -> moms[1] -> moms[0] over the same
    two phases."""
    a1 = int(total_step * pct_start)
    low = lr_max / div_factor
    if step < a1:
        pct = step / a1
        return annealing_cos(low, lr_max, pct), annealing_cos(moms[0], moms[1], pct)
    pct = (step - a1) / (total_step - a1)
    return annealing_cos(lr_max, low / 1e4, pct), annealing_cos(moms[1], moms[0], pct)


class AdamOneCycle:
    def __init__(self, params, wd, beta2=0.99, eps=1e-8):
        self.p = [np.asarray(p, dtype=np.float64).copy() for p in params]
        self.m = [np.zeros_like(p) for p in self.p]
        self.v = [np.zeros_like(p) for p in self.p]
        self.wd, self.beta2, self.eps = float(wd), float(beta2), float(eps)
        self.t, self.skipped, self.total_norm, self.clip_coef = 0, 0, 0.0, 1.0

    def step(self, grads, lr, mom, max_norm=None, norm_only=(), guard=0):
        """grads: one array or None per tensor -> whether the step was applied."""
        gs = [None if g is None else np.asarray(g, dtype=np.float64) for g in grads]
        with np.errstate(all='ignore'):
            sq = sum(float((g * g).sum()) for g in gs + [np.asarray(g, dtype=np.float64) for g in norm_only] if g is not None)
        self.total_norm = float(np.sqrt(sq))
        if not np.isfinite(self.total_norm) or guard:
            self.skipped += 1
            return False
        self.clip_coef = 1.0 if max_norm is None else min(1.0, max_norm / (self.total_norm + 1e-6))
        self.t += 1
        bc1, bc2 = 1 - mom ** self.t, 1 - self.beta2 ** self.t
        for i, g in enumerate(gs):
            self.p[i] *= 1 - self.wd * lr
            if g is None:
                continue
            gh = self.clip_coef * g
            self.m[i] += (1 - mom) * (gh - self.m[i])
            self.v[i] = self.beta2 * self.v[i] + (1 - self.beta2) * gh * gh
            self.p[i] -= lr / bc1 * self.m[i] / (np.sqrt(self.v[i]) / np.sqrt(bc2) + self.eps)
        return True
