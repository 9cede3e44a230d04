"""numpy restatement of what cleanrl/ppg_procgen.py adds to PPO: the auxiliary-phase loss with its gradient with respect
to the joint head output, and torch.optim.Adam's per-tensor semantics (one ``step`` per tensor, a tensor without a gradient
is skipped).  TEST INFRASTRUCTURE ONLY: validated against tests/golden/ppg_procgen_*.npz and torch autograd."""
from __future__ import annotations

import numpy as np


def _log_softmax(x):
    m = x.max(axis=-1, keepdims=True)
    m = np.where(np.isfinite(m), m, 0.0)
    return x - (np.log(np.exp(x - m).sum(axis=-1, keepdims=True)) + m)


def aux_loss(head, old_logits, returns, beta_clone=1.0, n_aux_grad_accum=1, dtype=np.float64):
    """head [n, A + 2] = [logits | value | aux_value]; returns ({kl_loss, aux_value_loss, real_value_loss}, dhead) where
    dhead = d((aux_value_loss + beta_clone * kl_loss + real_value_loss) / n_aux_grad_accum) / d(head)
    (cleanrl/ppg_procgen.py:449-461; KL edge cases as torch.distributions.kl._kl_categorical_categorical)."""
    head = np.asarray(head, dtype=dtype)
    old = np.asarray(old_logits, dtype=dtype)
    R = np.asarray(returns, dtype=dtype)
    n, A = old.shape
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        lp_new, lp_old = _log_softmax(head[:, :A]), _log_softmax(old)
        p_new, p_old = np.exp(lp_new), np.exp(lp_old)
        t = p_old * (lp_old - lp_new)
        t[p_new == 0] = np.inf
        t[p_old == 0] = 0
    v, aux = head[:, A], head[:, A + 1]
    stats = {"kl_loss": t.sum(-1).mean(), "aux_value_loss": 0.5 * ((aux - R) ** 2).mean(),
             "real_value_loss": 0.5 * ((v - R) ** 2).mean()}
    scale = 1.0 / (n * n_aux_grad_accum)
    dhead = np.empty_like(head)
    dhead[:, :A] = beta_clone * (p_new - p_old) * scale
    dhead[:, A] = (v - R) * scale
    dhead[:, A + 1] = (aux - R) * scale
    return stats, dhead


class Adam:
    """torch.optim.Adam (no weight decay, no amsgrad) over a list of arrays, float32 state, scalars in double as
    torch/optim/adam.py: every tensor has its own ``step``; a tensor whose gradient is None is skipped entirely."""

    def __init__(self, params, lr, beta1=0.9, beta2=0.999, eps=1e-8):
        self.params = [np.array(p, dtype=np.float32) for p in params]
        self.m = [np.zeros_like(p) for p in self.params]
        self.v = [np.zeros_like(p) for p in self.params]
        self.steps = [0] * len(self.params)
        self.lr, self.beta1, self.beta2, self.eps = lr, beta1, beta2, eps

    def step(self, grads, lr=None):
        lr = self.lr if lr is None else lr
        f = np.float32
        for i, g in enumerate(grads):
            if g is None:
                continue
            g = np.asarray(g, dtype=f)
            self.steps[i] += 1
            t = self.steps[i]
            self.m[i] = self.m[i] + f(1.0 - self.beta1) * (g - self.m[i])
            self.v[i] = self.v[i] * f(self.beta2) + f(1.0 - self.beta2) * g * g
            step_size = lr / (1.0 - self.beta1 ** t)
            bc2_sqrt = np.sqrt(1.0 - self.beta2 ** t)
            denom = np.sqrt(self.v[i]) / f(bc2_sqrt) + f(self.eps)
            self.params[i] = self.params[i] + f(-step_size) * (self.m[i] / denom)
        return self.params
