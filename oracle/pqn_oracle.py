"""numpy / torch-CPU restatement of cleanrl/pqn.py's update math.  TEST INFRASTRUCTURE ONLY.

* ``forward`` / ``loss_and_grads``: the LayerNorm Q-network (Linear 120 -> LayerNorm -> ReLU -> Linear 84 -> LayerNorm ->
  ReLU -> Linear A) and the gradient of ``F.mse_loss(b_returns[mb], Q[a])`` with respect to every parameter, in float64,
  with the LayerNorm backward written out (dz = rstd (dxhat - mean(dxhat) - xhat mean(dxhat xhat))).
* ``qlambda``: the reference's Q(lambda) loop in float32 with torch's rounding points.
* ``radam_step``: one ``torch.optim.RAdam`` step (``_single_tensor_radam``, no weight decay) in float32 numpy, with the
  python-double scalars rounded where the tensor operations round them.
"""
from __future__ import annotations

import math

import numpy as np

H1, H2, LN_EPS = 120, 84, 1e-5
PARAM_NAMES = ("network.0.weight", "network.0.bias", "network.1.weight", "network.1.bias", "network.3.weight",
               "network.3.bias", "network.4.weight", "network.4.bias", "network.6.weight", "network.6.bias")


def shapes(obs_dim, A):
    return [(H1, obs_dim), (H1,), (H1,), (H1,), (H2, H1), (H2,), (H2,), (H2,), (A, H2), (A,)]


def unflatten(flat, obs_dim, A):
    out, off = [], 0
    for s in shapes(obs_dim, A):
        n = int(np.prod(s))
        out.append(np.asarray(flat[off:off + n]).reshape(s))
        off += n
    return out


def _ln_fwd(z, g, b):
    mu = z.mean(1, keepdims=True)
    var = ((z - mu) ** 2).mean(1, keepdims=True)
    rstd = 1.0 / np.sqrt(var + LN_EPS)
    xh = (z - mu) * rstd
    return xh, rstd, xh * g + b


def forward(params, x, keep=False):
    w1, b1, g1, be1, w2, b2, g2, be2, w3, b3 = [np.asarray(p, np.float64) for p in params]
    x = np.asarray(x, np.float64)
    xh1, r1, y1 = _ln_fwd(x @ w1.T + b1, g1, be1)
    h1 = np.maximum(y1, 0)
    xh2, r2, y2 = _ln_fwd(h1 @ w2.T + b2, g2, be2)
    h2 = np.maximum(y2, 0)
    q = h2 @ w3.T + b3
    if keep:
        return q, dict(x=x, xh1=xh1, r1=r1, y1=y1, h1=h1, xh2=xh2, r2=r2, y2=y2, h2=h2)
    return q


def _ln_bwd(dy, xh, rstd, g):
    dxh = dy * g
    return rstd * (dxh - dxh.mean(1, keepdims=True) - xh * (dxh * xh).mean(1, keepdims=True))


def loss_and_grads(params, x, actions, returns):
    """(loss, mean q, [grad of every parameter]) of mse_loss(returns, Q[actions]) on the rows x, in float64."""
    params64 = [np.asarray(p, np.float64) for p in params]
    w1, b1, g1, be1, w2, b2, g2, be2, w3, b3 = params64
    q, k = forward(params64, x, keep=True)
    M = q.shape[0]
    a = np.asarray(actions).astype(np.int64)
    qa = q[np.arange(M), a]
    e = np.asarray(returns, np.float64) - qa
    loss = (e * e).mean()
    dqa = -2.0 * e / M
    dq = np.zeros_like(q)
    dq[np.arange(M), a] = dqa
    dw3, db3 = dq.T @ k["h2"], dq.sum(0)
    dy2 = (dq @ w3) * (k["y2"] > 0)
    dg2, dbe2 = (dy2 * k["xh2"]).sum(0), dy2.sum(0)
    dz2 = _ln_bwd(dy2, k["xh2"], k["r2"], g2)
    dw2, db2 = dz2.T @ k["h1"], dz2.sum(0)
    dy1 = (dz2 @ w2) * (k["y1"] > 0)
    dg1, dbe1 = (dy1 * k["xh1"]).sum(0), dy1.sum(0)
    dz1 = _ln_bwd(dy1, k["xh1"], k["r1"], g1)
    dw1, db1 = dz1.T @ k["x"], dz1.sum(0)
    return loss, qa.mean(), [dw1, db1, dg1, dbe1, dw2, db2, dg2, dbe2, dw3, db3]


def qlambda(rewards, values, dones, next_value, next_done, gamma, q_lambda):
    """pqn.py:205-218 in float32, each operation rounded as torch rounds it."""
    f = np.float32
    r, v, d = (np.asarray(t, f) for t in (rewards, values, dones))
    T = r.shape[0]
    g, ql, oml = f(gamma), f(q_lambda), f(1 - q_lambda)
    out = np.zeros_like(r)
    out[T - 1] = r[T - 1] + (g * np.asarray(next_value, f)) * (f(1.0) - np.asarray(next_done, f))
    for t in reversed(range(T - 1)):
        out[t] = r[t] + (g * ((ql * out[t + 1]) + (oml * v[t + 1]))) * (f(1.0) - d[t + 1])
    return out


def radam_scalars(step, lr, beta1=0.9, beta2=0.999):
    """(bc1, lr, bc2 ** 0.5, rect or None) in double, as _single_tensor_radam computes them."""
    step = float(step)
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    rho_inf = 2 / (1 - beta2) - 1
    rho_t = rho_inf - 2 * step * (beta2 ** step) / bc2
    rect = None
    if rho_t > 5.0:
        rect = ((rho_t - 4) * (rho_t - 2) * rho_inf / ((rho_inf - 4) * (rho_inf - 2) * rho_t)) ** 0.5
    return bc1, lr, bc2 ** 0.5, rect


def radam_step(p, g, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-8):
    """One RAdam step on float32 arrays (p, m, v updated in place)."""
    f = np.float32
    g = np.asarray(g, f)
    # exp_avg.lerp_(grad, 1 - beta1): torch's lerp for a weight < 0.5 is fma(weight, end - self, self)
    w = f(1 - beta1)
    m[...] = (np.float64(w) * (g - m).astype(np.float64) + m.astype(np.float64)).astype(f)
    v[...] = v * f(beta2)
    # exp_avg_sq.addcmul_(grad, grad, value=1 - beta2): CPU torch computes fma(value * grad, grad, self)
    v[...] = ((f(1 - beta2) * g).astype(np.float64) * g.astype(np.float64) + v.astype(np.float64)).astype(f)
    bc1, lr_, bc2s, rect = radam_scalars(step, lr, beta1, beta2)
    u = (m / f(bc1)) * f(lr_)
    if rect is None:
        p[...] = p - u
    else:
        adaptive = (f(1.0) / (np.sqrt(v) + f(eps))) * f(bc2s)
        p[...] = p - (u * adaptive) * f(rect)
    return p


def clip_coef(grads, max_norm):
    """clip_grad_norm_'s coefficient from the float64 total norm (the kernels fold the squares in double)."""
    norm = math.sqrt(sum(float((np.asarray(x, np.float64) ** 2).sum()) for x in grads))
    return norm, min(max_norm / (norm + 1e-6), 1.0)
