"""Thin torch-tensor front end over the C-ABI (device pointers + current stream).

PyTorch is plumbing here: it owns device memory and the stream; every function
below only validates arguments and enqueues libb200rl kernels on
``torch.cuda.current_stream()``.  CPU tensors are rejected loudly -- there is
no fallback path.
"""
from __future__ import annotations

import math

import torch

from . import _lib

STAT_NAMES = ("pg_loss", "v_loss", "entropy", "old_approx_kl", "approx_kl", "clipfrac", "loss",
              "adv_mean", "adv_std")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t, dtype=None, name="tensor", allow_none=False):
    if t is None:
        if allow_none:
            return None
        raise ValueError(f"{name} is None")
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"{name}: libb200rl kernels need a CUDA tensor (got {type(t).__name__} on "
                           f"{getattr(t, 'device', '?')}); there is no CPU fallback")
    if dtype is not None and t.dtype != dtype:
        raise TypeError(f"{name}: expected {dtype}, got {t.dtype}")
    return t.data_ptr()


def _contig(t, name):
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    return t


class Workspace:
    """Grow-only device scratch buffer owned by the caller side (never by the kernels)."""

    def __init__(self, device):
        self.device = device
        self.buf = None

    def get(self, nbytes):
        if self.buf is None or self.buf.numel() < nbytes:
            self.buf = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=self.device)
        return self.buf


_ws = {}


def _workspace(device, key, nbytes):
    w = _ws.setdefault((device, key), Workspace(device))
    return w.get(nbytes)


def gae(rewards, values, dones, next_value, next_done, gamma, gae_lambda, mode=0, out=None):
    """advantages, returns = GAE(...)  (reference loop: cleanrl/ppo.py:218-231)."""
    lib = _lib.load()
    T, N = rewards.shape
    for n, t in (("rewards", rewards), ("values", values), ("dones", dones)):
        _contig(t, n)
        assert t.shape == (T, N), f"{n} shape {tuple(t.shape)} != {(T, N)}"
    next_value = _contig(next_value.reshape(-1), "next_value")
    next_done = _contig(next_done.reshape(-1), "next_done")
    assert next_value.numel() == N and next_done.numel() == N
    if out is None:
        adv = torch.empty_like(rewards)
        ret = torch.empty_like(rewards)
    else:
        adv, ret = out
    f = torch.float32
    rc = lib.b200rl_gae_f32(_ptr(rewards, f, "rewards"), _ptr(values, f, "values"), _ptr(dones, f, "dones"),
                            _ptr(next_value, f, "next_value"), _ptr(next_done, f, "next_done"),
                            _ptr(adv, f, "advantages"), _ptr(ret, f, "returns"),
                            T, N, float(gamma), float(gae_lambda), int(mode), _stream())
    _lib.check(rc, "gae")
    return adv, ret


def categorical_sample(logits, noise, value_in=None, out=None):
    """action, logprob, entropy[, value] from raw logits and Exp(1) noise
    (reference: Categorical(logits).sample()/log_prob/entropy, ppo_atari_envpool.py:143-149)."""
    lib = _lib.load()
    n, A = logits.shape
    assert logits.stride(1) == 1
    _contig(noise, "noise")
    assert noise.shape == (n, A)
    dev = logits.device
    if out is None:
        action = torch.empty(n, dtype=torch.int64, device=dev)
        logprob = torch.empty(n, dtype=torch.float32, device=dev)
        entropy = torch.empty(n, dtype=torch.float32, device=dev)
        value = torch.empty(n, dtype=torch.float32, device=dev) if value_in is not None else None
    else:
        action, logprob, entropy, value = out
    f = torch.float32
    ldv = 0
    if value_in is not None:
        value_in = value_in.reshape(n, -1)
        ldv = value_in.stride(0)
    rc = lib.b200rl_categorical_sample_f32(
        _ptr(logits, f, "logits"), logits.stride(0), _ptr(noise, f, "noise"),
        _ptr(value_in, f, "value_in", True), ldv, n, A,
        _ptr(action, torch.int64, "action"), _ptr(logprob, f, "logprob"),
        _ptr(entropy, f, "entropy", True), _ptr(value, f, "value_out", True), _stream())
    _lib.check(rc, "categorical_sample")
    return action, logprob, entropy, value


def categorical_eval(logits, action):
    """logprob, entropy of given actions (reference: probs.log_prob(action), probs.entropy())."""
    lib = _lib.load()
    n, A = logits.shape
    assert logits.stride(1) == 1
    action = _contig(action.reshape(-1), "action")
    if action.dtype != torch.int64:
        action = action.long()
    f = torch.float32
    logprob = torch.empty(n, dtype=f, device=logits.device)
    entropy = torch.empty(n, dtype=f, device=logits.device)
    rc = lib.b200rl_categorical_eval_f32(_ptr(logits, f, "logits"), logits.stride(0), _ptr(action, torch.int64, "action"),
                                         n, A, _ptr(logprob, f, "logprob"), _ptr(entropy, f, "entropy"), _stream())
    _lib.check(rc, "categorical_eval")
    return logprob, entropy


def ppo_loss(new_logits, new_value, mb_inds, b_actions, b_logprobs, b_advantages, b_returns, b_values,
             clip_coef, ent_coef, vf_coef, norm_adv=True, clip_vloss=True, dlogits=None, dvalue=None, stats=None):
    """Fused PPO minibatch loss + gradients (reference: cleanrl/ppo.py:250-285).
    Returns (stats f32[16] device tensor, dlogits [M,A], dvalue [M])."""
    lib = _lib.load()
    M, A = new_logits.shape
    dev = new_logits.device
    assert new_logits.stride(1) == 1
    new_value = new_value.reshape(M, -1)
    f = torch.float32
    if dlogits is None:
        dlogits = torch.empty(M, A, dtype=f, device=dev)
    if dvalue is None:
        dvalue = torch.empty(M, dtype=f, device=dev)
    dv2 = dvalue.reshape(M, -1)
    if stats is None:
        stats = torch.zeros(16, dtype=f, device=dev)
    nbytes = lib.b200rl_ppo_loss_workspace_bytes(M)
    ws = _workspace(dev, "loss", nbytes)
    if mb_inds is not None:
        _contig(mb_inds, "mb_inds")
        assert mb_inds.numel() == M
    for n_, t in (("b_actions", b_actions), ("b_logprobs", b_logprobs), ("b_advantages", b_advantages),
                  ("b_returns", b_returns), ("b_values", b_values)):
        _contig(t, n_)
    rc = lib.b200rl_ppo_loss_f32(
        _ptr(new_logits, f, "new_logits"), new_logits.stride(0), _ptr(new_value, f, "new_value"), new_value.stride(0),
        _ptr(mb_inds, torch.int64, "mb_inds", True),
        _ptr(b_actions, torch.int64, "b_actions"), _ptr(b_logprobs, f, "b_logprobs"),
        _ptr(b_advantages, f, "b_advantages"), _ptr(b_returns, f, "b_returns"), _ptr(b_values, f, "b_values"),
        M, A, float(clip_coef), float(ent_coef), float(vf_coef), int(bool(norm_adv)), int(bool(clip_vloss)),
        _ptr(dlogits, f, "dlogits"), dlogits.stride(0), _ptr(dv2, f, "dvalue"), dv2.stride(0),
        _ptr(stats, f, "stats"), ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "ppo_loss")
    return stats, dlogits, dvalue


def clip_adam(params, grads, exp_avg, exp_avg_sq, step, lr, beta1=0.9, beta2=0.999, eps=1e-5,
              max_norm=0.5, world_size=1, norm_out=None):
    """In-place fused clip_grad_norm_ + Adam step on flat f32 vectors
    (reference: cleanrl/ppo.py:289-290; DP averaging ppo_atari_multigpu.py:369-373)."""
    lib = _lib.load()
    P = params.numel()
    f = torch.float32
    for n_, t in (("params", params), ("grads", grads), ("exp_avg", exp_avg), ("exp_avg_sq", exp_avg_sq)):
        _contig(t, n_)
        assert t.numel() == P
    nbytes = lib.b200rl_clip_adam_workspace_bytes(P)
    ws = _workspace(params.device, "adam", nbytes)
    rc = lib.b200rl_clip_adam_f32(
        _ptr(params, f, "params"), _ptr(grads, f, "grads"), _ptr(exp_avg, f, "exp_avg"),
        _ptr(exp_avg_sq, f, "exp_avg_sq"), P, int(step), float(lr), float(beta1), float(beta2), float(eps),
        -1.0 if max_norm is None else float(max_norm), int(world_size),
        _ptr(norm_out, f, "norm_out", True), ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "clip_adam")
    return params


def numpy_global_shuffle(arr):
    """``np.random.shuffle(arr)`` for a contiguous int64 vector, bit-exact (same permutation, same generator state afterwards)
    but 4-6x faster: libb200rl walks numpy's own algorithm over the global RandomState's MT19937 words.  Falls back to
    numpy itself for anything else (other dtypes / strides, a replaced bit generator)."""
    import ctypes
    import numpy as np
    if not (isinstance(arr, np.ndarray) and arr.dtype == np.int64 and arr.ndim == 1 and arr.flags.c_contiguous):
        return np.random.shuffle(arr)
    st = np.random.get_state(legacy=True)
    if st[0] != "MT19937":
        return np.random.shuffle(arr)
    key = np.ascontiguousarray(st[1], dtype=np.uint32).copy()
    pos = ctypes.c_int32(int(st[2]))
    rc = _lib.load().b200rl_mt19937_shuffle_i64(key.ctypes.data, ctypes.addressof(pos), arr.ctypes.data, arr.shape[0])
    _lib.check(rc, "mt19937_shuffle")
    np.random.set_state(("MT19937", key, int(pos.value), st[3], st[4]))


def adam_step_scalars(step, lr, beta1=0.9, beta2=0.999):
    """(sqrt(1 - beta2^step), -lr / (1 - beta1^step)) as float32, computed by the library in double as ``clip_adam`` does."""
    import ctypes
    out = (ctypes.c_float * 2)()
    _lib.check(_lib.load().b200rl_adam_step_scalars(int(step), float(lr), float(beta1), float(beta2), out), "adam_step_scalars")
    return float(out[0]), float(out[1])


def clip_adam_dyn(params, grads, exp_avg, exp_avg_sq, step_scalars, beta1=0.9, beta2=0.999, eps=1e-5, max_norm=0.5,
                  world_size=1, norm_out=None):
    """``clip_adam`` with the (step, lr)-dependent scalars in device memory (``step_scalars`` f32[2], see
    ``adam_step_scalars``): what a captured CUDA graph of the update replays."""
    lib = _lib.load()
    P = params.numel()
    f = torch.float32
    for n_, t in (("params", params), ("grads", grads), ("exp_avg", exp_avg), ("exp_avg_sq", exp_avg_sq)):
        _contig(t, n_)
        assert t.numel() == P
    assert step_scalars.numel() == 2 and step_scalars.is_contiguous()
    ws = _workspace(params.device, "adam", lib.b200rl_clip_adam_workspace_bytes(P))
    rc = lib.b200rl_clip_adam_dyn_f32(
        _ptr(params, f, "params"), _ptr(grads, f, "grads"), _ptr(exp_avg, f, "exp_avg"), _ptr(exp_avg_sq, f, "exp_avg_sq"), P,
        _ptr(step_scalars, f, "step_scalars"), float(beta1), float(beta2), float(eps),
        -1.0 if max_norm is None else float(max_norm), int(world_size), _ptr(norm_out, f, "norm_out", True),
        ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "clip_adam_dyn")
    return params


def clip_adam_ranges(params, grads, exp_avg, exp_avg_sq, step, lr, ranges, range_step, range_lr=0.0, beta1=0.9,
                     beta2=0.999, eps=1e-8, max_norm=0.5, norm_out=None):
    """``clip_adam`` with torch's per-tensor semantics for the element ranges ``ranges`` = [(lo, hi), ...] (at most 4) of
    the flat vector: ``range_step == 0`` freezes them (a tensor whose ``grad is None``: left out of the clip norm, weights
    and moments untouched), ``range_step >= 1`` updates them with their own ``(range_step, range_lr)`` while every other
    element uses ``(step, lr)`` (reference: cleanrl/ppg_procgen.py:393-394,465-466 with ``aux_critic``)."""
    import ctypes
    lib = _lib.load()
    P = params.numel()
    f = torch.float32
    for n_, t in (("params", params), ("grads", grads), ("exp_avg", exp_avg), ("exp_avg_sq", exp_avg_sq)):
        _contig(t, n_)
        assert t.numel() == P
    flat = [int(v) for r in ranges for v in r]
    arr = (ctypes.c_int64 * max(len(flat), 1))(*flat)
    ws = _workspace(params.device, "adam", lib.b200rl_clip_adam_workspace_bytes(P))
    rc = lib.b200rl_clip_adam_ranges_f32(
        _ptr(params, f, "params"), _ptr(grads, f, "grads"), _ptr(exp_avg, f, "exp_avg"), _ptr(exp_avg_sq, f, "exp_avg_sq"), P,
        int(step), float(lr), arr, len(ranges), int(range_step), float(range_lr), float(beta1), float(beta2), float(eps),
        -1.0 if max_norm is None else float(max_norm), _ptr(norm_out, f, "norm_out", True), ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "clip_adam_ranges")
    return params


def clip_adam_ranges_dyn(params, grads, exp_avg, exp_avg_sq, step_scalars, ranges, frozen=False, beta1=0.9, beta2=0.999,
                         eps=1e-8, max_norm=0.5, norm_out=None):
    """``clip_adam_ranges`` with the step-dependent scalars in device memory: ``step_scalars`` f32[4] =
    ``adam_step_scalars(step, lr) + adam_step_scalars(range_step, range_lr)``; what a captured CUDA graph replays."""
    import ctypes
    lib = _lib.load()
    P = params.numel()
    f = torch.float32
    for n_, t in (("params", params), ("grads", grads), ("exp_avg", exp_avg), ("exp_avg_sq", exp_avg_sq)):
        _contig(t, n_)
        assert t.numel() == P
    assert step_scalars.numel() == 4 and step_scalars.is_contiguous()
    flat = [int(v) for r in ranges for v in r]
    arr = (ctypes.c_int64 * max(len(flat), 1))(*flat)
    ws = _workspace(params.device, "adam", lib.b200rl_clip_adam_workspace_bytes(P))
    rc = lib.b200rl_clip_adam_ranges_dyn_f32(
        _ptr(params, f, "params"), _ptr(grads, f, "grads"), _ptr(exp_avg, f, "exp_avg"), _ptr(exp_avg_sq, f, "exp_avg_sq"), P,
        _ptr(step_scalars, f, "step_scalars"), arr, len(ranges), int(bool(frozen)), float(beta1), float(beta2), float(eps),
        -1.0 if max_norm is None else float(max_norm), _ptr(norm_out, f, "norm_out", True), ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "clip_adam_ranges_dyn")
    return params


PPG_AUX_STAT_NAMES = ("kl_loss", "aux_value_loss", "real_value_loss")


def ppg_aux_loss(head_out, rows, old_logits, returns, beta_clone, inv_accum=1.0, dhead=None, stats=None):
    """Fused auxiliary-phase loss of phasic policy gradient + its gradient (reference: cleanrl/ppg_procgen.py:449-461).
    ``head_out`` [n, A + 2] = [logits | value | aux_value]; row i is compared with ``old_logits[rows[i]]`` [*, A] and
    ``returns[rows[i]]``.  ``rows`` must index inside ``old_logits`` / ``returns``: the kernel does not check them.
    Returns (stats f32[>= 3]: kl_loss, aux_value_loss, real_value_loss; dhead [n, A + 2])."""
    lib = _lib.load()
    n, A2 = head_out.shape
    A = A2 - 2
    dev = head_out.device
    f = torch.float32
    assert head_out.stride(1) == 1
    if dhead is None:
        dhead = torch.empty(n, A2, dtype=f, device=dev)
    assert dhead.shape == (n, A2) and dhead.stride(1) == 1
    if stats is None:
        stats = torch.zeros(4, dtype=f, device=dev)
    old_logits = _contig(old_logits, "old_logits").view(-1, old_logits.shape[-1])
    returns = _contig(returns, "returns").view(-1)
    assert old_logits.shape[1] == A and old_logits.shape[0] == returns.numel()
    if rows is not None:
        _contig(rows, "rows")
        assert rows.numel() == n
    else:
        assert returns.numel() == n
    ws = _workspace(dev, "ppg_aux", lib.b200rl_ppg_aux_loss_workspace_bytes(n))
    rc = lib.b200rl_ppg_aux_loss_f32(
        _ptr(head_out, f, "head_out"), head_out.stride(0), _ptr(rows, torch.int64, "rows", True),
        _ptr(old_logits, f, "old_logits"), _ptr(returns, f, "returns"), n, A, float(beta_clone), float(inv_accum),
        _ptr(dhead, f, "dhead"), dhead.stride(0), _ptr(stats, f, "stats"), ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "ppg_aux_loss")
    return stats, dhead


# ----------------------------------------------------------------- fp32 layers
ACT = {None: 0, "none": 0, "relu": 1, "tanh": 2}


def _xdtype(x):
    if x.dtype == torch.uint8:
        return 1
    if x.dtype == torch.float32:
        return 0
    raise TypeError(f"unsupported input dtype {x.dtype} (need uint8 or float32)")


def conv2d_fwd(x, w, b, stride, act, rows=None, in_div=1.0, out=None, pad=0):
    """y = act(conv2d(x / in_div, w, padding=pad) + b), NCHW (reference: nn.Conv2d + ReLU, ppo_atari_envpool.py:126-132;
    padded 3x3: ppo_procgen.py:92-93).  ``rows`` (int64) gathers the batch dimension of x without materialising it (ppo.py:250)."""
    lib = _lib.load()
    _contig(x, "x"); _contig(w, "w")
    Cout, Cin, KH, KW = w.shape
    H, W = x.shape[-2:]
    assert x.shape[-3] == Cin
    n = rows.numel() if rows is not None else x.shape[0]
    OH, OW = (H + 2 * pad - KH) // stride + 1, (W + 2 * pad - KW) // stride + 1
    if out is None:
        out = torch.empty(n, Cout, OH, OW, dtype=torch.float32, device=x.device)
    rc = lib.b200rl_conv2d_fwd_pad_f32(_ptr(x, None, "x"), _xdtype(x), _ptr(rows, torch.int64, "rows", True), float(in_div),
                                       _ptr(w, torch.float32, "w"), _ptr(b, torch.float32, "b", True),
                                       _ptr(out, torch.float32, "y"), n, Cin, H, W, Cout, KH, KW, stride, int(pad), ACT[act], _stream())
    _lib.check(rc, "conv2d_fwd")
    return out


def conv2d_bwd_data(dy, w, x_post, prev_act, stride, out=None, pad=0, in_hw=None):
    """dx of the convolution; ``x_post`` / ``prev_act`` fold the derivative of the activation that produced the layer
    input (``prev_act=None``: pass ``in_hw=(H, W)`` instead of ``x_post``)."""
    lib = _lib.load()
    _contig(dy, "dy"); _contig(w, "w")
    Cout, Cin, KH, KW = w.shape
    n = dy.shape[0]
    H, W = x_post.shape[-2:] if x_post is not None else in_hw
    if out is None:
        out = torch.empty(n, Cin, H, W, dtype=torch.float32, device=dy.device)
    rc = lib.b200rl_conv2d_bwd_data_pad_f32(_ptr(dy, torch.float32, "dy"), _ptr(w, torch.float32, "w"),
                                            _ptr(x_post, torch.float32, "x_post", True), ACT[prev_act] if x_post is not None else 0,
                                            _ptr(out, torch.float32, "dx"), n, Cin, H, W, Cout, KH, KW, stride, int(pad), _stream())
    _lib.check(rc, "conv2d_bwd_data")
    return out


def conv2d_bwd_weight(x, dy, dw, db, stride, rows=None, in_div=1.0, pad=0):
    lib = _lib.load()
    _contig(x, "x"); _contig(dy, "dy"); _contig(dw, "dw")
    Cout, Cin, KH, KW = dw.shape
    H, W = x.shape[-2:]
    n = dy.shape[0]
    nbytes = lib.b200rl_conv2d_bwd_weight_pad_workspace_bytes(n, Cin, H, W, Cout, KH, KW, stride, int(pad))
    ws = _workspace(x.device, "wgrad", nbytes)
    rc = lib.b200rl_conv2d_bwd_weight_pad_f32(_ptr(x, None, "x"), _xdtype(x), _ptr(rows, torch.int64, "rows", True),
                                              float(in_div), _ptr(dy, torch.float32, "dy"), _ptr(dw, torch.float32, "dw"),
                                              _ptr(db, torch.float32, "db", True), n, Cin, H, W, Cout, KH, KW, stride, int(pad),
                                              ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "conv2d_bwd_weight")


def linear_fwd(x, w, b, act, rows=None, out=None):
    """y = act(x @ w.T + b) (reference: nn.Linear + activation)."""
    lib = _lib.load()
    _contig(x, "x"); _contig(w, "w")
    out_f, in_f = w.shape
    x2 = x.reshape(x.shape[0], -1)
    assert x2.shape[1] == in_f, f"linear_fwd: x has {x2.shape[1]} features, w expects {in_f}"
    n = rows.numel() if rows is not None else x2.shape[0]
    if out is None:
        out = torch.empty(n, out_f, dtype=torch.float32, device=x.device)
    rc = lib.b200rl_linear_fwd_f32(_ptr(x2, torch.float32, "x"), _ptr(rows, torch.int64, "rows", True),
                                   _ptr(w, torch.float32, "w"), _ptr(b, torch.float32, "b", True),
                                   _ptr(out, torch.float32, "y"), n, in_f, out_f, ACT[act], _stream())
    _lib.check(rc, "linear_fwd")
    return out


def linear_bwd_data(dy, w, x_post, prev_act, out=None):
    lib = _lib.load()
    _contig(dy, "dy"); _contig(w, "w")
    out_f, in_f = w.shape
    n = dy.shape[0]
    if out is None:
        out = torch.empty(n, in_f, dtype=torch.float32, device=dy.device)
    rc = lib.b200rl_linear_bwd_data_f32(_ptr(dy, torch.float32, "dy"), _ptr(w, torch.float32, "w"),
                                        _ptr(x_post, torch.float32, "x_post", True), ACT[prev_act],
                                        _ptr(out, torch.float32, "dx"), n, in_f, out_f, _stream())
    _lib.check(rc, "linear_bwd_data")
    return out


def linear_bwd_weight(x, dy, dw, db, rows=None):
    lib = _lib.load()
    _contig(x, "x"); _contig(dy, "dy"); _contig(dw, "dw")
    out_f, in_f = dw.shape
    n = dy.shape[0]
    nbytes = lib.b200rl_linear_bwd_weight_workspace_bytes(n, in_f, out_f)
    ws = _workspace(x.device, "wgrad", nbytes)
    rc = lib.b200rl_linear_bwd_weight_f32(_ptr(x, torch.float32, "x"), _ptr(rows, torch.int64, "rows", True),
                                          _ptr(dy, torch.float32, "dy"), _ptr(dw, torch.float32, "dw"),
                                          _ptr(db, torch.float32, "db", True), n, in_f, out_f,
                                          ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "linear_bwd_weight")


# ------------------------------------------------------------------ IMPALA-CNN glue
def maxpool3s2_fwd(x):
    """max_pool2d(x, kernel_size=3, stride=2, padding=1) on NCHW fp32 (ppo_procgen.py:113); returns (y, argmax u8)."""
    lib = _lib.load()
    _contig(x, "x")
    n, C, H, W = x.shape
    y = torch.empty(n, C, (H + 1) // 2, (W + 1) // 2, dtype=torch.float32, device=x.device)
    arg = torch.empty(y.shape, dtype=torch.uint8, device=x.device)
    _lib.check(lib.b200rl_maxpool3s2_fwd_f32(_ptr(x, torch.float32, "x"), n * C, H, W, _ptr(y, torch.float32, "y"),
                                             _ptr(arg, torch.uint8, "argmax"), _stream()), "maxpool_fwd")
    return y, arg


def maxpool3s2_bwd(dy, arg, in_hw):
    lib = _lib.load()
    _contig(dy, "dy")
    n, C = dy.shape[:2]
    H, W = in_hw
    dx = torch.empty(n, C, H, W, dtype=torch.float32, device=dy.device)
    _lib.check(lib.b200rl_maxpool3s2_bwd_f32(_ptr(dy, torch.float32, "dy"), _ptr(arg, torch.uint8, "argmax"), n * C, H, W,
                                             _ptr(dx, torch.float32, "dx"), _stream()), "maxpool_bwd")
    return dx


def relu(x):
    lib = _lib.load()
    y = torch.empty_like(_contig(x, "x"))
    _lib.check(lib.b200rl_relu_f32(_ptr(x, torch.float32, "x"), x.numel(), _ptr(y, torch.float32, "y"), _stream()), "relu")
    return y


def relu_bwd(dy, x, extra=None):
    """dx = dy * (x > 0) [+ extra]."""
    lib = _lib.load()
    dx = torch.empty_like(_contig(dy, "dy"))
    _lib.check(lib.b200rl_relu_bwd_f32(_ptr(dy, torch.float32, "dy"), _ptr(_contig(x, "x"), torch.float32, "x"),
                                       _ptr(extra, torch.float32, "extra", True), dy.numel(), _ptr(dx, torch.float32, "dx"),
                                       _stream()), "relu_bwd")
    return dx


def add(a, b):
    lib = _lib.load()
    y = torch.empty_like(_contig(a, "a"))
    _lib.check(lib.b200rl_add_f32(_ptr(a, torch.float32, "a"), _ptr(_contig(b, "b"), torch.float32, "b"), a.numel(),
                                  _ptr(y, torch.float32, "y"), _stream()), "add")
    return y


def nhwc_to_nchw_u8(x, rows=None):
    """uint8 frames [*, H, W, C] (optionally gathered through int64 ``rows``) -> [n, C, H, W] (ppo_procgen.py:143 permute)."""
    lib = _lib.load()
    _contig(x, "x")
    H, W, C = x.shape[-3:]
    n = rows.numel() if rows is not None else x.shape[0]
    y = torch.empty(n, C, H, W, dtype=torch.uint8, device=x.device)
    _lib.check(lib.b200rl_nhwc_to_nchw_u8(_ptr(x, torch.uint8, "x"), _ptr(rows, torch.int64, "rows", True), n, H, W, C,
                                          _ptr(y, torch.uint8, "y"), _stream()), "nhwc_to_nchw")
    return y


# ------------------------------------------------------------------------ LSTM cell
def lstm_mask_state(h, c, done, out=None):
    """(h', c') = (1 - done) * (h, c): the state reset of cleanrl/ppo_atari_lstm.py:137-142, [n, H] fp32."""
    lib = _lib.load()
    n, H = h.shape
    f = torch.float32
    hm, cm = out if out is not None else (torch.empty_like(h), torch.empty_like(c))
    rc = lib.b200rl_lstm_mask_state_f32(_ptr(_contig(h, "h"), f, "h"), _ptr(_contig(c, "c"), f, "c"),
                                        _ptr(_contig(done, "done"), f, "done"), n, H, _ptr(hm, f, "hm"), _ptr(cm, f, "cm"), _stream())
    _lib.check(rc, "lstm_mask_state")
    return hm, cm


def lstm_cell_fwd(gates_x, gates_h, c_masked, h_out, c_out, save=None):
    """One LSTM step from the two gate GEMMs (gate order i, f, g, o); ``save`` [n, 5H] keeps what the backward needs."""
    lib = _lib.load()
    n, H = c_masked.shape
    f = torch.float32
    for nm, t in (("gates_x", gates_x), ("gates_h", gates_h), ("c_masked", c_masked), ("h_out", h_out), ("c_out", c_out)):
        _contig(t, nm)
    assert gates_x.shape == (n, 4 * H) and gates_h.shape == (n, 4 * H)
    rc = lib.b200rl_lstm_cell_fwd_f32(_ptr(gates_x, f, "gates_x"), _ptr(gates_h, f, "gates_h"), _ptr(c_masked, f, "c_masked"), n, H,
                                      _ptr(h_out, f, "h_out"), _ptr(c_out, f, "c_out"), _ptr(save, f, "save", True), _stream())
    _lib.check(rc, "lstm_cell_fwd")


def lstm_cell_bwd(dh_heads, dh_rec_raw, done_next, dc_rec, save, c_masked, done, dgates, dc_rec_out):
    """One step of back-propagation through time (see include/b200rl.h)."""
    lib = _lib.load()
    n, H = c_masked.shape
    f = torch.float32
    for nm, t in (("dh_heads", dh_heads), ("save", save), ("c_masked", c_masked), ("done", done), ("dgates", dgates),
                  ("dc_rec_out", dc_rec_out)):
        _contig(t, nm)
    rc = lib.b200rl_lstm_cell_bwd_f32(_ptr(dh_heads, f, "dh_heads"), _ptr(dh_rec_raw, f, "dh_rec_raw", True),
                                      _ptr(done_next, f, "done_next", True), _ptr(dc_rec, f, "dc_rec", True), _ptr(save, f, "save"),
                                      _ptr(c_masked, f, "c_masked"), _ptr(done, f, "done"), n, H, _ptr(dgates, f, "dgates"),
                                      _ptr(dc_rec_out, f, "dc_rec_out"), _stream())
    _lib.check(rc, "lstm_cell_bwd")


# ------------------------------------------------------ tensor-core (bf16) network plans
class _TensorCorePlan:
    """Owns the device memory of one tensor-core network: the packed bf16 weights, the activation workspaces (one per
    batch shape) and the grow-only backward workspace.  Subclasses name their C entry points by ``NET``
    (``b200rl_<NET>_param_count``, ``b200rl_<NET>_bf16_{packed_bytes,pack,acts_bytes,acts_layout,workspace_bytes}``)
    and marshal the arguments of their forward / backward calls.

    A captured CUDA graph (and the CUtensorMaps baked into it) holds raw device pointers into these workspaces, so
    ``pin()`` runs after every capture: each workspace that exists at that moment then lives as long as the plan, whether
    it is an activation workspace of a batch shape or a backward workspace superseded by a larger one."""

    NET = NAME = None
    MAX_A = 23               # widest supported action space
    MAX_UNPINNED = 4         # activation workspaces kept for batch shapes that no captured graph references

    def __init__(self, A, device):
        self.A, self.device = int(A), device
        nbytes = self._c("packed_bytes")(self.A)
        if nbytes == 0:
            raise ValueError(f"{self.NAME} supports 1 <= A <= {self.MAX_A} actions (got {A})")
        self.param_count = getattr(_lib.load(), f"b200rl_{self.NET}_param_count")(self.A)
        self.packed = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self._acts = {}          # batch shape -> activation workspace, least-recently-used first
        self._pinned = set()     # batch shapes referenced by captured CUDA graphs: never evicted
        self._ws = None          # backward workspace (grow-only)
        self._pinned_ws = []     # backward workspaces referenced by captured CUDA graphs

    def _c(self, name):
        return getattr(_lib.load(), f"b200rl_{self.NET}_bf16_{name}")

    def pin(self):
        """Every workspace that exists now may be referenced by a captured CUDA graph: keep it alive."""
        self._pinned.update(self._acts)
        if self._ws is not None and all(w is not self._ws for w in self._pinned_ws):
            self._pinned_ws.append(self._ws)

    def acts(self, *shape):
        """The activation workspace of one batch shape, least recently used ones evicted unless pinned."""
        key = tuple(int(d) for d in shape)
        buf = self._acts.pop(key, None)
        if buf is None:
            unpinned = [k for k in self._acts if k not in self._pinned]
            while len(unpinned) >= self.MAX_UNPINNED:
                del self._acts[unpinned.pop(0)]
            nbytes = self._c("acts_bytes")(*key)
            if nbytes == 0:
                raise ValueError(f"{self.NAME}: batch shape {key} is out of range")
            # zero-initialised: the padded-grid gradient buffers rely on never-written positions being 0
            buf = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        self._acts[key] = buf    # most recently used = last
        return buf

    def _named_views(self, shape, specs):
        """``{name: view}`` of the activation workspace ``acts(*shape)``; ``specs`` lists ``(name, dtype, shape)`` in the
        order of the C layout table, whose negative offsets mark tensors the layout does not have."""
        import ctypes
        off = (ctypes.c_int64 * len(specs))()
        _lib.check(self._c("acts_layout")(*shape, off), f"{self.NET}_acts_layout")
        buf = self.acts(*shape)
        return {name: buf[o:o + math.prod(dims) * dtype.itemsize].view(dtype).view(*dims)
                for o, (name, dtype, dims) in zip(off, specs) if o >= 0}

    def workspace(self, *shape):
        """The backward workspace for one batch shape: grows, never shrinks."""
        nbytes = self._c("workspace_bytes")(*shape, self.A)
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        return self._ws

    def pack(self, flat_params):
        rc = self._c("pack")(_ptr(flat_params, torch.float32, "params"), self.A, self.packed.data_ptr(), _stream())
        _lib.check(rc, f"{self.NET}_bf16_pack")


class NatureCNNBf16(_TensorCorePlan):
    """The tensor-core NatureCNN; its activation workspaces are keyed by (n, obs format)."""

    NET, NAME, MAX_A = "naturecnn", "tensor-core NatureCNN", 2047

    @staticmethod
    def obs_format(obs):
        if obs.dtype == torch.uint8 and obs.dim() >= 4 and tuple(obs.shape[-3:]) == (4, 84, 84):
            return 0
        if obs.dtype == torch.bfloat16 and tuple(obs.shape[-3:]) == (21, 21, 64):
            return 1
        if obs.dtype == torch.uint8 and tuple(obs.shape[-2:]) == (441, 64):
            return 2
        raise TypeError("tensor-core NatureCNN path consumes uint8 [*,4,84,84] frames, uint8 space-to-depth rollout rows "
                        f"[*,441,64] or space-to-depth bf16 [*,21,21,64] (got {obs.dtype} {tuple(obs.shape)})")

    def forward(self, obs, rows, flat_params, head_out=None):
        lib = _lib.load()
        fmt = self.obs_format(obs)
        _contig(obs, "obs")
        n = rows.numel() if rows is not None else obs.shape[0]
        if head_out is None:
            head_out = torch.empty(n, self.A + 1, dtype=torch.float32, device=self.device)
        rc = lib.b200rl_naturecnn_bf16_forward(_ptr(obs, None, "obs"), fmt, _ptr(rows, torch.int64, "rows", True), n, self.A,
                                               _ptr(flat_params, torch.float32, "params"), self.packed.data_ptr(),
                                               self.acts(n, fmt).data_ptr(), _ptr(head_out, torch.float32, "head_out"), _stream())
        _lib.check(rc, "naturecnn_bf16_forward")
        return head_out

    def grad_tail_offset(self):
        """Element offset from which the flat gradient (fc + heads, 95 % of it) is final when ``tail_event`` fires."""
        return int(_lib.load().b200rl_naturecnn_grad_tail_offset(self.A))

    def backward(self, obs, rows, flat_params, dhead, flat_grads, tail_event=None, obs_aux=None):
        """``obs_aux``: the channel-major uint8 copy [*,64,448] of a uint8 space-to-depth rollout (format 2)."""
        lib = _lib.load()
        fmt = self.obs_format(obs)
        if fmt == 2:
            if obs_aux is None or obs_aux.dtype != torch.uint8 or tuple(obs_aux.shape[-2:]) != (64, 448) or \
                    obs_aux.shape[0] != obs.shape[0]:
                raise ValueError("uint8 rollout rows need their channel-major copy [*,64,448] (obs_aux) for the backward pass")
            _contig(obs_aux, "obs_aux")
        n = dhead.shape[0]
        _contig(dhead, "dhead")
        ws = self.workspace(n)
        rc = lib.b200rl_naturecnn_bf16_backward(_ptr(obs, None, "obs"), _ptr(obs_aux, None, "obs_aux", True), fmt,
                                                _ptr(rows, torch.int64, "rows", True), n, self.A,
                                                _ptr(flat_params, torch.float32, "params"), self.packed.data_ptr(),
                                                self.acts(n, fmt).data_ptr(), _ptr(dhead, torch.float32, "dhead"),
                                                _ptr(flat_grads, torch.float32, "grads"), ws.data_ptr(), ws.numel(),
                                                tail_event.cuda_event if tail_event is not None else None, _stream())
        _lib.check(rc, "naturecnn_bf16_backward")


class ImpalaCNNBf16(_TensorCorePlan):
    """The tensor-core IMPALA-CNN (procgen frames uint8 [*, 64, 64, 3]); its activation workspaces are keyed by n."""

    NET, NAME = "impala", "tensor-core IMPALA-CNN"
    VALUE_HEADS = 1          # head outputs = A + VALUE_HEADS

    def act_tensors(self, n):
        """Named views of the activation workspace of batch size ``n`` (layout: b200rl_impala_bf16_acts_layout)."""
        bf, u8, i32 = torch.bfloat16, torch.uint8, torch.int32
        specs = [("c0", bf, (n, 64, 64, 16)), ("c1", bf, (n, 32, 32, 32)), ("c2", bf, (n, 16, 16, 32))]
        for q, shp in enumerate(((n, 32, 32, 16), (n, 16, 16, 32), (n, 8, 8, 32))):
            specs += [(f"{name}_{q}", bf, shp) for name in ("s0", "s1", "s2", "y0", "y1")] + [(f"arg_{q}", u8, shp)]
        specs += [("h0", bf, (n, 2048)), ("mh0", i32, (n, 64)), ("hid", bf, (n, 256)), ("mhid", i32, (n, 8)),
                  ("dc", bf, (n, 65536)), ("ga", bf, (n, 16384)), ("gb", bf, (n, 16384)), ("gy", bf, (n, 16384)),
                  ("dhid", bf, (n, 256))]
        return self._named_views((n,), specs)

    @staticmethod
    def check_obs(obs):
        if obs.dtype != torch.uint8 or obs.dim() < 4 or tuple(obs.shape[-3:]) != (64, 64, 3):
            raise ValueError("tensor-core IMPALA-CNN consumes uint8 frames [*, 64, 64, 3] "
                             f"(got {obs.dtype} {tuple(obs.shape)})")

    def forward(self, obs, rows, flat_params, head_out=None):
        self.check_obs(obs)
        _contig(obs, "obs")
        n = rows.numel() if rows is not None else obs.shape[0]
        if rows is not None:
            _contig(rows, "rows")
        if head_out is None:
            head_out = torch.empty(n, self.A + self.VALUE_HEADS, dtype=torch.float32, device=self.device)
        rc = self._c("forward")(_ptr(obs, torch.uint8, "obs"), _ptr(rows, torch.int64, "rows", True), n,
                                self.A, _ptr(flat_params, torch.float32, "params"), self.packed.data_ptr(),
                                self.acts(n).data_ptr(), _ptr(head_out, torch.float32, "head_out"), _stream())
        _lib.check(rc, f"{self.NET}_bf16_forward")
        return head_out

    def backward(self, obs, rows, flat_params, dhead, flat_grads):
        """Gradient of the forward that last ran on (obs, rows) with this batch size; fills ``flat_grads``."""
        self.check_obs(obs)
        _contig(dhead, "dhead")
        n = dhead.shape[0]
        ws = self.workspace(n)
        rc = self._c("backward")(_ptr(obs, torch.uint8, "obs"), _ptr(rows, torch.int64, "rows", True), n,
                                 self.A, _ptr(flat_params, torch.float32, "params"), self.packed.data_ptr(),
                                 self.acts(n).data_ptr(), _ptr(dhead, torch.float32, "dhead"),
                                 _ptr(flat_grads, torch.float32, "grads"), ws.data_ptr(), ws.numel(), _stream())
        _lib.check(rc, f"{self.NET}_bf16_backward")


class ImpalaPPGBf16(ImpalaCNNBf16):
    """The tensor-core IMPALA-CNN of phasic policy gradient (cleanrl/ppg_procgen.py:168-211): the same trunk and activation
    workspace with the joint head [logits | value | aux_value] (A + 2 outputs); ``backward`` keeps the ``value`` column of
    ``dhead`` out of the hidden layer's gradient (``critic`` reads ``hidden.detach()``)."""

    NET, NAME, MAX_A, VALUE_HEADS = "impala_ppg", "tensor-core IMPALA-CNN (PPG heads)", 22, 2

    def _c(self, name):
        # the activation workspace does not depend on the heads: the IMPALA plan's layout serves both
        return super()._c(name) if not name.startswith("acts_") else getattr(_lib.load(), f"b200rl_impala_bf16_{name}")


class LSTMAgentBf16(_TensorCorePlan):
    """The tensor-core recurrent agent (single uint8 frames [*, 1, 84, 84], NatureCNN trunk, LSTM(512, 128), heads).
    Sequences are S steps x n envs, time-major; the activation workspaces are keyed by (S, n)."""

    NET, NAME = "lstm_agent", "tensor-core LSTM agent"
    H = 128

    def act_tensors(self, S, n):
        """Named views of the activation workspace of (S, n) (layout: b200rl_lstm_agent_bf16_acts_layout)."""
        M = S * n
        bf, f32, i32 = torch.bfloat16, torch.float32, torch.int32
        return self._named_views((S, n), [
            ("act1", bf, (M, 10, 10, 128)), ("m1", i32, (M, 400)), ("act2", bf, (M, 9, 9, 64)), ("act3", bf, (M, 7, 7, 64)),
            ("feats", bf, (M, 512)), ("m4", i32, (M, 16)),
            ("gx", f32, (M, 512)), ("hseq", bf, (M, 128)), ("hm", bf, (M, 128)), ("save", f32, (M, 5, 128)),
            ("cm", f32, (M, 128)), ("dgates", f32, (M, 512)), ("dfeats", bf, (M, 512))])

    @staticmethod
    def check_obs(obs):
        if obs.dtype != torch.uint8 or obs.dim() != 4 or tuple(obs.shape[-3:]) != (1, 84, 84):
            raise ValueError("tensor-core LSTM agent consumes uint8 frames [*, 1, 84, 84] "
                             f"(got {obs.dtype} {tuple(obs.shape)})")

    def forward(self, obs, rows, S, n, flat_params, h0, c0, done, head_out=None, h_out=None, c_out=None):
        """(head_out [S*n, A+1], h_S [n, 128], c_S [n, 128]); the sequence's activations stay in the workspace."""
        self.check_obs(obs)
        _contig(obs, "obs")
        f = torch.float32
        M = S * n
        if rows is not None:
            _contig(rows, "rows")
            if rows.numel() != M:
                raise ValueError(f"rows has {rows.numel()} entries for {S} steps x {n} envs")
        elif obs.shape[0] != M:
            raise ValueError(f"obs has {obs.shape[0]} frames for {S} steps x {n} envs")
        for nm, t, shape in (("h0", h0, (n, self.H)), ("c0", c0, (n, self.H)), ("done", done, (M,))):
            _contig(t, nm)
            if tuple(t.shape) != shape:
                raise ValueError(f"{nm}: expected shape {shape}, got {tuple(t.shape)}")
        if head_out is None:
            head_out = torch.empty(M, self.A + 1, dtype=f, device=self.device)
        if h_out is None:
            h_out = torch.empty(n, self.H, dtype=f, device=self.device)
        if c_out is None:
            c_out = torch.empty(n, self.H, dtype=f, device=self.device)
        rc = _lib.load().b200rl_lstm_agent_bf16_forward(
            _ptr(obs, torch.uint8, "obs"), _ptr(rows, torch.int64, "rows", True), S, n, self.A,
            _ptr(flat_params, f, "params"), self.packed.data_ptr(), _ptr(h0, f, "h0"), _ptr(c0, f, "c0"),
            _ptr(done, f, "done"), self.acts(S, n).data_ptr(), _ptr(head_out, f, "head_out"), _ptr(h_out, f, "h_out"),
            _ptr(c_out, f, "c_out"), _stream())
        _lib.check(rc, "lstm_agent_bf16_forward")
        return head_out, h_out, c_out

    def backward(self, obs, rows, S, n, flat_params, done, dhead, flat_grads):
        """Gradient of the forward that last ran on (obs, rows, S, n, done); fills ``flat_grads``."""
        self.check_obs(obs)
        _contig(dhead, "dhead")
        ws = self.workspace(S, n)
        f = torch.float32
        rc = _lib.load().b200rl_lstm_agent_bf16_backward(
            _ptr(obs, torch.uint8, "obs"), _ptr(rows, torch.int64, "rows", True), S, n, self.A,
            _ptr(flat_params, f, "params"), self.packed.data_ptr(), _ptr(done, f, "done"), self.acts(S, n).data_ptr(),
            _ptr(dhead, f, "dhead"), _ptr(flat_grads, f, "grads"), ws.data_ptr(), ws.numel(), _stream())
        _lib.check(rc, "lstm_agent_bf16_backward")


def frames_to_s2d(obs_u8, out=None, rows=None):
    """uint8 [n,4,84,84] frames -> bf16 [n,21,21,64] space-to-depth frames (once per env step)."""
    lib = _lib.load()
    _contig(obs_u8, "obs")
    n = rows.numel() if rows is not None else obs_u8.shape[0]
    if out is None:
        out = torch.empty(n, 21, 21, 64, dtype=torch.bfloat16, device=obs_u8.device)
    rc = lib.b200rl_frames_to_s2d_bf16(_ptr(obs_u8, torch.uint8, "obs"), _ptr(rows, torch.int64, "rows", True), n,
                                       _ptr(out, torch.bfloat16, "out"), _stream())
    _lib.check(rc, "frames_to_s2d")
    return out


def alloc_u8_rollout_rows(shape, device):
    """uint8 row-major rollout rows [..., 441, 64] with 256 bytes of slack behind the last frame: conv1 reads a frame as
    221 rows of 128 bytes (pairs of grid positions), and the second half of the last pair row lies 64 bytes past the frame."""
    n = 1
    for d in shape:
        n *= int(d)
    flat = torch.zeros(n + 256, dtype=torch.uint8, device=device)
    return flat[:n].view(*shape)


def frames_to_s2d_u8(obs_u8, out_rm=None, out_cm=None, rows=None):
    """uint8 [n,4,84,84] frames -> uint8 space-to-depth rollout rows: row-major [n,441,64] (conv1 forward on the integer
    tensor cores) and channel-major [n,64,448] (conv1 weight gradient); once per env step, 1 byte per pixel each."""
    lib = _lib.load()
    _contig(obs_u8, "obs")
    n = rows.numel() if rows is not None else obs_u8.shape[0]
    if out_rm is None:
        out_rm = alloc_u8_rollout_rows((n, 441, 64), obs_u8.device)
    if out_cm is None:
        out_cm = torch.empty(n, 64, 448, dtype=torch.uint8, device=obs_u8.device)
    _contig(out_rm, "out_rm"); _contig(out_cm, "out_cm")
    assert out_rm.shape[0] == n and out_cm.shape[0] == n
    rc = lib.b200rl_frames_to_s2d_u8(_ptr(obs_u8, torch.uint8, "obs"), _ptr(rows, torch.int64, "rows", True), n,
                                     _ptr(out_rm, torch.uint8, "out_rm"), _ptr(out_cm, torch.uint8, "out_cm"), _stream())
    _lib.check(rc, "frames_to_s2d_u8")
    return out_rm, out_cm


def frames_delta_s2d_u8(new_planes, prev_rm, prev_cm, out_rm, out_cm, full_slot=None, full_frames=None):
    """Rollout slot t from slot t-1 and the newest frame plane of every env (frame-stack delta upload, csrc/frame_stack.cu):
    ``new_planes`` u8 [n,7056]; envs with ``full_slot[i] = k >= 0`` take all four planes from ``full_frames[k]`` instead."""
    lib = _lib.load()
    n = new_planes.shape[0]
    for nm, t in (("new_planes", new_planes), ("prev_rm", prev_rm), ("prev_cm", prev_cm), ("out_rm", out_rm), ("out_cm", out_cm)):
        _contig(t, nm)
        assert t.shape[0] == n, nm
    if full_slot is not None:
        _contig(full_slot, "full_slot"); _contig(full_frames, "full_frames")
        assert full_slot.shape[0] == n
    rc = lib.b200rl_frames_delta_s2d_u8(_ptr(new_planes, torch.uint8, "new_planes"), _ptr(full_slot, torch.int32, "full_slot", True),
                                        _ptr(full_frames, torch.uint8, "full_frames", True), _ptr(prev_rm, torch.uint8, "prev_rm"),
                                        _ptr(prev_cm, torch.uint8, "prev_cm"), n, _ptr(out_rm, torch.uint8, "out_rm"),
                                        _ptr(out_cm, torch.uint8, "out_cm"), _stream())
    _lib.check(rc, "frames_delta_s2d_u8")


def h2d_rows_async(dst, src_ptr, src_pitch, row_bytes, rows, stream=None):
    """``rows`` rows of ``row_bytes`` from pitched host memory at address ``src_ptr`` into the dense device tensor ``dst``."""
    lib = _lib.load()
    assert dst.is_contiguous() and dst.numel() * dst.element_size() >= rows * row_bytes
    rc = lib.b200rl_h2d_rows_async(dst.data_ptr(), src_ptr, src_pitch, row_bytes, rows,
                                   stream.cuda_stream if stream is not None else _stream())
    _lib.check(rc, "h2d_rows_async")


class StackDeltaTracker:
    """Host side of the frame-stack delta upload for one vector env of ``n`` envs (b200rl_stackdelta_*): private mirror of
    every env's last observation + worker threads that verify, off the critical path, that the newest observation really
    is the previous one shifted by a plane for every env not flagged done."""

    def __init__(self, n, planes=4, plane_bytes=7056, threads=None, pinned=True):
        lib = _lib.load()
        if threads is None:
            import os
            ranks = max(1, int(os.environ.get("LOCAL_WORLD_SIZE", "1")))        # one process per GPU shares the host cores
            threads = int(os.environ.get("CLEANRL_B200_HOST_THREADS", min(8, max(2, (os.cpu_count() or 2) // (4 * ranks)))))
        self.n, self.planes, self.plane_bytes, self.threads = int(n), int(planes), int(plane_bytes), int(threads)
        self._h = lib.b200rl_stackdelta_create(self.n, self.planes, self.plane_bytes, int(threads))
        if not self._h:
            _lib.check(-1, "stackdelta_create")
        pin = pinned and torch.cuda.is_available()
        mk = lambda shape, dt: (torch.zeros(shape, dtype=dt).pin_memory() if pin else torch.zeros(shape, dtype=dt))
        self.new_h = mk((self.n, self.plane_bytes), torch.uint8)
        self.full_h = mk((self.n, self.planes * self.plane_bytes), torch.uint8)
        self.slot_h = mk((self.n,), torch.int32)
        self.mis_h = torch.zeros(self.n, dtype=torch.int32)
        self._pending = False

    def begin(self, obs, done=None, pack_new=True):
        """obs: uint8 ndarray [n, planes, ...] whose planes are contiguous per env (any env stride).  Returns the number of
        envs staged as full frames; ``slot_h`` / ``full_h`` (and ``new_h`` when ``pack_new``) are filled on return."""
        lib = _lib.load()
        assert obs.dtype.name == "uint8" and obs.shape[0] == self.n
        itemsz = self.planes * self.plane_bytes
        inner = 1
        for d, st in zip(obs.shape[:0:-1], obs.strides[:0:-1]):
            assert st == inner, "observation planes must be contiguous per env"
            inner *= d
        assert inner == itemsz, "observation size does not match the tracker geometry"
        d32 = None
        if done is not None:
            import numpy as np
            d32 = np.ascontiguousarray(done, dtype=np.float32).reshape(-1)
            assert d32.shape[0] == self.n
        self._keep = (obs, d32)                                  # the workers read these until wait()
        k = lib.b200rl_stackdelta_begin(self._h, obs.__array_interface__["data"][0], int(obs.strides[0]),
                                        d32.__array_interface__["data"][0] if d32 is not None else None,
                                        self.new_h.data_ptr() if pack_new else None, self.full_h.data_ptr(), self.slot_h.data_ptr())
        if k < 0:
            _lib.check(int(k), "stackdelta_begin")
        self._pending = True
        return int(k)

    def wait(self):
        """Join the verification; returns the (ascending) indices of envs that were NOT a shifted stack although not done."""
        if not self._pending:
            return self.mis_h[:0].numpy()
        m = _lib.load().b200rl_stackdelta_wait(self._h, self.mis_h.data_ptr())
        self._pending = False
        self._keep = None
        if m < 0:
            _lib.check(int(m), "stackdelta_wait")
        return self.mis_h[:int(m)].numpy()

    def invalidate(self):
        if self._pending:
            self.wait()
        _lib.load().b200rl_stackdelta_invalidate(self._h)

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                _lib.load().b200rl_stackdelta_destroy(h)
            except Exception:
                pass


# ----------------------------------------------------------- diagonal Gaussian policy
def gaussian_sample(mean, logstd, noise, value_in=None, out=None):
    """action, logprob, entropy[, value] for Normal(mean, exp(logstd)) with caller-supplied N(0,1) noise
    (reference: ppo_continuous_action.py:134-141)."""
    lib = _lib.load()
    n, D = mean.shape
    assert mean.stride(1) == 1
    _contig(noise, "noise"); _contig(logstd, "logstd")
    dev = mean.device
    f = torch.float32
    if out is None:
        action = torch.empty(n, D, dtype=f, device=dev)
        logprob = torch.empty(n, dtype=f, device=dev)
        entropy = torch.empty(n, dtype=f, device=dev)
        value = torch.empty(n, dtype=f, device=dev) if value_in is not None else None
    else:
        action, logprob, entropy, value = out
    ldv = 0
    if value_in is not None:
        value_in = value_in.reshape(n, -1)
        ldv = value_in.stride(0)
    rc = lib.b200rl_gaussian_sample_f32(_ptr(mean, f, "mean"), mean.stride(0), _ptr(logstd, f, "logstd"), _ptr(noise, f, "noise"),
                                        _ptr(value_in, f, "value_in", True), ldv, n, D, _ptr(action, f, "action"),
                                        _ptr(logprob, f, "logprob"), _ptr(entropy, f, "entropy", True),
                                        _ptr(value, f, "value_out", True), _stream())
    _lib.check(rc, "gaussian_sample")
    return action, logprob, entropy, value


def gaussian_eval(mean, logstd, action):
    lib = _lib.load()
    n, D = mean.shape
    f = torch.float32
    action = _contig(action.reshape(n, D), "action")
    logprob = torch.empty(n, dtype=f, device=mean.device)
    entropy = torch.empty(n, dtype=f, device=mean.device)
    rc = lib.b200rl_gaussian_eval_f32(_ptr(mean, f, "mean"), mean.stride(0), _ptr(logstd, f, "logstd"), _ptr(action, f, "action"),
                                      n, D, _ptr(logprob, f, "logprob"), _ptr(entropy, f, "entropy"), _stream())
    _lib.check(rc, "gaussian_eval")
    return logprob, entropy


def ppo_loss_gaussian(new_mean, logstd, new_value, mb_inds, b_actions, b_logprobs, b_advantages, b_returns, b_values,
                      clip_coef, ent_coef, vf_coef, norm_adv=True, clip_vloss=True, dmean=None, dlogstd=None, dvalue=None,
                      stats=None, mean_shift=None):
    """Continuous-action PPO loss + gradients (reference: ppo_continuous_action.py:262-300).  ``mean_shift`` [M, D]
    (minibatch row order): evaluate ``Normal(new_mean + mean_shift, std)`` instead, as RPO's update does
    (rpo_continuous_action.py:138-142); ``dmean`` stays the gradient w.r.t. ``new_mean``."""
    lib = _lib.load()
    M, D = new_mean.shape
    dev = new_mean.device
    f = torch.float32
    new_value = new_value.reshape(M, -1)
    if dmean is None:
        dmean = torch.empty(M, D, dtype=f, device=dev)
    if dlogstd is None:
        dlogstd = torch.empty(D, dtype=f, device=dev)
    if dvalue is None:
        dvalue = torch.empty(M, dtype=f, device=dev)
    dv2 = dvalue.reshape(M, -1)
    if stats is None:
        stats = torch.zeros(16, dtype=f, device=dev)
    ws = _workspace(dev, "gloss", lib.b200rl_ppo_loss_gaussian_workspace_bytes(M))
    inputs = (_ptr(new_mean, f, "new_mean"), new_mean.stride(0), _ptr(logstd, f, "logstd"),
              _ptr(new_value, f, "new_value"), new_value.stride(0), _ptr(mb_inds, torch.int64, "mb_inds", True),
              _ptr(b_actions, f, "b_actions"), _ptr(b_logprobs, f, "b_logprobs"), _ptr(b_advantages, f, "b_advantages"),
              _ptr(b_returns, f, "b_returns"), _ptr(b_values, f, "b_values"))
    rest = (M, D, float(clip_coef), float(ent_coef), float(vf_coef), int(bool(norm_adv)), int(bool(clip_vloss)),
            _ptr(dmean, f, "dmean"), dmean.stride(0), _ptr(dlogstd, f, "dlogstd"), _ptr(dv2, f, "dvalue"), dv2.stride(0),
            _ptr(stats, f, "stats"), ws.data_ptr(), ws.numel(), _stream())
    if mean_shift is None:
        rc = lib.b200rl_ppo_loss_gaussian_f32(*inputs, *rest)
        _lib.check(rc, "ppo_loss_gaussian")
    else:
        if tuple(mean_shift.shape) != (M, D) or mean_shift.stride(1) != 1:
            raise ValueError(f"ppo_loss_gaussian: mean_shift must be [{M}, {D}] with unit column stride, "
                             f"got {tuple(mean_shift.shape)} strides {mean_shift.stride()}")
        rc = lib.b200rl_ppo_loss_gaussian_shift_f32(*inputs, _ptr(mean_shift, f, "mean_shift"), mean_shift.stride(0),
                                                    *rest)
        _lib.check(rc, "ppo_loss_gaussian_shift")
    return stats, dmean, dlogstd, dvalue


# ------------------------------------------------------------------------ DQN
def dqn_td_loss(q, q_target_next, actions, rewards, dones, gamma, huber=False, dq=None, stats=None):
    """TD target, loss and dL/dQ (reference: dqn_atari.py:220-224).  Returns (stats[2] = td_loss, mean Q; dq)."""
    lib = _lib.load()
    B, A = q.shape
    f = torch.float32
    if dq is None:
        dq = torch.empty(B, A, dtype=f, device=q.device)
    if stats is None:
        stats = torch.zeros(2, dtype=f, device=q.device)
    ws = _workspace(q.device, "td", lib.b200rl_dqn_td_loss_workspace_bytes(B))
    rc = lib.b200rl_dqn_td_loss_f32(_ptr(q, f, "q"), q.stride(0), _ptr(q_target_next, f, "q_target_next"), q_target_next.stride(0),
                                    _ptr(_contig(actions.reshape(-1), "actions"), torch.int64, "actions"),
                                    _ptr(_contig(rewards.reshape(-1), "rewards"), f, "rewards"),
                                    _ptr(_contig(dones.reshape(-1), "dones"), f, "dones"), B, A, float(gamma), int(bool(huber)),
                                    _ptr(dq, f, "dq"), dq.stride(0), _ptr(stats, f, "stats"), ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "dqn_td_loss")
    return stats, dq


def argmax(q):
    lib = _lib.load()
    n, A = q.shape
    out = torch.empty(n, dtype=torch.int64, device=q.device)
    rc = lib.b200rl_argmax_f32(_ptr(q, torch.float32, "q"), q.stride(0), n, A, _ptr(out, torch.int64, "out"), _stream())
    _lib.check(rc, "argmax")
    return out


# ------------------------------------------------------------------------ C51
def c51_act(logits, atoms, action=None, want_q=False, want_pmf=True):
    """QNetwork.get_action (reference: c51_atari.py:131-138) from the head logits [n, A * n_atoms]: per action the
    softmax over atoms and q = sum(pmf * atoms); the first-max greedy action (or ``action``).
    Returns (action i64 [n], q f32 [n, A] or None, pmf f32 [n, n_atoms] of the chosen action or None)."""
    lib = _lib.load()
    n, W = logits.shape
    assert logits.stride(1) == 1
    atoms = _contig(atoms, "atoms")
    Z = atoms.numel()
    if W % Z != 0:
        raise ValueError(f"c51_act: {W} logits per row is not a multiple of n_atoms={Z}")
    A = W // Z
    f = torch.float32
    dev = logits.device
    if action is not None:
        action = _contig(action.reshape(-1), "action")
        if action.dtype != torch.int64:
            action = action.long()
    out_a = torch.empty(n, dtype=torch.int64, device=dev)
    q = torch.empty(n, A, dtype=f, device=dev) if want_q else None
    pmf = torch.empty(n, Z, dtype=f, device=dev) if want_pmf else None
    rc = lib.b200rl_c51_act_f32(_ptr(logits, f, "logits"), logits.stride(0), _ptr(atoms, f, "atoms"), n, A, Z,
                                _ptr(action, torch.int64, "action", True), _ptr(out_a, torch.int64, "action_out"),
                                _ptr(q, f, "q", True), _ptr(pmf, f, "pmf", True), _stream())
    _lib.check(rc, "c51_act")
    return out_a, q, pmf


def c51_loss(logits, next_logits, atoms, actions, rewards, dones, gamma, v_min, v_max, dlogits=None, stats=None):
    """Categorical projection + clamped cross-entropy + dloss/dlogits (reference: c51_atari.py:233-253).
    Returns (stats f32[2] = losses/loss, losses/q_values; dlogits [B, A * n_atoms])."""
    lib = _lib.load()
    B, W = logits.shape
    assert logits.stride(1) == 1 and next_logits.stride(1) == 1 and next_logits.shape == (B, W)
    atoms = _contig(atoms, "atoms")
    Z = atoms.numel()
    if W % Z != 0:
        raise ValueError(f"c51_loss: {W} logits per row is not a multiple of n_atoms={Z}")
    f = torch.float32
    dev = logits.device
    if dlogits is None:
        dlogits = torch.empty(B, W, dtype=f, device=dev)
    if stats is None:
        stats = torch.zeros(2, dtype=f, device=dev)
    actions = _contig(actions.reshape(-1), "actions")
    if actions.dtype != torch.int64:
        actions = actions.long()
    ws = _workspace(dev, "c51", lib.b200rl_c51_loss_workspace_bytes(B))
    rc = lib.b200rl_c51_loss_f32(_ptr(logits, f, "logits"), logits.stride(0), _ptr(next_logits, f, "next_logits"),
                                 next_logits.stride(0), _ptr(atoms, f, "atoms"), _ptr(actions, torch.int64, "actions"),
                                 _ptr(_contig(rewards.reshape(-1), "rewards"), f, "rewards"),
                                 _ptr(_contig(dones.reshape(-1), "dones"), f, "dones"), B, W // Z, Z,
                                 float(gamma), float(v_min), float(v_max), _ptr(dlogits, f, "dlogits"), dlogits.stride(0),
                                 _ptr(stats, f, "stats"), ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "c51_loss")
    return stats, dlogits


# ------------------------------------------------------------------------ SAC
SAC_CRITIC_STAT_NAMES = ("qf1_values", "qf2_values", "qf1_loss", "qf2_loss")
SAC_ACTOR_STAT_NAMES = ("actor_loss", "alpha_loss", "alpha", "log_alpha")


def sac_policy(logits):
    """Actor.get_action's (log_softmax, probs) of the logits [n, A] (reference: sac_atari.py:164-170)."""
    lib = _lib.load()
    n, A = logits.shape
    assert logits.stride(1) == 1
    f = torch.float32
    logp = torch.empty(n, A, dtype=f, device=logits.device)
    probs = torch.empty(n, A, dtype=f, device=logits.device)
    rc = lib.b200rl_sac_policy_f32(_ptr(logits, f, "logits"), logits.stride(0), n, A, _ptr(logp, f, "logp"), A,
                                   _ptr(probs, f, "probs"), A, _stream())
    _lib.check(rc, "sac_policy")
    return logp, probs


def sac_critic_loss(next_logits, q1_target, q2_target, q1, q2, actions, rewards, dones, gamma, alpha, y=None, dq1=None,
                    dq2=None, stats=None, workspace=None):
    """Soft-Q target, both critic losses and dL/dq1, dL/dq2 (reference: sac_atari.py:274-290); ``alpha`` is a device
    f32 [1].  ``workspace``: a caller-owned uint8 buffer (what a captured CUDA graph keeps), else a shared one.  Returns (stats f32[4] = qf1_values, qf2_values, qf1_loss, qf2_loss; y [B]; dq1 [B, A]; dq2 [B, A])."""
    lib = _lib.load()
    B, A = q1.shape
    for n_, t in (("next_logits", next_logits), ("q1_target", q1_target), ("q2_target", q2_target), ("q2", q2)):
        if tuple(t.shape) != (B, A):
            raise ValueError(f"sac_critic_loss: {n_} shape {tuple(t.shape)} != {(B, A)}")
    for t in (next_logits, q1_target, q2_target, q1, q2):
        assert t.stride(1) == 1
    f = torch.float32
    dev = q1.device
    y = torch.empty(B, dtype=f, device=dev) if y is None else y
    dq1 = torch.empty(B, A, dtype=f, device=dev) if dq1 is None else dq1
    dq2 = torch.empty(B, A, dtype=f, device=dev) if dq2 is None else dq2
    stats = torch.zeros(4, dtype=f, device=dev) if stats is None else stats
    actions = _contig(actions.reshape(-1), "actions")
    if actions.dtype != torch.int64:
        actions = actions.long()
    ws = workspace if workspace is not None else _workspace(dev, "sac_critic", lib.b200rl_sac_critic_loss_workspace_bytes(B))
    rc = lib.b200rl_sac_critic_loss_f32(
        _ptr(next_logits, f, "next_logits"), next_logits.stride(0), _ptr(q1_target, f, "q1_target"), q1_target.stride(0),
        _ptr(q2_target, f, "q2_target"), q2_target.stride(0), _ptr(q1, f, "q1"), q1.stride(0), _ptr(q2, f, "q2"),
        q2.stride(0), _ptr(actions, torch.int64, "actions"), _ptr(_contig(rewards.reshape(-1), "rewards"), f, "rewards"),
        _ptr(_contig(dones.reshape(-1), "dones"), f, "dones"), _ptr(alpha, f, "alpha"), B, A, float(gamma),
        _ptr(y, f, "y"), _ptr(dq1, f, "dq1"), dq1.stride(0), _ptr(dq2, f, "dq2"), dq2.stride(0), _ptr(stats, f, "stats"),
        ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "sac_critic_loss")
    return stats, y, dq1, dq2


def sac_actor_loss(logits, q1, q2, alpha, target_entropy=0.0, log_alpha=None, exp_avg=None, exp_avg_sq=None,
                   step_scalars=None, eps=1e-4, dlogits=None, stats=None, workspace=None):
    """Actor loss + dL/dlogits (reference: sac_atari.py:293-305) and, when ``log_alpha`` is given (autotune), the
    temperature loss, one Adam step of ``log_alpha`` (moments ``exp_avg`` / ``exp_avg_sq``, ``step_scalars`` f32[2] from
    ``adam_step_scalars``, all device memory) and ``alpha = exp(log_alpha)`` (sac_atari.py:307-314).  ``workspace`` as
    in ``sac_critic_loss``.
    Returns (stats f32[4] = actor_loss, alpha_loss, alpha, log_alpha; dlogits [B, A])."""
    lib = _lib.load()
    B, A = logits.shape
    for n_, t in (("q1", q1), ("q2", q2)):
        if tuple(t.shape) != (B, A):
            raise ValueError(f"sac_actor_loss: {n_} shape {tuple(t.shape)} != {(B, A)}")
    for t in (logits, q1, q2):
        assert t.stride(1) == 1
    f = torch.float32
    dev = logits.device
    dlogits = torch.empty(B, A, dtype=f, device=dev) if dlogits is None else dlogits
    stats = torch.zeros(4, dtype=f, device=dev) if stats is None else stats
    autotune = log_alpha is not None
    ws = workspace if workspace is not None else _workspace(dev, "sac_actor", lib.b200rl_sac_actor_loss_workspace_bytes(B))
    rc = lib.b200rl_sac_actor_loss_f32(
        _ptr(logits, f, "logits"), logits.stride(0), _ptr(q1, f, "q1"), q1.stride(0), _ptr(q2, f, "q2"), q2.stride(0), B, A,
        _ptr(alpha, f, "alpha"), int(autotune), _ptr(log_alpha, f, "log_alpha", True), _ptr(exp_avg, f, "exp_avg", True),
        _ptr(exp_avg_sq, f, "exp_avg_sq", True), _ptr(step_scalars, f, "step_scalars", True), float(target_entropy),
        0.9, 0.999, float(eps), _ptr(dlogits, f, "dlogits"), dlogits.stride(0), _ptr(stats, f, "stats"), ws.data_ptr(),
        ws.numel(), _stream())
    _lib.check(rc, "sac_actor_loss")
    return stats, dlogits


# ------------------------------------------------------------------------ continuous SAC (sac_continuous_action.py)
SACC_CRITIC_STAT_NAMES = SAC_CRITIC_STAT_NAMES
SACC_ACTOR_STAT_NAMES = SAC_ACTOR_STAT_NAMES
_F32 = torch.float32


def _o(t, name):
    return _ptr(t, _F32, name, allow_none=True)


def _rows(t, name="rows"):
    if t is None:
        return None
    return _ptr(_contig(t, name), torch.int64, name)


def _ld(t):
    if t.dim() != 2 or t.stride(1) != 1:
        raise ValueError("sac_continuous: row-major [n, d] tensor with unit column stride expected")
    return t.stride(0)


SACC_TD3_ACTOR = 2    # network kind of the deterministic TD3 actor (sacc_param_count / sacc_wgrad ``critic``)


def _net_kind(critic):
    """False / True: the tanh-Gaussian actor / a critic; ``SACC_TD3_ACTOR``: the deterministic actor."""
    return SACC_TD3_ACTOR if critic == SACC_TD3_ACTOR else int(bool(critic))


def sacc_param_count(obs_dim, act_dim, critic):
    n = _lib.load().b200rl_sacc_param_count(int(obs_dim), int(act_dim), _net_kind(critic))
    if n < 0:
        raise ValueError(f"sac_continuous: obs_dim={obs_dim}, act_dim={act_dim} outside the kernels' limits "
                         "(1 <= act_dim <= 32, obs_dim + act_dim <= 1024)")
    return n


def sacc_workspace(B, device):
    """Zeroed scratch of the row-mean kernels of a batch of B rows (one buffer serves all of them on one stream)."""
    return torch.zeros(max(int(_lib.load().b200rl_sacc_workspace_bytes(int(B))), 16), dtype=torch.uint8, device=device)


def sacc_critic_fwd(params, net_stride, obs, act, B, obs_dim, act_dim, obs_rows=None, act_rows=None, q=None, keep_x=None,
                    keep_h1=None, keep_h2=None):
    """q [2, B] of the twin critics on [obs[obs_rows] | act[act_rows]] (sac_continuous_action.py:94-99)."""
    q = torch.empty(2, B, dtype=_F32, device=params.device) if q is None else q
    rc = _lib.load().b200rl_sacc_critic_fwd_f32(
        _ptr(params, _F32, "params"), int(net_stride), _ptr(obs, _F32, "obs"), _ld(obs), _rows(obs_rows, "obs_rows"),
        _ptr(act, _F32, "act"), _ld(act), _rows(act_rows, "act_rows"), int(B), int(obs_dim), int(act_dim),
        _ptr(q, _F32, "q"), _o(keep_x, "keep_x"), _o(keep_h1, "keep_h1"), _o(keep_h2, "keep_h2"), _stream())
    _lib.check(rc, "sacc_critic_fwd")
    return q


def sacc_actor_fwd(params, obs, B, obs_dim, act_dim, eps, scale, bias, rows=None, action=None, log_pi=None,
                   mean_out=None, mean_logstd=None, keep_x=None, keep_h1=None, keep_h2=None, keep_head=None,
                   temperature=None, workspace=None):
    """Actor.get_action (sac_continuous_action.py:139-151) with noise ``eps`` [B, D].  ``temperature``: a dict(alpha,
    log_alpha, exp_avg, exp_avg_sq, step_scalars, target_entropy, stats) to take the autotune step on these log_pi
    (sac_continuous_action.py:289-297)."""
    t = temperature or {}
    rc = _lib.load().b200rl_sacc_actor_fwd_f32(
        _ptr(params, _F32, "params"), _ptr(obs, _F32, "obs"), _ld(obs), _rows(rows), int(B), int(obs_dim), int(act_dim),
        _o(eps, "eps"), _ptr(scale, _F32, "scale"), _ptr(bias, _F32, "bias"), _o(action, "action"), _o(log_pi, "log_pi"),
        _o(mean_out, "mean_out"), _o(mean_logstd, "mean_logstd"), _o(keep_x, "keep_x"), _o(keep_h1, "keep_h1"),
        _o(keep_h2, "keep_h2"), _o(keep_head, "keep_head"), int(bool(temperature)), float(t.get("target_entropy", 0.0)),
        _o(t.get("alpha"), "alpha"), _o(t.get("log_alpha"), "log_alpha"), _o(t.get("exp_avg"), "exp_avg"),
        _o(t.get("exp_avg_sq"), "exp_avg_sq"), _o(t.get("step_scalars"), "step_scalars"), 0.9, 0.999, 1e-8,
        _o(t.get("stats"), "stats"), workspace.data_ptr() if workspace is not None else None,
        workspace.numel() if workspace is not None else 0, _stream())
    _lib.check(rc, "sacc_actor_fwd")


def sacc_critic_loss(q_next, next_logpi, q, rewards, dones, alpha, gamma, rows=None, y=None, dq=None, stats=None,
                     workspace=None):
    """Soft-Q target and both MSE losses with dq [2, B] (sac_continuous_action.py:257-268).  ``rewards`` / ``dones``
    are 1-D (strided) views read at ``rows``.  ``next_logpi`` None: no entropy term (td3_continuous_action.py:241-242);
    ``alpha`` may then be None."""
    B = q.shape[1]
    dev = q.device
    dq = torch.empty(2, B, dtype=_F32, device=dev) if dq is None else dq
    stats = torch.zeros(4, dtype=_F32, device=dev) if stats is None else stats
    ws = sacc_workspace(B, dev) if workspace is None else workspace
    if rewards.stride() != dones.stride():
        raise ValueError("sacc_critic_loss: rewards and dones need the same stride")
    rc = _lib.load().b200rl_sacc_critic_loss_f32(
        _ptr(q_next, _F32, "q_next"), _o(next_logpi, "next_logpi"), _ptr(q, _F32, "q"),
        _ptr(rewards, _F32, "rewards"), _ptr(dones, _F32, "dones"), rewards.stride(0), _rows(rows), _o(alpha, "alpha"),
        int(B), float(gamma), _o(y, "y"), _ptr(dq, _F32, "dq"), _ptr(stats, _F32, "stats"), ws.data_ptr(), ws.numel(),
        _stream())
    _lib.check(rc, "sacc_critic_loss")
    return stats, dq


def sacc_critic_bwd(params, net_stride, B, obs_dim, act_dim, h1, h2, dq=None, q=None, dz1=None, dz2=None, dact=None):
    """Critic step (``dq``, ``dz1`` / ``dz2``), twin actor step (``q``, ``dact`` [2, B, D]) or, with ``net_stride`` 0
    and neither ``dq`` nor ``q``, the single-network actor step of -mean(q) (``dact`` [B, D])."""
    rc = _lib.load().b200rl_sacc_critic_bwd_f32(
        _ptr(params, _F32, "params"), int(net_stride), int(B), int(obs_dim), int(act_dim), _o(dq, "dq"), _o(q, "q"),
        _ptr(h1, _F32, "h1"), _ptr(h2, _F32, "h2"), _o(dz1, "dz1"), _o(dz2, "dz2"), _o(dact, "dact"), _stream())
    _lib.check(rc, "sacc_critic_bwd")


def sacc_actor_bwd(params, B, obs_dim, act_dim, head, eps, scale, dact, q, log_pi, alpha, h1, h2, dhead, dz1, dz2, stats,
                   workspace):
    rc = _lib.load().b200rl_sacc_actor_bwd_f32(
        _ptr(params, _F32, "params"), int(B), int(obs_dim), int(act_dim), _ptr(head, _F32, "head"), _ptr(eps, _F32, "eps"),
        _ptr(scale, _F32, "scale"), _ptr(dact, _F32, "dact"), _ptr(q, _F32, "q"), _ptr(log_pi, _F32, "log_pi"),
        _ptr(alpha, _F32, "alpha"), _ptr(h1, _F32, "h1"), _ptr(h2, _F32, "h2"), _ptr(dhead, _F32, "dhead"),
        _ptr(dz1, _F32, "dz1"), _ptr(dz2, _F32, "dz2"), _ptr(stats, _F32, "stats"), workspace.data_ptr(), workspace.numel(),
        _stream())
    _lib.check(rc, "sacc_actor_bwd")


def sacc_wgrad(critic, B, obs_dim, act_dim, x, h1, h2, dz1, dz2, dout, grad, net_stride=0):
    """Weight and bias gradients into the flat ``grad``: of the twin critics (``critic`` True, ``net_stride`` apart:
    dz1 / dz2 / h1 / h2 [2, B, 256], ``dout`` = dq [2, B]) or, with ``net_stride`` 0, of one critic (DDPG: [1, B, 256],
    dq [B]); of the tanh-Gaussian actor (False) or of the deterministic actor (``SACC_TD3_ACTOR``)."""
    rc = _lib.load().b200rl_sacc_wgrad_f32(
        _net_kind(critic), int(B), int(obs_dim), int(act_dim), _ptr(x, _F32, "x"), _ptr(h1, _F32, "h1"),
        _ptr(h2, _F32, "h2"), _ptr(dz1, _F32, "dz1"), _ptr(dz2, _F32, "dz2"), _ptr(dout, _F32, "dout"),
        _ptr(grad, _F32, "grad"), int(net_stride), _stream())
    _lib.check(rc, "sacc_wgrad")


def sacc_soft_update(src, dst, n, tau):
    """dst[:n] = tau * src[:n] + (1 - tau) * dst[:n] (sac_continuous_action.py:300-304)."""
    rc = _lib.load().b200rl_sacc_soft_update_f32(_ptr(src, _F32, "src"), _ptr(dst, _F32, "dst"), int(n), float(tau),
                                                 _stream())
    _lib.check(rc, "sacc_soft_update")


# ----------------------------------------------------------- TD3 (td3_continuous_action.py), kind SACC_TD3_ACTOR
def td3_actor_fwd(params, obs, B, obs_dim, act_dim, scale, bias, rows=None, mu=None, keep_y=None, keep_x=None,
                  keep_h1=None, keep_h2=None, smoothing=None):
    """Actor.forward (td3_continuous_action.py:128-132) on obs[rows]: ``mu`` [B, D] and the kept tanh ``keep_y``.
    ``smoothing``: a dict(eps [B, D], policy_noise, noise_clip, low, high, out [B, D]) for the smoothed target action
    of td3_continuous_action.py:232-238."""
    sm = smoothing or {}
    rc = _lib.load().b200rl_td3_actor_fwd_f32(
        _ptr(params, _F32, "params"), _ptr(obs, _F32, "obs"), _ld(obs), _rows(rows), int(B), int(obs_dim), int(act_dim),
        _ptr(scale, _F32, "scale"), _ptr(bias, _F32, "bias"), _o(mu, "mu"), _o(keep_y, "keep_y"), _o(keep_x, "keep_x"),
        _o(keep_h1, "keep_h1"), _o(keep_h2, "keep_h2"), _o(sm.get("eps"), "eps"), float(sm.get("policy_noise", 0.0)),
        float(sm.get("noise_clip", 0.0)), float(sm.get("low", 0.0)), float(sm.get("high", 0.0)), _o(sm.get("out"), "out"),
        _stream())
    _lib.check(rc, "td3_actor_fwd")


def td3_actor_bwd(params, B, obs_dim, act_dim, y, scale, dact, q, h1, h2, dhead, dz1, dz2, stats, workspace):
    """actor_loss = -qf1(obs, actor(obs)).mean() (td3_continuous_action.py:256) back through the deterministic head and
    the trunk; stats[0] = actor_loss."""
    rc = _lib.load().b200rl_td3_actor_bwd_f32(
        _ptr(params, _F32, "params"), int(B), int(obs_dim), int(act_dim), _ptr(y, _F32, "y"), _ptr(scale, _F32, "scale"),
        _ptr(dact, _F32, "dact"), _ptr(q, _F32, "q"), _ptr(h1, _F32, "h1"), _ptr(h2, _F32, "h2"),
        _ptr(dhead, _F32, "dhead"), _ptr(dz1, _F32, "dz1"), _ptr(dz2, _F32, "dz2"), _ptr(stats, _F32, "stats"),
        workspace.data_ptr(), workspace.numel(), _stream())
    _lib.check(rc, "td3_actor_bwd")


# ------------------------------------------------------------------ DDPG (ddpg_continuous_action.py), one critic
DDPG_CRITIC_STAT_NAMES = ("qf1_values", "qf1_loss")


def ddpg_critic_loss_bwd(params, B, obs_dim, act_dim, q_next, q, rewards, dones, gamma, h1, h2, rows=None, y=None,
                         dq=None, dz1=None, dz2=None, stats=None, workspace=None):
    """The one-critic step of ddpg_continuous_action.py:222-229 in one launch: y = r + (1 - d) gamma q_next, dq [B] of
    F.mse_loss(q, y) and the critic's data gradients dz1 / dz2 [B, 256] from its kept h1 / h2; ``stats`` [2] =
    ``DDPG_CRITIC_STAT_NAMES``.  ``q_next`` / ``q`` are [B] (or [1, B]); ``rewards`` / ``dones`` 1-D (strided) views
    read at ``rows``.  Returns (stats, dq, dz1, dz2)."""
    dev = q.device
    z = lambda *s: torch.empty(*s, dtype=_F32, device=dev)   # noqa: E731
    dq = z(B) if dq is None else dq
    dz1 = z(B, 256) if dz1 is None else dz1
    dz2 = z(B, 256) if dz2 is None else dz2
    stats = torch.zeros(2, dtype=_F32, device=dev) if stats is None else stats
    ws = sacc_workspace(B, dev) if workspace is None else workspace
    if rewards.stride() != dones.stride():
        raise ValueError("ddpg_critic_loss_bwd: rewards and dones need the same stride")
    rc = _lib.load().b200rl_ddpg_critic_loss_bwd_f32(
        _ptr(params, _F32, "params"), int(B), int(obs_dim), int(act_dim), _ptr(q_next, _F32, "q_next"),
        _ptr(q, _F32, "q"), _ptr(rewards, _F32, "rewards"), _ptr(dones, _F32, "dones"), rewards.stride(0), _rows(rows),
        float(gamma), _ptr(h1, _F32, "h1"), _ptr(h2, _F32, "h2"), _o(y, "y"), _ptr(dq, _F32, "dq"),
        _ptr(dz1, _F32, "dz1"), _ptr(dz2, _F32, "dz2"), _ptr(stats, _F32, "stats"), ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "ddpg_critic_loss_bwd")
    return stats, dq, dz1, dz2


# ------------------------------------------------------------------------------ RAdam (torch/optim/radam.py)
def radam_step_scalars(step, lr, beta1=0.9, beta2=0.999):
    """(bc1, lr, bc2 ** 0.5, rect) as float32 (rect 0 where rho_t <= 5), computed by the library in double as
    ``_single_tensor_radam`` computes them in python."""
    import ctypes
    out = (ctypes.c_float * 4)()
    _lib.check(_lib.load().b200rl_radam_step_scalars(int(step), float(lr), float(beta1), float(beta2), out),
               "radam_step_scalars")
    return tuple(float(x) for x in out)


def _radam_args(params, grads, exp_avg, exp_avg_sq):
    P = params.numel()
    for n_, t in (("params", params), ("grads", grads), ("exp_avg", exp_avg), ("exp_avg_sq", exp_avg_sq)):
        _contig(t, n_)
        assert t.numel() == P
    return (_ptr(params, _F32, "params"), _ptr(grads, _F32, "grads"), _ptr(exp_avg, _F32, "exp_avg"),
            _ptr(exp_avg_sq, _F32, "exp_avg_sq"), P)


def clip_radam(params, grads, exp_avg, exp_avg_sq, step, lr, beta1=0.9, beta2=0.999, eps=1e-8, max_norm=10.0,
               norm_out=None):
    """In-place clip_grad_norm_ + RAdam step on flat f32 vectors (cleanrl/pqn.py:239-240); ``max_norm`` None: no clip."""
    lib = _lib.load()
    *ptrs, P = _radam_args(params, grads, exp_avg, exp_avg_sq)
    ws = _workspace(params.device, "adam", lib.b200rl_clip_adam_workspace_bytes(P))
    rc = lib.b200rl_clip_radam_f32(*ptrs, P, int(step), float(lr), float(beta1), float(beta2), float(eps),
                                   -1.0 if max_norm is None else float(max_norm), _o(norm_out, "norm_out"),
                                   ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "clip_radam")
    return params


def clip_radam_dyn(params, grads, exp_avg, exp_avg_sq, step_scalars, beta1=0.9, beta2=0.999, eps=1e-8, max_norm=10.0,
                   norm_out=None):
    """``clip_radam`` with the four step scalars of ``radam_step_scalars`` in device memory (f32 [4]): what a captured
    CUDA graph of the update replays."""
    lib = _lib.load()
    *ptrs, P = _radam_args(params, grads, exp_avg, exp_avg_sq)
    assert step_scalars.numel() == 4 and step_scalars.is_contiguous()
    ws = _workspace(params.device, "adam", lib.b200rl_clip_adam_workspace_bytes(P))
    rc = lib.b200rl_clip_radam_dyn_f32(*ptrs, P, _ptr(step_scalars, _F32, "step_scalars"), float(beta1), float(beta2),
                                       float(eps), -1.0 if max_norm is None else float(max_norm),
                                       _o(norm_out, "norm_out"), ws.data_ptr(), ws.numel(), _stream())
    _lib.check(rc, "clip_radam_dyn")
    return params


# ------------------------------------------------------------------------------ PQN (cleanrl/pqn.py)
PQN_STAT_NAMES = ("td_loss", "q_values")


def pqn_param_count(obs_dim, A):
    n = _lib.load().b200rl_pqn_param_count(int(obs_dim), int(A))
    if n < 0:
        raise ValueError(f"pqn: obs_dim={obs_dim}, A={A} outside the kernels' limits (1 <= obs_dim <= 512, 2 <= A <= 64)")
    return n


def pqn_workspace(M, device):
    """Zeroed update workspace of a minibatch of up to M rows (one loss_bwd and the wgrad after it)."""
    return torch.zeros(int(_lib.load().b200rl_pqn_workspace_bytes(int(M))), dtype=torch.uint8, device=device)


def _obs2d(obs, obs_dim):
    if obs.dim() != 2 or obs.stride(1) != 1 or obs.shape[1] != obs_dim:
        raise ValueError(f"pqn: obs must be row-major [n, {obs_dim}] with unit column stride")
    return obs.stride(0)


def pqn_act(params, obs, obs_dim, A, values, random_actions=None, u=None, eps=0.0, actions=None, obs_slot=None,
            copy=None):
    """The rollout step (pqn.py:180-189) on obs [n, obs_dim]: ``values`` [n] = max Q and, with ``random_actions`` /
    ``u`` (the step's CPU draws), ``actions`` [n] int64 = u < eps ? random : argmax Q.  ``obs_slot`` [n, obs_dim] receives a
    copy of the rows and ``copy`` = (src, dst) f32 tensors of equal size is copied in the same launch."""
    n = obs.shape[0]
    src, dst = copy if copy is not None else (None, None)
    rc = _lib.load().b200rl_pqn_act_f32(
        _ptr(params, _F32, "params"), _ptr(obs, _F32, "obs"), _obs2d(obs, obs_dim), n, int(obs_dim), int(A),
        _rows(random_actions, "random_actions"), _o(u, "u"), float(eps), _o(obs_slot, "obs_slot"),
        _rows(actions, "actions"), _ptr(values, _F32, "values"), _o(src, "copy_in"), _o(dst, "copy_out"),
        0 if src is None else int(src.numel()), _stream())
    _lib.check(rc, "pqn_act")
    return actions, values


def pqn_forward(params, obs, obs_dim, A, q=None):
    """QNetwork.forward: q [n, A]."""
    n = obs.shape[0]
    q = torch.empty(n, A, dtype=_F32, device=obs.device) if q is None else q
    rc = _lib.load().b200rl_pqn_forward_f32(_ptr(params, _F32, "params"), _ptr(obs, _F32, "obs"), _obs2d(obs, obs_dim), n,
                                            int(obs_dim), int(A), _ptr(_contig(q, "q"), _F32, "q"), _stream())
    _lib.check(rc, "pqn_forward")
    return q


def pqn_loss_bwd(params, obs, obs_dim, A, mb_inds, b_actions, b_returns, stats, workspace):
    """One minibatch's loss, data backward and kept activations (pqn.py:233-238); ``stats`` [2] = ``PQN_STAT_NAMES``."""
    M = int(mb_inds.numel())
    rc = _lib.load().b200rl_pqn_loss_bwd_f32(
        _ptr(params, _F32, "params"), _ptr(obs, _F32, "obs"), _obs2d(obs, obs_dim), _rows(mb_inds, "mb_inds"),
        _rows(b_actions, "b_actions"), _ptr(_contig(b_returns, "b_returns"), _F32, "b_returns"), M, int(obs_dim), int(A),
        _ptr(stats, _F32, "stats"), workspace.data_ptr(), workspace.numel(), _stream())
    _lib.check(rc, "pqn_loss_bwd")
    return stats


def pqn_wgrad(obs, obs_dim, A, mb_inds, b_actions, workspace, grad):
    """Every weight / bias / gamma / beta gradient of the minibatch the last ``pqn_loss_bwd`` on ``workspace`` saw."""
    M = int(mb_inds.numel())
    rc = _lib.load().b200rl_pqn_wgrad_f32(
        _ptr(obs, _F32, "obs"), _obs2d(obs, obs_dim), _rows(mb_inds, "mb_inds"), _rows(b_actions, "b_actions"), M,
        int(obs_dim), int(A), workspace.data_ptr(), workspace.numel(), _ptr(grad, _F32, "grad"), _stream())
    _lib.check(rc, "pqn_wgrad")


def qlambda(rewards, values, dones, next_value, next_done, gamma, q_lambda, returns=None):
    """Q(lambda) returns (pqn.py:205-218), bit-identical to the reference loop."""
    T, N = rewards.shape
    for n_, t in (("rewards", rewards), ("values", values), ("dones", dones)):
        _contig(t, n_)
        assert t.shape == (T, N), f"{n_} shape {tuple(t.shape)} != {(T, N)}"
    next_value = _contig(next_value.reshape(-1), "next_value")
    next_done = _contig(next_done.reshape(-1), "next_done")
    assert next_value.numel() == N and next_done.numel() == N
    returns = torch.empty_like(rewards) if returns is None else returns
    rc = _lib.load().b200rl_qlambda_f32(
        _ptr(rewards, _F32, "rewards"), _ptr(values, _F32, "values"), _ptr(dones, _F32, "dones"),
        _ptr(next_value, _F32, "next_value"), _ptr(next_done, _F32, "next_done"), _ptr(returns, _F32, "returns"), T, N,
        float(gamma), float(q_lambda), _stream())
    _lib.check(rc, "qlambda")
    return returns
