"""TEST INFRASTRUCTURE: run the product's HOST logic (engine loop, rank seeding, flat-gradient
all-reduce over gloo, logging) on a CPU-only box by injecting oracle/torch-CPU implementations for the
device kernels.  The product itself has no such path: PPOEngine / agents / ops raise on CPU tensors
unless this module flips PPOEngine.ALLOW_NON_CUDA_FOR_TESTS and patches cleanrl_b200.ops."""
from __future__ import annotations

import numpy as np
import torch
from torch.distributions.categorical import Categorical

from cleanrl_b200 import agents, nets, ops, ppo_engine
from oracle import ppo_oracle as O


def _t(x, like=None):
    return torch.from_numpy(np.ascontiguousarray(x))


def gae(rewards, values, dones, next_value, next_done, gamma, gae_lambda, mode=0, out=None):
    adv, ret = O.gae(rewards.numpy(), values.numpy(), dones.numpy(), next_value.numpy().reshape(-1),
                     next_done.numpy().reshape(-1), gamma, gae_lambda)
    if out is None:
        return _t(adv), _t(ret)
    out[0].copy_(_t(adv)); out[1].copy_(_t(ret))
    return out


def categorical_sample(logits, noise, value_in=None, out=None):
    a, lp, ent = O.categorical_sample(logits.detach().numpy(), noise.numpy())
    v = value_in.detach().reshape(-1).clone() if value_in is not None else None
    if out is None:
        return _t(a), _t(lp), _t(ent), v
    out[0].copy_(_t(a)); out[1].copy_(_t(lp))
    if out[2] is not None:
        out[2].copy_(_t(ent))
    if out[3] is not None:
        out[3].copy_(v)
    return out


def categorical_eval(logits, action):
    lp, ent = O.categorical_eval(logits.detach().numpy(), action.numpy())
    return _t(lp), _t(ent)


def ppo_loss(new_logits, new_value, mb_inds, b_actions, b_logprobs, b_advantages, b_returns, b_values,
             clip_coef, ent_coef, vf_coef, norm_adv=True, clip_vloss=True, dlogits=None, dvalue=None, stats=None):
    st, dl, dv = O.ppo_loss(new_logits.detach().numpy(), new_value.detach().numpy().reshape(-1),
                            None if mb_inds is None else mb_inds.numpy(), b_actions.numpy(), b_logprobs.numpy(),
                            b_advantages.numpy(), b_returns.numpy(), b_values.numpy(), clip_coef, ent_coef, vf_coef,
                            norm_adv, clip_vloss)
    dlogits.copy_(_t(dl)); dvalue.copy_(_t(dv))
    for i, k in enumerate(ops.STAT_NAMES):
        stats[i] = float(st[k])
    return stats, dlogits, dvalue


def clip_adam(params, grads, exp_avg, exp_avg_sq, step, lr, beta1=0.9, beta2=0.999, eps=1e-5, max_norm=0.5,
              world_size=1, norm_out=None):
    p, m, v, tn = O.clip_adam(params.numpy(), grads.numpy(), exp_avg.numpy(), exp_avg_sq.numpy(), step, lr, beta1, beta2,
                              eps, max_norm, world_size)
    params.copy_(_t(p)); exp_avg.copy_(_t(m)); exp_avg_sq.copy_(_t(v))
    if norm_out is not None:
        norm_out.fill_(float(tn))
    return params


def _bind_cpu(self):
    dev = next(self.parameters()).device
    self._flat = nets.FlatParams(self._param_order(), dev)
    return self._flat


def _torch_heads(self, x, rows=None, keep=False):
    xx = x if rows is None else x[rows]
    with torch.set_grad_enabled(keep):
        if isinstance(self, agents.NatureCNNAgent):
            hidden = self.network(xx.float() / 255.0)
            logits, value = self.actor(hidden), self.critic(hidden)[:, 0]
        else:
            xf = xx.float().reshape(xx.shape[0], -1)
            logits, value = self.actor(xf), self.critic(xf)[:, 0]
    if keep:
        self._graph = (logits, value)
    return logits.detach() if not keep else logits, value.detach() if not keep else value


def _forward_train(self, b_obs, mb_inds):
    self.flat
    lg, v = _torch_heads(self, b_obs, rows=mb_inds, keep=True)
    return lg.detach(), v.detach()


def _alloc_head_grad(self, M, device):
    A = self.num_actions
    d = torch.empty(M, A + 1, dtype=torch.float32, device=device)
    return d, d[:, :A], d[:, A]


def _backward(self, dhead):
    logits, value = self._graph
    A = self.num_actions
    self._flat.grad.zero_()
    with torch.enable_grad():
        torch.autograd.backward([logits, value], [dhead[:, :A].contiguous(), dhead[:, A].contiguous()])
    self._graph = None


_saved = {}


def install():
    if _saved:
        return
    ppo_engine.PPOEngine.ALLOW_NON_CUDA_FOR_TESTS = True
    for name, fn in (("gae", gae), ("categorical_sample", categorical_sample), ("categorical_eval", categorical_eval),
                     ("ppo_loss", ppo_loss), ("clip_adam", clip_adam)):
        _saved[name] = getattr(ops, name)
        setattr(ops, name, fn)
    for cls in (agents.NatureCNNAgent, agents.MLPAgent):
        _saved[(cls, "bind")] = agents.KernelAgent.bind
        for attr, fn in (("_forward_heads", _torch_heads), ("forward_train", _forward_train),
                         ("alloc_head_grad", _alloc_head_grad), ("backward", _backward)):
            _saved[(cls, attr)] = cls.__dict__.get(attr)        # None: inherited from a base class
            setattr(cls, attr, fn)
    agents.KernelAgent.bind = _bind_cpu
    _saved[(agents.KernelAgent, "_build_plan")] = agents.KernelAgent._build_plan
    agents.KernelAgent._build_plan = lambda self: None


def uninstall():
    if not _saved:
        return
    ppo_engine.PPOEngine.ALLOW_NON_CUDA_FOR_TESTS = False
    for k, v in list(_saved.items()):
        if isinstance(k, str):
            setattr(ops, k, v)
        elif k[1] == "bind":
            agents.KernelAgent.bind = v
        elif v is None:
            delattr(k[0], k[1])
        else:
            setattr(k[0], k[1], v)
    _saved.clear()
