"""Numpy restatement of RPO's update loss (cleanrl/rpo_continuous_action.py:138-144,269-304).  TEST INFRASTRUCTURE ONLY.

RPO evaluates the stored actions under ``Normal(action_mean + z, action_std)``.  The shifted mean is the reference's
separate fp32 add; everything after it is continuous PPO's loss, so this is ``ppo_oracle.ppo_loss_gaussian`` on
``fl(new_mean + mean_shift)``.  Its ``dmean`` is the gradient w.r.t. the shifted mean, which equals the gradient w.r.t.
``new_mean``.
"""
from __future__ import annotations

import numpy as np

from oracle.ppo_oracle import f32, ppo_loss_gaussian


def ppo_loss_gaussian_shift(new_mean, mean_shift, logstd, new_value, mb_inds, b_actions, b_logprobs, b_advantages,
                            b_returns, b_values, clip_coef, ent_coef, vf_coef, norm_adv=True, clip_vloss=True):
    """Returns (stats, dmean [M,D], dlogstd [D], dvalue [M]) of the loss of ``Normal(new_mean + mean_shift, std)``;
    ``mean_shift`` is [M, D] in minibatch row order."""
    mu = (np.asarray(new_mean, dtype=f32) + np.asarray(mean_shift, dtype=f32)).astype(f32)
    return ppo_loss_gaussian(mu, logstd, new_value, mb_inds, b_actions, b_logprobs, b_advantages, b_returns, b_values,
                             clip_coef, ent_coef, vf_coef, norm_adv, clip_vloss)
