"""Generate the RPO fixtures from the UNMODIFIED reference (build container only).  TEST INFRASTRUCTURE ONLY.

    python -m oracle.make_golden_rpo_continuous

* tests/golden/rpo_continuous_n4_t64_seed2.npz: cleanrl/rpo_continuous_action.py on the HalfCheetah-shaped synthetic
  gymnasium env (obs 17, act 6), 2 iterations of 2 epochs x 4 minibatches.  Per iteration the rollout tensors and the
  parameter sums; per update the logged losses, the parameter sums after the step, the iteration it belongs to, the
  head of its mb_inds and the first ``Z_HEAD`` rows of its mean shift ``z``; for the first update the full ``z``,
  ``mb_inds``, ``newlogprob``, ``newvalue``, the minibatch's observations, the parameters before the step and the
  gradients after clipping.  Also the shuffles, the state_dict keys and the TensorBoard series.
* tests/golden/rpo_continuous_n4_t64_seed5_kl.npz: seed 5, ``--rpo-alpha 0.3`` and a ``--target-kl`` that ends an
  iteration's update after its first epoch (asserted below), 3 iterations of 3 epochs: the draws of the iterations
  after the early stop show that ``z`` is consumed per epoch.
* tests/golden/rpo_continuous_surface.json: the script's Args fields (default, help text) and top-level names.

``z`` is recorded by wrapping ``torch.Tensor.uniform_`` (the reference draws it with
``torch.FloatTensor(shape).uniform_(-rpo_alpha, rpo_alpha)``, rpo_continuous_action.py:140).  The .npz files are written
with fixed zip timestamps, so a rerun reproduces them byte for byte.
"""
from __future__ import annotations

import sys

import numpy as np

from oracle.make_golden import OUT
from oracle.make_golden_c51 import surface
from oracle.make_golden_ddpg_continuous import _savez
from oracle.ref_harness import _main_globals, run_reference

COMMON = ["--no-cuda", "--num-envs", "4", "--num-steps", "64", "--num-minibatches", "4"]
ARGV = COMMON + ["--total-timesteps", "512", "--seed", "2", "--update-epochs", "2"]
ARGV_KL = COMMON + ["--total-timesteps", "768", "--seed", "5", "--update-epochs", "3", "--rpo-alpha", "0.3",
                    "--target-kl", "0.095"]
Z_HEAD = 8


def rpo_continuous(name, argv, expect_early_stop=False):
    import torch
    zs, extra = [], []
    orig_uniform, orig_step = torch.Tensor.uniform_, torch.optim.Adam.step

    def uniform_(self_, *a, **k):
        out = orig_uniform(self_, *a, **k)
        g = _main_globals()
        if g is not None and "mb_inds" in g and "b_obs" in g:      # inside the update loop: the mean shift z
            zs.append(out.detach().numpy().copy())
        return out

    def step(self_, *a, **k):
        g = _main_globals()
        if g is not None:
            rec = {"iteration": int(g["update"]), "epoch": int(g["epoch"])}
            if not extra:
                rec["b_obs_mb"] = g["b_obs"][g["mb_inds"]].detach().numpy().copy()
            extra.append(rec)
        return orig_step(self_, *a, **k)

    torch.Tensor.uniform_, torch.optim.Adam.step = uniform_, step
    try:
        rec, g = run_reference("rpo_continuous_action.py", argv, gymnasium_kind="continuous", keep_params=True)
    finally:
        torch.Tensor.uniform_, torch.optim.Adam.step = orig_uniform, orig_step
    n_upd = len(rec.updates)
    assert len(zs) == n_upd == len(extra), (len(zs), n_upd, len(extra))
    args = g["args"]
    full = args.update_epochs * args.num_minibatches
    per_iter = np.bincount([e["iteration"] for e in extra], minlength=len(rec.iterations) + 1)[1:]
    assert len(per_iter) == len(rec.iterations)
    if expect_early_stop:
        assert (per_iter < full).any() and per_iter[-1] > 0, per_iter
        assert (per_iter[:-1] < full).any(), "the early stop must come before the last iteration's draws"
    else:
        assert (per_iter == full).all(), per_iter
    out = {"argv": np.array(argv), "updates_per_iteration": per_iter}
    for k in ("actions", "logprobs", "rewards", "dones", "values", "advantages", "returns", "next_value", "next_done",
              "param_sums"):
        out[k] = np.stack([r[k] for r in rec.iterations])
    for k in ("pg_loss", "v_loss", "entropy_loss", "old_approx_kl", "approx_kl", "loss", "clipfrac", "lr",
              "grad_norm_postclip"):
        out["upd_" + k] = np.array([u[k] for u in rec.updates])
    out["upd_param_sums"] = np.stack([u["param_sums"] for u in rec.updates])
    out["upd_mb_inds_head"] = np.stack([u["mb_inds_head"] for u in rec.updates])
    out["upd_iteration"] = np.array([e["iteration"] for e in extra])
    out["upd_epoch"] = np.array([e["epoch"] for e in extra])
    out["upd_z_head"] = np.stack([z[:Z_HEAD] for z in zs])
    u1 = rec.updates[0]
    out["u1_z"] = zs[0]
    out["u1_b_obs"] = extra[0]["b_obs_mb"]
    for k in ("mb_inds", "newlogprob", "newvalue", "b_logprobs", "b_advantages", "b_returns", "b_values", "b_actions"):
        out["u1_" + k] = u1[k]
    flat = lambda lst: np.concatenate([x.reshape(-1) for x in lst])
    out["u1_params_before_flat"] = flat(u1["params_before"])
    out["u1_grads_flat"] = flat(u1["grads"])               # after clip_grad_norm_
    out["param_shapes"] = np.array([list(x.shape) + [0] * (2 - x.ndim) for x in u1["params"]])
    out["final_param_sums"] = np.array([p.detach().double().sum().item() for p in g["agent"].parameters()])
    out["shuffles"] = np.stack(rec.shuffles)
    out["state_dict_keys"] = np.array(list(g["agent"].state_dict().keys()))
    for t in sorted({t for t, _, _ in rec.scalars}):      # charts/SPS is wall-clock: its steps are kept, values zeroed
        out["tb/" + t] = np.array([(s_, 0.0 if t == "charts/SPS" else v) for tt, v, s_ in rec.scalars if tt == t],
                                  dtype=np.float64)
    _savez(OUT / name, out)
    print("wrote", name, n_upd, "updates", per_iter.tolist())


def main():
    surface("rpo_continuous_surface.json", "rpo_continuous_action.py")
    rpo_continuous("rpo_continuous_n4_t64_seed2.npz", ARGV)
    rpo_continuous("rpo_continuous_n4_t64_seed5_kl.npz", ARGV_KL, expect_early_stop=True)


if __name__ == "__main__":
    sys.exit(main())
