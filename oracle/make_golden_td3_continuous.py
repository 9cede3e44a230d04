"""Generate the TD3 fixtures from the UNMODIFIED reference (build container only).  TEST INFRASTRUCTURE ONLY.

    python -m oracle.make_golden_td3_continuous

* tests/golden/td3_continuous_n2_seed1.npz (defaults but ``--num-envs 2``, a 32-slot ring that wraps, batch 8) and
  td3_continuous_seed2_pf3.npz (seed 2, ``--policy-frequency 3 --policy-noise 0.4 --noise-clip 0.1
  --exploration-noise 0.3``: both smoothing clamps bind and actor_loss is stale at step 100):
  cleanrl/td3_continuous_action.py (+ the reference's own ReplayBuffer) on the synthetic HalfCheetah-shaped gymnasium
  env.  Per update: both critic losses and the logged q means, actor_loss on policy steps (NaN otherwise), and the
  parameter sums after the update of the actor (NaN on critic-only updates), the critics and the three targets; the
  first update's full tensors (the sampled batch, its smoothing draw, next_state_actions, y, the fc3 bias gradients);
  every exploration draw, the per-step action stream, the randint heads, the state_dict keys and the TensorBoard
  series.
* tests/golden/td3_continuous_surface.json: the script's Args fields (default, help text) and top-level names.
"""
from __future__ import annotations

import sys

import numpy as np

from oracle.make_golden import OUT
from oracle.make_golden_c51 import surface
from oracle.ref_harness import run_reference

COMMON = ["--no-cuda", "--total-timesteps", "120", "--learning-starts", "40", "--buffer-size", "64", "--batch-size", "8"]
ARGV = COMMON + ["--num-envs", "2", "--seed", "1"]
ARGV_PF3 = COMMON + ["--seed", "2", "--policy-frequency", "3", "--policy-noise", "0.4", "--noise-clip", "0.1",
                     "--exploration-noise", "0.3"]


def _script_globals():
    f = sys._getframe(1)
    while f is not None:
        if f.f_globals.get("__name__") == "__main__" and "qf1" in f.f_globals and "q_optimizer" in f.f_globals:
            return f.f_globals
        f = f.f_back
    return None


def _sums(*nets):
    return np.array([p.detach().double().sum().item() for n in nets for p in n.parameters()])


def td3_continuous(name, argv):
    import torch
    from cleanrl_b200 import synthetic_envs as S
    updates, samples, actions, explore, smooth = [], [], [], [], []
    orig_step, orig_randint, orig_env_step = torch.optim.Adam.step, np.random.randint, S.SyntheticGymnasiumVec.step
    orig_randn_like, orig_normal = torch.randn_like, torch.normal

    def np_(t):
        return t.detach().numpy().copy()

    def randn_like(*a, **k):
        out = orig_randn_like(*a, **k)
        smooth.append(np_(out))
        return out

    def normal(*a, **k):
        out = orig_normal(*a, **k)
        explore.append(np_(out))
        return out

    def target_sums(g):
        return _sums(g["target_actor"], g["qf1_target"], g["qf2_target"])

    def adam_step(self_, *a, **k):
        g = _script_globals()
        if g is None:
            return orig_step(self_, *a, **k)
        if self_ is g["q_optimizer"]:
            if updates:                   # the targets as the previous update's soft update left them
                updates[-1]["target_sums"] = target_sums(g)
            rec = {"qf1_loss": float(g["qf1_loss"].detach()), "qf2_loss": float(g["qf2_loss"].detach()),
                   "qf1_values": float(g["qf1_a_values"].detach().mean()),
                   "qf2_values": float(g["qf2_a_values"].detach().mean()), "actor_loss": np.nan}
            if not updates:
                d = g["data"]
                rec.update(obs=np_(d.observations), next_obs=np_(d.next_observations), actions=np_(d.actions),
                           rewards=np_(d.rewards).reshape(-1), dones=np_(d.dones).reshape(-1), smooth_draw=smooth[-1],
                           next_state_actions=np_(g["next_state_actions"]), y=np_(g["next_q_value"]),
                           dq1_bias=np_(g["qf1"].fc3.bias.grad), dq2_bias=np_(g["qf2"].fc3.bias.grad))
            out = orig_step(self_, *a, **k)
            rec["q_sums"], rec["actor_sums"] = _sums(g["qf1"], g["qf2"]), np.full(6, np.nan)
            updates.append(rec)
            return out
        if self_ is g["actor_optimizer"]:
            rec = updates[-1]
            rec["actor_loss"] = float(g["actor_loss"].detach())
            out = orig_step(self_, *a, **k)
            rec["actor_sums"] = _sums(g["actor"])
            return out
        return orig_step(self_, *a, **k)

    def randint(*a, **k):
        out = orig_randint(*a, **k)
        samples.append(np.array(out).reshape(-1)[:8].copy())
        return out

    def env_step(self_, act):
        actions.append(np.asarray(act, dtype=np.float32).copy())
        return orig_env_step(self_, act)

    torch.optim.Adam.step, np.random.randint, S.SyntheticGymnasiumVec.step = adam_step, randint, env_step
    torch.randn_like, torch.normal = randn_like, normal
    try:
        rec, g = run_reference("td3_continuous_action.py", argv, gymnasium_kind="continuous")
    finally:
        torch.optim.Adam.step, np.random.randint, S.SyntheticGymnasiumVec.step = orig_step, orig_randint, orig_env_step
        torch.randn_like, torch.normal = orig_randn_like, orig_normal
    updates[-1]["target_sums"] = target_sums(g)
    out = {"argv": np.array(argv), "action_stream": np.stack(actions), "explore_draws": np.stack(explore),
           "randint_heads": np.stack(samples) if samples else np.zeros((0, 8)),
           "actor_keys": np.array(list(g["actor"].state_dict().keys())),
           "qf_keys": np.array(list(g["qf1"].state_dict().keys())),
           "final_sums_actor": _sums(g["actor"]), "final_sums_q": _sums(g["qf1"], g["qf2"])}
    for k in ("qf1_loss", "qf2_loss", "qf1_values", "qf2_values", "actor_loss"):
        out[k] = np.array([u[k] for u in updates])
    for k in ("q_sums", "actor_sums", "target_sums"):
        out[k] = np.stack([u[k] for u in updates])
    first = updates[0]
    for k, v in first.items():
        if isinstance(v, np.ndarray) and k not in ("q_sums", "actor_sums", "target_sums"):
            out["u1_" + k] = v
    for t in sorted({t for t, _, _ in rec.scalars}):      # charts/SPS is wall-clock: its steps are kept, values zeroed
        out["tb/" + t] = np.array([(s_, 0.0 if t == "charts/SPS" else v) for tt, v, s_ in rec.scalars if tt == t],
                                  dtype=np.float64)
    np.savez_compressed(OUT / name, **out)
    print("wrote", name, len(updates), "updates")


def main():
    surface("td3_continuous_surface.json", "td3_continuous_action.py")
    td3_continuous("td3_continuous_n2_seed1.npz", ARGV)
    td3_continuous("td3_continuous_seed2_pf3.npz", ARGV_PF3)


if __name__ == "__main__":
    sys.exit(main())
