"""Generate the continuous-SAC fixtures from the UNMODIFIED reference (build container only).  TEST INFRASTRUCTURE ONLY.

    python -m oracle.make_golden_sac_continuous

* tests/golden/sac_continuous_n2_seed1.npz (autotune, ``--num-envs 2``, a 32-slot ring that wraps) and
  sac_continuous_seed2_alpha01.npz (seed 2, ``--no-autotune --alpha 0.1 --policy-frequency 3
  --target-network-frequency 2``): cleanrl/sac_continuous_action.py (+ the reference's own ReplayBuffer) on the synthetic
  HalfCheetah-shaped gymnasium env.  Per update: both critic losses, the logged q means, alpha before the update and,
  on updates with actor steps, the last actor loss, alpha_loss and log_alpha (NaN otherwise), and each network's
  parameter sums after the update; the first update's full tensors (the sampled batch, every standard-normal draw of the
  update in order, next-state log_pi, y, the fc3 bias gradients); the randint heads, the per-step action stream, the state_dict keys and the TensorBoard series.
* tests/golden/sac_continuous_surface.json: the script's Args fields (default, help text) and top-level names.
"""
from __future__ import annotations

import sys

import numpy as np

from oracle.make_golden import OUT
from oracle.make_golden_c51 import surface
from oracle.ref_harness import run_reference

ARGV = ["--no-cuda", "--total-timesteps", "120", "--learning-starts", "40", "--buffer-size", "64", "--batch-size", "8",
        "--num-envs", "2", "--seed", "1"]
ARGV_FIXED_ALPHA = ["--no-cuda", "--total-timesteps", "120", "--learning-starts", "40", "--buffer-size", "64",
                    "--batch-size", "8", "--seed", "2", "--no-autotune", "--alpha", "0.1", "--policy-frequency", "3",
                    "--target-network-frequency", "2"]


def _script_globals():
    f = sys._getframe(1)
    while f is not None:
        if f.f_globals.get("__name__") == "__main__" and "qf1" in f.f_globals and "q_optimizer" in f.f_globals:
            return f.f_globals
        f = f.f_back
    return None


def _sums(*nets):
    return np.array([p.detach().double().sum().item() for n in nets for p in n.parameters()])


def sac_continuous(name, argv):
    import torch
    import torch.distributions.normal as normal_mod
    from cleanrl_b200 import synthetic_envs as S
    updates, samples, actions, draws = [], [], [], []
    orig_step, orig_randint, orig_env_step = torch.optim.Adam.step, np.random.randint, S.SyntheticGymnasiumVec.step
    orig_std_normal = normal_mod._standard_normal

    def np_(t):
        return t.detach().numpy().copy()

    def std_normal(*a, **k):
        out = orig_std_normal(*a, **k)
        draws.append(out.detach().numpy().copy())
        return out

    def adam_step(self_, *a, **k):
        g = _script_globals()
        if g is None:
            return orig_step(self_, *a, **k)
        if self_ is g["q_optimizer"]:
            rec = {"qf1_loss": float(g["qf1_loss"].detach()), "qf2_loss": float(g["qf2_loss"].detach()),
                   "qf1_values": float(g["qf1_a_values"].detach().mean()),
                   "qf2_values": float(g["qf2_a_values"].detach().mean()), "alpha": float(g["alpha"]),
                   "actor_loss": np.nan, "alpha_loss": np.nan, "log_alpha": np.nan, "n_draws": len(draws)}
            if not updates:
                d = g["data"]
                rec.update(obs=np_(d.observations), next_obs=np_(d.next_observations), actions=np_(d.actions),
                           rewards=np_(d.rewards).reshape(-1), dones=np_(d.dones).reshape(-1),
                           next_logpi=np_(g["next_state_log_pi"]).reshape(-1), y=np_(g["next_q_value"]),
                           dq1_bias=np_(g["qf1"].fc3.bias.grad), dq2_bias=np_(g["qf2"].fc3.bias.grad))
            out = orig_step(self_, *a, **k)
            rec["q_sums"], rec["actor_sums"] = _sums(g["qf1"], g["qf2"]), np.full(8, np.nan)
            updates.append(rec)
            return out
        rec = updates[-1]
        if self_ is g["actor_optimizer"]:
            rec["actor_loss"] = float(g["actor_loss"].detach())
            out = orig_step(self_, *a, **k)
            rec["actor_sums"] = _sums(g["actor"])
            return out
        if self_ is g["a_optimizer"]:
            rec["alpha_loss"] = float(g["alpha_loss"].detach())
            out = orig_step(self_, *a, **k)
            rec["log_alpha"] = float(g["log_alpha"].detach())
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
    normal_mod._standard_normal = std_normal
    try:
        rec, g = run_reference("sac_continuous_action.py", argv, gymnasium_kind="continuous")
    finally:
        torch.optim.Adam.step, np.random.randint, S.SyntheticGymnasiumVec.step = orig_step, orig_randint, orig_env_step
        normal_mod._standard_normal = orig_std_normal
    out = {"argv": np.array(argv), "action_stream": np.stack(actions),
           "randint_heads": np.stack(samples) if samples else np.zeros((0, 8)),
           "actor_keys": np.array(list(g["actor"].state_dict().keys())),
           "qf_keys": np.array(list(g["qf1"].state_dict().keys())),
           "final_sums_actor": _sums(g["actor"]), "final_sums_q": _sums(g["qf1"], g["qf2"]),
           "final_sums_qt": _sums(g["qf1_target"], g["qf2_target"])}
    for k in ("qf1_loss", "qf2_loss", "qf1_values", "qf2_values", "alpha", "actor_loss", "alpha_loss", "log_alpha"):
        out[k] = np.array([u[k] for u in updates])
    for k in ("q_sums", "actor_sums"):
        out[k] = np.stack([u[k] for u in updates])
    # an update's draws: its next_obs draw (the last one before its q step) up to the next step's rollout draw
    def update_draws(k):
        return np.stack(draws[updates[k]["n_draws"] - 1:updates[k + 1]["n_draws"] - 2])

    first = updates[0]
    out["u1_draws"] = update_draws(0)
    for k, v in first.items():
        if isinstance(v, np.ndarray) and k not in ("q_sums", "actor_sums"):
            out["u1_" + k] = v
    for t in sorted({t for t, _, _ in rec.scalars}):      # charts/SPS is wall-clock: its steps are kept, values zeroed
        out["tb/" + t] = np.array([(s_, 0.0 if t == "charts/SPS" else v) for tt, v, s_ in rec.scalars if tt == t],
                                  dtype=np.float64)
    np.savez_compressed(OUT / name, **out)
    print("wrote", name, len(updates), "updates")


def main():
    surface("sac_continuous_surface.json", "sac_continuous_action.py")
    sac_continuous("sac_continuous_n2_seed1.npz", ARGV)
    sac_continuous("sac_continuous_seed2_alpha01.npz", ARGV_FIXED_ALPHA)


if __name__ == "__main__":
    sys.exit(main())
