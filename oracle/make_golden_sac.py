"""Generate the SAC fixtures from the UNMODIFIED reference (build container only).  TEST INFRASTRUCTURE ONLY.

    python -m oracle.make_golden_sac

* tests/golden/sac_atari_b8_seed1.npz (autotune) and sac_atari_b8_seed2_alpha01.npz (seed 2, ``--no-autotune --alpha 0.1``):
  cleanrl/sac_atari.py (+ the reference's own ReplayBuffer) on the synthetic gymnasium Atari env.  Per update: both
  critic losses, the logged q means, the actor loss, alpha before the update, alpha_loss, log_alpha and its gradient, and
  each network's parameter sums after its optimiser step; the first update's full tensors (sampled actions / rewards / dones, target-side logp /
  probs / Q, y, pre- and post-step Q values, actor logp / probs, head bias gradients); the randint heads, the per-step
  action stream, the state_dict keys and the TensorBoard series.  The three optimisers are told apart by identity.
* tests/golden/sac_atari_surface.json: the script's Args fields (default, help text) and top-level names.
"""
from __future__ import annotations

import sys

import numpy as np

from oracle.make_golden import OUT
from oracle.make_golden_c51 import surface
from oracle.ref_harness import run_reference

ARGV = ["--no-cuda", "--total-timesteps", "300", "--learning-starts", "40", "--buffer-size", "64", "--batch-size", "8",
        "--update-frequency", "4", "--target-network-frequency", "40", "--seed", "1"]
ARGV_FIXED_ALPHA = ARGV[:-1] + ["2", "--no-autotune", "--alpha", "0.1"]


def _script_globals():
    f = sys._getframe(1)
    while f is not None:
        if f.f_globals.get("__name__") == "__main__" and "qf1" in f.f_globals and "q_optimizer" in f.f_globals:
            return f.f_globals
        f = f.f_back
    return None


def _sums(net):
    return np.array([p.detach().double().sum().item() for p in net.parameters()])


def sac(name, argv):
    import torch
    from cleanrl_b200 import synthetic_envs as S
    updates, samples, actions = [], [], []
    orig_step, orig_randint, orig_env_step = torch.optim.Adam.step, np.random.randint, S.SyntheticGymnasiumVec.step

    def np_(t):
        return t.detach().numpy().copy()

    def adam_step(self_, *a, **k):
        g = _script_globals()
        if g is None:
            return orig_step(self_, *a, **k)
        if self_ is g["q_optimizer"]:
            rec = {"qf1_loss": float(g["qf1_loss"].detach()), "qf2_loss": float(g["qf2_loss"].detach()),
                   "qf1_values": float(g["qf1_a_values"].detach().mean()),
                   "qf2_values": float(g["qf2_a_values"].detach().mean()), "alpha": float(g["alpha"])}
            if not updates:
                d = g["data"]
                rec.update(actions=d.actions.view(-1).numpy().copy(), rewards=d.rewards.view(-1).numpy().copy(),
                           dones=d.dones.view(-1).numpy().copy(), next_logp=np_(g["next_state_log_pi"]),
                           next_probs=np_(g["next_state_action_probs"]), q1t=np_(g["qf1_next_target"]),
                           q2t=np_(g["qf2_next_target"]), y=np_(g["next_q_value"]), q1=np_(g["qf1_values"]),
                           q2=np_(g["qf2_values"]), dq1_bias=np_(g["qf1"].fc_q.bias.grad),
                           dq2_bias=np_(g["qf2"].fc_q.bias.grad))
            out = orig_step(self_, *a, **k)
            rec["qf1_sums"], rec["qf2_sums"] = _sums(g["qf1"]), _sums(g["qf2"])
            updates.append(rec)
            return out
        rec = updates[-1]
        if self_ is g["actor_optimizer"]:
            rec["actor_loss"] = float(g["actor_loss"].detach())
            if len(updates) == 1:
                rec.update(post_q1=np_(g["qf1_values"]), post_q2=np_(g["qf2_values"]), logp=np_(g["log_pi"]),
                           probs=np_(g["action_probs"]), dl_bias=np_(g["actor"].fc_logits.bias.grad))
            out = orig_step(self_, *a, **k)
            rec["actor_sums"] = _sums(g["actor"])
            return out
        if self_ is g["a_optimizer"]:
            rec["alpha_loss"] = float(g["alpha_loss"].detach())
            rec["log_alpha_grad"] = float(g["log_alpha"].grad)
            out = orig_step(self_, *a, **k)
            rec["log_alpha"] = float(g["log_alpha"].detach())
            return out
        return orig_step(self_, *a, **k)

    def randint(*a, **k):
        out = orig_randint(*a, **k)
        samples.append(np.array(out).reshape(-1)[:8].copy())
        return out

    def env_step(self_, act):
        actions.append(int(np.asarray(act).reshape(-1)[0]))
        return orig_env_step(self_, act)

    torch.optim.Adam.step, np.random.randint, S.SyntheticGymnasiumVec.step = adam_step, randint, env_step
    try:
        rec, g = run_reference("sac_atari.py", argv, gymnasium_kind="atari")
    finally:
        torch.optim.Adam.step, np.random.randint, S.SyntheticGymnasiumVec.step = orig_step, orig_randint, orig_env_step
    out = {"argv": np.array(argv), "action_stream": np.array(actions, dtype=np.int64),
           "randint_heads": np.stack(samples[:96]) if samples else np.zeros((0, 8)),
           "actor_keys": np.array(list(g["actor"].state_dict().keys())),
           "qf_keys": np.array(list(g["qf1"].state_dict().keys())),
           "target_entropy": np.float32(g["target_entropy"]) if "target_entropy" in g else np.float32(0)}
    for k in ("qf1_loss", "qf2_loss", "qf1_values", "qf2_values", "alpha", "actor_loss", "alpha_loss", "log_alpha",
              "log_alpha_grad"):
        if k in updates[0]:
            out[k] = np.array([u[k] for u in updates])
    for k in ("qf1_sums", "qf2_sums", "actor_sums"):
        out[k] = np.stack([u[k] for u in updates])
    for k, v in updates[0].items():
        if isinstance(v, np.ndarray) and k not in ("qf1_sums", "qf2_sums", "actor_sums"):
            out["u1_" + k] = v
    for t in sorted({t for t, _, _ in rec.scalars}):
        out["tb/" + t] = np.array([(s_, v) for tt, v, s_ in rec.scalars if tt == t], dtype=np.float64)
    np.savez_compressed(OUT / name, **out)
    print("wrote", name, len(updates), "updates")


def main():
    surface("sac_atari_surface.json", "sac_atari.py")
    sac("sac_atari_b8_seed1.npz", ARGV)
    sac("sac_atari_b8_seed2_alpha01.npz", ARGV_FIXED_ALPHA)


if __name__ == "__main__":
    sys.exit(main())
