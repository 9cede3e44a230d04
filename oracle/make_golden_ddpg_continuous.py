"""Generate the DDPG fixtures from the UNMODIFIED reference (build container only).  TEST INFRASTRUCTURE ONLY.

    python -m oracle.make_golden_ddpg_continuous

* tests/golden/ddpg_continuous_seed1.npz (the defaults with a 64-slot ring that wraps, batch 8) and
  ddpg_continuous_seed2_pf3.npz (seed 2, ``--policy-frequency 3 --exploration-noise 0.3 --tau 0.02``, with the vector
  env's ``action_space`` batched to (1, D) as gymnasium's one-env ``SyncVectorEnv`` has it, so the actor's buffers and
  the exploration draws are [1, D]): cleanrl/ddpg_continuous_action.py (+ the reference's own ReplayBuffer) on the
  synthetic HalfCheetah-shaped gymnasium env.  Per update: qf1_loss and the logged q mean, actor_loss on policy steps
  (NaN otherwise), and the parameter sums after the update of the actor (NaN on critic-only updates), qf1 and both
  targets; the first update's full tensors (the sampled batch, next_state_actions, y, the fc3 bias gradient); every
  exploration draw, the per-step action stream, the randint heads, the state_dict keys and shapes and the TensorBoard
  series.
* tests/golden/ddpg_continuous_surface.json: the script's Args fields (default, help text) and top-level names.

The .npz files are written with fixed zip timestamps, so a rerun reproduces them byte for byte.
"""
from __future__ import annotations

import sys
import zipfile

import numpy as np

from oracle.make_golden import OUT
from oracle.make_golden_c51 import surface
from oracle.ref_harness import run_reference

COMMON = ["--no-cuda", "--total-timesteps", "120", "--learning-starts", "40", "--buffer-size", "64", "--batch-size", "8"]
ARGV = COMMON + ["--seed", "1"]
ARGV_PF3 = COMMON + ["--seed", "2", "--policy-frequency", "3", "--exploration-noise", "0.3", "--tau", "0.02"]


def _script_globals():
    f = sys._getframe(1)
    while f is not None:
        if f.f_globals.get("__name__") == "__main__" and "qf1" in f.f_globals and "q_optimizer" in f.f_globals:
            return f.f_globals
        f = f.f_back
    return None


def _sums(*nets):
    return np.array([p.detach().double().sum().item() for n in nets for p in n.parameters()])


def _savez(path, arrays):
    """np.savez_compressed's layout with a fixed timestamp per member."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for k, v in arrays.items():
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            with zf.open(info, "w", force_zip64=True) as f:
                np.lib.format.write_array(f, np.asanyarray(v), allow_pickle=False)


def ddpg_continuous(name, argv, batched_action_space=False):
    import torch
    from cleanrl_b200 import synthetic_envs as S
    updates, samples, actions, explore = [], [], [], []
    orig_step, orig_randint, orig_env_step = torch.optim.Adam.step, np.random.randint, S.SyntheticGymnasiumVec.step
    orig_init, orig_normal = S.SyntheticGymnasiumVec.__init__, torch.normal

    def np_(t):
        return t.detach().numpy().copy()

    def init(self_, *a, **k):
        orig_init(self_, *a, **k)
        if batched_action_space:          # gymnasium's SyncVectorEnv: action_space is the batched Box [num_envs, D]
            sp = self_.single_action_space
            self_.action_space = S.Box(-1.0, 1.0, (self_.num_envs,) + sp.shape, np.float32)

    def normal(*a, **k):
        out = orig_normal(*a, **k)
        explore.append(np_(out))
        return out

    def target_sums(g):
        return _sums(g["target_actor"], g["qf1_target"])

    def adam_step(self_, *a, **k):
        g = _script_globals()
        if g is None:
            return orig_step(self_, *a, **k)
        if self_ is g["q_optimizer"]:
            if updates:                   # the targets as the previous update's soft update left them
                updates[-1]["target_sums"] = target_sums(g)
            rec = {"qf1_loss": float(g["qf1_loss"].detach()), "qf1_values": float(g["qf1_a_values"].detach().mean()),
                   "actor_loss": np.nan}
            if not updates:
                d = g["data"]
                rec.update(obs=np_(d.observations), next_obs=np_(d.next_observations), actions=np_(d.actions),
                           rewards=np_(d.rewards).reshape(-1), dones=np_(d.dones).reshape(-1),
                           next_state_actions=np_(g["next_state_actions"]), y=np_(g["next_q_value"]),
                           dq1_bias=np_(g["qf1"].fc3.bias.grad))
            out = orig_step(self_, *a, **k)
            rec["q_sums"], rec["actor_sums"] = _sums(g["qf1"]), np.full(6, np.nan)
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
    S.SyntheticGymnasiumVec.__init__, torch.normal = init, normal
    try:
        rec, g = run_reference("ddpg_continuous_action.py", argv, gymnasium_kind="continuous")
    finally:
        torch.optim.Adam.step, np.random.randint, S.SyntheticGymnasiumVec.step = orig_step, orig_randint, orig_env_step
        S.SyntheticGymnasiumVec.__init__, torch.normal = orig_init, orig_normal
    updates[-1]["target_sums"] = target_sums(g)
    asd, qsd = g["actor"].state_dict(), g["qf1"].state_dict()
    out = {"argv": np.array(argv), "action_stream": np.stack(actions), "explore_draws": np.stack(explore),
           "randint_heads": np.stack(samples) if samples else np.zeros((0, 8)),
           "actor_keys": np.array(list(asd.keys())), "qf_keys": np.array(list(qsd.keys())),
           "actor_shapes": np.array([str(tuple(v.shape)) for v in asd.values()]),
           "qf_shapes": np.array([str(tuple(v.shape)) for v in qsd.values()]),
           "action_scale": np_(g["actor"].action_scale), "action_bias": np_(g["actor"].action_bias),
           "final_sums_actor": _sums(g["actor"]), "final_sums_q": _sums(g["qf1"])}
    for k in ("qf1_loss", "qf1_values", "actor_loss"):
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
    _savez(OUT / name, out)
    print("wrote", name, len(updates), "updates")


def main():
    surface("ddpg_continuous_surface.json", "ddpg_continuous_action.py")
    ddpg_continuous("ddpg_continuous_seed1.npz", ARGV)
    ddpg_continuous("ddpg_continuous_seed2_pf3.npz", ARGV_PF3, batched_action_space=True)


if __name__ == "__main__":
    sys.exit(main())
