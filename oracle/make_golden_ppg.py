"""Generate the PPG fixtures from the UNMODIFIED reference (build container only).  TEST INFRASTRUCTURE ONLY.

    python -m oracle.make_golden_ppg

* tests/golden/ppg_procgen_n4_t8_seed3.npz and ..._accum2.npz: cleanrl/ppg_procgen.py on the procgen-shaped synthetic
  env, two phases of (2 policy iterations x 2 minibatches, then 2 auxiliary epochs x 4 minibatches of 2 rollouts), the
  second with ``--n-aux-grad-accum 2``.  Recorded: the rollout tensors of every policy iteration; per Adam step the phase
  it belongs to, every parameter tensor's sum before / after, the post-clip gradient and the values before / after of the
  head tensors but the actor weight (the trajectory the Adam oracle replays: ``aux_critic`` has no gradient in a policy phase), Adam's
  per-tensor ``step``; per auxiliary minibatch the three losses, the rollout columns and, for the first one of each phase,
  the head outputs, old logits and returns the losses were computed from; ``aux_pi`` and ``aux_returns`` of each phase;
  the logged scalars; a SHA-256 of every freshly initialised parameter tensor.
* tests/golden/ppg_procgen_surface.json: the script's Args fields (default, help text) and top-level names.
"""
from __future__ import annotations

import hashlib
import sys

import numpy as np

from oracle.make_golden import OUT
from oracle.make_golden_c51 import surface
from oracle import ref_harness
from oracle.ref_harness import _main_globals, _np, run_reference

ARGV = ["--no-cuda", "--num-envs", "4", "--num-steps", "8", "--total-timesteps", "128", "--seed", "3",
        "--n-iteration", "2", "--e-auxiliary", "2", "--num-aux-rollouts", "2", "--num-minibatches", "2"]
HEADS = ("actor.bias", "critic.weight", "critic.bias", "aux_critic.weight", "aux_critic.bias")


class _Space:
    def __init__(self, shape=None, n=None):
        self.shape, self.n = shape, n


class _Envs:
    single_observation_space = _Space(shape=(64, 64, 3))
    single_action_space = _Space(shape=(), n=15)


def ppg(name, argv):
    import torch
    from torch import distributions as td
    steps, aux, phases = [], [], []
    state = {"kl": None, "phase_first": True}
    orig_step, orig_kl, orig_backward = torch.optim.Adam.step, td.kl_divergence, torch.Tensor.backward

    def kl_divergence(p, q):
        out = orig_kl(p, q)
        state["kl"] = (p.logits.detach(), q.logits.detach())
        return out

    def backward(self_, *a, **k):
        g = _main_globals() if state["kl"] is not None else None
        if g is not None:
            rec = {"kl_loss": float(g["kl_loss"].detach()), "aux_value_loss": float(g["aux_value_loss"].detach()),
                   "real_value_loss": float(g["real_value_loss"].detach()), "cols": _np(g["aux_minibatch_ind"]),
                   "phase": int(g["phase"])}
            if not aux or aux[-1]["phase"] != rec["phase"]:
                old, new = state["kl"]
                rec["first"] = {"old_logits": _np(old), "new_logits": _np(new), "new_values": _np(g["new_values"]),
                                "new_aux_values": _np(g["new_aux_values"]), "returns": _np(g["m_aux_returns"])}
                phases.append({"aux_pi": _np(g["aux_pi"]), "aux_returns": _np(g["aux_returns"])})
            aux.append(rec)
        out = orig_backward(self_, *a, **k)
        if g is not None:
            state["kl"] = None
            if "first" in aux[-1]:
                # d(loss)/d(head outputs) is not retained by autograd: the agent's head gradients identify it instead
                aux[-1]["first"]["critic_bias_grad"] = _np(g["agent"].critic.bias.grad)
        return out

    def adam_step(self_, *a, **k):
        g = _main_globals()
        sd = dict(g["agent"].named_parameters())
        rec = {"aux": len(aux) > 0 and aux[-1]["phase"] == int(g["phase"]), "lr": float(self_.param_groups[0]["lr"]),
               "has_grad": np.array([p.grad is not None for p in sd.values()]),
               "sums_before": np.array([p.detach().double().sum().item() for p in sd.values()]),
               "before": np.concatenate([_np(sd[k]).reshape(-1) for k in HEADS]),
               "grad": np.concatenate([(_np(sd[k].grad) if sd[k].grad is not None else np.full(sd[k].shape, np.nan, np.float32)
                                        ).reshape(-1) for k in HEADS])}
        out = orig_step(self_, *a, **k)
        rec["sums_after"] = np.array([p.detach().double().sum().item() for p in sd.values()])
        rec["after"] = np.concatenate([_np(sd[k]).reshape(-1) for k in HEADS])
        rec["adam_step"] = np.array([float(self_.state[p]["step"]) if p in self_.state and len(self_.state[p]) else 0.0
                                     for p in sd.values()])
        steps.append(rec)
        return out

    # the harness's own per-step record reads every parameter's gradient; ``aux_critic`` has none in a policy phase
    orig_rec = ref_harness.Recorder.on_adam_step
    ref_harness.Recorder.on_adam_step = lambda self_, g, before: None
    torch.optim.Adam.step, td.kl_divergence, torch.Tensor.backward = adam_step, kl_divergence, backward
    try:
        rec, g = run_reference("ppg_procgen.py", argv)
    finally:
        torch.optim.Adam.step, td.kl_divergence, torch.Tensor.backward = orig_step, orig_kl, orig_backward
        ref_harness.Recorder.on_adam_step = orig_rec

    torch.manual_seed(3)
    fresh = g["Agent"](_Envs())
    out = {"argv": np.array(argv), "param_names": np.array([k for k, _ in g["agent"].named_parameters()]),
           "head_names": np.array(HEADS),
           "head_sizes": np.array([dict(g["agent"].named_parameters())[k].numel() for k in HEADS]),
           "init_seed": np.array(3),
           "init_sha256": np.array([hashlib.sha256(v.detach().numpy().tobytes()).hexdigest() for v in fresh.state_dict().values()]),
           "init_keys": np.array(list(fresh.state_dict().keys()))}
    for k in ("actions", "logprobs", "rewards", "dones", "values", "advantages", "returns", "next_done"):
        out[k] = np.stack([r[k] for r in rec.iterations])
    for k in ("aux", "lr", "has_grad", "sums_before", "sums_after", "before", "after", "grad", "adam_step"):
        out["step_" + k] = np.stack([np.asarray(s[k]) for s in steps])
    for k in ("kl_loss", "aux_value_loss", "real_value_loss", "cols", "phase"):
        out["aux_" + k] = np.stack([np.asarray(a[k]) for a in aux])
    firsts = [a["first"] for a in aux if "first" in a]
    for k in firsts[0]:
        out["first_" + k] = np.stack([f[k] for f in firsts])
    out["aux_pi"] = np.stack([p["aux_pi"] for p in phases])
    out["aux_returns"] = np.stack([p["aux_returns"] for p in phases])
    out["shuffles"] = np.stack([s[:8] for s in rec.shuffles])
    for t in sorted({t for t, _, _ in rec.scalars}):
        out["tb/" + t] = np.array([(s_, v) for tt, v, s_ in rec.scalars if tt == t], dtype=np.float64)
    np.savez_compressed(OUT / name, **out)
    print("wrote", name, len(steps), "Adam steps,", len(aux), "auxiliary minibatches")


def main():
    surface("ppg_procgen_surface.json", script="ppg_procgen.py")
    ppg("ppg_procgen_n4_t8_seed3.npz", ARGV)
    ppg("ppg_procgen_n4_t8_seed3_accum2.npz", ARGV + ["--n-aux-grad-accum", "2"])


if __name__ == "__main__":
    sys.exit(main())
