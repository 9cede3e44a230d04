"""Generate the C51 fixtures from the UNMODIFIED reference (build container only).  TEST INFRASTRUCTURE ONLY.

    python -m oracle.make_golden_c51

* tests/golden/c51_atari_b8_seed1.npz: cleanrl/c51_atari.py (+ the reference's own ReplayBuffer) on the synthetic
  gymnasium Atari env: per update the loss, the logged q_values and the sampled index heads; the first update's
  online / target logits, actions, rewards, dones and target_pmfs; the per-step action stream; the final parameter
  sums; the state_dict keys; the TensorBoard series.
* tests/golden/c51_atari_surface.json: the script's Args fields (default, help text) and top-level names.
"""
from __future__ import annotations

import ast
import json
import sys

import numpy as np

from oracle.make_golden import OUT
from oracle.ref_harness import REFERENCE_ROOT, run_reference

ARGV = ["--no-cuda", "--total-timesteps", "260", "--learning-starts", "40", "--buffer-size", "64", "--batch-size", "8",
        "--train-frequency", "4", "--target-network-frequency", "20", "--seed", "1"]


def _script_globals():
    f = sys._getframe(1)
    while f is not None:
        if f.f_globals.get("__name__") == "__main__" and "q_network" in f.f_globals and "target_pmfs" in f.f_globals:
            return f.f_globals
        f = f.f_back
    return None


def c51(name, argv):
    import torch
    from cleanrl_b200 import synthetic_envs as S
    updates, samples, actions = [], [], []
    orig_step, orig_randint, orig_env_step = torch.optim.Adam.step, np.random.randint, S.SyntheticGymnasiumVec.step

    def adam_step(self_, *a, **k):
        g = _script_globals()
        if g is not None:
            rec = {"loss": float(g["loss"].detach()),
                   "q_values": float((g["old_pmfs"].detach() * g["q_network"].atoms).sum(1).mean())}
            if not updates:
                data = g["data"]
                with torch.no_grad():
                    rec["logits"] = g["q_network"].network(data.observations / 255.0).numpy()
                    rec["next_logits"] = g["target_network"].network(data.next_observations / 255.0).numpy()
                rec["actions"] = data.actions.view(-1).numpy().copy()
                rec["rewards"] = data.rewards.view(-1).numpy().copy()
                rec["dones"] = data.dones.view(-1).numpy().copy()
                rec["target_pmfs"] = g["target_pmfs"].numpy().copy()
            updates.append(rec)
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
        rec, g = run_reference("c51_atari.py", argv, gymnasium_kind="atari")
    finally:
        torch.optim.Adam.step, np.random.randint, S.SyntheticGymnasiumVec.step = orig_step, orig_randint, orig_env_step
    qn = g["q_network"]
    first = updates[0]
    out = {"argv": np.array(argv), "losses": np.array([u["loss"] for u in updates]),
           "q_values": np.array([u["q_values"] for u in updates]),
           "randint_heads": np.stack(samples[:64]) if samples else np.zeros((0, 8)),
           "action_stream": np.array(actions, dtype=np.int64),
           "param_sums": np.array([p.detach().double().sum().item() for p in qn.parameters()]),
           "param_abs_sums": np.array([p.detach().double().abs().sum().item() for p in qn.parameters()]),
           "atoms": qn.atoms.numpy().copy(),
           "state_dict_keys": np.array(list(qn.state_dict().keys()))}
    for k in ("logits", "next_logits", "actions", "rewards", "dones", "target_pmfs"):
        out["u1_" + k] = first[k]
    for t in sorted({t for t, _, _ in rec.scalars}):
        out["tb/" + t] = np.array([(s_, v) for tt, v, s_ in rec.scalars if tt == t], dtype=np.float64)
    np.savez_compressed(OUT / name, **out)
    print("wrote", name, len(updates), "updates")


def surface(name, script="c51_atari.py"):
    """Args fields of the reference script (default, or "<expr>" where the default is not a literal, and the help
    string) and its top-level class / function names."""
    tree = ast.parse((REFERENCE_ROOT / "cleanrl" / script).read_text())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "Args")
    fields = []
    for i, node in enumerate(cls.body):
        if isinstance(node, ast.AnnAssign):
            try:
                default = ast.literal_eval(node.value)
            except Exception:
                default = "<expr>"
            doc = None
            if i + 1 < len(cls.body) and isinstance(cls.body[i + 1], ast.Expr) and isinstance(cls.body[i + 1].value, ast.Constant):
                doc = cls.body[i + 1].value.value
            fields.append([node.target.id, default, doc])
    names = [n.name for n in tree.body if isinstance(n, (ast.ClassDef, ast.FunctionDef))]
    (OUT / name).write_text(json.dumps({script: {"args": fields, "names": names}}, indent=1, sort_keys=True) + "\n")


def main():
    surface("c51_atari_surface.json")
    c51("c51_atari_b8_seed1.npz", ARGV)


if __name__ == "__main__":
    sys.exit(main())
