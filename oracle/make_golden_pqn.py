"""Generate the PQN fixtures from the UNMODIFIED reference (build container only).  TEST INFRASTRUCTURE ONLY.

    python -m oracle.make_golden_pqn

* tests/golden/pqn_seed1.npz and pqn_seed2_mb.npz: cleanrl/pqn.py on the CartPole-v1 dynamics of
  ``synthetic_envs.CartPoleVec``.  Recorded: the initial parameters (flat, nn.Module order) and state_dict keys; per
  iteration obs / actions / rewards / dones / values / returns / next_obs / next_done; per env step the
  ``torch.randint`` and ``torch.rand`` draws and epsilon; per RAdam step mb_inds (padded with -1), the loss, mean(q),
  the pre-clip norm and the parameter sums after the step; the TensorBoard series.
* tests/golden/pqn_surface.json: the script's Args fields (default, help text) and top-level names.

The script's ``torch.optim.RAdam.step``, ``torch.randint``, ``torch.rand``, ``torch.argmax`` and
``nn.utils.clip_grad_norm_`` are wrapped here (``ref_harness`` hooks Adam and ends an iteration on
``charts/learning_rate``, which pqn.py never logs; an iteration ends here on ``losses/td_loss``).  The generator
asserts each run's update count, how often the clip binds, the RAdam steps at rho_t > 5, the minibatch sizes, and that
the smallest greedy Q margin (top-1 minus top-2) exceeds 1e-3 so an exact action comparison is fair.  The .npz files are
written with fixed zip timestamps, so a rerun reproduces them byte for byte.
"""
from __future__ import annotations

import sys

import numpy as np

from oracle.make_golden_c51 import surface
from oracle.make_golden_ddpg_continuous import _savez
from oracle.make_golden import OUT
from oracle.ref_harness import run_reference

ARGV1 = ["--no-cuda", "--seed", "1", "--num-envs", "4", "--num-steps", "16", "--total-timesteps", "192"]
ARGV2 = ["--no-cuda", "--seed", "2", "--num-envs", "3", "--num-steps", "10", "--total-timesteps", "90",
         "--num-minibatches", "4", "--update-epochs", "3", "--q-lambda", "0.3", "--gamma", "0.9", "--max-grad-norm",
         "1000", "--no-anneal-lr", "--exploration-fraction", "0.2", "--learning-rate", "1e-3"]
# (updates, clip binds, RAdam steps at rho_t > 5, minibatch sizes) the issue's table states for each run
EXPECT = {"pqn_seed1.npz": (48, 48, 43, {16}), "pqn_seed2_mb.npz": (45, 0, 40, {7, 2})}


def _script_globals():
    f = sys._getframe(1)
    while f is not None:
        if f.f_globals.get("__name__") == "__main__" and "q_network" in f.f_globals:
            return f.f_globals
        f = f.f_back
    return None


def _sums(net):
    return np.array([p.detach().double().sum().item() for p in net.parameters()])


def pqn(name, argv):
    import torch
    from oracle import pqn_oracle as O
    iters, steps, updates, margins, init = [], [], [], [], {}
    orig = dict(step=torch.optim.RAdam.step, randint=torch.randint, rand=torch.rand, argmax=torch.argmax,
                clip=torch.nn.utils.clip_grad_norm_)
    norms = []

    def np_(t):
        return t.detach().cpu().numpy().copy()

    def randint(*a, **k):
        out = orig["randint"](*a, **k)
        g = _script_globals()
        if g is not None:
            if not init:
                net = g["q_network"]
                init["flat"] = np.concatenate([np_(p).reshape(-1) for p in net.parameters()])
                init["keys"] = list(net.state_dict().keys())
            steps.append({"randint": np_(out), "eps": float(g["epsilon"])})
        return out

    def rand(*a, **k):
        out = orig["rand"](*a, **k)
        if _script_globals() is not None and steps and "rand" not in steps[-1]:
            steps[-1]["rand"] = np_(out)
        return out

    def argmax(x, *a, **k):
        if _script_globals() is not None and x.dim() == 2:
            s = torch.sort(x.detach(), dim=1, descending=True).values
            margins.append(float((s[:, 0] - s[:, 1]).min()))
        return orig["argmax"](x, *a, **k)

    def clip(parameters, *a, **k):
        out = orig["clip"](parameters, *a, **k)
        norms.append(float(out))
        return out

    def radam_step(self_, *a, **k):
        g = _script_globals()
        out = orig["step"](self_, *a, **k)
        if g is not None:
            mb = np.asarray(g["mb_inds"]).copy()
            updates.append({"mb": mb, "loss": float(g["loss"].detach()), "qmean": float(g["old_val"].detach().mean()),
                            "norm": norms[-1], "sums": _sums(g["q_network"]), "lr": float(self_.param_groups[0]["lr"])})
        return out

    def end_of_iteration():
        g = _script_globals()
        iters.append({k: np_(g[k]) for k in ("obs", "actions", "rewards", "dones", "values", "returns", "next_obs",
                                              "next_done")})

    torch.randint, torch.rand, torch.argmax = randint, rand, argmax
    torch.nn.utils.clip_grad_norm_, torch.optim.RAdam.step = clip, radam_step
    try:
        rec, g = _run_with_iteration_hook(end_of_iteration, argv)
    finally:
        torch.randint, torch.rand, torch.argmax = orig["randint"], orig["rand"], orig["argmax"]
        torch.nn.utils.clip_grad_norm_, torch.optim.RAdam.step = orig["clip"], orig["step"]

    args = g["args"]
    n_upd, n_clip, n_rect, sizes = EXPECT[name]
    assert len(updates) == n_upd, (name, len(updates))
    assert sum(u["norm"] > args.max_grad_norm for u in updates) == n_clip, name
    assert sum(O.radam_scalars(i + 1, 1.0)[3] is not None for i in range(len(updates))) == n_rect, name
    assert {len(u["mb"]) for u in updates} == sizes, name
    assert min(margins) > 1e-3, (name, min(margins))
    mbs = max(len(u["mb"]) for u in updates)
    out = {"argv": np.array(argv), "init_flat": init["flat"], "keys": np.array(init["keys"]),
           "min_margin": np.float64(min(margins)),
           "randint": np.stack([s["randint"] for s in steps]), "rand": np.stack([s["rand"] for s in steps]),
           "eps": np.array([s["eps"] for s in steps]),
           "mb_inds": np.stack([np.pad(u["mb"], (0, mbs - len(u["mb"])), constant_values=-1) for u in updates]),
           "mb_len": np.array([len(u["mb"]) for u in updates]),
           "loss": np.array([u["loss"] for u in updates]), "qmean": np.array([u["qmean"] for u in updates]),
           "norm": np.array([u["norm"] for u in updates]), "lr": np.array([u["lr"] for u in updates]),
           "param_sums": np.stack([u["sums"] for u in updates])}
    for k in iters[0]:
        out["it_" + k] = np.stack([it[k] for it in iters])
    for t in sorted({t for t, _, _ in rec.scalars}):      # charts/SPS is wall-clock: its steps are kept, values zeroed
        out["tb/" + t] = np.array([(s_, 0.0 if t == "charts/SPS" else v) for tt, v, s_ in rec.scalars if tt == t],
                                  dtype=np.float64)
    _savez(OUT / name, out)
    print("wrote", name, len(updates), "updates, min margin", min(margins))


def _run_with_iteration_hook(on_td_loss, argv):
    """run_reference with ``on_td_loss()`` called whenever the script logs losses/td_loss (the end of an iteration's
    update, before its rollout buffers are reused).  ref_harness installs its capturing writer class just before it
    calls ``runpy.run_path``; the wrapper below extends that class's add_scalar at that point."""
    import runpy

    import torch.utils.tensorboard as tb
    orig_run_path = runpy.run_path

    def run_path(path, *a, **k):
        writer_cls = tb.SummaryWriter
        orig_add = writer_cls.add_scalar

        def add_scalar(self_, tag, value, step=None, *a_, **k_):
            if tag == "losses/td_loss":
                on_td_loss()
            return orig_add(self_, tag, value, step, *a_, **k_)

        writer_cls.add_scalar = add_scalar
        return orig_run_path(path, *a, **k)

    runpy.run_path = run_path
    try:
        return run_reference("pqn.py", argv, gymnasium_kind="cartpole")
    finally:
        runpy.run_path = orig_run_path


def main():
    surface("pqn_surface.json", "pqn.py")
    pqn("pqn_seed1.npz", ARGV1)
    pqn("pqn_seed2_mb.npz", ARGV2)


if __name__ == "__main__":
    sys.exit(main())
