"""CLI surface of the drop-in scripts: same flag names, types, defaults and help
text as the reference ``Args`` dataclasses (cleanrl/ppo.py:17-78,
ppo_atari_envpool.py:19-80, ppo_atari_multigpu.py:29-102,
ppo_continuous_action.py:17-84), parsed by ``tyro.cli`` like the reference.

The dataclasses are generated from one table so the four scripts cannot drift
apart; script-specific defaults are overrides on top of the common PPO block.
Extra (non-reference) flags default to reference behaviour.
"""
from __future__ import annotations

import dataclasses
from typing import Annotated, List, Literal, Optional

import tyro

_COMMON = [
    # name, type, default, help
    ("exp_name", str, None, "the name of this experiment"),
    ("seed", int, 1, "seed of the experiment"),
    ("torch_deterministic", bool, True, "if toggled, `torch.backends.cudnn.deterministic=False`"),
    ("cuda", bool, True, "if toggled, cuda will be enabled by default"),
    ("track", bool, False, "if toggled, this experiment will be tracked with Weights and Biases"),
    ("wandb_project_name", str, "cleanRL", "the wandb's project name"),
    ("wandb_entity", Optional[str], None, "the entity (team) of wandb's project"),
    ("capture_video", bool, False, "whether to capture videos of the agent performances (check out `videos` folder)"),
]
_ALGO = [
    ("env_id", str, "CartPole-v1", "the id of the environment"),
    ("total_timesteps", int, 500000, "total timesteps of the experiments"),
    ("learning_rate", float, 2.5e-4, "the learning rate of the optimizer"),
    ("num_envs", int, 4, "the number of parallel game environments"),
    ("num_steps", int, 128, "the number of steps to run in each environment per policy rollout"),
    ("anneal_lr", bool, True, "Toggle learning rate annealing for policy and value networks"),
    ("gamma", float, 0.99, "the discount factor gamma"),
    ("gae_lambda", float, 0.95, "the lambda for the general advantage estimation"),
    ("num_minibatches", int, 4, "the number of mini-batches"),
    ("update_epochs", int, 4, "the K epochs to update the policy"),
    ("norm_adv", bool, True, "Toggles advantages normalization"),
    ("clip_coef", float, 0.2, "the surrogate clipping coefficient"),
    ("clip_vloss", bool, True, "Toggles whether or not to use a clipped loss for the value function, as per the paper."),
    ("ent_coef", float, 0.01, "coefficient of the entropy"),
    ("vf_coef", float, 0.5, "coefficient of the value function"),
    ("max_grad_norm", float, 0.5, "the maximum norm for the gradient clipping"),
    ("target_kl", Optional[float], None, "the target KL divergence threshold"),
]
_RUNTIME = [
    ("batch_size", int, 0, "the batch size (computed in runtime)"),
    ("minibatch_size", int, 0, "the mini-batch size (computed in runtime)"),
    ("num_iterations", int, 0, "the number of iterations (computed in runtime)"),
]
# flags the reference does not have; defaults keep reference behaviour
_EXTRA = [
    ("precision", Literal["fp32", "bf16"], "fp32",
     "[b200] network arithmetic: fp32 = exact CUDA-core kernels (reference numerics), "
     "bf16 = wgmma tensor-core kernels with fp32 accumulation"),
    ("gae_kernel", Literal["sequential", "scan"], "sequential",
     "[b200] GAE kernel: sequential = bit-identical to the reference loop, scan = chunked affine scan"),
    ("synthetic_env", bool, False,
     "[b200] train on the built-in synthetic vector env instead of the real env library "
     "(never chosen silently: without this flag a missing env library is an error)"),
]


def _make(name, rows):
    fields = []
    for fname, ftype, default, help_ in rows:
        ann = Annotated[ftype, tyro.conf.arg(help=help_)]
        if isinstance(default, list):
            fields.append((fname, ann, dataclasses.field(default_factory=lambda d=default: list(d))))
        else:
            fields.append((fname, ann, dataclasses.field(default=default)))
    return dataclasses.make_dataclass(name, fields)


def _override(rows, **kw):
    out = []
    for r in rows:
        out.append((r[0], r[1], kw.pop(r[0]), r[3]) if r[0] in kw else r)
    assert not kw, kw
    return out


def ppo_args(exp_name="ppo"):
    return _make("Args", _override(_COMMON, exp_name=exp_name) + _ALGO + _RUNTIME + _EXTRA)


_ENV_GROUPS = [
    ("env_groups", int, 1,
     "[b200] split the envs into this many independent vector envs and software-pipeline them: while one group's frames "
     "are evaluated and its env steps on the host, the next group's frames cross PCIe (1 = the reference's loop order)"),
]


def ppo_atari_envpool_args(exp_name="ppo_atari_envpool"):
    algo = _override(_ALGO, env_id="Breakout-v5", total_timesteps=10000000, num_envs=8, clip_coef=0.1)
    return _make("Args", _override(_COMMON, exp_name=exp_name) + algo + _RUNTIME + _EXTRA + _ENV_GROUPS)


def ppo_atari_args(exp_name="ppo_atari"):
    """cleanrl/ppo_atari.py:20-90."""
    algo = _override(_ALGO, env_id="BreakoutNoFrameskip-v4", total_timesteps=10000000, num_envs=8, clip_coef=0.1)
    return _make("Args", _override(_COMMON, exp_name=exp_name) + algo + _RUNTIME + _EXTRA)


def ppo_atari_multigpu_args(exp_name="ppo_atari_multigpu"):
    algo = _override(_ALGO, env_id="BreakoutNoFrameskip-v4", total_timesteps=10000000, clip_coef=0.1)
    algo = [r if r[0] != "num_envs" else
            ("local_num_envs", int, 8, "the number of parallel game environments (in the local rank)") for r in algo]
    dist = [
        ("device_ids", List[int], [], "the device ids that subprocess workers will use"),
        ("backend", Literal["gloo", "nccl", "mpi"], "gloo", "the backend for distributed training"),
    ]
    runtime = [
        ("local_batch_size", int, 0, "the local batch size in the local rank (computed in runtime)"),
        ("local_minibatch_size", int, 0, "the local mini-batch size in the local rank (computed in runtime)"),
        ("num_envs", int, 0, "the number of parallel game environments (computed in runtime)"),
    ] + _RUNTIME + [("world_size", int, 0, "the number of processes (computed in runtime)")]
    return _make("Args", _override(_COMMON, exp_name=exp_name) + algo + dist + runtime + _EXTRA)


def ppo_procgen_args(exp_name="ppo_procgen"):
    """cleanrl/ppo_procgen.py:16-79."""
    algo = _override(_ALGO, env_id="starpilot", total_timesteps=int(25e6), learning_rate=5e-4, num_envs=64, num_steps=256,
                     anneal_lr=False, gamma=0.999, num_minibatches=8, update_epochs=3)
    return _make("Args", _override(_COMMON, exp_name=exp_name) + algo + _RUNTIME + _EXTRA)


def ppo_atari_multigpu_envpool_args(exp_name="ppo_atari_multigpu_envpool"):
    """The script the reference defers (docs/rl-algorithms/ppo.md:1020): ppo_atari_multigpu.py's data parallelism over
    ppo_atari_envpool.py's vector env.  Fields = the multi-GPU script's, env defaults = the envpool script's."""
    algo = _override(_ALGO, env_id="Breakout-v5", total_timesteps=10000000, clip_coef=0.1)
    algo = [r if r[0] != "num_envs" else
            ("local_num_envs", int, 8, "the number of parallel game environments (in the local rank)") for r in algo]
    dist = [
        ("device_ids", List[int], [], "the device ids that subprocess workers will use"),
        ("backend", Literal["gloo", "nccl", "mpi"], "nccl", "the backend for distributed training"),
        ("env_threads", int, 0, "[b200] envpool worker threads per rank (0 = host cores / world size)"),
        ("pin_env_threads", bool, True,
         "[b200] pin each rank (and the env worker threads it spawns) to its own slice of the host cores, so the "
         "ranks' env pools do not fight each other (docs/rl-algorithms/ppo.md:1020)"),
    ]
    runtime = [
        ("local_batch_size", int, 0, "the local batch size in the local rank (computed in runtime)"),
        ("local_minibatch_size", int, 0, "the local mini-batch size in the local rank (computed in runtime)"),
        ("num_envs", int, 0, "the number of parallel game environments (computed in runtime)"),
    ] + _RUNTIME + [("world_size", int, 0, "the number of processes (computed in runtime)")]
    return _make("Args", _override(_COMMON, exp_name=exp_name) + algo + dist + runtime + _EXTRA)


def ppo_continuous_action_args(exp_name="ppo_continuous_action"):
    common = list(_override(_COMMON, exp_name=exp_name))
    common += [
        ("save_model", bool, False, "whether to save model into the `runs/{run_name}` folder"),
        ("upload_model", bool, False, "whether to upload the saved model to huggingface"),
        ("hf_entity", str, "", "the user or org name of the model repository from the Hugging Face Hub"),
    ]
    algo = _override(_ALGO, env_id="HalfCheetah-v4", total_timesteps=1000000, learning_rate=3e-4, num_envs=1,
                     num_steps=2048, num_minibatches=32, update_epochs=10, ent_coef=0.0)
    return _make("Args", common + algo + _RUNTIME + _EXTRA)


def dqn_atari_args(exp_name="dqn_atari"):
    """cleanrl/dqn_atari.py:27-80."""
    common = list(_override(_COMMON, exp_name=exp_name))
    common += [
        ("save_model", bool, False, "whether to save model into the `runs/{run_name}` folder"),
        ("upload_model", bool, False, "whether to upload the saved model to huggingface"),
        ("hf_entity", str, "", "the user or org name of the model repository from the Hugging Face Hub"),
    ]
    algo = [
        ("env_id", str, "BreakoutNoFrameskip-v4", "the id of the environment"),
        ("total_timesteps", int, 10000000, "total timesteps of the experiments"),
        ("learning_rate", float, 1e-4, "the learning rate of the optimizer"),
        ("num_envs", int, 1, "the number of parallel game environments"),
        ("buffer_size", int, 1000000, "the replay memory buffer size"),
        ("gamma", float, 0.99, "the discount factor gamma"),
        ("tau", float, 1.0, "the target network update rate"),
        ("target_network_frequency", int, 1000, "the timesteps it takes to update the target network"),
        ("batch_size", int, 32, "the batch size of sample from the reply memory"),
        ("start_e", float, 1, "the starting epsilon for exploration"),
        ("end_e", float, 0.01, "the ending epsilon for exploration"),
        ("exploration_fraction", float, 0.10, "the fraction of `total-timesteps` it takes from start-e to go end-e"),
        ("learning_starts", int, 80000, "timestep to start learning"),
        ("train_frequency", int, 4, "the frequency of training"),
    ]
    extra = [r for r in _EXTRA if r[0] != "gae_kernel"] + [
        ("huber_loss", bool, False, "[b200] smooth-L1 TD loss instead of the reference's MSE (dqn_atari.py:224)")]
    return _make("Args", common + algo + extra)


def parse(cls, argv=None):
    return tyro.cli(cls, args=argv)


def use_synthetic(args):
    """The synthetic envs are used ONLY on request: ``--synthetic-env`` or ``CLEANRL_B200_SYNTHETIC_ENV=1``.
    A run that asks for Breakout must never quietly train on synthetic frames."""
    import os
    if os.environ.get("CLEANRL_B200_SYNTHETIC_ENV", "0") not in ("", "0"):
        args.synthetic_env = True
    return bool(args.synthetic_env)


def env_import_error(what, err):
    """Re-raise a missing env dependency with an actionable message (instead of falling back to synthetic data)."""
    return ImportError(f"{what} could not be imported ({err}). Install the reference's env extras "
                       f"(e.g. `pip install envpool` / `gymnasium[atari,accept-rom-license]` / `gymnasium[mujoco]`) "
                       f"or pass --synthetic-env (or CLEANRL_B200_SYNTHETIC_ENV=1) to run on the built-in synthetic "
                       f"vector env.")


def run_name_for(args):
    """runs/{run_name}: the reference's pattern (ppo.py:140); runs on synthetic data are tagged as such."""
    import time
    env = args.env_id + ("-synthetic" if getattr(args, "synthetic_env", False) else "")
    return f"{env}__{args.exp_name}__{args.seed}__{int(time.time())}"
