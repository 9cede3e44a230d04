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


def ppg_procgen_args(exp_name="ppg_procgen"):
    """cleanrl/ppg_procgen.py:19-98."""
    algo = [r for r in _override(_ALGO, env_id="starpilot", total_timesteps=int(25e6), learning_rate=5e-4, num_envs=64,
                                 num_steps=256, anneal_lr=False, gamma=0.999, num_minibatches=8)
            if r[0] not in ("update_epochs", "norm_adv")]
    at = [r[0] for r in algo].index("clip_coef")
    algo.insert(at, ("adv_norm_fullbatch", bool, True, "Toggle full batch advantage normalization as used in PPG code"))
    ppg = [
        ("n_iteration", int, 32, "N_pi: the number of policy update in the policy phase "),
        ("e_policy", int, 1, "E_pi: the number of policy update in the policy phase "),
        ("v_value", int, 1, "E_V: the number of policy update in the policy phase "),
        ("e_auxiliary", int, 6, "E_aux:the K epochs to update the policy"),
        ("beta_clone", float, 1.0, "the behavior cloning coefficient"),
        ("num_aux_rollouts", int, 4, "the number of mini batch in the auxiliary phase"),
        ("n_aux_grad_accum", int, 1, "the number of gradient accumulation in mini batch"),
    ]
    runtime = _RUNTIME + [
        ("num_phases", int, 0, "the number of phases (computed in runtime)"),
        ("aux_batch_rollouts", int, 0, "the number of rollouts in the auxiliary phase (computed in runtime)"),
    ]
    return _make("Args", _override(_COMMON, exp_name=exp_name) + algo + ppg + runtime + _EXTRA)


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


def rpo_continuous_action_args(exp_name="rpo_continuous_action"):
    """cleanrl/rpo_continuous_action.py:17-80: ppo_continuous_action.py's fields without save_model / upload_model /
    hf_entity, total_timesteps 8e6, and rpo_alpha after target_kl."""
    algo = _override(_ALGO, env_id="HalfCheetah-v4", total_timesteps=8000000, learning_rate=3e-4, num_envs=1,
                     num_steps=2048, num_minibatches=32, update_epochs=10, ent_coef=0.0)
    algo += [("rpo_alpha", float, 0.5, "the alpha parameter for RPO")]
    return _make("Args", _override(_COMMON, exp_name=exp_name) + algo + _RUNTIME + _EXTRA)


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


def c51_atari_args(exp_name="c51_atari"):
    """cleanrl/c51_atari.py:25-82."""
    common = list(_override(_COMMON, exp_name=exp_name))
    common += [
        ("save_model", bool, False, "whether to save model into the `runs/{run_name}` folder"),
        ("upload_model", bool, False, "whether to upload the saved model to huggingface"),
        ("hf_entity", str, "", "the user or org name of the model repository from the Hugging Face Hub"),
    ]
    algo = [
        ("env_id", str, "BreakoutNoFrameskip-v4", "the id of the environment"),
        ("total_timesteps", int, 10000000, "total timesteps of the experiments"),
        ("learning_rate", float, 2.5e-4, "the learning rate of the optimizer"),
        ("num_envs", int, 1, "the number of parallel game environments"),
        ("n_atoms", int, 51, "the number of atoms"),
        ("v_min", float, -10, "the return lower bound"),
        ("v_max", float, 10, "the return upper bound"),
        ("buffer_size", int, 1000000, "the replay memory buffer size"),
        ("gamma", float, 0.99, "the discount factor gamma"),
        ("target_network_frequency", int, 10000, "the timesteps it takes to update the target network"),
        ("batch_size", int, 32, "the batch size of sample from the reply memory"),
        ("start_e", float, 1, "the starting epsilon for exploration"),
        ("end_e", float, 0.01, "the ending epsilon for exploration"),
        ("exploration_fraction", float, 0.10, "the fraction of `total-timesteps` it takes from start-e to go end-e"),
        ("learning_starts", int, 80000, "timestep to start learning"),
        ("train_frequency", int, 4, "the frequency of training"),
    ]
    extra = [r for r in _EXTRA if r[0] != "gae_kernel"]
    return _make("Args", common + algo + extra)


def sac_atari_args(exp_name="sac_atari"):
    """cleanrl/sac_atari.py:27-74."""
    common = list(_override(_COMMON, exp_name=exp_name))
    algo = [
        ("env_id", str, "BeamRiderNoFrameskip-v4", "the id of the environment"),
        ("total_timesteps", int, 5000000, "total timesteps of the experiments"),
        ("buffer_size", int, int(1e6), "the replay memory buffer size"),
        ("gamma", float, 0.99, "the discount factor gamma"),
        ("tau", float, 1.0, "target smoothing coefficient (default: 1)"),
        ("batch_size", int, 64, "the batch size of sample from the reply memory"),
        ("learning_starts", int, 2e4, "timestep to start learning"),
        ("policy_lr", float, 3e-4, "the learning rate of the policy network optimizer"),
        ("q_lr", float, 3e-4, "the learning rate of the Q network network optimizer"),
        ("update_frequency", int, 4, "the frequency of training updates"),
        ("target_network_frequency", int, 8000, "the frequency of updates for the target networks"),
        ("alpha", float, 0.2, "Entropy regularization coefficient."),
        ("autotune", bool, True, "automatic tuning of the entropy coefficient"),
        ("target_entropy_scale", float, 0.89, "coefficient for scaling the autotune entropy target"),
    ]
    extra = [r for r in _EXTRA if r[0] != "gae_kernel"]
    return _make("Args", common + algo + extra)


def sac_continuous_action_args(exp_name="sac_continuous_action"):
    """cleanrl/sac_continuous_action.py:19-66."""
    common = list(_override(_COMMON, exp_name=exp_name))
    algo = [
        ("env_id", str, "Hopper-v4", "the environment id of the task"),
        ("total_timesteps", int, 1000000, "total timesteps of the experiments"),
        ("num_envs", int, 1, "the number of parallel game environments"),
        ("buffer_size", int, int(1e6), "the replay memory buffer size"),
        ("gamma", float, 0.99, "the discount factor gamma"),
        ("tau", float, 0.005, "target smoothing coefficient (default: 0.005)"),
        ("batch_size", int, 256, "the batch size of sample from the reply memory"),
        ("learning_starts", int, 5e3, "timestep to start learning"),
        ("policy_lr", float, 3e-4, "the learning rate of the policy network optimizer"),
        ("q_lr", float, 1e-3, "the learning rate of the Q network network optimizer"),
        ("policy_frequency", int, 2, "the frequency of training policy (delayed)"),
        ("target_network_frequency", int, 1, "the frequency of updates for the target nerworks"),
        ("alpha", float, 0.2, "Entropy regularization coefficient."),
        ("autotune", bool, True, "automatic tuning of the entropy coefficient"),
    ]
    extra = [r for r in _EXTRA if r[0] == "synthetic_env"]
    return _make("Args", common + algo + extra)


def td3_continuous_action_args(exp_name="td3_continuous_action"):
    """cleanrl/td3_continuous_action.py:19-70."""
    common = list(_override(_COMMON, exp_name=exp_name))
    common += [
        ("save_model", bool, False, "whether to save model into the `runs/{run_name}` folder"),
        ("upload_model", bool, False, "whether to upload the saved model to huggingface"),
        ("hf_entity", str, "", "the user or org name of the model repository from the Hugging Face Hub"),
    ]
    algo = [
        ("env_id", str, "Hopper-v4", "the id of the environment"),
        ("total_timesteps", int, 1000000, "total timesteps of the experiments"),
        ("learning_rate", float, 3e-4, "the learning rate of the optimizer"),
        ("num_envs", int, 1, "the number of parallel game environments"),
        ("buffer_size", int, int(1e6), "the replay memory buffer size"),
        ("gamma", float, 0.99, "the discount factor gamma"),
        ("tau", float, 0.005, "target smoothing coefficient (default: 0.005)"),
        ("batch_size", int, 256, "the batch size of sample from the reply memory"),
        ("policy_noise", float, 0.2, "the scale of policy noise"),
        ("exploration_noise", float, 0.1, "the scale of exploration noise"),
        ("learning_starts", int, 25e3, "timestep to start learning"),
        ("policy_frequency", int, 2, "the frequency of training policy (delayed)"),
        ("noise_clip", float, 0.5, "noise clip parameter of the Target Policy Smoothing Regularization"),
    ]
    extra = [r for r in _EXTRA if r[0] == "synthetic_env"]
    return _make("Args", common + algo + extra)


def ddpg_continuous_action_args(exp_name="ddpg_continuous_action"):
    """cleanrl/ddpg_continuous_action.py:19-64 (one env: no num_envs; env_id keeps the reference's help text)."""
    common = list(_override(_COMMON, exp_name=exp_name))
    common += [
        ("save_model", bool, False, "whether to save model into the `runs/{run_name}` folder"),
        ("upload_model", bool, False, "whether to upload the saved model to huggingface"),
        ("hf_entity", str, "", "the user or org name of the model repository from the Hugging Face Hub"),
    ]
    algo = [
        ("env_id", str, "Hopper-v4", "the environment id of the Atari game"),
        ("total_timesteps", int, 1000000, "total timesteps of the experiments"),
        ("learning_rate", float, 3e-4, "the learning rate of the optimizer"),
        ("buffer_size", int, int(1e6), "the replay memory buffer size"),
        ("gamma", float, 0.99, "the discount factor gamma"),
        ("tau", float, 0.005, "target smoothing coefficient (default: 0.005)"),
        ("batch_size", int, 256, "the batch size of sample from the reply memory"),
        ("exploration_noise", float, 0.1, "the scale of exploration noise"),
        ("learning_starts", int, 25e3, "timestep to start learning"),
        ("policy_frequency", int, 2, "the frequency of training policy (delayed)"),
    ]
    extra = [r for r in _EXTRA if r[0] == "synthetic_env"]
    return _make("Args", common + algo + extra)


def pqn_args(exp_name="pqn"):
    """cleanrl/pqn.py:17-64."""
    algo = [
        ("env_id", str, "CartPole-v1", "the id of the environment"),
        ("total_timesteps", int, 500000, "total timesteps of the experiments"),
        ("learning_rate", float, 2.5e-4, "the learning rate of the optimizer"),
        ("num_envs", int, 4, "the number of parallel game environments"),
        ("num_steps", int, 128, "the number of steps to run for each environment per update"),
        ("num_minibatches", int, 4, "the number of mini-batches"),
        ("update_epochs", int, 4, "the K epochs to update the policy"),
        ("anneal_lr", bool, True, "Toggle learning rate annealing"),
        ("gamma", float, 0.99, "the discount factor gamma"),
        ("start_e", float, 1, "the starting epsilon for exploration"),
        ("end_e", float, 0.05, "the ending epsilon for exploration"),
        ("exploration_fraction", float, 0.5, "the fraction of `total_timesteps` it takes from start_e to end_e"),
        ("max_grad_norm", float, 10.0, "the maximum norm for the gradient clipping"),
        ("q_lambda", float, 0.65, "the lambda for Q(lambda)"),
    ]
    extra = [r for r in _EXTRA if r[0] == "synthetic_env"]
    return _make("Args", _override(_COMMON, exp_name=exp_name) + algo + extra)


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
