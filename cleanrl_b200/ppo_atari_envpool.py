"""Drop-in for cleanrl/ppo_atari_envpool.py on the H100-native PPO engine.

Same CLI flags (``Args``), same ``Agent`` surface / ``state_dict`` keys, same
TensorBoard tags and stdout lines as the reference script
(cleanrl/ppo_atari_envpool.py:19-80,123-149,332-341), launched the same way
(``python cleanrl_b200/ppo_atari_envpool.py --flags`` or ``runpy.run_path`` as
cleanrl_utils/tuner.py:90-95 does; ``run_name`` is left in the module globals).
The loop body runs on libb200rl kernels through ``PPOEngine`` instead of torch
autograd / cuDNN; environments stay on the host.
"""
from __future__ import annotations

import os
import random
import sys
import time
from collections import deque

if __package__ in (None, ""):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

from cleanrl_b200 import cli
from cleanrl_b200.agents import NatureCNNAgent as Agent, layer_init  # noqa: F401  (reference module-level names)
from cleanrl_b200.ppo_engine import PPOEngine

Args = cli.ppo_atari_envpool_args(os.path.basename(__file__)[: -len(".py")])
run_name = None


class RecordEpisodeStatistics:
    """Host-side episode accounting for envpool's gym API (raw, unclipped score keyed on
    ``info["reward"]`` / ``info["terminated"]``; reference: ppo_atari_envpool.py:83-114)."""

    def __init__(self, env, deque_size=100):
        self.env = env
        self.num_envs = getattr(env, "num_envs", 1)
        self.episode_returns = None
        self.episode_lengths = None

    def __getattr__(self, name):
        if name.startswith("_") or name == "env":
            raise AttributeError(name)
        return getattr(self.env, name)

    def reset(self, **kwargs):
        observations = self.env.reset(**kwargs)
        n = self.num_envs
        self.episode_returns = np.zeros(n, dtype=np.float32)
        self.episode_lengths = np.zeros(n, dtype=np.int32)
        self.lives = np.zeros(n, dtype=np.int32)
        self.returned_episode_returns = np.zeros(n, dtype=np.float32)
        self.returned_episode_lengths = np.zeros(n, dtype=np.int32)
        return observations

    def step(self, action):
        observations, rewards, dones, infos = self.env.step(action)
        self.episode_returns += infos["reward"]
        self.episode_lengths += 1
        self.returned_episode_returns[:] = self.episode_returns
        self.returned_episode_lengths[:] = self.episode_lengths
        alive = 1 - infos["terminated"]
        self.episode_returns *= alive
        self.episode_lengths *= alive
        infos["r"] = self.returned_episode_returns
        infos["l"] = self.returned_episode_lengths
        return observations, rewards, dones, infos

    def close(self):
        return self.env.close()


def make_envs(args, pinned=True, mode=None):
    """envpool.make(...) as the reference (ppo_atari_envpool.py:185-196); when envpool is not
    installed (this image) or --synthetic-env is set, a seeded synthetic Breakout-shaped env."""
    envs = None
    if not cli.use_synthetic(args):
        try:
            import envpool  # type: ignore
        except ImportError as e:
            raise cli.env_import_error("envpool", e) from e
        envs = envpool.make(args.env_id, env_type="gym", num_envs=args.num_envs, episodic_life=True,
                            reward_clip=True, seed=args.seed)
    if envs is None:
        from cleanrl_b200.synthetic_envs import SyntheticAtariVec

        mode = mode or os.environ.get("CLEANRL_B200_SYNTH_MODE", "fresh")
        envs = SyntheticAtariVec(args.num_envs, seed=args.seed, mode=mode, pinned=pinned)
    envs.num_envs = args.num_envs
    envs.single_action_space = envs.action_space
    envs.single_observation_space = envs.observation_space
    envs = RecordEpisodeStatistics(envs)
    assert hasattr(envs.action_space, "n"), "only discrete action space is supported"
    return envs


def make_env_groups(args, groups, pinned=True, mode=None):
    """``groups`` independent vector envs over contiguous slices of the envs.  Group g is seeded ``seed + g * n`` so that,
    with envpool's per-env seeding (seed + env index), every env keeps the stream it has in the single-pool run."""
    import copy
    assert args.num_envs % groups == 0, "--num-envs must be divisible by --env-groups"
    n = args.num_envs // groups
    parts = []
    for g in range(groups):
        sub = copy.copy(args)
        sub.num_envs, sub.seed = n, args.seed + g * n
        parts.append(make_envs(sub, pinned=pinned, mode=mode))
    return parts


def main(argv=None, writer_factory=None, env_factory=None, on_iteration=None):
    global run_name
    args = cli.parse(Args, argv)
    args.batch_size = int(args.num_envs * args.num_steps)
    args.minibatch_size = int(args.batch_size // args.num_minibatches)
    args.num_iterations = args.total_timesteps // args.batch_size
    cli.use_synthetic(args)
    run_name = cli.run_name_for(args)
    if args.track:
        import wandb

        wandb.init(project=args.wandb_project_name, entity=args.wandb_entity, sync_tensorboard=True,
                   config=vars(args), name=run_name, monitor_gym=True, save_code=True)
    if writer_factory is None:
        from torch.utils.tensorboard import SummaryWriter as writer_factory
    writer = writer_factory(f"runs/{run_name}")
    writer.add_text("hyperparameters",
                    "|param|value|\n|-|-|\n%s" % ("\n".join([f"|{key}|{value}|" for key, value in vars(args).items()])))

    # seeding: same generators, same order as the reference (ppo_atari_envpool.py:177-180)
    random.seed(args.seed)
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)
    torch.backends.cudnn.deterministic = args.torch_deterministic

    if not (torch.cuda.is_available() and args.cuda) and not PPOEngine.ALLOW_NON_CUDA_FOR_TESTS:
        raise RuntimeError("cleanrl_b200.ppo_atari_envpool runs on libb200rl CUDA kernels: a CUDA device and "
                           "--cuda are required (no CPU fallback). Use the reference script for CPU runs.")
    # "cpu" is only reachable from the CPU test harness (tests/cpu_backend.py drives the host logic with injected ops)
    device = torch.device("cuda" if torch.cuda.is_available() else "cpu")

    groups = int(getattr(args, "env_groups", 1))
    env_parts = None
    if groups > 1:
        env_parts = make_env_groups(args, groups)
        envs = env_parts[0]
    else:
        envs = env_factory(args) if env_factory else make_envs(args)
    agent = Agent(envs).to(device)   # CPU init (same RNG stream as the reference), then moved
    agent.precision = args.precision
    engine = PPOEngine(agent, args, envs.single_observation_space.shape, envs.single_observation_space.dtype,
                       args.num_envs, device, gae_mode=0 if args.gae_kernel == "sequential" else 1)
    avg_returns = deque(maxlen=20)

    global_step = 0
    start_time = time.time()
    if env_parts is not None:
        obs_parts = [e.reset() for e in env_parts]
        done_parts = [np.zeros(e.num_envs, dtype=np.float32) for e in env_parts]
    else:
        next_obs = envs.reset()
        next_done = np.zeros(args.num_envs, dtype=np.float32)
    lrnow = args.learning_rate

    def log_episodes(step_global, next_done, info):
        finished = np.nonzero(np.logical_and(next_done, info["lives"] == 0))[0]
        for idx in finished:
            print(f"global_step={step_global}, episodic_return={info['r'][idx]}")
            avg_returns.append(info["r"][idx])
            writer.add_scalar("charts/avg_episodic_return", np.average(avg_returns), step_global)
            writer.add_scalar("charts/episodic_return", info["r"][idx], step_global)
            writer.add_scalar("charts/episodic_length", info["l"][idx], step_global)

    for iteration in range(1, args.num_iterations + 1):
        if args.anneal_lr:
            frac = 1.0 - (iteration - 1.0) / args.num_iterations
            lrnow = frac * args.learning_rate

        if env_parts is not None:
            # grouped, software-pipelined rollout (PPOEngine.collect); global_step advances by num_envs per step as in the
            # reference (ppo_atari_envpool.py:225)
            base = global_step
            obs_parts, done_parts = engine.collect(
                env_parts, obs_parts, done_parts,
                on_step=lambda t, p, reward, done, info: log_episodes(base + (t + 1) * args.num_envs, done, info))
            global_step = base + args.num_steps * args.num_envs
            engine.finish_rollout_parts(obs_parts, done_parts)

        for step in range(0, args.num_steps if env_parts is None else 0):
            global_step += args.num_envs
            action = engine.policy_step(step, next_obs, next_done)
            next_obs, reward, next_done, info = envs.step(action)
            engine.record_reward(step, reward)
            log_episodes(global_step, next_done, info)

        if env_parts is None:
            engine.finish_rollout(next_obs, next_done)
        st = engine.update(lrnow)
        explained_var = engine.explained_variance()

        writer.add_scalar("charts/learning_rate", lrnow, global_step)
        writer.add_scalar("losses/value_loss", st["v_loss"], global_step)
        writer.add_scalar("losses/policy_loss", st["pg_loss"], global_step)
        writer.add_scalar("losses/entropy", st["entropy"], global_step)
        writer.add_scalar("losses/old_approx_kl", st["old_approx_kl"], global_step)
        writer.add_scalar("losses/approx_kl", st["approx_kl"], global_step)
        writer.add_scalar("losses/clipfrac", st["clipfrac_mean"], global_step)
        writer.add_scalar("losses/explained_variance", explained_var, global_step)
        sps = int(global_step / (time.time() - start_time))
        print("SPS:", sps)
        writer.add_scalar("charts/SPS", sps, global_step)
        if on_iteration is not None:
            on_iteration(iteration, engine, st)

    for e in (env_parts or [envs]):
        e.close()
    writer.close()
    return engine


if __name__ == "__main__":
    main()
