"""Drop-in for cleanrl/rpo_continuous_action.py (robust policy optimization for MuJoCo-style tasks) on libb200rl.

Same flags (no --save-model: the reference has none), Agent surface (``Agent(envs, rpo_alpha)`` with ``critic`` /
``actor_mean`` / ``actor_logstd`` => same state_dict keys), env stack, TensorBoard tags and stdout as the reference
(cleanrl/rpo_continuous_action.py:17-80,108-144,311-329).  The loop is ppo_continuous_action.py's; the update evaluates
the stored actions under ``Normal(mean + z, std)`` with ``z ~ U(-rpo_alpha, rpo_alpha)`` from the CPU generator, drawn
once per epoch and uploaded in one copy (agents.RPOAgent), inside the fused Gaussian loss
(b200rl_ppo_loss_gaussian_shift_f32).
"""
from __future__ import annotations

import os
import random
import sys
import time

if __package__ in (None, ""):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

from cleanrl_b200 import cli
from cleanrl_b200.agents import RPOAgent as Agent, layer_init  # noqa: F401
from cleanrl_b200.ppo_engine import PPOEngine

Args = cli.rpo_continuous_action_args(os.path.basename(__file__)[: -len(".py")])
run_name = None


def make_env(env_id, idx, capture_video, run_name, gamma):
    """gymnasium thunk with the reference's wrapper stack (rpo_continuous_action.py:83-99)."""
    def thunk():
        import gymnasium as gym  # type: ignore

        if capture_video and idx == 0:
            env = gym.make(env_id, render_mode="rgb_array")
            env = gym.wrappers.RecordVideo(env, f"videos/{run_name}")
        else:
            env = gym.make(env_id)
        env = gym.wrappers.FlattenObservation(env)
        env = gym.wrappers.RecordEpisodeStatistics(env)
        env = gym.wrappers.ClipAction(env)
        env = gym.wrappers.NormalizeObservation(env)
        env = gym.wrappers.TransformObservation(env, lambda obs: np.clip(obs, -10, 10))
        env = gym.wrappers.NormalizeReward(env, gamma=gamma)
        env = gym.wrappers.TransformReward(env, lambda reward: np.clip(reward, -10, 10))
        return env

    return thunk


def make_envs(args, run_name, num_envs=None):
    n = num_envs or args.num_envs
    if not cli.use_synthetic(args):
        try:
            import gymnasium as gym  # type: ignore  # noqa: F401
        except ImportError as e:
            raise cli.env_import_error("gymnasium (+ mujoco)", e) from e
        return gym.vector.SyncVectorEnv([make_env(args.env_id, i, args.capture_video, run_name, args.gamma)
                                         for i in range(n)])
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec

    return SyntheticGymnasiumVec(n, kind="continuous")


def main(argv=None, writer_factory=None, env_factory=None, on_iteration=None, agent_hook=None):
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

    random.seed(args.seed)
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)
    torch.backends.cudnn.deterministic = args.torch_deterministic

    if not (torch.cuda.is_available() and args.cuda) and not PPOEngine.ALLOW_NON_CUDA_FOR_TESTS:
        raise RuntimeError("cleanrl_b200.rpo_continuous_action runs on libb200rl CUDA kernels: a CUDA device and --cuda "
                           "are required (no CPU fallback). Use the reference script for CPU runs.")
    device = torch.device("cuda" if torch.cuda.is_available() else "cpu")

    envs = env_factory(args) if env_factory else make_envs(args, run_name)
    assert hasattr(envs.single_action_space, "low"), "only continuous action space is supported"
    agent = Agent(envs, args.rpo_alpha).to(device)
    if agent_hook:
        agent_hook(agent)
    engine = PPOEngine(agent, args, envs.single_observation_space.shape, np.float32, args.num_envs, device,
                       gae_mode=0 if args.gae_kernel == "sequential" else 1)

    global_step = 0
    start_time = time.time()
    next_obs, _ = envs.reset(seed=args.seed)
    next_done = np.zeros(args.num_envs, dtype=np.float32)
    lrnow = args.learning_rate

    for iteration in range(1, args.num_iterations + 1):
        if args.anneal_lr:
            frac = 1.0 - (iteration - 1.0) / args.num_iterations
            lrnow = frac * args.learning_rate

        for step in range(0, args.num_steps):
            global_step += args.num_envs
            action = engine.policy_step(step, next_obs, next_done)
            next_obs, reward, terminations, truncations, infos = envs.step(action)
            next_done = np.logical_or(terminations, truncations)
            engine.record_reward(step, reward)
            if "final_info" in infos:
                for info in infos["final_info"]:
                    if info and "episode" in info:
                        print(f"global_step={global_step}, episodic_return={info['episode']['r']}")
                        writer.add_scalar("charts/episodic_return", info["episode"]["r"], global_step)
                        writer.add_scalar("charts/episodic_length", info["episode"]["l"], global_step)

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

    envs.close()
    writer.close()
    return engine


if __name__ == "__main__":
    main()
