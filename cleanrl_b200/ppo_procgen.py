"""Drop-in for cleanrl/ppo_procgen.py: PPO with the IMPALA-CNN agent on libb200rl.

Same CLI flags (``Args``), ``Agent`` / ``ResidualBlock`` / ``ConvSequence`` module tree and ``state_dict`` keys,
TensorBoard tags and stdout lines as the reference (cleanrl/ppo_procgen.py:16-79,89-150,320-343).  The loop is the shared
``PPOEngine`` (rollout storage as uint8, one-launch GAE, fused loss + hand-written backward + fused clip/Adam); procgen's
old-gym vector API (``step -> obs, reward, done, info`` with a list of per-env info dicts) and its wrapper stack stay on the
host exactly as in the reference (:176-186).
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
from cleanrl_b200.agents import ConvSequence, ImpalaAgent as Agent, ResidualBlock, layer_init  # noqa: F401
from cleanrl_b200.ppo_engine import PPOEngine

Args = cli.ppo_procgen_args(os.path.basename(__file__)[: -len(".py")])
run_name = None


def make_envs(args, run_name):
    """ProcgenEnv + the reference's wrappers (cleanrl/ppo_procgen.py:176-186); synthetic only on request."""
    if not cli.use_synthetic(args):
        try:
            import gym  # type: ignore
            from procgen import ProcgenEnv  # type: ignore
        except ImportError as e:
            raise cli.env_import_error("procgen / gym", e) from e
        envs = ProcgenEnv(num_envs=args.num_envs, env_name=args.env_id, num_levels=0, start_level=0, distribution_mode="easy")
        envs = gym.wrappers.TransformObservation(envs, lambda obs: obs["rgb"])
        envs.single_action_space = envs.action_space
        envs.single_observation_space = envs.observation_space["rgb"]
        envs.is_vector_env = True
        envs = gym.wrappers.RecordEpisodeStatistics(envs)
        if args.capture_video:
            envs = gym.wrappers.RecordVideo(envs, f"videos/{run_name}")
        envs = gym.wrappers.NormalizeReward(envs, gamma=args.gamma)
        envs = gym.wrappers.TransformReward(envs, lambda reward: np.clip(reward, -10, 10))
        return envs
    from cleanrl_b200.synthetic_envs import SyntheticProcgenVec

    return SyntheticProcgenVec(args.num_envs)


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
    if not (torch.cuda.is_available() and args.cuda):
        raise RuntimeError("cleanrl_b200.ppo_procgen runs on libb200rl CUDA kernels: a CUDA device and --cuda are required "
                           "(no CPU fallback). Use the reference script for CPU runs.")
    device = torch.device("cuda")

    envs = env_factory(args) if env_factory else make_envs(args, run_name)
    assert hasattr(envs.single_action_space, "n"), "only discrete action space is supported"
    agent = Agent(envs).to(device)
    agent.precision = args.precision
    if agent_hook:
        agent_hook(agent)
    engine = PPOEngine(agent, args, envs.single_observation_space.shape, np.uint8, args.num_envs, device,
                       gae_mode=0 if args.gae_kernel == "sequential" else 1)

    global_step = 0
    start_time = time.time()
    next_obs = np.asarray(envs.reset())
    next_done = np.zeros(args.num_envs, dtype=np.float32)
    lrnow = args.learning_rate

    for iteration in range(1, args.num_iterations + 1):
        if args.anneal_lr:
            frac = 1.0 - (iteration - 1.0) / args.num_iterations
            lrnow = frac * args.learning_rate

        for step in range(0, args.num_steps):
            global_step += args.num_envs
            action = engine.policy_step(step, next_obs, next_done)
            next_obs, reward, next_done, info = envs.step(action)
            next_obs = np.asarray(next_obs)
            engine.record_reward(step, reward)
            for item in info:
                if "episode" in item.keys():
                    print(f"global_step={global_step}, episodic_return={item['episode']['r']}")
                    writer.add_scalar("charts/episodic_return", item["episode"]["r"], global_step)
                    writer.add_scalar("charts/episodic_length", item["episode"]["l"], global_step)
                    break

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
        print("SPS:", int(global_step / (time.time() - start_time)))
        writer.add_scalar("charts/SPS", int(global_step / (time.time() - start_time)), global_step)
        if on_iteration is not None:
            on_iteration(iteration, engine, st)

    envs.close()
    writer.close()
    return engine


if __name__ == "__main__":
    main()
