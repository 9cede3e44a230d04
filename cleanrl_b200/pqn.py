"""Drop-in for cleanrl/pqn.py (parallel Q-learning with a LayerNorm Q-network and Q(lambda) targets) on libb200rl.

Same flags, ``QNetwork`` surface and state_dict keys, initialisation, exploration draws, TensorBoard tags and stdout as
the reference (cleanrl/pqn.py:17-109,112-248).  The rollout, the Q(lambda) scan and the update run on the fp32
kernels of cleanrl_b200/csrc/pqn.cu and the clip + RAdam step of optim.cu through ``pqn_engine.PQNEngine``; each update
epoch is replayed as one CUDA graph.
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
from cleanrl_b200.agents import PQNQNetwork as QNetwork, layer_init  # noqa: F401
from cleanrl_b200.pqn_engine import PQNEngine

Args = cli.pqn_args(os.path.basename(__file__)[: -len(".py")])
run_name = None


def make_env(env_id, seed, idx, capture_video, run_name):
    """gymnasium thunk of the reference (pqn.py:67-79)."""
    def thunk():
        import gymnasium as gym  # type: ignore

        if capture_video and idx == 0:
            env = gym.make(env_id, render_mode="rgb_array")
            env = gym.wrappers.RecordVideo(env, f"videos/{run_name}")
        else:
            env = gym.make(env_id)
        env = gym.wrappers.RecordEpisodeStatistics(env)
        env.action_space.seed(seed)
        return env

    return thunk


def linear_schedule(start_e: float, end_e: float, duration: int, t: int):
    slope = (end_e - start_e) / duration
    return max(slope * t + start_e, end_e)


def make_envs(args, run_name):
    """The reference's ``SyncVectorEnv`` (pqn.py:145-147), or ``synthetic_envs.CartPoleVec`` on request."""
    if not cli.use_synthetic(args):
        try:
            import gymnasium as gym  # type: ignore
        except ImportError as e:
            raise cli.env_import_error("gymnasium", e) from e
        return gym.vector.SyncVectorEnv([make_env(args.env_id, args.seed + i, i, args.capture_video, run_name)
                                         for i in range(args.num_envs)])
    from cleanrl_b200.synthetic_envs import CartPoleVec

    return CartPoleVec(args.num_envs)


def main(argv=None, writer_factory=None, env_factory=None, on_iteration=None):
    """``on_iteration(iteration, engine, stats)`` runs after every iteration's update with the ``PQNEngine`` and the
    logged (td_loss, q_values)."""
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
        raise RuntimeError("cleanrl_b200.pqn runs on libb200rl CUDA kernels: a CUDA device and --cuda are required "
                           "(no CPU fallback).")
    device = torch.device("cuda")

    envs = env_factory(args) if env_factory else make_envs(args, run_name)
    assert hasattr(envs.single_action_space, "n"), "only discrete action space is supported"

    q_network = QNetwork(envs).to(device)           # layer_init draws from the CPU generator, as the reference
    engine = PQNEngine(q_network, args, args.num_envs, device)

    global_step = 0
    start_time = time.time()
    next_obs, _ = envs.reset(seed=args.seed)
    next_done = np.zeros(args.num_envs, dtype=np.float32)
    reward = np.zeros(args.num_envs, dtype=np.float32)
    lrnow = args.learning_rate

    for iteration in range(1, args.num_iterations + 1):
        if args.anneal_lr:
            frac = 1.0 - (iteration - 1.0) / args.num_iterations
            lrnow = frac * args.learning_rate

        for step in range(0, args.num_steps):
            global_step += args.num_envs
            epsilon = linear_schedule(args.start_e, args.end_e, args.exploration_fraction * args.total_timesteps,
                                      global_step)
            action = engine.policy_step(step, next_obs, next_done, reward, epsilon)
            next_obs, reward, terminations, truncations, infos = envs.step(action)
            next_done = np.logical_or(terminations, truncations)
            if "final_info" in infos:
                for info in infos["final_info"]:
                    if info and "episode" in info:
                        print(f"global_step={global_step}, episodic_return={info['episode']['r']}")
                        writer.add_scalar("charts/episodic_return", info["episode"]["r"], global_step)
                        writer.add_scalar("charts/episodic_length", info["episode"]["l"], global_step)

        engine.finish_rollout(next_obs, next_done, reward)
        td_loss, q_values = engine.update(lrnow).tolist()

        writer.add_scalar("losses/td_loss", td_loss, global_step)
        writer.add_scalar("losses/q_values", q_values, global_step)
        print("SPS:", int(global_step / (time.time() - start_time)))
        writer.add_scalar("charts/SPS", int(global_step / (time.time() - start_time)), global_step)
        if on_iteration is not None:
            on_iteration(iteration, engine, (td_loss, q_values))

    envs.close()
    writer.close()
    return q_network, engine


if __name__ == "__main__":
    main()
