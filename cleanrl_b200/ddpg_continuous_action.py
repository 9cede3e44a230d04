"""Drop-in for cleanrl/ddpg_continuous_action.py (deep deterministic policy gradient) on libb200rl.

Same flags, ``Actor`` / ``QNetwork`` surface and state_dict keys, initialisation, TensorBoard tags and stdout as the
reference (cleanrl/ddpg_continuous_action.py:19-116,119-263).  The numpy ``ReplayBuffer`` becomes the device-resident
float32 ring in the reference's ``optimize_memory_usage=False`` layout (``cleanrl_b200.replay.DeviceReplayRing``),
sampled with the same numpy index stream; the sampled rows are gathered inside the MLP kernels.  qf1, qf1_target and
the actor target each live in one flat buffer, and every update -- the critic step with its loss fused into the critic
data backward, the delayed actor step and the soft update of both targets -- is replayed as one CUDA graph of fp32
kernels (cleanrl_b200/csrc/sac_continuous.cu).
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

from cleanrl_b200 import agents, cli
from cleanrl_b200.agents import DDPGActor as Actor, DDPGState, SoftQNetworkMLP as QNetwork, ddpg_update
from cleanrl_b200.replay import DeviceReplayRing

Args = cli.ddpg_continuous_action_args(os.path.basename(__file__)[: -len(".py")])
run_name = None


def make_env(env_id, seed, idx, capture_video, run_name):
    """gymnasium thunk of the reference (ddpg_continuous_action.py:67-78)."""
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


def make_envs(args, run_name):
    """The reference's one-env ``SyncVectorEnv`` (ddpg_continuous_action.py:148)."""
    if not cli.use_synthetic(args):
        try:
            import gymnasium as gym  # type: ignore
        except ImportError as e:
            raise cli.env_import_error("gymnasium (+ mujoco)", e) from e
        return gym.vector.SyncVectorEnv([make_env(args.env_id, args.seed, 0, args.capture_video, run_name)])
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec

    return SyntheticGymnasiumVec(1, kind="continuous")


def main(argv=None, writer_factory=None, env_factory=None, on_update=None):
    """``on_update(global_step, state)`` runs after every update with the ``DDPGState``."""
    global run_name
    args = cli.parse(Args, argv)
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
        raise RuntimeError("cleanrl_b200.ddpg_continuous_action runs on libb200rl CUDA kernels: a CUDA device and "
                           "--cuda are required (no CPU fallback).")
    device = torch.device("cuda")

    envs = env_factory(args) if env_factory else make_envs(args, run_name)
    assert hasattr(envs.single_action_space, "low"), "only continuous action space is supported"
    low, high = envs.single_action_space.low, envs.single_action_space.high

    # construction order of the reference (ddpg_continuous_action.py:151-154): it fixes the generator stream
    nets = [Actor(envs), QNetwork(envs), QNetwork(envs), Actor(envs)]
    actor, qf1, qf1_target, target_actor = [n.to(device) for n in nets]
    target_actor.load_state_dict(actor.state_dict())
    qf1_target.load_state_dict(qf1.state_dict())
    state = DDPGState(actor, qf1, qf1_target, target_actor, device)

    envs.single_observation_space.dtype = np.float32
    rb = DeviceReplayRing(args.buffer_size, envs.single_observation_space.shape, envs.num_envs, device,
                          optimize_memory_usage=False, obs_dtype=torch.float32,
                          action_shape=envs.single_action_space.shape)
    start_time = time.time()

    obs, _ = envs.reset(seed=args.seed)
    for global_step in range(args.total_timesteps):
        if global_step < args.learning_starts:
            actions = np.array([envs.single_action_space.sample() for _ in range(envs.num_envs)])
        else:
            actions = actor(torch.from_numpy(np.asarray(obs, dtype=np.float32)).to(device))
            actions += agents._exploration_noise(actor.action_scale * args.exploration_noise)
            actions = actions.cpu().numpy().clip(low, high)

        next_obs, rewards, terminations, truncations, infos = envs.step(actions)
        if "final_info" in infos:
            for info in infos["final_info"]:
                if info is not None:
                    print(f"global_step={global_step}, episodic_return={info['episode']['r']}")
                    writer.add_scalar("charts/episodic_return", info["episode"]["r"], global_step)
                    writer.add_scalar("charts/episodic_length", info["episode"]["l"], global_step)
                    break

        real_next_obs = next_obs.copy()
        for idx, trunc in enumerate(truncations):
            if trunc:
                real_next_obs[idx] = infos["final_observation"][idx]
        rb.add(obs, real_next_obs, actions, rewards, terminations, infos)
        obs = next_obs

        if global_step > args.learning_starts:
            data = rb.sample(args.batch_size)
            ddpg_update(state, rb, data, global_step, args)
            if on_update is not None:
                on_update(global_step, state)

            if global_step % 100 == 0:
                q1v, q1l = state.qstats.cpu().tolist()
                (actor_loss,) = state.astats.cpu().tolist()        # the latest actor step's, as the reference logs
                writer.add_scalar("losses/qf1_values", q1v, global_step)
                writer.add_scalar("losses/qf1_loss", q1l, global_step)
                writer.add_scalar("losses/actor_loss", actor_loss, global_step)
                print("SPS:", int(global_step / (time.time() - start_time)))
                writer.add_scalar("charts/SPS", int(global_step / (time.time() - start_time)), global_step)

    if args.save_model:
        os.makedirs(f"runs/{run_name}", exist_ok=True)
        model_path = f"runs/{run_name}/{args.exp_name}.cleanrl_model"
        torch.save((actor.state_dict(), qf1.state_dict()), model_path)
        print(f"model saved to {model_path}")
        # evaluation of the saved model as the reference does (ddpg_continuous_action.py:249-262)
        from cleanrl_b200.evals import evaluate_ddpg

        eval_envs = env_factory(args) if env_factory else make_envs(args, f"{run_name}-eval")
        episodic_returns = evaluate_ddpg(model_path, make_env, args.env_id, eval_episodes=10,
                                         run_name=f"{run_name}-eval", Model=(Actor, QNetwork), device=device,
                                         exploration_noise=args.exploration_noise, envs=eval_envs)
        eval_envs.close()
        for idx, episodic_return in enumerate(episodic_returns):
            writer.add_scalar("eval/episodic_return", float(np.asarray(episodic_return).reshape(-1)[0]), idx)
        if args.upload_model:
            print("[cleanrl_b200] --upload-model needs cleanrl_utils.huggingface (not part of the hot path); skipped",
                  file=sys.stderr)

    envs.close()
    writer.close()
    return actor, qf1, state


if __name__ == "__main__":
    main()
