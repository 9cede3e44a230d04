"""Drop-in for cleanrl/c51_atari.py (distributional Q-learning, Bellemare et al. 2017) on libb200rl.

Same flags, ``QNetwork`` surface / state_dict keys, epsilon schedule, TensorBoard tags and stdout as the reference
(cleanrl/c51_atari.py:25-138,199-299).  The numpy ``ReplayBuffer`` becomes the device-resident uint8 ring
(``cleanrl_b200.replay.DeviceReplayRing``) sampled with the same numpy index stream; the sampled frames are gathered
inside the conv kernels; the target projection (the reference's per-row ``index_add_`` loop), the cross-entropy and
dL/dlogits are one kernel; Adam is the fused flat step.
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
from cleanrl_b200.agents import C51QNetwork as QNetwork, c51_update, dqn_sync_target
from cleanrl_b200.dqn_atari import linear_schedule, make_env, make_envs
from cleanrl_b200.replay import DeviceReplayRing

Args = cli.c51_atari_args(os.path.basename(__file__)[: -len(".py")])
run_name = None


def main(argv=None, writer_factory=None, env_factory=None, on_update=None):
    global run_name
    args = cli.parse(Args, argv)
    assert args.num_envs == 1, "vectorized envs are not supported at the moment"   # c51_atari.py:148
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
        raise RuntimeError("cleanrl_b200.c51_atari runs on libb200rl CUDA kernels: a CUDA device and --cuda are "
                           "required (no CPU fallback).")
    device = torch.device("cuda")

    envs = env_factory(args) if env_factory else make_envs(args, run_name)
    assert hasattr(envs.single_action_space, "n"), "only discrete action space is supported"
    q_network = QNetwork(envs, n_atoms=args.n_atoms, v_min=args.v_min, v_max=args.v_max).to(device)
    target_network = QNetwork(envs, n_atoms=args.n_atoms, v_min=args.v_min, v_max=args.v_max).to(device)
    q_network.precision = target_network.precision = args.precision
    target_network.load_state_dict(q_network.state_dict())
    q_network.flat, target_network.flat
    rb = DeviceReplayRing(args.buffer_size, envs.single_observation_space.shape, args.num_envs, device)
    stats = torch.zeros(2, dtype=torch.float32, device=device)
    start_time = time.time()

    obs, _ = envs.reset(seed=args.seed)
    for global_step in range(args.total_timesteps):
        epsilon = linear_schedule(args.start_e, args.end_e, args.exploration_fraction * args.total_timesteps, global_step)
        if random.random() < epsilon:
            actions = np.array([envs.single_action_space.sample() for _ in range(envs.num_envs)])
        else:
            actions, pmf = q_network.get_action(torch.from_numpy(np.ascontiguousarray(obs)).to(device))
            actions = actions.cpu().numpy()

        next_obs, rewards, terminations, truncations, infos = envs.step(actions)
        if "final_info" in infos:
            for info in infos["final_info"]:
                if info and "episode" in info:
                    print(f"global_step={global_step}, episodic_return={info['episode']['r']}")
                    writer.add_scalar("charts/episodic_return", info["episode"]["r"], global_step)
                    writer.add_scalar("charts/episodic_length", info["episode"]["l"], global_step)

        real_next_obs = next_obs.copy()
        for idx, trunc in enumerate(truncations):
            if trunc:
                real_next_obs[idx] = infos["final_observation"][idx]
        rb.add(obs, real_next_obs, actions, rewards, terminations, infos)
        obs = next_obs

        if global_step > args.learning_starts:
            if global_step % args.train_frequency == 0:
                data = rb.sample(args.batch_size)
                c51_update(q_network, target_network, rb, data, args.gamma, args.learning_rate, args.v_min, args.v_max,
                           args.batch_size, stats=stats)
                if on_update is not None:
                    on_update(global_step, stats, q_network)
                if global_step % 100 == 0:
                    loss, q_mean = stats.cpu().tolist()
                    writer.add_scalar("losses/loss", loss, global_step)
                    writer.add_scalar("losses/q_values", q_mean, global_step)
                    sps = int(global_step / (time.time() - start_time))
                    print("SPS:", sps)
                    writer.add_scalar("charts/SPS", sps, global_step)
            # hard target copy (c51_atari.py:268-269)
            if global_step % args.target_network_frequency == 0:
                dqn_sync_target(q_network, target_network, 1.0)

    if args.save_model:
        os.makedirs(f"runs/{run_name}", exist_ok=True)
        model_path = f"runs/{run_name}/{args.exp_name}.cleanrl_model"
        model_data = {
            "model_weights": {k: v.detach().cpu() for k, v in q_network.state_dict().items()},
            "args": vars(args),
        }
        torch.save(model_data, model_path)
        print(f"model saved to {model_path}")
        # evaluation of the saved model as the reference does (c51_atari.py:279-292): 10 episodes, epsilon = end_e
        from cleanrl_b200.evals import evaluate_c51

        eval_args = type(args)(**{**vars(args), "num_envs": 1})
        eval_envs = env_factory(eval_args) if env_factory else make_envs(eval_args, f"{run_name}-eval")
        episodic_returns = evaluate_c51(model_path, None, args.env_id, eval_episodes=10, run_name=f"{run_name}-eval",
                                        Model=QNetwork, device=device, epsilon=args.end_e, envs=eval_envs)
        eval_envs.close()
        for idx, episodic_return in enumerate(episodic_returns):
            writer.add_scalar("eval/episodic_return", float(np.asarray(episodic_return).reshape(-1)[0]), idx)
        if args.upload_model:
            print("[cleanrl_b200] --upload-model needs cleanrl_utils.huggingface (not part of the hot path); skipped",
                  file=sys.stderr)

    envs.close()
    writer.close()
    return q_network


if __name__ == "__main__":
    main()
