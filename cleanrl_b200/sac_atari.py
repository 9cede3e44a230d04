"""Drop-in for cleanrl/sac_atari.py (discrete soft actor-critic, Christodoulou 2019) on libb200rl.

Same flags, ``Actor`` / ``SoftQNetwork`` surface and state_dict keys, initialisation, TensorBoard tags and stdout as the
reference (cleanrl/sac_atari.py:27-74,102-171,174-320).  The numpy ``ReplayBuffer`` becomes the device-resident uint8
ring in the reference's ``optimize_memory_usage=False`` layout (``cleanrl_b200.replay.DeviceReplayRing``), sampled with
the same numpy index stream; the sampled frames are gathered inside the conv kernels.  The soft-Q target with both
critic losses, and the actor loss with the temperature step, are one kernel each; the temperature stays on the device
(the host reads it only at logging steps); Adam is the fused flat step.  With ``--precision bf16`` the whole update is
replayed as one CUDA graph.
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
from cleanrl_b200.agents import SACActor as Actor, SACState, SoftQNetwork, dqn_sync_target, sac_update
from cleanrl_b200.agents import sac_layer_init as layer_init  # noqa: F401  (the reference's module-level name)
from cleanrl_b200.dqn_atari import make_env, make_envs  # noqa: F401
from cleanrl_b200.replay import DeviceReplayRing

Args = cli.sac_atari_args(os.path.basename(__file__)[: -len(".py")])
run_name = None


def main(argv=None, writer_factory=None, env_factory=None, on_update=None):
    """``on_update(global_step, state, nets)`` runs after every update with the ``SACState`` and
    ``(actor, qf1, qf2, qf1_target, qf2_target)``."""
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
        raise RuntimeError("cleanrl_b200.sac_atari runs on libb200rl CUDA kernels: a CUDA device and --cuda are "
                           "required (no CPU fallback).")
    device = torch.device("cuda")

    args.num_envs = 1
    envs = env_factory(args) if env_factory else make_envs(args, run_name)
    assert hasattr(envs.single_action_space, "n"), "only discrete action space is supported"

    # construction order of the reference (sac_atari.py:207-213): it fixes the generator stream
    nets = [Actor(envs), SoftQNetwork(envs), SoftQNetwork(envs), SoftQNetwork(envs), SoftQNetwork(envs)]
    actor, qf1, qf2, qf1_target, qf2_target = [n.to(device) for n in nets]
    qf1_target.load_state_dict(qf1.state_dict())
    qf2_target.load_state_dict(qf2.state_dict())
    for n in (actor, qf1, qf2, qf1_target, qf2_target):
        n.precision = args.precision
        n.flat
    A = int(envs.single_action_space.n)
    state = SACState(A, device, autotune=args.autotune, alpha=args.alpha, target_entropy_scale=args.target_entropy_scale)

    rb = DeviceReplayRing(args.buffer_size, envs.single_observation_space.shape, 1, device, optimize_memory_usage=False)
    start_time = time.time()

    obs, _ = envs.reset(seed=args.seed)
    for global_step in range(args.total_timesteps):
        if global_step < args.learning_starts:
            actions = np.array([envs.single_action_space.sample() for _ in range(envs.num_envs)])
        else:
            actions, _, _ = actor.get_action(torch.from_numpy(np.ascontiguousarray(obs)).to(device))
            actions = actions.detach().cpu().numpy()

        next_obs, rewards, terminations, truncations, infos = envs.step(actions)
        if "final_info" in infos:
            for info in infos["final_info"]:
                if not info or "episode" not in info:
                    continue
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
            if global_step % args.update_frequency == 0:
                data = rb.sample(args.batch_size)
                sac_update(actor, qf1, qf2, qf1_target, qf2_target, rb, data, state, args.gamma, args.q_lr, args.policy_lr)
                if on_update is not None:
                    on_update(global_step, state, (actor, qf1, qf2, qf1_target, qf2_target))

            # hard (tau = 1) or soft target update (sac_atari.py:317-321)
            if global_step % args.target_network_frequency == 0:
                dqn_sync_target(qf1, qf1_target, args.tau)
                dqn_sync_target(qf2, qf2_target, args.tau)

            if global_step % 100 == 0:
                q1v, q2v, q1l, q2l = state.qstats.cpu().tolist()
                actor_loss, alpha_loss, alpha, _ = state.astats.cpu().tolist()
                writer.add_scalar("losses/qf1_values", q1v, global_step)
                writer.add_scalar("losses/qf2_values", q2v, global_step)
                writer.add_scalar("losses/qf1_loss", q1l, global_step)
                writer.add_scalar("losses/qf2_loss", q2l, global_step)
                writer.add_scalar("losses/qf_loss", float(np.float32(q1l) + np.float32(q2l)) / 2.0, global_step)
                writer.add_scalar("losses/actor_loss", actor_loss, global_step)
                writer.add_scalar("losses/alpha", alpha if args.autotune else args.alpha, global_step)
                print("SPS:", int(global_step / (time.time() - start_time)))
                writer.add_scalar("charts/SPS", int(global_step / (time.time() - start_time)), global_step)
                if args.autotune:
                    writer.add_scalar("losses/alpha_loss", alpha_loss, global_step)

    envs.close()
    writer.close()
    return actor, qf1, qf2, state


if __name__ == "__main__":
    main()
