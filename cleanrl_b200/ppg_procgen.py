"""Drop-in for cleanrl/ppg_procgen.py: phasic policy gradient with the IMPALA-CNN agent on libb200rl.

Same CLI flags (``Args``), module-level names, ``Agent`` module tree and ``state_dict`` keys, asserts, TensorBoard tags and
stdout lines as the reference (cleanrl/ppg_procgen.py:19-98,101-211,285-477).  The policy phase is the shared engine's
rollout, GAE and fused PPO loss; the auxiliary buffer (uint8 frames, returns, old logits) stays on the device and the
auxiliary phase runs forward, fused distillation loss, hand-written backward and clip + Adam per minibatch without a
host synchronisation inside an epoch (cleanrl_b200/ppg_engine.py).
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
from cleanrl_b200.agents import PPGAgent as Agent, PPGConvSequence as ConvSequence, PPGResidualBlock as ResidualBlock  # noqa: F401
from cleanrl_b200.agents import layer_init_normed  # noqa: F401
from cleanrl_b200.ppg_engine import PPGEngine
from cleanrl_b200.ppo_procgen import make_envs

Args = cli.ppg_procgen_args(os.path.basename(__file__)[: -len(".py")])
run_name = None


def flatten01(arr):
    return arr.reshape((-1, *arr.shape[2:]))


def unflatten01(arr, targetshape):
    return arr.reshape((*targetshape, *arr.shape[1:]))


def flatten_unflatten_test():
    a = torch.rand(40, 3, 10, 10, 5)
    b = flatten01(a)
    c = unflatten01(b, a.shape[:2])
    assert torch.equal(a, c)


def main(argv=None, writer_factory=None, env_factory=None, on_iteration=None, on_aux_phase=None, agent_hook=None):
    global run_name
    args = cli.parse(Args, argv)
    args.batch_size = int(args.num_envs * args.num_steps)
    args.minibatch_size = int(args.batch_size // args.num_minibatches)
    args.num_iterations = args.total_timesteps // args.batch_size
    args.num_phases = int(args.num_iterations // args.n_iteration)
    args.aux_batch_rollouts = int(args.num_envs * args.n_iteration)
    assert args.v_value == 1, "Multiple value epoch (v_value != 1) is not supported yet"
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

    flatten_unflatten_test()

    random.seed(args.seed)
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)
    torch.backends.cudnn.deterministic = args.torch_deterministic
    if not (torch.cuda.is_available() and args.cuda):
        raise RuntimeError("cleanrl_b200.ppg_procgen runs on libb200rl CUDA kernels: a CUDA device and --cuda are required "
                           "(no CPU fallback). Use the reference script for CPU runs.")
    device = torch.device("cuda")

    envs = env_factory(args) if env_factory else make_envs(args, run_name)
    assert hasattr(envs.single_action_space, "n"), "only discrete action space is supported"
    agent = Agent(envs).to(device)
    agent.precision = args.precision
    if agent_hook:
        agent_hook(agent)
    engine = PPGEngine(agent, args, envs.single_observation_space.shape, args.num_envs, device,
                       gae_mode=0 if args.gae_kernel == "sequential" else 1)

    global_step = 0
    start_time = time.time()
    next_obs = np.asarray(envs.reset())
    next_done = np.zeros(args.num_envs, dtype=np.float32)
    lrnow = args.learning_rate

    for phase in range(1, args.num_phases + 1):

        # POLICY PHASE
        for update in range(1, args.n_iteration + 1):
            if args.anneal_lr:
                frac = 1.0 - (update - 1.0) / args.num_iterations
                lrnow = frac * args.learning_rate

            for step in range(0, args.num_steps):
                global_step += 1 * args.num_envs
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

            engine.store_rollout(update)
            if on_iteration is not None:
                on_iteration(phase, update, engine, st)

        # AUXILIARY PHASE
        aux = engine.aux_phase(lrnow, on_epoch=lambda k: print(f"aux epoch {k}"))
        writer.add_scalar("losses/aux/kl_loss", aux["kl_loss"], global_step)
        writer.add_scalar("losses/aux/aux_value_loss", aux["aux_value_loss"], global_step)
        writer.add_scalar("losses/aux/real_value_loss", aux["real_value_loss"], global_step)
        if on_aux_phase is not None:
            on_aux_phase(phase, engine, aux)

    envs.close()
    writer.close()
    return engine


if __name__ == "__main__":
    main()
