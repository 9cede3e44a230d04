"""Drop-in for cleanrl/ppo_atari_lstm.py: recurrent PPO (NatureCNN trunk -> LSTM(512, 128) -> actor / critic) on libb200rl.

Same CLI flags (``Args``), ``Agent`` surface (``get_states`` / ``get_value`` / ``get_action_and_value`` taking and
returning the LSTM state), ``state_dict`` keys, TensorBoard tags and stdout lines as the reference
(cleanrl/ppo_atari_lstm.py:26-83,117-160,197-375).  The loop keeps the reference's structure -- LSTM state carried across
the rollout, ``initial_lstm_state`` snapshot per iteration, minibatches over whole ENV sequences (``envsperbatch`` envs x
all steps, time-major indices, :297-312) -- and runs on the same kernels as the feed-forward scripts: the one-launch GAE,
the fused loss (+ its gradient), hand-written backward (back-propagation through time in ``LSTMAgent``), fused clip + Adam
over one flat parameter vector.  Observations stay uint8 on the device; ``b_obs[mb_inds]`` is a row gather inside the first
conv kernel.
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

from cleanrl_b200 import cli, ops
from cleanrl_b200.agents import LSTMAgent as Agent, layer_init  # noqa: F401  (reference module-level names)

Args = cli.ppo_atari_args(os.path.basename(__file__)[: -len(".py")])
run_name = None


def make_env(env_id, idx, capture_video, run_name):
    """The reference's wrapper stack with a single-frame stack (cleanrl/ppo_atari_lstm.py:86-108)."""
    def thunk():
        import gymnasium as gym  # type: ignore
        from cleanrl_utils.atari_wrappers import (ClipRewardEnv, EpisodicLifeEnv, FireResetEnv, MaxAndSkipEnv,  # type: ignore
                                                  NoopResetEnv)
        if capture_video and idx == 0:
            env = gym.make(env_id, render_mode="rgb_array")
            env = gym.wrappers.RecordVideo(env, f"videos/{run_name}")
        else:
            env = gym.make(env_id)
        env = gym.wrappers.RecordEpisodeStatistics(env)
        env = NoopResetEnv(env, noop_max=30)
        env = MaxAndSkipEnv(env, skip=4)
        env = EpisodicLifeEnv(env)
        if "FIRE" in env.unwrapped.get_action_meanings():
            env = FireResetEnv(env)
        env = ClipRewardEnv(env)
        env = gym.wrappers.ResizeObservation(env, (84, 84))
        env = gym.wrappers.GrayScaleObservation(env)
        env = gym.wrappers.FrameStack(env, 1)
        return env

    return thunk


def make_envs(args, run_name):
    if not cli.use_synthetic(args):
        try:
            import gymnasium as gym  # type: ignore  # noqa: F401
        except ImportError as e:
            raise cli.env_import_error("gymnasium (+ ale-py, cleanrl_utils.atari_wrappers)", e) from e
        return gym.vector.SyncVectorEnv([make_env(args.env_id, i, args.capture_video, run_name) for i in range(args.num_envs)])
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec

    return SyntheticGymnasiumVec(args.num_envs, kind="atari1")


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
        raise RuntimeError("cleanrl_b200.ppo_atari_lstm runs on libb200rl CUDA kernels: a CUDA device and --cuda are "
                           "required (no CPU fallback). Use the reference script for CPU runs.")
    device = torch.device("cuda")

    envs = env_factory(args) if env_factory else make_envs(args, run_name)
    assert hasattr(envs.single_action_space, "n"), "only discrete action space is supported"
    agent = Agent(envs).to(device)
    agent.precision = args.precision
    if agent_hook:
        agent_hook(agent)
    flat = agent.flat
    T, N = args.num_steps, args.num_envs
    B = T * N
    H = agent.hidden_size
    obs_shape = tuple(envs.single_observation_space.shape)
    f32 = torch.float32

    # storage (ppo_atari_lstm.py:214-220): frames stay uint8
    obs = torch.zeros((T, N) + obs_shape, dtype=torch.uint8, device=device)
    actions = torch.zeros((T, N), dtype=torch.int64, device=device)
    logprobs = torch.zeros((T, N), dtype=f32, device=device)
    rewards = torch.zeros((T, N), dtype=f32, device=device)
    dones = torch.zeros((T, N), dtype=f32, device=device)
    values = torch.zeros((T, N), dtype=f32, device=device)
    advantages = torch.zeros((T, N), dtype=f32, device=device)
    returns = torch.zeros((T, N), dtype=f32, device=device)
    n_upd = int(args.update_epochs) * int(args.num_minibatches)
    stats = torch.zeros(max(n_upd, 1), 16, dtype=f32, device=device)
    rewards_h = torch.zeros((T, N), dtype=f32).pin_memory()

    global_step = 0
    start_time = time.time()
    next_obs_np, _ = envs.reset(seed=args.seed)
    next_obs = torch.from_numpy(np.ascontiguousarray(next_obs_np)).to(device=device, dtype=torch.uint8)
    next_done = torch.zeros(N, dtype=f32, device=device)
    next_lstm_state = (torch.zeros(1, N, H, dtype=f32, device=device), torch.zeros(1, N, H, dtype=f32, device=device))
    lrnow = args.learning_rate
    scratch = {}

    for iteration in range(1, args.num_iterations + 1):
        initial_lstm_state = (next_lstm_state[0].clone(), next_lstm_state[1].clone())
        if args.anneal_lr:
            frac = 1.0 - (iteration - 1.0) / args.num_iterations
            lrnow = frac * args.learning_rate

        with torch.no_grad():
            for step in range(0, T):
                global_step += N
                obs[step].copy_(next_obs)
                dones[step].copy_(next_done)
                action, logprob, _, value, next_lstm_state = agent.get_action_and_value(next_obs, next_lstm_state, next_done)
                values[step].copy_(value.flatten())
                actions[step].copy_(action)
                logprobs[step].copy_(logprob)
                next_obs_np, reward, terminations, truncations, infos = envs.step(action.cpu().numpy())
                rewards_h[step].copy_(torch.as_tensor(np.asarray(reward, dtype=np.float32).reshape(-1)))
                next_done_np = np.logical_or(terminations, truncations)
                next_obs = torch.from_numpy(np.ascontiguousarray(next_obs_np)).to(device=device, dtype=torch.uint8)
                next_done = torch.from_numpy(next_done_np.astype(np.float32)).to(device)
                if "final_info" in infos:
                    for info in infos["final_info"]:
                        if info and "episode" in info:
                            print(f"global_step={global_step}, episodic_return={info['episode']['r']}")
                            writer.add_scalar("charts/episodic_return", info["episode"]["r"], global_step)
                            writer.add_scalar("charts/episodic_length", info["episode"]["l"], global_step)

            # bootstrap value + GAE (ppo_atari_lstm.py:262-280): one kernel
            rewards.copy_(rewards_h, non_blocking=True)
            next_value = agent.get_value(next_obs, next_lstm_state, next_done).reshape(-1)
            ops.gae(rewards, values, dones, next_value, next_done, args.gamma, args.gae_lambda,
                    mode=0 if args.gae_kernel == "sequential" else 1, out=(advantages, returns))

            # flatten the batch; minibatches are whole env sequences (ppo_atari_lstm.py:283-312)
            b_obs = obs.reshape((-1,) + obs_shape)
            b = {"actions": actions.view(B), "logprobs": logprobs.view(B), "advantages": advantages.view(B),
                 "returns": returns.view(B), "values": values.view(B)}
            assert N % args.num_minibatches == 0
            envsperbatch = N // args.num_minibatches
            envinds = np.arange(N)
            flatinds = np.arange(B).reshape(T, N)
            k = 0
            stop = False
            for epoch in range(args.update_epochs):
                np.random.shuffle(envinds)
                for start in range(0, N, envsperbatch):
                    mbenvinds = envinds[start:start + envsperbatch]
                    mb_inds_np = flatinds[:, mbenvinds].ravel()            # time-major: be really careful about the index
                    mb_inds = torch.from_numpy(mb_inds_np).to(device)
                    env_t = torch.from_numpy(mbenvinds).to(device)
                    state = (initial_lstm_state[0][:, env_t].contiguous(), initial_lstm_state[1][:, env_t].contiguous())
                    logits, value = agent.forward_train(b_obs, mb_inds, state, dones.view(B))
                    agent.loss_backward(logits, value, mb_inds, b, args, stats[k], scratch)
                    flat.step += 1
                    ops.clip_adam(flat.flat, flat.grad, flat.exp_avg, flat.exp_avg_sq, flat.step, lrnow, eps=1e-5,
                                  max_norm=args.max_grad_norm)
                    agent.params_updated()
                    k += 1
                if args.target_kl is not None and stats[k - 1, 4].item() > args.target_kl:
                    stop = True
                if stop:
                    break
        s = stats[:k].cpu().numpy()
        st = {name: float(s[k - 1, i]) for i, name in enumerate(ops.STAT_NAMES)}
        st["clipfrac_mean"] = float(np.mean(s[:, 5].astype(np.float64)))
        st["per_update"], st["num_updates"] = s.copy(), k

        y_pred, y_true = values.view(-1).cpu().numpy(), returns.view(-1).cpu().numpy()
        var_y = np.var(y_true)
        explained_var = np.nan if var_y == 0 else 1 - np.var(y_true - y_pred) / var_y

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
            on_iteration(iteration, dict(actions=actions, logprobs=logprobs, values=values, rewards=rewards, dones=dones,
                                         advantages=advantages, returns=returns, agent=agent,
                                         lstm_state=next_lstm_state), st)

    envs.close()
    writer.close()
    return agent


if __name__ == "__main__":
    main()
