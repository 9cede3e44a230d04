"""Post-training evaluation with the call surfaces of cleanrl_utils/evals/ppo_eval.py:7-36, dqn_eval.py:9-44, c51_eval.py,
td3_eval.py and ddpg_eval.py (SURVEY.md 8f rank 1).

``evaluate(model_path, make_env, env_id, eval_episodes, run_name, Model, device, capture_video, gamma)`` rebuilds
the agent from a ``.cleanrl_model`` file (a plain ``state_dict`` whose keys equal the reference's, so files written
by either implementation load in both) and plays until ``eval_episodes`` episode returns have been collected.
The policy runs on libb200rl kernels through ``Model.get_action_and_value``.
"""
from __future__ import annotations

import numpy as np
import torch


def _single_env(make_env, env_id, capture_video, run_name, gamma):
    import gymnasium as gym  # type: ignore

    return gym.vector.SyncVectorEnv([make_env(env_id, 0, capture_video, run_name, gamma)])


def _finished_returns(infos):
    """Episode returns reported by gymnasium's RecordEpisodeStatistics in this step (possibly none)."""
    out = []
    for info in infos.get("final_info", ()):
        if info and "episode" in info:
            out.append(info["episode"]["r"])
    return out


def evaluate(model_path, make_env, env_id, eval_episodes, run_name, Model, device=torch.device("cuda"),
             capture_video=True, gamma=0.99, envs=None, max_steps=100000):
    envs = envs if envs is not None else _single_env(make_env, env_id, capture_video, run_name, gamma)
    agent = Model(envs).to(device)
    agent.load_state_dict(torch.load(model_path, map_location=device))
    agent.eval()

    episodic_returns = []
    obs, _ = envs.reset()
    for _ in range(max_steps):
        if len(episodic_returns) >= eval_episodes:
            break
        with torch.no_grad():
            action = agent.get_action_and_value(torch.as_tensor(np.asarray(obs)).to(device))[0]
        obs, _, _, _, infos = envs.step(action.cpu().numpy())
        for ret in _finished_returns(infos):
            print(f"eval_episode={len(episodic_returns)}, episodic_return={ret}")
            episodic_returns.append(ret)
    return episodic_returns


def evaluate_q(model_path, make_env, env_id, eval_episodes, run_name, Model, device=torch.device("cuda"),
               epsilon=0.05, capture_video=True, envs=None, max_steps=1000000):
    """Epsilon-greedy rollout of a saved Q-network (cleanrl_utils/evals/dqn_eval.py): ``Model(envs)`` is rebuilt from
    the ``.cleanrl_model`` state_dict, greedy actions come from ``Model.forward`` (libb200rl kernels + argmax), with
    probability ``epsilon`` every env takes a uniformly sampled action instead (python's ``random`` as the reference)."""
    import random

    if envs is None:
        import gymnasium as gym  # type: ignore

        envs = gym.vector.SyncVectorEnv([make_env(env_id, 0, 0, capture_video, run_name)])
    model = Model(envs).to(device)
    model.load_state_dict(torch.load(model_path, map_location=device))
    model.eval()

    returns = []
    obs, _ = envs.reset()
    for _ in range(max_steps):
        if len(returns) >= eval_episodes:
            break
        if random.random() < epsilon:
            actions = np.array([envs.single_action_space.sample() for _ in range(envs.num_envs)])
        else:
            with torch.no_grad():
                q = model(torch.as_tensor(np.asarray(obs)).to(device))
            actions = q.argmax(dim=1).cpu().numpy()
        obs, _, _, _, infos = envs.step(actions)
        for ret in _finished_returns(infos):
            print(f"eval_episode={len(returns)}, episodic_return={ret}")
            returns.append(ret)
    return returns


def evaluate_c51(model_path, make_env, env_id, eval_episodes, run_name, Model, device=torch.device("cuda"),
                 epsilon=0.05, capture_video=True, envs=None, max_steps=1000000):
    """Epsilon-greedy rollout of a saved C51 network (cleanrl_utils/evals/c51_eval.py): the file holds
    ``{"model_weights": state_dict, "args": vars(args)}``; ``Model(envs, n_atoms=, v_min=, v_max=)`` is rebuilt from the
    saved args and acts through ``Model.get_action`` (libb200rl kernels)."""
    import random
    from argparse import Namespace

    if envs is None:
        import gymnasium as gym  # type: ignore

        envs = gym.vector.SyncVectorEnv([make_env(env_id, 0, 0, capture_video, run_name)])
    model_data = torch.load(model_path, map_location="cpu")
    args = Namespace(**model_data["args"])
    model = Model(envs, n_atoms=args.n_atoms, v_min=args.v_min, v_max=args.v_max)
    model.load_state_dict(model_data["model_weights"])
    model = model.to(device)
    model.eval()

    returns = []
    obs, _ = envs.reset()
    for _ in range(max_steps):
        if len(returns) >= eval_episodes:
            break
        if random.random() < epsilon:
            actions = np.array([envs.single_action_space.sample() for _ in range(envs.num_envs)])
        else:
            with torch.no_grad():
                actions, _ = model.get_action(torch.as_tensor(np.asarray(obs)).to(device))
            actions = actions.cpu().numpy()
        obs, _, _, _, infos = envs.step(actions)
        for ret in _finished_returns(infos):
            print(f"eval_episode={len(returns)}, episodic_return={ret}")
            returns.append(ret)
    return returns


def _noisy_actor_returns(actor, envs, eval_episodes, exploration_noise, device, max_steps):
    """The rollout of cleanrl_utils/evals/td3_eval.py and ddpg_eval.py: reset without a seed, then each step adds one
    ``torch.normal(0, action_scale * exploration_noise)`` draw to the actor's actions (libb200rl kernels) and clips
    them to the single action space on the host, until ``eval_episodes`` returns are in."""
    returns = []
    obs, _ = envs.reset()
    for _ in range(max_steps):
        if len(returns) >= eval_episodes:
            break
        with torch.no_grad():
            actions = actor(torch.as_tensor(np.asarray(obs, dtype=np.float32)).to(device))
            actions += torch.normal(0, actor.action_scale * exploration_noise)
            actions = actions.cpu().numpy().clip(envs.single_action_space.low, envs.single_action_space.high)
        obs, _, _, _, infos = envs.step(actions)
        for ret in _finished_returns(infos):
            print(f"eval_episode={len(returns)}, episodic_return={ret}")
            returns.append(ret)
    return returns


def _load_actor_and_critics(model_path, envs, Model, n_critics, device):
    """Rebuild ``Model[0]`` (the actor) and ``n_critics`` ``Model[1]`` critics from a file holding their state_dicts in
    that order; the critics are loaded but not used, as in the reference."""
    nets_ = [Model[0](envs).to(device)] + [Model[1](envs).to(device) for _ in range(n_critics)]
    for m, sd in zip(nets_, torch.load(model_path, map_location=device)):
        m.load_state_dict(sd)
        m.eval()
    return nets_[0]


def _gymnasium_env(make_env, env_id, capture_video, run_name):
    import gymnasium as gym  # type: ignore

    return gym.vector.SyncVectorEnv([make_env(env_id, 0, 0, capture_video, run_name)])


def evaluate_td3(model_path, make_env, env_id, eval_episodes, run_name, Model, device=torch.device("cuda"),
                 capture_video=True, exploration_noise=0.1, envs=None, max_steps=1000000):
    """Noisy deterministic rollout of a saved TD3 actor (cleanrl_utils/evals/td3_eval.py): the file holds
    ``(actor.state_dict(), qf1.state_dict(), qf2.state_dict())``; ``Model = (Actor, QNetwork)``.  Each step adds one
    ``torch.normal(0, action_scale * exploration_noise)`` draw to the actor's actions (libb200rl kernels) and clips
    them to the action space on the host; the critics are loaded but not used, as in the reference."""
    envs = envs if envs is not None else _gymnasium_env(make_env, env_id, capture_video, run_name)
    actor = _load_actor_and_critics(model_path, envs, Model, 2, device)
    return _noisy_actor_returns(actor, envs, eval_episodes, exploration_noise, device, max_steps)


def evaluate_ddpg(model_path, make_env, env_id, eval_episodes, run_name, Model, device=torch.device("cuda"),
                  capture_video=True, exploration_noise=0.1, envs=None, max_steps=1000000):
    """Noisy deterministic rollout of a saved DDPG actor (cleanrl_utils/evals/ddpg_eval.py): the file holds
    ``(actor.state_dict(), qf1.state_dict())``; ``Model = (Actor, QNetwork)``; the rollout is ``evaluate_td3``'s."""
    envs = envs if envs is not None else _gymnasium_env(make_env, env_id, capture_video, run_name)
    actor = _load_actor_and_critics(model_path, envs, Model, 1, device)
    return _noisy_actor_returns(actor, envs, eval_episodes, exploration_noise, device, max_steps)
