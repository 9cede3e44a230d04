"""DDPG (cleanrl/ddpg_continuous_action.py) without a GPU: the oracle's one-critic loss and gradient against autograd,
the oracle against the first update of the reference runs, the replay ring's index stream, the CLI / module surface,
the networks' construction (the actor's buffers from the batched or unbatched ``action_space``), and argument
validation of the new C entry point and mode."""
from __future__ import annotations

import dataclasses
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import ddpg_continuous_oracle as O

GOLDEN = Path(__file__).resolve().parent / "golden"
FIXTURES = ["ddpg_continuous_seed1.npz", "ddpg_continuous_seed2_pf3.npz"]


def test_critic_loss_matches_autograd():
    g = torch.Generator().manual_seed(5)
    B = 32
    q, qn = torch.randn(B, generator=g), torch.randn(B, generator=g)
    r, d = torch.randn(B, generator=g), (torch.rand(B, generator=g) < 0.2).float()
    y, loss, dq = O.critic_loss(q, qn, r, d, 0.99)
    assert torch.equal(y, r.flatten() + (1 - d.flatten()) * 0.99 * qn.view(-1))   # ddpg_continuous_action.py:219
    a = q.clone().requires_grad_(True)
    ref = torch.nn.functional.mse_loss(a, y)
    ref.backward()
    assert torch.equal(loss, ref.detach())
    torch.testing.assert_close(dq, a.grad, rtol=1e-6, atol=0)


def _flag(argv, name, default, cast=int):
    return cast(argv[argv.index(name) + 1]) if name in argv else default


def _env(batched):
    """The synthetic HalfCheetah-shaped env; ``batched``: ``action_space`` as gymnasium's one-env SyncVectorEnv has
    it, the [1, D] Box."""
    from cleanrl_b200.synthetic_envs import Box, SyntheticGymnasiumVec
    env = SyntheticGymnasiumVec(1, kind="continuous")
    if batched:
        env.action_space = Box(-1.0, 1.0, (1, 6), np.float32)
    return env


def _reference_nets(seed, batched):
    """The reference's networks on the CPU: torch.manual_seed(seed), then actor, qf1, qf1_target, target_actor in its
    construction order (ddpg_continuous_action.py:139,151-156)."""
    from cleanrl_b200.agents import DDPGActor, SoftQNetworkMLP
    env = _env(batched)
    torch.manual_seed(seed)
    nets = [DDPGActor(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env), DDPGActor(env)]
    nets[3].load_state_dict(nets[0].state_dict())
    nets[2].load_state_dict(nets[1].state_dict())
    return nets


def _vec(*ns):
    return torch.cat([torch.nn.utils.parameters_to_vector(n.parameters()) for n in ns])


def _batched(z):
    return z["action_scale"].ndim == 2


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_the_reference_first_update(name):
    z = np.load(GOLDEN / name)
    argv = z["argv"].tolist()
    nets = _reference_nets(_flag(argv, "--seed", 1), _batched(z))
    assert list(nets[0].state_dict()) == z["actor_keys"].tolist() and list(nets[1].state_dict()) == z["qf_keys"].tolist()
    assert [str(tuple(v.shape)) for v in nets[0].state_dict().values()] == z["actor_shapes"].tolist()
    assert [str(tuple(v.shape)) for v in nets[1].state_dict().values()] == z["qf_shapes"].tolist()
    ref = O.EagerDDPG(_vec(nets[0]), _vec(nets[1]), _vec(nets[2]), _vec(nets[3]), 17, 6, nets[0].action_scale,
                      nets[0].action_bias, "cpu", tau=_flag(argv, "--tau", 0.005, float),
                      policy_frequency=_flag(argv, "--policy-frequency", 2))
    step = _flag(argv, "--learning-starts", 40) + 1           # the first update runs at global_step learning_starts + 1
    ref.update(step, torch.from_numpy(z["u1_obs"]), torch.from_numpy(z["u1_actions"]), torch.from_numpy(z["u1_next_obs"]),
               torch.from_numpy(z["u1_rewards"]), torch.from_numpy(z["u1_dones"]))
    np.testing.assert_allclose(ref.stats["next_state_actions"].numpy(), z["u1_next_state_actions"], rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(ref.stats["y"].numpy(), z["u1_y"], rtol=1e-6, atol=1e-6)
    for k in ("qf1_loss", "qf1_values"):
        assert ref.stats[k]() == pytest.approx(z[k][0], rel=1e-5, abs=1e-6), k
    np.testing.assert_allclose(_sums(ref.qf1), z["q_sums"][0], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(ref.qf1.fc3.bias.grad.numpy(), z["u1_dq1_bias"], rtol=1e-5, atol=1e-7)
    assert np.isnan(z["actor_loss"][0])                       # a critic-only update leaves the targets alone
    np.testing.assert_allclose(_sums(ref.target_actor, ref.qf1_target), z["target_sums"][0], rtol=1e-6, atol=1e-6)


def _sums(*nets):
    return np.array([p.detach().double().sum().item() for n in nets for p in n.parameters()])


def test_fixtures_cover_the_delayed_actor_step_and_both_buffer_shapes():
    z = np.load(GOLDEN / "ddpg_continuous_seed2_pf3.npz")
    ls = _flag(z["argv"].tolist(), "--learning-starts", 40)
    steps = np.arange(ls + 1, ls + 1 + len(z["actor_loss"]))
    assert np.array_equal(~np.isnan(z["actor_loss"]), steps % 3 == 0)
    # step 100 is not a policy step: the logged actor_loss is the one of step 99
    assert z["tb/losses/actor_loss"][0, 0] == 100
    assert z["tb/losses/actor_loss"][0, 1] == pytest.approx(z["actor_loss"][steps == 99][0], rel=1e-6)
    # gymnasium's batched action_space: [1, D] buffers and [1, D] exploration draws; unbatched: [D]
    assert z["action_scale"].shape == (1, 6) and z["explore_draws"].shape == (len(z["action_stream"]) - ls, 1, 6)
    z1 = np.load(GOLDEN / "ddpg_continuous_seed1.npz")
    assert z1["action_scale"].shape == (6,) and z1["explore_draws"].shape == (len(z1["action_stream"]) - ls, 6)
    assert set(k[3:] for k in z1.files if k.startswith("tb/")) == {
        "charts/SPS", "charts/episodic_length", "charts/episodic_return", "losses/actor_loss", "losses/qf1_loss",
        "losses/qf1_values"}


@pytest.mark.parametrize("name", FIXTURES)
def test_replay_index_stream_matches_the_reference_run(name):
    from cleanrl_b200.replay import DeviceReplayRing
    z = np.load(GOLDEN / name)
    argv = z["argv"].tolist()
    bs = _flag(argv, "--batch-size", 256)
    rb = DeviceReplayRing(_flag(argv, "--buffer-size", 10 ** 6), (17,), 1, "cpu", optimize_memory_usage=False,
                          obs_dtype=torch.float32, action_shape=(6,))
    np.random.seed(_flag(argv, "--seed", 1))
    heads = []
    for step in range(_flag(argv, "--total-timesteps", 0)):
        rb.add(np.zeros((1, 17)), np.zeros((1, 17)), np.zeros((1, 6)), np.zeros(1), np.zeros(1))
        if step > _flag(argv, "--learning-starts", 0):
            bi, ei = rb.sample_indices(bs)
            heads += [bi[:8], ei[:8]]
    assert rb.full
    assert np.array_equal(np.stack(heads), z["randint_heads"])


def test_cli_fields_and_names_match_the_reference_surface():
    from cleanrl_b200 import cli, ddpg_continuous_action as m
    surf = json.loads((GOLDEN / "ddpg_continuous_surface.json").read_text())["ddpg_continuous_action.py"]
    fields = {f.name: f for f in dataclasses.fields(cli.ddpg_continuous_action_args())}
    for name, default, doc in surf["args"]:
        f = fields[name]
        if default != "<expr>":
            assert f.default == default, name
        assert f.type.__metadata__[0].help == doc, name
    assert fields["exp_name"].default == "ddpg_continuous_action" and fields["learning_starts"].default == 25e3
    assert fields["env_id"].type.__metadata__[0].help == "the environment id of the Atari game"
    assert set(fields) == {a[0] for a in surf["args"]} | {"synthetic_env"}
    assert "num_envs" not in fields
    for n in surf["names"]:
        assert hasattr(m, n), n
    assert m.Args is not None and m.QNetwork.__name__ == "SoftQNetworkMLP"


@pytest.mark.parametrize("batched", [False, True])
def test_networks_keep_the_reference_modules_and_init(batched):
    from cleanrl_b200.agents import DDPGActor
    nets = _reference_nets(4, batched)
    assert list(nets[0].state_dict()) == ["action_scale", "action_bias", "fc1.weight", "fc1.bias", "fc2.weight",
                                          "fc2.bias", "fc_mu.weight", "fc_mu.bias"]
    assert list(nets[1].state_dict()) == ["fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias", "fc3.weight", "fc3.bias"]
    shape = (1, 6) if batched else (6,)
    assert nets[0].action_scale.shape == shape and nets[3].action_bias.shape == shape
    assert torch.equal(nets[0].action_scale, torch.ones(shape)) and torch.equal(nets[0].action_bias, torch.zeros(shape))
    torch.manual_seed(4)
    a = [torch.nn.Linear(17, 256), torch.nn.Linear(256, 256), torch.nn.Linear(256, 6)]
    q = [[torch.nn.Linear(23, 256), torch.nn.Linear(256, 256), torch.nn.Linear(256, 1)] for _ in range(2)]
    t = [torch.nn.Linear(17, 256)]
    assert torch.equal(a[0].weight, nets[0].fc1.weight) and torch.equal(a[2].bias, nets[0].fc_mu.bias)
    assert torch.equal(q[0][0].weight, nets[1].fc1.weight) and torch.equal(q[0][2].bias, nets[2].fc3.bias)
    assert not torch.equal(q[1][0].weight, nets[2].fc1.weight)        # qf1_target was loaded from qf1
    assert not torch.equal(t[0].weight, nets[3].fc1.weight)            # the target actor was loaded from the actor
    assert torch.equal(nets[3].fc1.weight, nets[0].fc1.weight)
    with pytest.raises(RuntimeError, match="CUDA"):
        DDPGActor(_env(batched))(torch.zeros(2, 17))


@pytest.fixture(scope="module")
def lib():
    from cleanrl_b200 import _lib, build

    build.build()
    return _lib.load()


def test_entry_point_refuses_bad_arguments_without_gpu(lib):
    E, W = -1, -4
    assert lib.b200rl_sacc_param_count(17, 6, 3) == -1               # no new network kind
    P = 1 << 12
    ws = lib.b200rl_sacc_workspace_bytes(8)
    # ddpg_critic_loss_bwd(params, B, obs_dim, act_dim, q_next, q, r, d, ld_rd, rows, gamma, h1, h2, y, dq, dz1, dz2,
    #                      stats, ws, ws_bytes, stream)
    ok = [P, 8, 17, 6, P, P, P, P, 1, None, 0.99, P, P, None, P, P, P, P, P, ws, None]
    bad_args = [(1, 0), (1, 8193), (3, 0), (3, 33), (2, 1019), (2, 0), (8, 0), (9, P + 4), (4, P + 2)]
    bad_args += [(i, None) for i in (0, 4, 5, 6, 7, 11, 12, 14, 15, 16, 17, 18)]
    for i, bad in bad_args:
        a = list(ok)
        a[i] = bad
        assert lib.b200rl_ddpg_critic_loss_bwd_f32(*a) == E, (i, bad)
        assert "ddpg_critic_loss_bwd" in lib.b200rl_last_error().decode()
    a = list(ok)
    a[19] = ws - 1                                                    # short workspace
    assert lib.b200rl_ddpg_critic_loss_bwd_f32(*a) == W
    # the one-critic weight gradient (kind 1, net_stride 0) is new; a nonzero stride below one critic is still refused
    assert lib.b200rl_sacc_wgrad_f32(1, 8, 17, 6, P, P, P, P, P, P, P, 5, None) == E
    assert "net_stride" in lib.b200rl_last_error().decode()
    from cleanrl_b200 import ops
    assert ops.DDPG_CRITIC_STAT_NAMES == ("qf1_values", "qf1_loss")
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.ddpg_critic_loss_bwd(torch.zeros(8), 2, 17, 6, torch.zeros(2), torch.zeros(2), torch.zeros(2),
                                 torch.zeros(2), 0.99, torch.zeros(2, 256), torch.zeros(2, 256))
