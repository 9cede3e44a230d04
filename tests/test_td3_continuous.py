"""TD3 (cleanrl/td3_continuous_action.py) without a GPU: the oracle's deterministic head, its gradient and the target
policy smoothing against autograd on the reference's own expressions, the oracle against the first update of the
reference runs, the replay ring's index stream, the CLI / module surface, the networks' construction, and argument
validation of the new C entry points and modes."""
from __future__ import annotations

import dataclasses
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import td3_continuous_oracle as O

GOLDEN = Path(__file__).resolve().parent / "golden"
FIXTURES = ["td3_continuous_n2_seed1.npz", "td3_continuous_seed2_pf3.npz"]


@pytest.mark.parametrize("regime", ["typical", "saturated"])
def test_head_restatement_matches_autograd(regime):
    g = torch.Generator().manual_seed(3)
    B, D = 64, 6
    z = torch.randn(B, D, generator=g) * (12.0 if regime == "saturated" else 1.0)   # tanh(z) == +-1 in fp32 for many
    scale, bias = torch.linspace(0.5, 2.0, D), torch.linspace(-0.3, 0.4, D)
    dmu = torch.randn(B, D, generator=g) / B
    zl = z.clone().requires_grad_(True)
    ref = torch.tanh(zl) * scale + bias          # Actor.forward (td3_continuous_action.py:131-132)
    (ref * dmu).sum().backward()
    mu, y = O.head_forward(z, scale, bias)
    assert torch.equal(mu, ref.detach())
    # tanh_backward's vectorised CPU kernel may fuse (1 - y^2) * g: agreement to the last bits, not bitwise
    torch.testing.assert_close(O.head_backward(y, scale, dmu), zl.grad, rtol=1e-6, atol=1e-8)


@pytest.mark.parametrize("case", ["typical", "noise_beyond_clip", "actions_beyond_bounds", "per_dimension_box"])
def test_smoothing_matches_the_reference_expression(case):
    g = torch.Generator().manual_seed(7)
    B, D = 32, 5
    mu = torch.rand(B, D, generator=g) * 2 - 1
    eps = torch.randn(B, D, generator=g)
    scale = torch.ones(D)
    low, high = np.full(D, -1.0, np.float32), np.full(D, 1.0, np.float32)
    policy_noise, noise_clip = 0.2, 0.5
    if case == "noise_beyond_clip":
        policy_noise, noise_clip = 0.4, 0.1
    if case == "actions_beyond_bounds":
        mu = mu * 0.999 + torch.sign(mu) * 0.0005
        policy_noise, noise_clip = 1.0, 0.5
    if case == "per_dimension_box":
        low = np.array([-0.5, -2.0, -1.0, -3.0, 0.0], np.float32)
        high = np.array([0.5, 2.0, 1.0, 3.0, 4.0], np.float32)
        scale = torch.tensor((high - low) / 2.0)
        mu = mu * scale + torch.tensor((high + low) / 2.0)
        policy_noise, noise_clip = 0.5, 0.3
    # td3_continuous_action.py:232-238 verbatim on the same standard normals
    clipped_noise = (eps * policy_noise).clamp(-noise_clip, noise_clip) * scale
    want = (mu + clipped_noise).clamp(low[0], high[0])
    got = O.smooth(mu, eps, scale, policy_noise, noise_clip, float(low[0]), float(high[0]))
    assert torch.equal(got, want)
    if case == "noise_beyond_clip":
        assert bool(((eps * policy_noise).abs() > noise_clip).any())
    if case == "actions_beyond_bounds":
        assert bool(((mu + clipped_noise).abs() > 1.0).any())
    if case == "per_dimension_box":       # the scalar bounds of the first dimension, not each dimension's own
        per_dim = torch.max(torch.min(mu + clipped_noise, torch.tensor(high)), torch.tensor(low))
        assert not torch.equal(got, per_dim)


def test_critic_and_actor_losses_match_autograd():
    g = torch.Generator().manual_seed(5)
    B = 32
    q1, q2, q1t, q2t = (torch.randn(B, generator=g) for _ in range(4))
    r, d = torch.randn(B, generator=g), (torch.rand(B, generator=g) < 0.2).float()
    y, l1, l2, dq1, dq2 = O.critic_loss(q1, q2, q1t, q2t, r, d, 0.99)
    assert torch.equal(y, r + (1 - d) * 0.99 * torch.min(q1t, q2t))
    a, b = q1.clone().requires_grad_(True), q2.clone().requires_grad_(True)
    (torch.nn.functional.mse_loss(a, y) + torch.nn.functional.mse_loss(b, y)).backward()
    torch.testing.assert_close(dq1, a.grad, rtol=1e-6, atol=0)
    torch.testing.assert_close(dq2, b.grad, rtol=1e-6, atol=0)
    c = q1.clone().requires_grad_(True)
    O.actor_loss(c).backward()             # -mean(q1): -1/B to every row of qf1, nothing to qf2
    assert torch.equal(c.grad, torch.full((B,), -1.0 / B))


def test_exploration_draw_is_a_scaled_standard_normal():
    std = torch.tensor([0.1, 0.2, 0.05, 0.3, 0.1, 0.7])
    torch.manual_seed(3)
    a = torch.normal(0, std)
    torch.manual_seed(3)
    assert torch.equal(a, torch.empty(6).normal_() * std)


def _flag(argv, name, default, cast=int):
    return cast(argv[argv.index(name) + 1]) if name in argv else default


def _reference_nets(seed, num_envs):
    """The reference's networks on the CPU: torch.manual_seed(seed), then actor, qf1, qf2, qf1_target, qf2_target,
    target_actor in its construction order (td3_continuous_action.py:160,171-179)."""
    from cleanrl_b200.agents import SoftQNetworkMLP, TD3Actor
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    env = SyntheticGymnasiumVec(num_envs, kind="continuous")
    torch.manual_seed(seed)
    nets = [TD3Actor(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env),
            TD3Actor(env)]
    nets[5].load_state_dict(nets[0].state_dict())
    nets[3].load_state_dict(nets[1].state_dict())
    nets[4].load_state_dict(nets[2].state_dict())
    return nets


def _vec(*ns):
    return torch.cat([torch.nn.utils.parameters_to_vector(n.parameters()) for n in ns])


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_the_reference_first_update(name):
    z = np.load(GOLDEN / name)
    argv = z["argv"].tolist()
    nets = _reference_nets(_flag(argv, "--seed", 1), _flag(argv, "--num-envs", 1))
    assert list(nets[0].state_dict()) == z["actor_keys"].tolist() and list(nets[1].state_dict()) == z["qf_keys"].tolist()
    ref = O.EagerTD3(_vec(nets[0]), _vec(nets[1], nets[2]), _vec(nets[3], nets[4]), _vec(nets[5]), 17, 6,
                     nets[0].action_scale, nets[0].action_bias, "cpu",
                     policy_noise=_flag(argv, "--policy-noise", 0.2, float),
                     noise_clip=_flag(argv, "--noise-clip", 0.5, float),
                     policy_frequency=_flag(argv, "--policy-frequency", 2))
    step = _flag(argv, "--learning-starts", 40) + 1           # the first update runs at global_step learning_starts + 1
    ref.update(step, torch.from_numpy(z["u1_obs"]), torch.from_numpy(z["u1_actions"]), torch.from_numpy(z["u1_next_obs"]),
               torch.from_numpy(z["u1_rewards"]), torch.from_numpy(z["u1_dones"]),
               lambda shape: torch.from_numpy(z["u1_smooth_draw"]).reshape(shape))
    assert torch.equal(ref.stats["next_state_actions"], torch.from_numpy(z["u1_next_state_actions"]))
    np.testing.assert_allclose(ref.stats["y"].numpy(), z["u1_y"], rtol=1e-6, atol=1e-6)
    for k in ("qf1_loss", "qf2_loss", "qf1_values", "qf2_values"):
        assert ref.stats[k]() == pytest.approx(z[k][0], rel=1e-5, abs=1e-6), k
    sums = np.array([p.detach().double().sum().item() for q in (ref.qf1, ref.qf2) for p in q.parameters()])
    np.testing.assert_allclose(sums, z["q_sums"][0], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(ref.qf1.fc3.bias.grad.numpy(), z["u1_dq1_bias"], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(ref.qf2.fc3.bias.grad.numpy(), z["u1_dq2_bias"], rtol=1e-5, atol=1e-7)
    if np.isnan(z["actor_loss"][0]):                          # a critic-only update leaves the targets alone
        tsums = np.array([p.detach().double().sum().item()
                          for n in (ref.target_actor, ref.qf1_target, ref.qf2_target) for p in n.parameters()])
        np.testing.assert_allclose(tsums, z["target_sums"][0], rtol=1e-6, atol=1e-6)


def test_fixtures_cover_the_delayed_actor_step():
    z = np.load(GOLDEN / "td3_continuous_seed2_pf3.npz")
    ls = _flag(z["argv"].tolist(), "--learning-starts", 40)
    steps = np.arange(ls + 1, ls + 1 + len(z["actor_loss"]))
    assert np.array_equal(~np.isnan(z["actor_loss"]), steps % 3 == 0)
    # step 100 is not a policy step: the logged actor_loss is the one of step 99
    assert z["tb/losses/actor_loss"][0, 0] == 100
    assert z["tb/losses/actor_loss"][0, 1] == pytest.approx(z["actor_loss"][steps == 99][0], rel=1e-6)
    # the smoothing noise is clipped at noise_clip in the first update
    assert float(np.abs(z["u1_smooth_draw"] * 0.4).max()) > 0.1
    assert z["explore_draws"].shape == (len(z["action_stream"]) - ls, 6)


@pytest.mark.parametrize("name", FIXTURES)
def test_replay_index_stream_matches_the_reference_run(name):
    from cleanrl_b200.replay import DeviceReplayRing
    z = np.load(GOLDEN / name)
    argv = z["argv"].tolist()
    n_envs, bs = _flag(argv, "--num-envs", 1), _flag(argv, "--batch-size", 256)
    rb = DeviceReplayRing(_flag(argv, "--buffer-size", 10 ** 6), (17,), n_envs, "cpu", optimize_memory_usage=False,
                          obs_dtype=torch.float32, action_shape=(6,))
    np.random.seed(_flag(argv, "--seed", 1))
    heads = []
    for step in range(_flag(argv, "--total-timesteps", 0)):
        rb.add(np.zeros((n_envs, 17)), np.zeros((n_envs, 17)), np.zeros((n_envs, 6)), np.zeros(n_envs), np.zeros(n_envs))
        if step > _flag(argv, "--learning-starts", 0):
            bi, ei = rb.sample_indices(bs)
            heads += [bi[:8], ei[:8]]
    assert rb.full
    assert np.array_equal(np.stack(heads), z["randint_heads"])


def test_cli_fields_and_names_match_the_reference_surface():
    from cleanrl_b200 import cli, td3_continuous_action as m
    surf = json.loads((GOLDEN / "td3_continuous_surface.json").read_text())["td3_continuous_action.py"]
    fields = {f.name: f for f in dataclasses.fields(cli.td3_continuous_action_args())}
    for name, default, doc in surf["args"]:
        f = fields[name]
        if default != "<expr>":
            assert f.default == default, name
        assert f.type.__metadata__[0].help == doc, name
    assert fields["exp_name"].default == "td3_continuous_action" and fields["learning_starts"].default == 25e3
    assert set(fields) == {a[0] for a in surf["args"]} | {"synthetic_env"}
    for n in surf["names"]:
        assert hasattr(m, n), n
    assert m.Args is not None and m.QNetwork.__name__ == "SoftQNetworkMLP"


def test_networks_keep_the_reference_modules_and_init():
    from cleanrl_b200.agents import TD3Actor
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    env = SyntheticGymnasiumVec(1, kind="continuous")
    nets = _reference_nets(4, 1)
    assert list(nets[0].state_dict()) == ["action_scale", "action_bias", "fc1.weight", "fc1.bias", "fc2.weight",
                                          "fc2.bias", "fc_mu.weight", "fc_mu.bias"]
    assert list(nets[1].state_dict()) == ["fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias", "fc3.weight", "fc3.bias"]
    torch.manual_seed(4)
    a = [torch.nn.Linear(17, 256), torch.nn.Linear(256, 256), torch.nn.Linear(256, 6)]
    q = [[torch.nn.Linear(23, 256), torch.nn.Linear(256, 256), torch.nn.Linear(256, 1)] for _ in range(4)]
    t = [torch.nn.Linear(17, 256)]
    assert torch.equal(a[0].weight, nets[0].fc1.weight) and torch.equal(a[2].bias, nets[0].fc_mu.bias)
    assert torch.equal(q[1][0].weight, nets[2].fc1.weight) and torch.equal(q[1][2].bias, nets[4].fc3.bias)
    assert not torch.equal(t[0].weight, nets[5].fc1.weight)            # the target actor was loaded from the actor
    assert torch.equal(nets[5].fc1.weight, nets[0].fc1.weight)
    assert torch.equal(nets[0].action_scale, torch.ones(6)) and torch.equal(nets[0].action_bias, torch.zeros(6))
    with pytest.raises(RuntimeError, match="CUDA"):
        TD3Actor(env)(torch.zeros(2, 17))


@pytest.fixture(scope="module")
def lib():
    from cleanrl_b200 import _lib, build

    build.build()
    return _lib.load()


def test_entry_points_refuse_bad_arguments_without_gpu(lib):
    E = -1
    H = 256
    assert lib.b200rl_sacc_param_count(17, 6, 2) == H * 17 + H + H * H + H + 6 * H + 6
    assert lib.b200rl_sacc_param_count(17, 6, 3) == -1 and lib.b200rl_sacc_param_count(17, 6, -1) == -1
    assert lib.b200rl_sacc_param_count(1000, 25, 2) == -1 and lib.b200rl_sacc_param_count(4, 33, 2) == -1
    P = 1 << 12
    # td3_actor_fwd(params, obs, ld, rows, B, obs_dim, act_dim, scale, bias, mu, keep_y, x, h1, h2, eps, pn, nc, lo, hi,
    #               smoothed, stream)
    ok = [P, P, 17, None, 8, 17, 6, P, P, P, None, None, None, None, None, 0.2, 0.5, -1.0, 1.0, None, None]
    for i, bad in ((4, 0), (4, 8193), (6, 0), (6, 33), (5, 1024), (0, None), (7, None), (2, 10), (1, P + 2),
                   (14, P), (19, P), (12, P), (3, P + 4)):
        a = list(ok)
        a[i] = bad
        assert lib.b200rl_td3_actor_fwd_f32(*a) == E, (i, bad)
    a = list(ok)
    a[14], a[19], a[16] = P, P, -0.1                                   # negative noise_clip
    assert lib.b200rl_td3_actor_fwd_f32(*a) == E
    a[16], a[17], a[18] = 0.5, 1.0, -1.0                                # low > high
    assert lib.b200rl_td3_actor_fwd_f32(*a) == E
    # td3_actor_bwd(params, B, obs_dim, act_dim, y, scale, dact, q, h1, h2, dhead, dz1, dz2, stats, ws, ws_bytes, stream)
    okb = [P, 8, 17, 6, P, P, P, P, P, P, P, P, P, P, P, 64, None]
    for i, bad in ((1, 0), (3, 33), (4, None), (7, None), (13, None), (14, None), (15, 1)):
        a = list(okb)
        a[i] = bad
        assert lib.b200rl_td3_actor_bwd_f32(*a) in (E, -4), (i, bad)
    assert lib.b200rl_td3_actor_bwd_f32(*[15 == i and 1 or v for i, v in enumerate(okb)]) == -4
    # critic loss: next_logpi without alpha is refused; dq / stats still required
    assert lib.b200rl_sacc_critic_loss_f32(P, P, P, P, P, 1, None, None, 8, 0.99, None, P, P, P, 64, None) == E
    assert lib.b200rl_sacc_critic_loss_f32(P, None, P, P, P, 1, None, None, 8, 0.99, None, None, P, P, 64, None) == E
    # critic bwd(params, stride, B, obs, act, dq, q, h1, h2, dz1, dz2, dact, stream): the single-network mode needs
    # net_stride 0 and dact, and takes neither dq nor q nor dz1 / dz2
    S = lib.b200rl_sacc_param_count(17, 6, 1)
    assert lib.b200rl_sacc_critic_bwd_f32(P, S, 8, 17, 6, None, None, P, P, None, None, P, None) == E
    assert lib.b200rl_sacc_critic_bwd_f32(P, 0, 8, 17, 6, None, None, P, P, None, None, None, None) == E
    assert lib.b200rl_sacc_critic_bwd_f32(P, 0, 8, 17, 6, None, None, P, P, P, P, P, None) == E
    assert lib.b200rl_sacc_critic_bwd_f32(P, 0, 8, 17, 6, P, P, P, P, P, P, P, None) == E      # both modes at once
    # wgrad: kinds outside 0..2
    assert lib.b200rl_sacc_wgrad_f32(3, 8, 17, 6, P, P, P, P, P, P, P, 0, None) == E
    assert "kind" in lib.b200rl_last_error().decode()
    from cleanrl_b200 import ops
    assert ops.sacc_param_count(17, 6, ops.SACC_TD3_ACTOR) == H * 17 + H + H * H + H + 6 * H + 6
    assert ops.sacc_param_count(17, 6, True) == S
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.td3_actor_fwd(torch.zeros(8), torch.zeros(2, 17), 2, 17, 6, torch.ones(6), torch.zeros(6))
