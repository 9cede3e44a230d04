"""Continuous SAC (cleanrl/sac_continuous_action.py) without a GPU: the oracle's restated head gradient against autograd on
the reference's own expressions, the replay ring's index stream, the CLI / module surface, argument validation of the
C entry points and the synthetic Box's sampler."""
from __future__ import annotations

import dataclasses

import numpy as np
import pytest
import torch

from oracle import sac_continuous_oracle as O


def _autograd_head(mean, raw, eps, scale, bias, g, dpi):
    mean, raw = mean.clone().requires_grad_(True), raw.clone().requires_grad_(True)
    # Actor.forward / get_action verbatim (sac_continuous_action.py:129-151)
    log_std = torch.tanh(raw)
    log_std = O.LOG_STD_MIN + 0.5 * (O.LOG_STD_MAX - O.LOG_STD_MIN) * (log_std + 1)
    std = log_std.exp()
    normal = torch.distributions.Normal(mean, std)
    x_t = mean + eps * std                     # Normal.rsample: loc + eps * scale, with the given eps
    y_t = torch.tanh(x_t)
    action = y_t * scale + bias
    log_prob = normal.log_prob(x_t)
    log_prob = log_prob - torch.log(scale * (1 - y_t.pow(2)) + 1e-6)
    log_prob = log_prob.sum(1, keepdim=True)
    ((g * log_prob).sum() + (dpi * action).sum()).backward()
    return log_prob.detach(), action.detach(), mean.grad, raw.grad


@pytest.mark.parametrize("regime", ["typical", "saturated", "clamps"])
def test_head_restatement_matches_autograd(regime):
    g = torch.Generator().manual_seed(3)
    B, D = 64, 6
    mean = torch.randn(B, D, generator=g)
    raw = torch.randn(B, D, generator=g)
    if regime == "saturated":
        mean = mean * 12.0                        # tanh(x_t) == +-1 in fp32 for many elements
    if regime == "clamps":
        raw = torch.sign(raw) * 30.0              # log_std at LOG_STD_MIN / LOG_STD_MAX
    eps = torch.randn(B, D, generator=g)
    scale, bias = torch.full((D,), 2.0), torch.full((D,), 0.5)
    gl = torch.full((B, 1), 0.2 / B)
    dpi = torch.randn(B, D, generator=g) / B
    lp, act, dm_ref, dr_ref = _autograd_head(mean, raw, eps, scale, bias, gl, dpi)
    a, lp_o, _, _ = O.head_forward(mean, raw, eps, scale, bias)
    assert torch.equal(a, act)
    torch.testing.assert_close(lp_o, lp, rtol=1e-6, atol=1e-5)
    dm, dr = O.head_backward(mean, raw, eps, scale, gl, dpi)
    tol = 1e-5 * max(1.0, float(dm_ref.abs().max()))
    assert float((dm - dm_ref).abs().max()) <= tol
    tol = 1e-5 * max(1.0, float(dr_ref.abs().max()))
    assert float((dr - dr_ref).abs().max()) <= tol


def test_min_splits_the_gradient_at_ties():
    q1 = torch.tensor([1.0, 2.0, 3.0], requires_grad=True)
    q2 = torch.tensor([1.0, 1.0, 4.0], requires_grad=True)
    torch.min(q1, q2).sum().backward()
    # what sacc_critic_bwd_kernel gives each critic: all of it to the smaller, half to each at a tie
    assert q1.grad.tolist() == [0.5, 0.0, 1.0] and q2.grad.tolist() == [0.5, 1.0, 0.0]


def test_critic_and_actor_losses_match_autograd():
    g = torch.Generator().manual_seed(5)
    B = 32
    q1, q2, q1t, q2t, lp = (torch.randn(B, generator=g) for _ in range(5))
    r, d = torch.randn(B, generator=g), (torch.rand(B, generator=g) < 0.2).float()
    y, l1, l2, dq1, dq2 = O.critic_loss(q1, q2, q1t, q2t, lp, r, d, 0.2, 0.99)
    a, b = q1.clone().requires_grad_(True), q2.clone().requires_grad_(True)
    (torch.nn.functional.mse_loss(a, y) + torch.nn.functional.mse_loss(b, y)).backward()
    torch.testing.assert_close(dq1, a.grad, rtol=1e-6, atol=0)
    torch.testing.assert_close(dq2, b.grad, rtol=1e-6, atol=0)
    assert float(O.actor_loss(lp, q1, q2, 0.2)) == pytest.approx(float((0.2 * lp - torch.min(q1, q2)).mean()))


def test_temperature_step_is_torch_adam():
    la, m, v = torch.zeros(1), torch.zeros(1), torch.zeros(1)
    lp = torch.randn(16, 1, generator=torch.Generator().manual_seed(1))
    ref = torch.zeros(1, requires_grad=True)
    opt = torch.optim.Adam([ref], lr=1e-3)
    for step in (1, 2, 3):
        loss, la, m, v = O.temperature_step(la, m, v, step, lp, -6.0, 1e-3)
        opt.zero_grad()
        (-ref.exp() * (lp + -6.0)).mean().backward()
        opt.step()
        assert torch.equal(la, ref.detach())


def test_replay_index_stream_is_the_reference_buffers():
    from cleanrl_b200.replay import DeviceReplayRing

    rb = DeviceReplayRing(12, (3,), 2, "cpu", optimize_memory_usage=False, obs_dtype=torch.float32, action_shape=(2,))
    for t in range(9):
        rb.add(np.full((2, 3), t), np.full((2, 3), t + 0.5), np.full((2, 2), -t), np.full(2, t), np.zeros(2))
    np.random.seed(7)
    got = rb.sample(5)
    np.random.seed(7)
    # buffers.py BaseBuffer.sample / ReplayBuffer._get_samples: randint(0, size if full else pos), then the env index
    bi = np.random.randint(0, rb.buffer_size, size=5)
    ei = np.random.randint(0, high=2, size=(5,))
    assert rb.full and np.array_equal(got["batch_inds"], bi) and np.array_equal(got["env_indices"], ei)
    assert torch.equal(got["rows"], torch.from_numpy(bi * 2 + ei))
    slot = rb.observations[bi, ei]
    assert torch.equal(rb.frames[got["rows"]], slot.reshape(5, 3))
    assert torch.equal(rb.action_rows[got["rows"]], rb.actions[bi, ei].reshape(5, 2))
    assert torch.equal(rb.next_frames[got["rows"]], rb.next_observations[bi, ei].reshape(5, 3))
    assert float(rb.rewards[0, 0]) == 6.0            # the 7th add wrapped onto slot 0 (6 slots per env)


def test_cli_and_module_surface():
    from cleanrl_b200 import cli, sac_continuous_action as m

    fields = {f.name: f.default for f in dataclasses.fields(cli.sac_continuous_action_args())}
    want = dict(seed=1, torch_deterministic=True, cuda=True, track=False, wandb_project_name="cleanRL", wandb_entity=None,
                capture_video=False, env_id="Hopper-v4", total_timesteps=1000000, num_envs=1, buffer_size=int(1e6),
                gamma=0.99, tau=0.005, batch_size=256, learning_starts=5e3, policy_lr=3e-4, q_lr=1e-3,
                policy_frequency=2, target_network_frequency=1, alpha=0.2, autotune=True)
    for k, v in want.items():
        assert fields[k] == v, k
    assert fields["exp_name"] == "sac_continuous_action"
    assert (m.LOG_STD_MAX, m.LOG_STD_MIN) == (2, -5)
    for n in ("Args", "make_env", "SoftQNetwork", "Actor"):
        assert hasattr(m, n), n


def test_networks_keep_the_reference_modules_and_init():
    from cleanrl_b200.agents import SACContinuousActor, SoftQNetworkMLP
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec

    env = SyntheticGymnasiumVec(1, kind="continuous")
    torch.manual_seed(4)
    a, q = SACContinuousActor(env), SoftQNetworkMLP(env)
    # the module's own buffers come before its children's parameters, as in the reference's Actor
    assert list(a.state_dict()) == ["action_scale", "action_bias", "fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias",
                                    "fc_mean.weight", "fc_mean.bias", "fc_logstd.weight", "fc_logstd.bias"]
    assert list(q.state_dict()) == ["fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias", "fc3.weight", "fc3.bias"]
    torch.manual_seed(4)
    ref = [torch.nn.Linear(17, 256), torch.nn.Linear(256, 256), torch.nn.Linear(256, 6), torch.nn.Linear(256, 6),
           torch.nn.Linear(23, 256)]
    assert torch.equal(ref[0].weight, a.fc1.weight) and torch.equal(ref[3].bias, a.fc_logstd.bias)
    assert torch.equal(ref[4].weight, q.fc1.weight)
    assert torch.equal(a.action_scale, torch.ones(6)) and torch.equal(a.action_bias, torch.zeros(6))


@pytest.fixture(scope="module")
def lib():
    from cleanrl_b200 import _lib, build

    build.build()
    return _lib.load()


def test_entry_points_refuse_out_of_range_shapes_without_gpu(lib):
    E = -1
    assert lib.b200rl_sacc_param_count(17, 6, 1) == 256 * 23 + 256 + 256 * 256 + 256 + 257
    assert lib.b200rl_sacc_param_count(17, 6, 0) == 256 * 17 + 256 + 256 * 256 + 256 + 2 * (6 * 256 + 6)
    assert lib.b200rl_sacc_param_count(1000, 25, 1) == -1 and lib.b200rl_sacc_param_count(4, 33, 0) == -1
    assert lib.b200rl_sacc_workspace_bytes(0) == 0
    P = 1 << 12
    # critic_fwd(params, stride, obs, ld, rows, act, ld, rows, B, obs_dim, act_dim, q, x, h1, h2, stream)
    ok = [P, 0, P, 17, None, P, 6, None, 8, 17, 6, P, None, None, None, None]
    for i, bad in ((8, 0), (8, 8193), (10, 0), (10, 33), (9, 1000), (11, None), (2, P + 2), (3, 10)):
        a = list(ok)
        a[i] = bad
        assert lib.b200rl_sacc_critic_fwd_f32(*a) == E, (i, bad)
    msg = lib.b200rl_last_error().decode()
    assert "strides" in msg
    a = list(ok)
    a[10] = 33
    assert lib.b200rl_sacc_critic_fwd_f32(*a) == E and "act_dim=33 outside [1, 32]" in lib.b200rl_last_error().decode()
    a = list(ok)
    a[9] = 1019
    assert lib.b200rl_sacc_critic_fwd_f32(*a) == E and "1024" in lib.b200rl_last_error().decode()
    assert lib.b200rl_sacc_critic_loss_f32(P, P, P, P, P, 1, None, P, 9000, 0.99, None, P, P, P, 64, None) == E
    assert lib.b200rl_sacc_critic_loss_f32(P, P, P, P, P, 1, None, P, 8, 0.99, None, P, P, P, 1, None) == -4
    assert lib.b200rl_sacc_critic_bwd_f32(P, 0, 8, 17, 6, P, P, P, P, P, P, P, None) == E    # both modes at once
    assert lib.b200rl_sacc_soft_update_f32(P, P, 0, 0.005, None) == E
    assert lib.b200rl_sacc_wgrad_f32(1, 0, 17, 6, P, P, P, P, P, P, P, 0, None) == E
    from cleanrl_b200 import ops
    with pytest.raises(ValueError, match="act_dim"):
        ops.sacc_param_count(17, 40, True)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.sacc_soft_update(torch.zeros(4), torch.zeros(4), 4, 0.005)


def test_box_sample_is_uniform_in_bounds_and_seeded():
    from cleanrl_b200.synthetic_envs import Box

    b = Box(-2.0, 3.0, (6,), np.float32)
    b.seed(11)
    s = np.stack([b.sample() for _ in range(2000)])
    assert s.dtype == np.float32 and s.shape == (2000, 6)
    assert s.min() >= -2.0 and s.max() <= 3.0 and abs(float(s.mean()) - 0.5) < 0.1
    b.seed(11)
    assert np.array_equal(b.sample(), s[0])
    with pytest.raises(ValueError):
        Box(-np.inf, np.inf, (2,), np.float32).sample()


# ------------------------------------------------------------ against runs of the unmodified reference script
from pathlib import Path  # noqa: E402
import json  # noqa: E402

GOLDEN = Path(__file__).resolve().parent / "golden"
FIXTURES = ["sac_continuous_n2_seed1.npz", "sac_continuous_seed2_alpha01.npz"]


def _flag(argv, name, default, cast=int):
    return cast(argv[argv.index(name) + 1]) if name in argv else default


def _reference_nets(seed, num_envs):
    """The reference's networks on the CPU: torch.manual_seed(seed), then Actor, qf1, qf2, qf1_target, qf2_target in its
    construction order (sac_continuous_action.py:179,192-197), each from the reference's default nn.Linear init."""
    from cleanrl_b200.agents import SACContinuousActor, SoftQNetworkMLP
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    env = SyntheticGymnasiumVec(num_envs, kind="continuous")
    torch.manual_seed(seed)
    nets = [SACContinuousActor(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env)]
    nets[3].load_state_dict(nets[1].state_dict())
    nets[4].load_state_dict(nets[2].state_dict())
    vec = lambda *ns: torch.cat([torch.nn.utils.parameters_to_vector(n.parameters()) for n in ns])   # noqa: E731
    return nets, vec(nets[0]), vec(nets[1], nets[2]), vec(nets[3], nets[4])


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_the_reference_first_update(name):
    z = np.load(GOLDEN / name)
    argv = z["argv"].tolist()
    autotune = "--no-autotune" not in argv
    nets, af, qf, qtf = _reference_nets(_flag(argv, "--seed", 1), _flag(argv, "--num-envs", 1))
    assert list(nets[0].state_dict()) == z["actor_keys"].tolist() and list(nets[1].state_dict()) == z["qf_keys"].tolist()
    ref = O.EagerSAC(af, qf, qtf, 17, 6, nets[0].action_scale, nets[0].action_bias, "cpu", autotune=autotune,
                     alpha=_flag(argv, "--alpha", 0.2, float), policy_frequency=_flag(argv, "--policy-frequency", 2),
                     target_network_frequency=_flag(argv, "--target-network-frequency", 1))
    draws = iter(torch.from_numpy(d) for d in z["u1_draws"])
    step = _flag(argv, "--learning-starts", 40) + 1           # the first update runs at global_step learning_starts + 1
    ref.update(step, torch.from_numpy(z["u1_obs"]), torch.from_numpy(z["u1_actions"]), torch.from_numpy(z["u1_next_obs"]),
               torch.from_numpy(z["u1_rewards"]), torch.from_numpy(z["u1_dones"]), lambda shape: next(draws))
    assert next(draws, None) is None                          # every draw of the update was consumed, in order
    for k in ("qf1_loss", "qf2_loss", "qf1_values", "qf2_values"):
        assert ref.stats[k]() == pytest.approx(z[k][0], rel=1e-5, abs=1e-6), k
    sums = np.array([p.detach().double().sum().item() for q in (ref.qf1, ref.qf2) for p in q.parameters()])
    np.testing.assert_allclose(sums, z["q_sums"][0], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(ref.qf1.fc3.bias.grad.numpy(), z["u1_dq1_bias"], rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("name", FIXTURES)
def test_replay_index_stream_matches_the_reference_run(name):
    """The ring's index draws reproduce the randint calls the reference's ReplayBuffer made in the recorded run."""
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
    assert rb.full                                            # the fixture's ring wrapped
    assert np.array_equal(np.stack(heads), z["randint_heads"])


def test_cli_fields_and_names_match_the_reference_surface():
    from cleanrl_b200 import cli, sac_continuous_action as m
    surf = json.loads((GOLDEN / "sac_continuous_surface.json").read_text())["sac_continuous_action.py"]
    fields = {f.name: f for f in dataclasses.fields(cli.sac_continuous_action_args())}
    for name, default, doc in surf["args"]:
        f = fields[name]
        if default != "<expr>":
            assert f.default == default, name
        assert f.type.__metadata__[0].help == doc, name
    for n in surf["names"]:
        assert hasattr(m, n), n
