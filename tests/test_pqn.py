"""PQN (cleanrl/pqn.py) without a GPU: the oracle against autograd and torch.optim.RAdam, Q(lambda) against the reference
runs, the Q-network's keys and initial weights, the CLI surface, the epsilon boundary and argument validation."""
from __future__ import annotations

import dataclasses
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import pqn_oracle as O

GOLDEN = Path(__file__).resolve().parent / "golden"
FIXTURES = ["pqn_seed1.npz", "pqn_seed2_mb.npz"]


def _argv(z):
    a = list(z["argv"])
    return {k.lstrip("-").replace("-", "_"): v for k, v in zip(a[1::2], a[2::2])} | {"seed": int(a[a.index("--seed") + 1])}


def _torch_net(params, dtype):
    d, A = params[0].shape[1], params[8].shape[0]
    net = torch.nn.Sequential(torch.nn.Linear(d, 120), torch.nn.LayerNorm(120), torch.nn.ReLU(), torch.nn.Linear(120, 84),
                              torch.nn.LayerNorm(84), torch.nn.ReLU(), torch.nn.Linear(84, A)).to(dtype)
    with torch.no_grad():
        for p, v in zip(net.parameters(), params):
            p.copy_(torch.as_tensor(np.asarray(v)))
    return net


def _random_params(rng, d, A):
    ps = [rng.standard_normal(s) * (0.3 if len(s) == 2 else 0.1) for s in O.shapes(d, A)]
    ps[2] += 1.0                                        # LayerNorm gammas around 1
    ps[6] += 1.0
    return ps


@pytest.mark.parametrize("d,A,M", [(4, 2, 16), (8, 4, 7), (6, 3, 1)])
def test_oracle_loss_and_grads_match_autograd(d, A, M):
    rng = np.random.default_rng(d * 100 + M)
    ps = _random_params(rng, d, A)
    x, a, R = rng.standard_normal((M, d)), rng.integers(0, A, M), rng.standard_normal(M)
    loss, qmean, grads = O.loss_and_grads(ps, x, a, R)
    net = _torch_net(ps, torch.float64)
    q = net(torch.as_tensor(x)).gather(1, torch.as_tensor(a).unsqueeze(-1)).squeeze(-1)
    ref = torch.nn.functional.mse_loss(torch.as_tensor(R), q)
    ref.backward()
    assert abs(loss - ref.item()) < 1e-12 and abs(qmean - q.mean().item()) < 1e-12
    for g, p in zip(grads, net.parameters()):
        np.testing.assert_allclose(g, p.grad.numpy(), rtol=1e-9, atol=1e-12)


def test_oracle_radam_is_torch_radam_bit_for_bit():
    """steps 1-12 cover both sides of rho_t > 5 (rectification from step 6 at beta2 = 0.999)."""
    rng = np.random.default_rng(3)
    p0 = rng.standard_normal(11342).astype(np.float32)
    t = torch.nn.Parameter(torch.as_tensor(p0.copy()))
    opt = torch.optim.RAdam([t], lr=2.5e-4, foreach=False)
    p, m, v = p0.copy(), np.zeros_like(p0), np.zeros_like(p0)
    rect_steps = 0
    for step in range(1, 13):
        g = (rng.standard_normal(11342) * 10 ** rng.uniform(-3, 1)).astype(np.float32)
        t.grad = torch.as_tensor(g.copy())
        opt.step()
        O.radam_step(p, g, m, v, step, 2.5e-4)
        st = opt.state[t]
        assert np.array_equal(m, st["exp_avg"].numpy()) and np.array_equal(v, st["exp_avg_sq"].numpy()), step
        assert np.array_equal(p, t.detach().numpy()), step
        rect_steps += O.radam_scalars(step, 2.5e-4)[3] is not None
    assert rect_steps == 7


def test_library_radam_scalars_are_the_python_doubles_rounded(lib):
    from cleanrl_b200 import ops
    for step in (1, 2, 5, 6, 7, 12, 100, 10 ** 6):
        for lr in (2.5e-4, 1e-3, 0.123456789):
            bc1, lr_, bc2s, rect = O.radam_scalars(step, lr)
            got = ops.radam_step_scalars(step, lr)
            want = (np.float32(bc1), np.float32(lr_), np.float32(bc2s), np.float32(rect if rect is not None else 0.0))
            assert tuple(np.float32(x) for x in got) == want, (step, lr)


@pytest.mark.parametrize("name", FIXTURES)
def test_qlambda_oracle_reproduces_the_reference_returns(name):
    """Iteration 1: next_value = max Q(next_obs) under the initial parameters (CPU torch, the reference's own op),
    then the Q(lambda) loop in float32 with torch's rounding points gives the recorded returns bit for bit."""
    z = np.load(GOLDEN / name)
    a = _argv(z)
    d, A = z["it_obs"].shape[-1], 2
    net = _torch_net(O.unflatten(z["init_flat"], d, A), torch.float32)
    with torch.no_grad():
        nv, _ = torch.max(net(torch.as_tensor(z["it_next_obs"][0])), dim=-1)
    gamma, ql = float(a.get("gamma", 0.99)), float(a.get("q_lambda", 0.65))
    R = O.qlambda(z["it_rewards"][0], z["it_values"][0], z["it_dones"][0], nv.numpy(), z["it_next_done"][0], gamma, ql)
    assert np.array_equal(R, z["it_returns"][0])


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_the_first_update(name):
    """The first minibatch of iteration 1: loss, mean q and the pre-clip norm from the fp64 oracle."""
    z = np.load(GOLDEN / name)
    d, A = z["it_obs"].shape[-1], 2
    ps = O.unflatten(z["init_flat"], d, A)
    mb = z["mb_inds"][0][:z["mb_len"][0]]
    x = z["it_obs"][0].reshape(-1, d)[mb]
    loss, qmean, grads = O.loss_and_grads(ps, x, z["it_actions"][0].reshape(-1)[mb], z["it_returns"][0].reshape(-1)[mb])
    norm, _ = O.clip_coef(grads, 10.0)
    assert abs(loss - z["loss"][0]) <= 1e-5 * max(1.0, abs(z["loss"][0]))
    assert abs(qmean - z["qmean"][0]) <= 1e-5
    assert abs(norm - z["norm"][0]) <= 1e-4 * z["norm"][0]


def test_fixtures_cover_clipping_rectification_and_ragged_minibatches():
    a, b = (np.load(GOLDEN / n) for n in FIXTURES)
    assert len(a["loss"]) == 48 and (a["norm"] > 10.0).all() and set(a["mb_len"]) == {16}
    assert len(b["loss"]) == 45 and (b["norm"] < 1000.0).all() and set(b["mb_len"]) == {7, 2}
    for z in (a, b):
        assert z["min_margin"] > 1e-3
        assert z["randint"].shape == z["rand"].shape == (len(z["eps"]), z["it_obs"].shape[2])


@pytest.mark.parametrize("name", FIXTURES)
def test_qnetwork_keys_and_initial_weights_match_the_reference(name, lib):
    from cleanrl_b200.agents import PQNQNetwork
    from cleanrl_b200.synthetic_envs import CartPoleVec
    z = np.load(GOLDEN / name)
    torch.manual_seed(_argv(z)["seed"])
    net = PQNQNetwork(CartPoleVec(z["it_obs"].shape[2]))
    assert list(net.state_dict()) == list(z["keys"]) == list(O.PARAM_NAMES)
    flat = np.concatenate([p.detach().numpy().reshape(-1) for p in net.parameters()])
    assert np.array_equal(flat, z["init_flat"])
    with pytest.raises(RuntimeError, match="CUDA"):
        net(torch.zeros(2, 4))


def test_qnetwork_refuses_shapes_outside_the_kernel_limits(lib):
    from cleanrl_b200.agents import PQNQNetwork
    from cleanrl_b200.synthetic_envs import Box, Discrete, SyntheticGymnasiumVec
    env = SyntheticGymnasiumVec(1, kind="discrete")
    env.single_action_space = Discrete(65)
    with pytest.raises(ValueError, match="2 <= A <= 64"):
        PQNQNetwork(env)
    env.single_action_space = Discrete(2)
    env.single_observation_space = Box(-1, 1, (513,), np.float32)
    with pytest.raises(ValueError, match="obs_dim <= 512"):
        PQNQNetwork(env)


def test_cli_fields_and_names_match_the_reference_surface():
    from cleanrl_b200 import cli, pqn as m
    surf = json.loads((GOLDEN / "pqn_surface.json").read_text())["pqn.py"]
    fields = {f.name: f for f in dataclasses.fields(cli.pqn_args())}
    for name, default, doc in surf["args"]:
        f = fields[name]
        if default != "<expr>":
            assert f.default == default, name
        assert f.type.__metadata__[0].help == doc, name
    assert fields["exp_name"].default == "pqn"
    assert set(fields) == {a[0] for a in surf["args"]} | {"synthetic_env"}
    for n in surf["names"]:
        assert hasattr(m, n), n
    assert m.linear_schedule(1, 0.05, 100.0, 50) == 0.525 and m.linear_schedule(1, 0.05, 100.0, 500) == 0.05


@pytest.mark.parametrize("eps", [1.0, 0.05, 0.1, 1 / 3, 0.525, 0.9999999, 0.6180339887498949])
def test_epsilon_boundary_rule_is_torchs_comparison(eps):
    """torch.rand(...) < epsilon compares in float32: u == fl32(eps) is greedy, the float below explores."""
    e32 = np.float32(eps)
    for u in (e32, np.nextafter(e32, np.float32(0)), np.nextafter(e32, np.float32(2))):
        torch_explore = bool((torch.tensor([u], dtype=torch.float32) < eps)[0])
        assert torch_explore == bool(u < e32), (eps, u)
    assert not bool((torch.tensor([e32]) < eps)[0])


@pytest.fixture(scope="module")
def lib():
    from cleanrl_b200 import _lib, build

    build.build()
    return _lib.load()


def test_entry_points_refuse_bad_arguments_without_gpu(lib):
    E, W = -1, -4
    P = 1 << 12
    assert lib.b200rl_pqn_param_count(4, 2) == 120 * 4 + 120 * 3 + 84 * 120 + 84 * 3 + 2 * 84 + 2
    for d, A in ((0, 2), (513, 2), (4, 1), (4, 65)):
        assert lib.b200rl_pqn_param_count(d, A) == -1
    assert lib.b200rl_pqn_workspace_bytes(0) == 0
    ws = lib.b200rl_pqn_workspace_bytes(16)

    def refused(fn, ok, bad_args, what, code=E):
        for i, bad in bad_args:
            a = list(ok)
            a[i] = bad
            assert fn(*a) == code, (what, i, bad)
            assert what in lib.b200rl_last_error().decode(), (what, i)

    # act(params, obs, ld_obs, n, obs_dim, A, random_actions, u, eps, obs_slot, actions_slot, values_slot, copy_in,
    #     copy_out, copy_n, stream)
    ok = [P, P, 4, 4, 4, 2, P, P, 0.5, P, P, P, None, None, 0, None]
    refused(lib.b200rl_pqn_act_f32, ok, [(3, 0), (4, 0), (4, 513), (5, 1), (5, 65), (2, 3), (0, None), (1, None),
                                         (11, None), (6, None), (7, None), (10, None), (14, 4), (14, -1), (1, P + 2),
                                         (10, P + 4)], "pqn_act")
    # forward(params, obs, ld_obs, n, obs_dim, A, q, stream)
    ok = [P, P, 4, 4, 4, 2, P, None]
    refused(lib.b200rl_pqn_forward_f32, ok, [(3, 0), (4, 0), (5, 65), (2, 3), (0, None), (1, None), (6, None),
                                             (6, P + 1)], "pqn_forward")
    # loss_bwd(params, obs, ld_obs, mb_inds, b_actions, b_returns, M, obs_dim, A, stats, ws, ws_bytes, stream)
    ok = [P, P, 4, P, P, P, 16, 4, 2, P, P, ws, None]
    refused(lib.b200rl_pqn_loss_bwd_f32, ok, [(6, 0), (7, 0), (8, 1), (2, 3), (0, None), (1, None), (4, None),
                                              (5, None), (9, None), (10, None), (10, P + 8), (3, P + 4)],
            "pqn_loss_bwd")
    refused(lib.b200rl_pqn_loss_bwd_f32, ok, [(11, ws - 1)], "pqn_loss_bwd", W)
    # wgrad(obs, ld_obs, mb_inds, b_actions, M, obs_dim, A, ws, ws_bytes, grad, stream)
    ok = [P, 4, P, P, 16, 4, 2, P, ws, P, None]
    refused(lib.b200rl_pqn_wgrad_f32, ok, [(4, 0), (5, 513), (6, 65), (1, 3), (0, None), (3, None), (9, None),
                                           (7, None), (3, P + 4)], "pqn_wgrad")
    refused(lib.b200rl_pqn_wgrad_f32, ok, [(8, ws - 1)], "pqn_wgrad", W)
    # qlambda(rewards, values, dones, next_value, next_done, returns, T, N, gamma, q_lambda, stream)
    ok = [P, P, P, P, P, P, 4, 4, 0.99, 0.65, None]
    refused(lib.b200rl_qlambda_f32, ok, [(6, 0), (7, 0)] + [(i, None) for i in range(6)] + [(5, P + 2)], "qlambda")
    # clip_radam(params, grads, m, v, P, step, lr, b1, b2, eps, max_norm, norm_out, ws, ws_bytes, stream)
    aws = lib.b200rl_clip_adam_workspace_bytes(64)
    ok = [P, P, P, P, 64, 1, 1e-3, 0.9, 0.999, 1e-8, 10.0, None, P, aws, None]
    refused(lib.b200rl_clip_radam_f32, ok, [(5, 0), (0, None), (3, None), (1, P + 4), (12, None)], "clip_radam")
    refused(lib.b200rl_clip_radam_f32, ok, [(13, aws - 1)], "clip_radam", W)
    ok = [P, P, P, P, 64, P, 0.9, 0.999, 1e-8, 10.0, None, P, aws, None]
    refused(lib.b200rl_clip_radam_dyn_f32, ok, [(5, None), (5, P + 2), (0, None)], "clip_radam")
    assert lib.b200rl_radam_step_scalars(0, 1e-3, 0.9, 0.999, None) == E
    from cleanrl_b200 import ops
    assert ops.PQN_STAT_NAMES == ("td_loss", "q_values")
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.qlambda(torch.zeros(2, 2), torch.zeros(2, 2), torch.zeros(2, 2), torch.zeros(2), torch.zeros(2), 0.99, 0.65)
