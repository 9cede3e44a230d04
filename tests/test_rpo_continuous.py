"""CPU tests of the rpo_continuous_action.py drop-in: the oracle's shifted Gaussian loss against autograd and against
the reference's first update, the per-epoch draw of the mean shifts against the reference's per-minibatch draws, the
agent's construction, the CLI / module surface, and argument validation of the shift entry point."""
from __future__ import annotations

import dataclasses
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from oracle import rpo_continuous_oracle as R

GOLDEN = Path(__file__).resolve().parent / "golden"
FIXTURES = ["rpo_continuous_n4_t64_seed2.npz", "rpo_continuous_n4_t64_seed5_kl.npz"]


def _flag(argv, name, default):
    return type(default)(argv[argv.index(name) + 1]) if name in argv else default


def _reference_loss(mean, z, logstd, nv, mb_inds, b_act, b_lp, b_adv, b_ret, b_val, clip, ent_coef, vf_coef,
                    norm_adv, clip_vloss):
    """rpo_continuous_action.py:131-144,270-304 in torch (autograd)."""
    from torch.distributions.normal import Normal
    action_mean = mean + z
    action_std = torch.exp(logstd.expand_as(action_mean))
    probs = Normal(action_mean, action_std)
    newlogprob = probs.log_prob(b_act[mb_inds]).sum(1)
    entropy = probs.entropy().sum(1)
    logratio = newlogprob - b_lp[mb_inds]
    ratio = logratio.exp()
    mb_adv = b_adv[mb_inds]
    if norm_adv:
        mb_adv = (mb_adv - mb_adv.mean()) / (mb_adv.std() + 1e-8)
    pg_loss = torch.max(-mb_adv * ratio, -mb_adv * torch.clamp(ratio, 1 - clip, 1 + clip)).mean()
    nv = nv.view(-1)
    if clip_vloss:
        vu = (nv - b_ret[mb_inds]) ** 2
        vc = (b_val[mb_inds] + torch.clamp(nv - b_val[mb_inds], -clip, clip) - b_ret[mb_inds]) ** 2
        v_loss = 0.5 * torch.max(vu, vc).mean()
    else:
        v_loss = 0.5 * ((nv - b_ret[mb_inds]) ** 2).mean()
    loss = pg_loss - ent_coef * entropy.mean() + v_loss * vf_coef
    return loss, pg_loss, v_loss, ((ratio - 1) - logratio).mean()


@pytest.mark.parametrize("norm_adv,clip_vloss", [(True, True), (False, False)])
def test_oracle_shifted_loss_matches_autograd(norm_adv, clip_vloss):
    g = torch.Generator().manual_seed(11)
    M, D, B = 48, 6, 160
    mean = torch.randn(M, D, generator=g, requires_grad=True)
    z = torch.empty(M, D).uniform_(-0.5, 0.5, generator=g)
    logstd = (torch.randn(1, D, generator=g) * 0.2).requires_grad_(True)
    nv = torch.randn(M, 1, generator=g, requires_grad=True)
    b_act = torch.randn(B, D, generator=g)
    b_lp = torch.randn(B, generator=g) * 0.2 - 1.4 * D
    b_adv, b_ret = torch.randn(B, generator=g), torch.randn(B, generator=g)
    b_val = b_ret + 0.3 * torch.randn(B, generator=g)
    inds = torch.randperm(B, generator=g)[:M]
    loss, pg, vl, kl = _reference_loss(mean, z, logstd, nv, inds, b_act, b_lp, b_adv, b_ret, b_val, 0.2, 0.01, 0.5,
                                       norm_adv, clip_vloss)
    loss.backward()
    st, dm, dls, dv = R.ppo_loss_gaussian_shift(mean.detach().numpy(), z.numpy(), logstd.detach().numpy(),
                                                nv.detach().numpy(), inds.numpy(), b_act.numpy(), b_lp.numpy(),
                                                b_adv.numpy(), b_ret.numpy(), b_val.numpy(), 0.2, 0.01, 0.5, norm_adv,
                                                clip_vloss)
    for k, ref in (("loss", loss), ("pg_loss", pg), ("v_loss", vl), ("approx_kl", kl)):
        assert abs(float(st[k]) - ref.item()) <= 1e-5 * max(1.0, abs(ref.item())), k
    assert np.allclose(dm, mean.grad.numpy(), rtol=1e-4, atol=1e-7)
    assert np.allclose(dls, logstd.grad.numpy().reshape(-1), rtol=1e-4, atol=1e-6)
    assert np.allclose(dv, nv.grad.numpy().reshape(-1), rtol=1e-5, atol=1e-8)
    # a shift moves the loss: the argument is not ignored
    st0 = O.ppo_loss_gaussian(mean.detach().numpy(), logstd.detach().numpy(), nv.detach().numpy(), inds.numpy(),
                              b_act.numpy(), b_lp.numpy(), b_adv.numpy(), b_ret.numpy(), b_val.numpy(), 0.2, 0.01, 0.5,
                              norm_adv, clip_vloss)[0]
    assert st0["approx_kl"] != st["approx_kl"]


def _env():
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    return SyntheticGymnasiumVec(4, kind="continuous")


def _unflat(flat, shapes):
    out, o = [], 0
    for s in shapes:
        shape = tuple(int(x) for x in s if x)
        n = int(np.prod(shape))
        out.append(flat[o:o + n].reshape(shape))
        o += n
    assert o == flat.size
    return out


def test_oracle_reproduces_the_reference_first_update():
    z = np.load(GOLDEN / FIXTURES[0])
    from cleanrl_b200.agents import RPOAgent
    agent = RPOAgent(_env(), 0.5)
    params = list(agent.parameters())
    for p, v in zip(params, _unflat(z["u1_params_before_flat"], z["param_shapes"])):
        p.data.copy_(torch.from_numpy(v))
    obs = torch.from_numpy(z["u1_b_obs"])
    mean, value = agent.actor_mean(obs), agent.critic(obs)
    st, dm, dls, dv = R.ppo_loss_gaussian_shift(mean.detach().numpy(), z["u1_z"], agent.actor_logstd.detach().numpy(),
                                                value.detach().numpy(), z["u1_mb_inds"], z["u1_b_actions"],
                                                z["u1_b_logprobs"], z["u1_b_advantages"], z["u1_b_returns"],
                                                z["u1_b_values"], 0.2, 0.0, 0.5, True, True)
    for k in ("pg_loss", "v_loss", "approx_kl", "loss"):
        ref = float(z["upd_" + k][0])
        assert abs(float(st[k]) - ref) <= 2e-6 * max(1.0, abs(ref)), (k, st[k], ref)
    torch.autograd.backward([mean, value], [torch.from_numpy(dm), torch.from_numpy(dv).view(-1, 1)])
    agent.actor_logstd.grad = torch.from_numpy(dls).view(1, -1)
    grads = [p.grad.double() for p in params]
    norm = torch.sqrt(sum((x ** 2).sum() for x in grads))
    coef = min(1.0, 0.5 / (norm.item() + 1e-6))                      # clip_grad_norm_(max_norm=0.5)
    got = np.concatenate([(x * coef).numpy().reshape(-1) for x in grads])
    ref = z["u1_grads_flat"]
    assert np.abs(got - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


def test_one_cpu_draw_per_epoch_equals_per_minibatch_draws():
    """CPU uniform_ fills in order: one [B, D] draw is the concatenation of the reference's [M, D] draws."""
    B, M, D = 100_000, 3125, 6
    torch.manual_seed(123)
    whole = torch.empty(B, D).uniform_(-0.5, 0.5)
    torch.manual_seed(123)
    parts = torch.cat([torch.empty(M, D).uniform_(-0.5, 0.5) for _ in range(B // M)])
    assert torch.equal(whole, parts)


@pytest.mark.parametrize("name", FIXTURES)
def test_per_epoch_draws_reproduce_the_reference_stream(name):
    """Replay the run's CPU generator: construction, one Normal draw per rollout step (the reference samples actions on
    the CPU generator), then RPOAgent's one [B, D] draw per update epoch.  Every update's z head matches, including the
    iterations after a target_kl stop."""
    from cleanrl_b200.agents import RPOAgent
    z = np.load(GOLDEN / name)
    argv = z["argv"].tolist()
    N, T = _flag(argv, "--num-envs", 1), _flag(argv, "--num-steps", 2048)
    nmb, alpha = _flag(argv, "--num-minibatches", 32), _flag(argv, "--rpo-alpha", 0.5)
    B, M = N * T, N * T // nmb
    torch.manual_seed(_flag(argv, "--seed", 1))
    env = _env()
    RPOAgent(env, alpha)
    heads, epochs = z["upd_z_head"], z["upd_epoch"]
    u = 0
    for n_upd in z["updates_per_iteration"]:
        for _ in range(T):
            torch.randn(N, env.single_action_space.shape[0])
        for _ in range(int(n_upd) // nmb):
            drawn = torch.empty(B, 6).uniform_(-alpha, alpha).numpy()
            for start in range(0, B, M):
                assert np.array_equal(drawn[start:start + heads.shape[1]], heads[u]), (u, int(epochs[u]))
                if u == 0:
                    assert np.array_equal(drawn[:M], z["u1_z"])
                u += 1
    assert u == len(heads)
    if "--target-kl" in argv:
        assert (z["updates_per_iteration"] < _flag(argv, "--update-epochs", 10) * nmb).any()


def test_agent_keeps_the_reference_modules_and_init():
    from cleanrl_b200.agents import ContinuousMLPAgent, RPOAgent
    z = np.load(GOLDEN / FIXTURES[0])
    torch.manual_seed(_flag(z["argv"].tolist(), "--seed", 1))
    agent = RPOAgent(_env(), 0.25)
    assert agent.rpo_alpha == 0.25 and isinstance(agent, ContinuousMLPAgent)
    assert list(agent.state_dict().keys()) == z["state_dict_keys"].tolist()
    init = _unflat(z["u1_params_before_flat"], z["param_shapes"])
    assert [float(np.sum(v, dtype=np.float64)) for v in init] == \
        [p.detach().double().sum().item() for p in agent.parameters()]
    for p, v in zip(agent.parameters(), init):
        assert np.array_equal(p.detach().numpy(), v)


def test_cli_fields_and_names_match_the_reference_surface():
    from cleanrl_b200 import cli, rpo_continuous_action as m
    surf = json.loads((GOLDEN / "rpo_continuous_surface.json").read_text())["rpo_continuous_action.py"]
    fields = {f.name: f for f in dataclasses.fields(cli.rpo_continuous_action_args())}
    for name, default, doc in surf["args"]:
        f = fields[name]
        if default != "<expr>":
            assert f.default == default, name
        assert f.type.__metadata__[0].help == doc, name
    assert [a[0] for a in surf["args"]] == [n for n in fields if n not in ("precision", "gae_kernel", "synthetic_env")]
    assert fields["exp_name"].default == "rpo_continuous_action" and fields["total_timesteps"].default == 8000000
    assert "save_model" not in fields and fields["rpo_alpha"].default == 0.5
    for n in surf["names"]:
        assert hasattr(m, n), n
    assert m.Agent.__name__ == "RPOAgent"
    args = cli.parse(m.Args, ["--rpo-alpha", "0.3", "--target-kl", "0.02", "--synthetic-env"])
    assert args.rpo_alpha == 0.3 and args.target_kl == 0.02 and args.synthetic_env


@pytest.fixture(scope="module")
def lib():
    from cleanrl_b200 import _lib, build

    build.build()
    return _lib.load()


def test_shift_entry_point_refuses_bad_arguments_without_gpu(lib):
    E, W = -1, -4
    P = 1 << 12
    ws = lib.b200rl_ppo_loss_gaussian_workspace_bytes(64)
    # (new_mean, ld_mean, logstd, new_value, ld_value, mb_inds, b_actions, b_logprobs, b_advantages, b_returns, b_values,
    #  mean_shift, ld_shift, M, D, clip, ent, vf, norm_adv, clip_vloss, dmean, ld_dmean, dlogstd, dvalue, ld_dvalue,
    #  stats, ws, ws_bytes, stream)
    ok = [P, 6, P, P, 1, P, P, P, P, P, P, P, 6, 64, 6, 0.2, 0.0, 0.5, 1, 1, P, 6, P, P, 1, P, P, ws, None]
    bad_args = [(11, None), (12, 5), (13, 0), (14, 0), (14, 33), (1, 5), (0, None), (20, None), (26, None), (26, P + 4)]
    for i, bad in bad_args:
        a = list(ok)
        a[i] = bad
        if i == 14 and bad == 33:
            a[12] = a[1] = a[21] = 33
        assert lib.b200rl_ppo_loss_gaussian_shift_f32(*a) == E, (i, bad)
        assert "ppo_loss_gaussian_shift" in lib.b200rl_last_error().decode()
    a = list(ok)
    a[27] = ws - 1
    assert lib.b200rl_ppo_loss_gaussian_shift_f32(*a) == W
    assert "ppo_loss_gaussian_shift" in lib.b200rl_last_error().decode()
