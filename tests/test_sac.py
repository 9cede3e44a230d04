"""Discrete SAC without a GPU: the numpy oracle against torch autograd on the reference's own expressions, the oracle
against the recorded reference run, the replay layout's index stream against the reference ReplayBuffer's, the CLI /
module surface, and argument validation of the new C entry points."""
import json

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import sac_oracle as O

FIXTURES = ["sac_atari_b8_seed1.npz", "sac_atari_b8_seed2_alpha01.npz"]


def _case(B, A, seed, sharp=False):
    g = torch.Generator().manual_seed(seed)
    scale = 40.0 if sharp else 2.0
    return (torch.randn(B, A, generator=g) * scale, torch.randn(B, A, generator=g), torch.randn(B, A, generator=g),
            torch.randn(B, A, generator=g), torch.randn(B, A, generator=g), torch.randint(0, A, (B,), generator=g),
            torch.randint(-1, 2, (B,), generator=g).float(), (torch.rand(B, generator=g) < 0.3).float(),
            torch.randn(B, A, generator=g) * scale)


@pytest.mark.parametrize("A", [2, 4, 18])
@pytest.mark.parametrize("sharp", [False, True])
@pytest.mark.parametrize("autotune", [True, False])
def test_oracle_vs_torch_autograd(A, sharp, autotune):
    B = 64
    nl, q1t, q2t, q1, q2, a, r, d, lo = _case(B, A, A * 7 + sharp, sharp)
    alpha, gamma = (0.83 if autotune else 0.1), 0.99
    # critic
    q1v, q2v = q1.clone().requires_grad_(True), q2.clone().requires_grad_(True)
    l1, l2, y_t, q1a, q2a = O.torch_critic(nl, q1t, q2t, q1v, q2v, a, r, d, gamma, alpha)
    (l1 + l2).backward()
    st, y, dq1, dq2 = O.critic_loss(nl.numpy(), q1t.numpy(), q2t.numpy(), q1.numpy(), q2.numpy(), a.numpy(), r.numpy(),
                                    d.numpy(), gamma, alpha)
    assert np.abs(y - y_t.numpy()).max() <= 1e-6 * max(1.0, np.abs(y).max())
    ref = [float(q1a.detach().mean()), float(q2a.detach().mean()), float(l1), float(l2)]
    assert np.allclose(st, ref, rtol=1e-6, atol=1e-6)
    assert np.abs(dq1 - q1v.grad.numpy()).max() <= 1e-6 and np.abs(dq2 - q2v.grad.numpy()).max() <= 1e-6
    assert (dq1[np.arange(B), a.numpy()] != 0).any() and (np.count_nonzero(dq1, 1) <= 1).all()
    # actor (+ temperature)
    te = O.target_entropy(A)
    lg = lo.clone().requires_grad_(True)
    la = torch.tensor([np.log(alpha)], dtype=torch.float32, requires_grad=True)
    loss, a_loss = O.torch_actor(lg, q1, q2, alpha, la if autotune else None, te)
    loss.backward()
    out = O.actor_loss(lo.numpy(), q1.numpy(), q2.numpy(), alpha, te if autotune else None,
                       la.detach().numpy()[0] if autotune else None)
    assert abs(out[0] - float(loss)) <= 1e-6 * max(1.0, abs(float(loss)))
    assert np.abs(out[1] - lg.grad.numpy()).max() <= 1e-6 * max(np.abs(lg.grad.numpy()).max(), 1e-6)
    if autotune:
        a_loss.backward()
        assert abs(out[2] - float(a_loss)) <= 1e-6 * max(1.0, abs(float(a_loss)))
        assert abs(out[3] - float(la.grad)) <= 1e-6 * max(1.0, abs(float(la.grad)))
        opt = torch.optim.Adam([la], lr=3e-4, eps=1e-4)
        opt.step()
        assert abs(out[4][0] - float(la.detach())) <= 1e-7
    else:
        assert out[2] is None


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_reference_first_update(name):
    z = np.load(GOLDEN / name)
    autotune = "--no-autotune" not in z["argv"].tolist()
    A = z["u1_q1"].shape[1]
    # the actor's next-obs logits are recovered from its log_softmax (a logit shift leaves every output unchanged)
    st, y, dq1, dq2 = O.critic_loss(z["u1_next_logp"], z["u1_q1t"], z["u1_q2t"], z["u1_q1"], z["u1_q2"], z["u1_actions"],
                                    z["u1_rewards"], z["u1_dones"], 0.99, z["alpha"][0])
    assert np.abs(y - z["u1_y"]).max() <= 1e-5 * max(1.0, np.abs(z["u1_y"]).max())
    ref = [z["qf1_values"][0], z["qf2_values"][0], z["qf1_loss"][0], z["qf2_loss"][0]]
    assert np.allclose(st, ref, rtol=1e-5, atol=1e-6), (st, ref)
    assert np.allclose(dq1.sum(0), z["u1_dq1_bias"], atol=1e-6) and np.allclose(dq2.sum(0), z["u1_dq2_bias"], atol=1e-6)
    te = O.target_entropy(A)
    assert np.float32(te) == z["target_entropy"] or not autotune
    out = O.actor_loss(z["u1_logp"], z["u1_post_q1"], z["u1_post_q2"], z["alpha"][0], te if autotune else None,
                       0.0 if autotune else None, step=1, lr=3e-4)
    assert abs(out[0] - z["actor_loss"][0]) <= 1e-5 * max(1.0, abs(z["actor_loss"][0]))
    assert np.allclose(out[1].sum(0), z["u1_dl_bias"], atol=1e-6)
    if autotune:
        assert abs(out[2] - z["alpha_loss"][0]) <= 1e-6 * max(1.0, abs(z["alpha_loss"][0]))
        assert abs(out[3] - z["log_alpha_grad"][0]) <= 1e-6 * max(1.0, abs(z["log_alpha_grad"][0]))
        assert abs(out[4][0] - z["log_alpha"][0]) <= 1e-8
        assert abs(out[5] - z["alpha"][1]) <= 1.2e-7          # exp(log_alpha): numpy and torch may differ by one ulp


def test_replay_layout_draws_the_reference_indices():
    """optimize_memory_usage=False: randint(0, size if full else pos), then the env index -- the reference ReplayBuffer's
    stream over a run that wraps (buffers.py:217-225, 397-415); the default layout is unchanged."""
    from cleanrl_b200.replay import DeviceReplayRing
    ring = DeviceReplayRing.__new__(DeviceReplayRing)
    ring.buffer_size, ring.n_envs, ring.optimize_memory_usage = 16, 1, False
    draws, ref = [], []
    np.random.seed(5)
    for step in range(60):
        ring.pos, ring.full = (step + 1) % 16, step + 1 >= 16
        draws.append(ring.sample_indices(8))
    np.random.seed(5)
    for step in range(60):
        pos, full = (step + 1) % 16, step + 1 >= 16
        bi = np.random.randint(0, 16 if full else pos, size=8)
        ref.append((bi, np.random.randint(0, high=1, size=(8,))))
    for (a, b), (c, d) in zip(draws, ref):
        assert np.array_equal(a, c) and np.array_equal(b, d)
    # the default (DQN / C51) layout keeps its own draw
    ring.optimize_memory_usage = True
    ring.pos, ring.full = 3, True
    np.random.seed(5)
    bi, _ = ring.sample_indices(8)
    np.random.seed(5)
    assert np.array_equal(bi, (np.random.randint(1, 16, size=8) + 3) % 16)


def test_reference_run_sample_heads_follow_the_layout():
    """Replays the recorded run's buffer positions: every sample's index draw equals what the ring draws from the same
    numpy state (the heads were recorded from the reference's own np.random.randint calls)."""
    z = np.load(GOLDEN / FIXTURES[0])
    heads = z["randint_heads"]
    ls = int(z["argv"].tolist()[z["argv"].tolist().index("--learning-starts") + 1])
    size = int(z["argv"].tolist()[z["argv"].tolist().index("--buffer-size") + 1])
    # updates happen at steps > learning_starts divisible by 4; the buffer holds step + 1 transitions then
    steps = [s for s in range(ls + 1, 300) if s % 4 == 0]
    for k, s in enumerate(steps[: heads.shape[0] // 2]):
        upper = size if s + 1 >= size else s + 1
        assert heads[2 * k].max() < upper and (heads[2 * k + 1] == 0).all()


def test_cli_fields_and_names_match_reference():
    import dataclasses
    from cleanrl_b200 import cli, sac_atari
    surf = json.loads((GOLDEN / "sac_atari_surface.json").read_text())["sac_atari.py"]
    fields = {f.name: f for f in dataclasses.fields(cli.sac_atari_args())}
    for name, default, doc in surf["args"]:
        assert name in fields, name
        f = fields[name]
        if default != "<expr>":
            assert f.default == default, (name, f.default, default)
        helps = [m.help for m in getattr(f.type, "__metadata__", ()) if hasattr(m, "help")]
        assert helps and helps[0] == doc, (name, helps, doc)
    assert set(fields) - {n for n, _, _ in surf["args"]} == {"precision", "synthetic_env"}
    for n in ("make_env", "layer_init", "SoftQNetwork", "Actor"):
        assert n in surf["names"] and hasattr(sac_atari, n), n


def test_networks_surface_and_init_without_gpu():
    """state_dict keys of the reference, kaiming init in its construction order (same generator consumption)."""
    import torch.nn as nn
    from cleanrl_b200.agents import SACActor, SoftQNetwork, sac_layer_init
    from cleanrl_b200.synthetic_envs import Box, Discrete

    class Envs:
        single_observation_space = Box(0, 255, (4, 84, 84), np.uint8)
        single_action_space = Discrete(6)
    z = np.load(GOLDEN / FIXTURES[0])
    torch.manual_seed(3)
    actor, qf = SACActor(Envs()), SoftQNetwork(Envs())
    assert list(actor.state_dict().keys()) == z["actor_keys"].tolist()
    assert list(qf.state_dict().keys()) == z["qf_keys"].tolist()
    torch.manual_seed(3)
    ref = []
    for _ in range(2):
        conv = [sac_layer_init(nn.Conv2d(4, 32, 8, stride=4)), sac_layer_init(nn.Conv2d(32, 64, 4, stride=2)),
                sac_layer_init(nn.Conv2d(64, 64, 3, stride=1))]
        ref.append(conv + [sac_layer_init(nn.Linear(3136, 512)), sac_layer_init(nn.Linear(512, 6))])
    for net, layers in zip((actor, qf), ref):
        got = list(net.parameters())
        want = [p for m in layers for p in m.parameters()]
        assert all(torch.equal(a, b) for a, b in zip(got, want))
    assert float(qf.conv[0].bias.abs().sum()) == 0.0
    with pytest.raises(RuntimeError, match="CUDA"):
        actor.get_action(torch.zeros(1, 4, 84, 84))


def test_sac_entry_points_validate_arguments_without_gpu(lib):
    from cleanrl_b200 import ops
    E = -1
    # sac_policy(logits, ld, n, A, logp, ld_logp, probs, ld_probs, stream)
    assert lib.b200rl_sac_policy_f32(16, 4, 4, 1, 16, 4, 16, 4, None) == E              # A < 2
    assert lib.b200rl_sac_policy_f32(16, 33, 4, 33, 16, 33, 16, 33, None) == E          # A > 32
    assert b"outside" in lib.b200rl_last_error()
    assert lib.b200rl_sac_policy_f32(16, 4, 4, 4, None, 4, None, 4, None) == E          # no output
    assert lib.b200rl_sac_policy_f32(18, 4, 4, 4, 16, 4, 16, 4, None) == E              # misaligned
    ws = lib.b200rl_sac_critic_loss_workspace_bytes(8)
    crit = [16, 4, 16, 4, 16, 4, 16, 4, 16, 4, 64, 16, 16, 16, 8, 4, 0.99, None, 16, 4, 16, 4, 16, 256, ws, None]
    W = -4      # B200RL_ERR_WORKSPACE
    for k, bad, err in ((15, 1, E), (15, 33, E), (14, 0, E), (13, None, E), (1, 3, E), (10, 68, E), (24, ws - 4, W),
                        (23, 260, E)):
        a = list(crit); a[k] = bad
        assert lib.b200rl_sac_critic_loss_f32(*a) == err, (k, bad)
    wa = lib.b200rl_sac_actor_loss_workspace_bytes(8)
    act = [16, 4, 16, 4, 16, 4, 8, 4, 16, 1, 16, 16, 16, 16, 1.23, 0.9, 0.999, 1e-4, 16, 4, 16, 256, wa, None]
    for k, bad, err in ((7, 1, E), (7, 40, E), (6, 0, E), (10, None, E), (13, None, E), (8, None, E), (19, 2, E),
                        (22, wa - 4, W)):
        a = list(act); a[k] = bad
        assert lib.b200rl_sac_actor_loss_f32(*a) == err, (k, bad)
    assert lib.b200rl_sac_critic_loss_workspace_bytes(-1) == 0 and lib.b200rl_sac_actor_loss_workspace_bytes(-1) == 0
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.sac_policy(torch.zeros(2, 4))
    z = torch.zeros(2, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.sac_critic_loss(z, z, z, z, z, torch.zeros(2, dtype=torch.long), torch.zeros(2), torch.zeros(2), 0.99,
                            torch.ones(1))
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.sac_actor_loss(z, z, z, torch.ones(1))
