"""C51 without a GPU: the numpy oracle against torch autograd on the reference's own expressions, the oracle against
the recorded reference run, the CLI / module surface, and argument validation of the new C entry points."""
import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import c51_oracle as O


def _autograd(logits, nlogits, atoms, a, r, d, gamma, v_min, v_max, Z):
    lg = logits.clone().requires_grad_(True)
    loss, old, target = O.torch_update_loss(lg, nlogits, atoms, a, r, d, gamma, v_min, v_max, Z)
    loss.backward()
    return float(loss.detach()), float((old.detach() * atoms).sum(1).mean()), lg.grad.numpy(), target.numpy()


def _check(logits, nlogits, atoms, a, r, d, gamma=0.99, v_min=-10.0, v_max=10.0):
    Z = atoms.numel()
    l_t, q_t, g_t, tgt_t = _autograd(logits, nlogits, atoms, a, r, d, gamma, v_min, v_max, Z)
    l_o, q_o, g_o, tgt_o = O.loss_and_grad(logits.numpy(), nlogits.numpy(), atoms.numpy(), a.numpy(), r.numpy(), d.numpy(),
                                           gamma, v_min, v_max)
    assert np.abs(tgt_o - tgt_t).max() <= 1e-6
    assert abs(l_o - l_t) <= 1e-6 * max(1.0, abs(l_t)) and abs(q_o - q_t) <= 1e-6 * max(1.0, abs(q_t))
    assert np.abs(g_o - g_t).max() <= 1e-6 * max(np.abs(g_t).max(), 1e-30)
    return tgt_o


@pytest.mark.parametrize("A,Z", [(4, 51), (18, 51), (6, 101)])
def test_oracle_vs_torch_autograd(A, Z):
    g = torch.Generator().manual_seed(A * Z)
    B = 64
    atoms = torch.linspace(-10, 10, Z)
    logits = torch.randn(B, A * Z, generator=g) * 3
    nlogits = torch.randn(B, A * Z, generator=g) * 3
    a = torch.randint(0, A, (B, 1), generator=g)
    r = torch.randn(B, generator=g) * 4
    d = (torch.rand(B, generator=g) < 0.3).float()
    _check(logits, nlogits, atoms, a, r, d)


def test_oracle_edge_cases():
    """b exactly an integer, clamping at both ends, done = 1 and pmfs beyond the clamp bounds."""
    A, Z, B = 4, 51, 8
    g = torch.Generator().manual_seed(7)
    atoms = torch.linspace(-10, 10, Z)
    logits = torch.randn(B, A * Z, generator=g)
    logits[:4] *= 40.0                              # near one-hot pmfs: entries below 1e-5 and above 1 - 1e-5
    nlogits = torch.randn(B, A * Z, generator=g)
    a = torch.randint(0, A, (B, 1), generator=g)
    dz = atoms[1] - atoms[0]
    r = torch.tensor([0.0, 50.0, -50.0, float(-10 + 5 * dz), 1.0, 0.0, 25.0, -25.0])
    d = torch.tensor([1.0, 0.0, 0.0, 1.0, 0.0, 1.0, 1.0, 1.0])
    tgt = _check(logits, nlogits, atoms, a, r, d, gamma=1.0)
    next_atoms = r.numpy()[:, None] + atoms.numpy()[None] * (1 - d.numpy()[:, None])
    b = (np.clip(next_atoms, -10, 10) + np.float32(10)) / dz.numpy()
    assert (b == np.floor(b)).any(), "an exactly integer b must occur"
    assert (next_atoms < -10).any() and (next_atoms > 10).any(), "clamping at both ends must occur"
    p = O.get_action(logits.numpy(), atoms.numpy(), a.numpy())[1]
    assert (p < 1e-5).any() and (p > 1 - 1e-5).any()
    assert np.allclose(tgt.sum(1), 1.0, atol=1e-5)


def test_oracle_reproduces_reference_first_update():
    z = np.load(GOLDEN / "c51_atari_b8_seed1.npz")
    gamma, v_min, v_max = 0.99, -10.0, 10.0
    loss, qv, _, tgt = O.loss_and_grad(z["u1_logits"], z["u1_next_logits"], z["atoms"], z["u1_actions"], z["u1_rewards"],
                                       z["u1_dones"], gamma, v_min, v_max)
    assert np.abs(tgt - z["u1_target_pmfs"]).max() <= 1e-6
    assert abs(loss - z["losses"][0]) <= 1e-6 * max(1.0, abs(z["losses"][0]))
    assert abs(qv - z["q_values"][0]) <= 1e-6


def test_cli_fields_and_names_match_reference():
    import dataclasses
    import json
    from cleanrl_b200 import c51_atari, cli
    surf = json.loads((GOLDEN / "c51_atari_surface.json").read_text())["c51_atari.py"]
    fields = {f.name: f for f in dataclasses.fields(cli.c51_atari_args())}
    for name, default, doc in surf["args"]:
        assert name in fields, name
        f = fields[name]
        if default != "<expr>":
            assert f.default == default, (name, f.default, default)
        helps = [m.help for m in getattr(f.type, "__metadata__", ()) if hasattr(m, "help")]
        assert helps and helps[0] == doc, (name, helps, doc)
    assert set(fields) - {n for n, _, _ in surf["args"]} == {"precision", "synthetic_env"}
    missing = [n for n in surf["names"] if not hasattr(c51_atari, n)]
    assert surf["names"] and not missing, missing


def test_qnetwork_surface_without_gpu():
    from cleanrl_b200.agents import C51QNetwork
    from cleanrl_b200.synthetic_envs import Box, Discrete

    class Envs:
        single_observation_space = Box(0, 255, (4, 84, 84), np.uint8)
        single_action_space = Discrete(6)
    torch.manual_seed(0)
    net = C51QNetwork(Envs())
    keys = list(net.state_dict().keys())
    assert keys[0] == "atoms" and keys[1:] == [f"network.{i}.{p}" for i in (0, 2, 4, 7, 9) for p in ("weight", "bias")]
    assert torch.equal(net.atoms, torch.linspace(-100, 100, steps=101))
    assert net.network[9].out_features == 6 * 101
    with pytest.raises(RuntimeError, match="CUDA"):
        net.get_action(torch.zeros(1, 4, 84, 84))


def test_c51_entry_points_validate_arguments_without_gpu(lib):
    from cleanrl_b200 import ops
    E = -1
    # c51_act(logits, ld, atoms, n, A, n_atoms, action_in, action_out, q_out, pmf_out, stream)
    assert lib.b200rl_c51_act_f32(16, 204, 16, 4, 4, 51, None, None, None, None, None) == E           # null action_out
    assert lib.b200rl_c51_act_f32(16, 4, 16, 4, 4, 1, None, 64, None, None, None) == E               # n_atoms < 2
    assert lib.b200rl_c51_act_f32(16, 257 * 4, 16, 4, 4, 257, None, 64, None, None, None) == E       # n_atoms > 256
    assert lib.b200rl_c51_act_f32(18, 204, 16, 4, 4, 51, None, 64, None, None, None) == E            # misaligned
    assert b"misaligned" in lib.b200rl_last_error()
    ws = lib.b200rl_c51_loss_workspace_bytes(8)
    args = [16, 204, 16, 204, 16, 64, 16, 16, 8, 4, 51, 0.99, -10.0, 10.0, 16, 204, 16, 256, ws, None]
    for k, bad in ((10, 1), (10, 300), (0, None), (6, 18), (17, 4)):
        a = list(args); a[k] = bad
        assert lib.b200rl_c51_loss_f32(*a) == E, (k, bad)
    # wide heads: 24..2048 outputs accepted, wider rejected before any CUDA call
    assert lib.b200rl_naturecnn_bf16_packed_bytes(2048) == 0 and lib.b200rl_naturecnn_bf16_workspace_bytes(8, 2048) == 0
    assert lib.b200rl_naturecnn_bf16_packed_bytes(203) > lib.b200rl_naturecnn_bf16_packed_bytes(23)
    assert lib.b200rl_naturecnn_bf16_packed_bytes(23) == lib.b200rl_naturecnn_bf16_packed_bytes(3)
    assert lib.b200rl_naturecnn_bf16_forward(16, 0, None, 4, 2048, 16, 16, 16, 16, None) == E
    assert b"outside" in lib.b200rl_last_error()
    assert lib.b200rl_naturecnn_bf16_pack(16, 2048, 16, None) == E
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.c51_act(torch.zeros(2, 204), torch.linspace(-10, 10, 51))
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.c51_loss(torch.zeros(2, 204), torch.zeros(2, 204), torch.linspace(-10, 10, 51), torch.zeros(2, dtype=torch.long),
                     torch.zeros(2), torch.zeros(2), 0.99, -10, 10)
