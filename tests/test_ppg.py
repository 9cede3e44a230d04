"""CPU tests of phasic policy gradient: the numpy oracle (auxiliary loss, per-tensor Adam) against the fixtures recorded
from the unmodified cleanrl/ppg_procgen.py and against torch autograd; the drop-in's CLI / module surface and its agent's
initialisation against the reference; the new C-ABI entry points' argument validation."""
import ctypes
import dataclasses
import hashlib
import json
import re

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle import ppg_oracle

FIXTURES = ["ppg_procgen_n4_t8_seed3.npz", "ppg_procgen_n4_t8_seed3_accum2.npz"]


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_aux_loss_reproduces_reference_minibatches(name):
    """The first auxiliary minibatch of each phase, from its recorded head outputs, old logits and returns."""
    z = np.load(GOLDEN / name)
    firsts = [i for i in range(len(z["aux_phase"])) if i == 0 or z["aux_phase"][i] != z["aux_phase"][i - 1]]
    for f, i in enumerate(firsts):
        head = np.concatenate([z["first_new_logits"][f], z["first_new_values"][f][:, None], z["first_new_aux_values"][f][:, None]], 1)
        st, dhead = ppg_oracle.aux_loss(head, z["first_old_logits"][f], z["first_returns"][f], 1.0, 1)
        for k in ("kl_loss", "aux_value_loss", "real_value_loss"):
            ref = float(z["aux_" + k][i])
            assert abs(st[k] - ref) <= 1e-6 * max(1.0, abs(ref)) + 2e-7, (k, st[k], ref)
        # the recorded old logits are the buffer's rows of those rollouts, step-major (normalised once more by Categorical)
        cols = z["aux_cols"][i]
        assert np.allclose(z["first_old_logits"][f], z["aux_pi"][f][:, cols].reshape(-1, z["aux_pi"].shape[-1]), rtol=0, atol=1e-6)
        assert np.array_equal(z["first_returns"][f], z["aux_returns"][f][:, cols].reshape(-1))
        # d loss / d value summed over rows is what this backward adds to the critic bias's gradient.  The reference zeroes
        # gradients before a policy backward and after an auxiliary step only, so the first auxiliary backward of a phase
        # accumulates onto the (clipped) gradient the last policy update left behind.
        accum = 2 if "accum2" in name else 1
        _, dh = ppg_oracle.aux_loss(head, z["first_old_logits"][f], z["first_returns"][f], 1.0, accum)
        A = z["aux_pi"].shape[-1]
        aux_steps = z["step_aux"]
        last_policy = [s - 1 for s in range(1, len(aux_steps)) if aux_steps[s] and not aux_steps[s - 1]][f]
        cb = list(z["head_names"]).index("critic.bias")
        left = z["step_grad"][last_policy][int(z["head_sizes"][:cb].sum())]
        assert abs(left + dh[:, A].sum() - float(z["first_critic_bias_grad"][f][0])) <= 1e-6


def test_oracle_aux_gradient_matches_autograd_fp64():
    from torch import distributions as td
    g = torch.Generator().manual_seed(0)
    for n, A, beta, accum in ((7, 15, 1.0, 1), (33, 4, 0.5, 2), (5, 22, 2.0, 3)):
        head = torch.randn(n, A + 2, generator=g, dtype=torch.float64).requires_grad_(True)
        old = torch.randn(n, A, generator=g, dtype=torch.float64) * 3
        old[0, 1] = -float("inf")                      # an old action of probability zero
        old[2, 0] = -800.0                             # ... and one that underflows to zero
        R = torch.randn(n, generator=g, dtype=torch.float64)
        kl = td.kl_divergence(td.Categorical(logits=old), td.Categorical(logits=head[:, :A])).mean()
        real = 0.5 * ((head[:, A] - R) ** 2).mean()
        aux = 0.5 * ((head[:, A + 1] - R) ** 2).mean()
        ((aux + beta * kl + real) / accum).backward()
        st, dhead = ppg_oracle.aux_loss(head.detach().numpy(), old.numpy(), R.numpy(), beta, accum)
        assert np.isfinite(dhead).all()
        assert np.abs(dhead - head.grad.numpy()).max() <= 1e-12
        for k, v in (("kl_loss", kl), ("aux_value_loss", aux), ("real_value_loss", real)):
            assert abs(st[k] - float(v.detach())) <= 1e-12
    # a new action of probability zero under a positive old probability: +inf, as torch
    head = np.zeros((1, 5)); head[0, 0] = -np.inf
    st, _ = ppg_oracle.aux_loss(head, np.zeros((1, 3)), np.zeros(1))
    assert st["kl_loss"] == np.inf


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_adam_reproduces_policy_aux_policy_trajectory(name):
    """Adam with a ``step`` per tensor and tensors without a gradient skipped, replayed over every recorded Adam step
    (policy -> auxiliary -> policy -> auxiliary) from the recorded post-clip gradients."""
    z = np.load(GOLDEN / name)
    names, sizes = list(z["head_names"]), z["head_sizes"]
    offs = np.concatenate([[0], np.cumsum(sizes)])
    split = lambda v: [v[offs[i]:offs[i + 1]] for i in range(len(names))]
    opt = ppg_oracle.Adam(split(z["step_before"][0]), lr=5e-4)
    flat = ppg_oracle.Adam([z["step_before"][0]], lr=5e-4)          # one step count for every element, nothing skipped
    aux_i = [names.index("aux_critic.weight"), names.index("aux_critic.bias")]
    flat_err = 0.0
    for s in range(z["step_before"].shape[0]):
        grads = split(z["step_grad"][s])
        has = [not np.isnan(g).any() for g in grads]
        assert all(has[i] == bool(z["step_aux"][s]) for i in aux_i) and all(h for i, h in enumerate(has) if i not in aux_i)
        for i, p in enumerate(opt.params):
            assert np.array_equal(p, split(z["step_before"][s])[i]) or np.abs(p - split(z["step_before"][s])[i]).max() <= 2e-7
        opt.params = [np.array(p) for p in split(z["step_before"][s])]
        after = opt.step([g if h else None for g, h in zip(grads, has)], lr=float(z["step_lr"][s]))
        for i, p in enumerate(after):
            assert np.abs(p - split(z["step_after"][s])[i]).max() <= 2e-7, (s, names[i])
        if not z["step_aux"][s]:
            for i in aux_i:                                           # bit-untouched across a policy step
                assert np.array_equal(after[i], split(z["step_before"][s])[i])
        flat.params = [z["step_before"][s].copy()]
        fa = flat.step([np.nan_to_num(z["step_grad"][s], nan=0.0)], lr=float(z["step_lr"][s]))[0]
        flat_err = max(flat_err, np.abs(split(fa)[aux_i[0]] - split(z["step_after"][s])[aux_i[0]]).max())
    # the recorded per-tensor step counts: aux_critic counts auxiliary updates only
    pn = list(z["param_names"])
    n_aux = np.cumsum(z["step_aux"])
    assert np.array_equal(z["step_adam_step"][:, pn.index("aux_critic.weight")], n_aux)
    assert np.array_equal(z["step_adam_step"][:, pn.index("critic.weight")], np.arange(1, len(n_aux) + 1))
    # the check a flat single-step Adam fails: zero gradients still move aux_critic through its decaying moments in
    # the second policy phase, and its bias corrections use the wrong count in the auxiliary phases
    assert flat_err > 1e-5, flat_err


def test_cli_and_module_surface_match_reference():
    from cleanrl_b200 import cli, ppg_procgen as S
    ref = json.loads((GOLDEN / "ppg_procgen_surface.json").read_text())["ppg_procgen.py"]
    fields = {f.name: f for f in dataclasses.fields(cli.ppg_procgen_args())}
    assert [n for n, _, _ in ref["args"]] == [n for n in fields if n not in ("precision", "gae_kernel", "synthetic_env")]
    for name, default, doc in ref["args"]:
        f = fields[name]
        if default != "<expr>":
            assert f.default == default, (name, f.default, default)
        helps = [m.help for m in getattr(f.type, "__metadata__", ()) if hasattr(m, "help")]
        assert helps and helps[0] == doc, (name, helps, doc)
    assert dataclasses.fields(S.Args)[0].default == "ppg_procgen"
    missing = [n for n in ref["names"] if not hasattr(S, n)]
    assert ref["names"] and not missing, missing
    S.flatten_unflatten_test()


def test_script_asserts_v_value_and_refuses_to_run_without_cuda():
    from cleanrl_b200 import ppg_procgen as S
    with pytest.raises(AssertionError, match="v_value"):
        S.main(["--v-value", "2"])
    if torch.cuda.is_available():
        pytest.skip("CUDA present")

    class W:
        def __init__(self, *a): pass
        def add_text(self, *a): pass
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        S.main(["--num-envs", "2", "--num-steps", "4", "--total-timesteps", "16", "--n-iteration", "2"], writer_factory=W)


class _Envs:
    def __init__(self, A):
        from cleanrl_b200.synthetic_envs import Box, Discrete
        self.single_observation_space = Box(0, 255, (64, 64, 3), np.uint8)
        self.single_action_space = Discrete(A)


def test_agent_initialisation_is_the_references_bit_for_bit():
    from cleanrl_b200.agents import PPGAgent
    z = np.load(GOLDEN / FIXTURES[0])
    torch.manual_seed(int(z["init_seed"]))
    sd = PPGAgent(_Envs(15)).state_dict()
    assert list(sd.keys()) == list(z["init_keys"])
    for k, h in zip(z["init_keys"], z["init_sha256"]):
        assert hashlib.sha256(sd[k].numpy().tobytes()).hexdigest() == h, k
    with pytest.raises(ValueError, match="22 actions"):
        PPGAgent(_Envs(23))


def test_param_order_puts_the_three_heads_last():
    from cleanrl_b200.agents import PPGAgent
    a = PPGAgent(_Envs(15))
    order = a._param_order()
    tail = [a.actor.weight, a.critic.weight, a.aux_critic.weight, a.actor.bias, a.critic.bias, a.aux_critic.bias]
    assert all(x is y for x, y in zip(order[-6:], tail)) and len(order) == 38


def test_new_entry_points_are_declared_and_validate_before_launch(lib):
    txt = (ROOT / "include" / "b200rl.h").read_text()
    names = ["b200rl_ppg_aux_loss_workspace_bytes", "b200rl_ppg_aux_loss_f32", "b200rl_clip_adam_ranges_f32",
             "b200rl_impala_ppg_param_count", "b200rl_impala_ppg_bf16_packed_bytes", "b200rl_impala_ppg_bf16_workspace_bytes",
             "b200rl_impala_ppg_bf16_pack", "b200rl_impala_ppg_bf16_forward", "b200rl_impala_ppg_bf16_backward"]
    for n in names:
        assert re.search(r"\b%s\s*\(" % n, txt), n
        assert hasattr(lib, n)
    bad = -1                                                   # B200RL_ERR_INVALID_ARGUMENT
    aux = lambda *a: lib.b200rl_ppg_aux_loss_f32(*a)
    ok = dict(head=64, ld=17, rows=64, old=64, ret=64, n=8, A=15, dhead=64, ldd=17, stats=64, ws=64, wsb=1 << 16)

    def call(**kw):
        q = dict(ok, **kw)
        return aux(q["head"], q["ld"], q["rows"], q["old"], q["ret"], q["n"], q["A"], 1.0, 1.0, q["dhead"], q["ldd"],
                   q["stats"], q["ws"], q["wsb"], None)
    assert call(head=None) == bad and b"null" in lib.b200rl_last_error()
    assert call(dhead=None) == bad and call(stats=None) == bad and call(old=None) == bad
    assert call(head=66) == bad and b"misaligned" in lib.b200rl_last_error()
    assert call(rows=68) == bad and call(ws=72) == bad
    assert call(A=23, ld=25, ldd=25) == bad and b"outside" in lib.b200rl_last_error()
    assert call(A=0) == bad and call(n=0) == bad and call(n=(1 << 22) + 1) == bad
    assert call(ld=16) == bad and b"strides" in lib.b200rl_last_error()
    assert call(wsb=8) == -4                                   # workspace too small
    assert lib.b200rl_ppg_aux_loss_workspace_bytes(0) == 0 and lib.b200rl_ppg_aux_loss_workspace_bytes(1024) == 8 * 12

    rng = (ctypes.c_int64 * 4)(0, 4, 6, 8)
    adam = lambda p=64, step=1, nr=2, rs=0, r=rng, ws=64, P=8: lib.b200rl_clip_adam_ranges_f32(
        p, 64, 64, 64, P, step, 1e-3, r, nr, rs, 1e-3, 0.9, 0.999, 1e-8, 0.5, None, ws, 1 << 20, None)
    assert adam(p=None) == bad and adam(p=66) == bad and adam(step=0) == bad and adam(rs=-1) == bad
    assert adam(nr=5) == bad and adam(nr=2, r=None) == bad and adam(ws=None) == bad
    assert adam(P=7) == bad and b"range" in lib.b200rl_last_error()     # a range past the end of the vector

    assert lib.b200rl_impala_ppg_param_count(15) == lib.b200rl_impala_param_count(15) + 257
    assert lib.b200rl_impala_ppg_bf16_packed_bytes(22) == lib.b200rl_impala_bf16_packed_bytes(15) > 0
    assert lib.b200rl_impala_ppg_bf16_packed_bytes(23) == 0 and lib.b200rl_impala_ppg_bf16_workspace_bytes(64, 23) == 0
    assert lib.b200rl_impala_ppg_bf16_workspace_bytes(0, 15) == 0
    assert lib.b200rl_impala_ppg_bf16_workspace_bytes(1024, 15) >= lib.b200rl_impala_bf16_workspace_bytes(1024, 15)
    assert lib.b200rl_impala_ppg_bf16_forward(256, None, 8, 23, 256, 256, 256, 256, None) == bad
    assert lib.b200rl_impala_ppg_bf16_forward(None, None, 8, 15, 256, 256, 256, 256, None) == bad
    assert lib.b200rl_impala_ppg_bf16_forward(256, None, (1 << 17) + 1, 15, 256, 256, 256, 256, None) == bad
    assert lib.b200rl_impala_ppg_bf16_forward(256, None, 8, 15, 260, 256, 256, 256, None) == bad
    assert lib.b200rl_impala_ppg_bf16_backward(256, None, 8, 23, 256, 256, 256, 256, 256, 256, 1 << 30, None) == bad
    assert lib.b200rl_impala_ppg_bf16_backward(256, None, 0, 15, 256, 256, 256, 256, 256, 256, 1 << 30, None) == bad
    assert lib.b200rl_impala_ppg_bf16_backward(256, None, 8, 15, 256, 256, 256, 256, 256, 256, 16, None) == -4
    assert lib.b200rl_impala_ppg_bf16_pack(None, 15, 256, None) == bad and lib.b200rl_impala_ppg_bf16_pack(256, 23, 256, None) == bad


def test_plan_class_shares_the_workspace_rules(lib):
    from cleanrl_b200 import ops
    cpu = torch.device("cpu")
    with pytest.raises(ValueError, match="22 actions"):
        ops.ImpalaPPGBf16(23, cpu)
    plan = ops.ImpalaPPGBf16(15, cpu)
    assert plan.param_count == ops.ImpalaCNNBf16(15, cpu).param_count + 257
    first = plan.acts(4)
    assert first.numel() == ops.ImpalaCNNBf16(15, cpu).acts(4).numel() and not first.any()
    ws = plan.workspace(4)
    plan.pin()
    assert plan.workspace(2048).numel() >= ws.numel() and plan._pinned_ws[0] is ws


def test_bench_ppg_needs_a_cuda_device():
    import subprocess
    import sys
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    r = subprocess.run([sys.executable, str(ROOT / "bench_ppg.py")], capture_output=True, text=True)
    assert r.returncode != 0 and "needs a CUDA device" in (r.stderr + r.stdout)
