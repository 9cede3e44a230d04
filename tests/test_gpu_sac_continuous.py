"""Continuous SAC kernels (csrc/sac_continuous.cu) on the GPU: each kernel against the fp32 oracle over batch sizes and
(obs, act) shapes, bitwise repeatability, graph replay against eager launches, the device noise against
``Normal.rsample``, the launch budget, refused shapes, and the drop-in end to end on the synthetic HalfCheetah env."""
from __future__ import annotations

import types

import numpy as np
import pytest
import torch

from oracle import sac_continuous_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
SHAPES = [(17, 6), (3, 1), (376, 17), (1000, 24), (1023, 1)]     # the last two at the 1024-column limit
BATCHES = [1, 7, 256, 1000, 8192]


def _close(got, want, rtol=1e-5):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    err = float((got - want).abs().max()) if got.numel() else 0.0
    assert err <= rtol * max(1.0, float(want.abs().max())), (err, float(want.abs().max()), got.shape)


def _setup(od, D, seed=0):
    """Flat actor and twin-critic parameters with the reference's default nn.Linear initialisation (the regime the
    networks train in; saturated heads are covered on the CPU against autograd)."""
    torch.manual_seed(seed)
    vec = torch.nn.utils.parameters_to_vector
    actor = vec(O._Actor(od, D, torch.ones(D), torch.zeros(D)).parameters()).detach()
    q = torch.cat([vec(O._Q(od, D).parameters()).detach() for _ in range(2)])
    return actor.to(DEV), q.to(DEV), q.numel() // 2


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("od,D", SHAPES)
def test_kernels_match_the_oracle(B, od, D):
    from cleanrl_b200 import ops
    g = torch.Generator().manual_seed(B + od)
    af, qf, S = _setup(od, D)
    N = B + 5
    obs = torch.randn(N, od, generator=g).to(DEV)
    act = torch.rand(N, D, generator=g).to(DEV) * 2 - 1
    rows = torch.randint(0, N, (B,), generator=g).to(DEV)
    eps = torch.randn(B, D, generator=g).to(DEV)
    scale, bias = torch.full((D,), 1.5, device=DEV), torch.full((D,), 0.25, device=DEV)
    x, xa = obs[rows], act[rows]
    # twin critic forward with gather
    keep = dict(keep_x=torch.empty(B, od + D, device=DEV), keep_h1=torch.empty(2, B, 256, device=DEV),
                keep_h2=torch.empty(2, B, 256, device=DEV))
    q = ops.sacc_critic_fwd(qf, S, obs, act, B, od, D, obs_rows=rows, act_rows=rows, **keep)
    for n in range(2):
        p, _ = O.mlp_params(qf[n * S:(n + 1) * S], od + D, 1)
        _close(q[n], O.critic_forward(p, x, xa).view(-1))
    assert torch.equal(keep["keep_x"], torch.cat([x, xa], 1))
    # actor forward + head
    pa, _ = O.mlp_params(af, od, D, heads=2)
    out = {k: torch.empty(B, D, device=DEV) for k in ("action", "mean_out")}
    out["log_pi"], out["mean_logstd"] = torch.empty(B, device=DEV), torch.empty(B, 2 * D, device=DEV)
    kh = dict(keep_x=torch.empty(B, od, device=DEV), keep_h1=torch.empty(B, 256, device=DEV),
              keep_h2=torch.empty(B, 256, device=DEV), keep_head=torch.empty(B, 2 * D, device=DEV))
    ops.sacc_actor_fwd(af, obs, B, od, D, eps, scale, bias, rows=rows, **out, **kh)
    m, raw = O.actor_head(pa, x)
    a_o, lp_o, sm_o, ls_o = O.head_forward(m, raw, eps, scale, bias)
    _close(out["action"], a_o)
    _close(out["log_pi"], lp_o.view(-1))
    _close(out["mean_out"], sm_o)
    _close(out["mean_logstd"], torch.cat([m, ls_o], 1))
    # critic loss
    alpha = torch.full((1,), 0.3, device=DEV)
    rew, done = torch.randn(N, generator=g).to(DEV), (torch.rand(N, generator=g) < 0.1).float().to(DEV)
    qn = torch.randn(2, B, generator=g).to(DEV)
    stats, dq = ops.sacc_critic_loss(qn, out["log_pi"], q, rew, done, alpha, 0.99, rows=rows)
    y, l1, l2, d1, d2 = O.critic_loss(q[0], q[1], qn[0], qn[1], out["log_pi"], rew[rows], done[rows], 0.3, 0.99)
    _close(dq, torch.stack([d1, d2]))
    _close(stats, torch.stack([q[0].mean(), q[1].mean(), l1, l2]))
    # critic backward + weight gradients against autograd on the oracle's networks
    dz1, dz2 = torch.empty(2, B, 256, device=DEV), torch.empty(2, B, 256, device=DEV)
    ops.sacc_critic_bwd(qf, S, B, od, D, keep["keep_h1"], keep["keep_h2"], dq=dq, dz1=dz1, dz2=dz2)
    grad = torch.full_like(qf, float("nan"))
    ops.sacc_wgrad(True, B, od, D, keep["keep_x"], keep["keep_h1"], keep["keep_h2"], dz1, dz2, dq, grad, S)
    qleaf = qf.clone().requires_grad_(True)
    loss = 0
    for n in range(2):
        p, _ = O.mlp_params(qleaf[n * S:(n + 1) * S], od + D, 1)
        loss = loss + (O.critic_forward(p, x, xa).view(-1) * dq[n]).sum()
    loss.backward()
    _close(grad, qleaf.grad)
    # actor step: critics to the action columns, head and actor backward, actor weight gradients
    qpi = ops.sacc_critic_fwd(qf, S, obs, out["action"], B, od, D, obs_rows=rows, keep_h1=keep["keep_h1"],
                              keep_h2=keep["keep_h2"])
    dact = torch.empty(2, B, D, device=DEV)
    ops.sacc_critic_bwd(qf, S, B, od, D, keep["keep_h1"], keep["keep_h2"], q=qpi, dact=dact)
    dhead, dz1a, dz2a = torch.empty(B, 2 * D, device=DEV), torch.empty(B, 256, device=DEV), torch.empty(B, 256, device=DEV)
    ast = torch.zeros(4, device=DEV)
    ops.sacc_actor_bwd(af, B, od, D, kh["keep_head"], eps, scale, dact, qpi, out["log_pi"], alpha, kh["keep_h1"],
                       kh["keep_h2"], dhead, dz1a, dz2a, ast, ops.sacc_workspace(B, DEV))
    agrad = torch.full_like(af, float("nan"))
    ops.sacc_wgrad(False, B, od, D, kh["keep_x"], kh["keep_h1"], kh["keep_h2"], dz1a, dz2a, dhead, agrad)
    aleaf = af.clone().requires_grad_(True)
    pa2, _ = O.mlp_params(aleaf, od, D, heads=2)
    m2, raw2 = O.actor_head(pa2, x)
    pi, lp, _, _ = O.head_forward(m2, raw2, eps, scale, bias)
    qs = []
    for n in range(2):
        p, _ = O.mlp_params(qf[n * S:(n + 1) * S], od + D, 1)
        qs.append(O.critic_forward(p, x, pi))
    al = O.actor_loss(lp, qs[0], qs[1], 0.3)
    al.backward()
    _close(ast[0:1], al.detach().view(1))
    _close(agrad, aleaf.grad)
    # the autotune step on a fresh sample, against the oracle's torch.optim.Adam step
    la, m1, v1 = torch.full((1,), -0.3, device=DEV), torch.full((1,), 0.01, device=DEV), torch.full((1,), 2e-4, device=DEV)
    t = dict(alpha=torch.zeros(1, device=DEV), log_alpha=la.clone(), exp_avg=m1.clone(), exp_avg_sq=v1.clone(),
             step_scalars=torch.tensor(ops.adam_step_scalars(3, 1e-3), device=DEV), target_entropy=-float(D),
             stats=torch.zeros(4, device=DEV))
    lp_t = torch.empty(B, device=DEV)
    ops.sacc_actor_fwd(af, obs, B, od, D, eps, scale, bias, rows=rows, log_pi=lp_t, temperature=t,
                       workspace=ops.sacc_workspace(B, DEV))
    loss, la_o, m_o, v_o = O.temperature_step(la, m1, v1, 3, lp_o, -float(D), 1e-3)
    _close(t["stats"][1], loss)
    _close(t["log_alpha"], la_o)
    _close(t["alpha"], la_o.exp())
    _close(t["exp_avg"], m_o)


def test_soft_update_rounds_like_the_reference():
    from cleanrl_b200 import ops
    g = torch.Generator().manual_seed(1)
    src, dst = torch.randn(100003, generator=g).to(DEV), torch.randn(100003, generator=g).to(DEV)
    want = 0.005 * src + (1 - 0.005) * dst
    ops.sacc_soft_update(src, dst, src.numel(), 0.005)
    assert torch.equal(dst, want)


def test_out_of_range_shapes_are_refused():
    from cleanrl_b200 import ops
    z = torch.zeros(8, 1100, device=DEV)
    p = torch.zeros(1 << 20, device=DEV)
    for od, D, B in ((1000, 25, 8), (17, 33, 8), (17, 6, 8193)):
        with pytest.raises(RuntimeError, match="outside"):
            ops.sacc_critic_fwd(p, 0, torch.zeros(B, od, device=DEV), torch.zeros(B, D, device=DEV), B, od, D)


def test_noise_equals_normal_rsample():
    from cleanrl_b200.agents import SACContinuousActor
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    env = SyntheticGymnasiumVec(4, kind="continuous")
    actor = SACContinuousActor(env).to(DEV)
    obs = torch.randn(4, 17, device=DEV)
    mean, log_std = actor(obs)
    torch.manual_seed(9)
    a, lp, _ = actor.get_action(obs)
    torch.manual_seed(9)
    x_t = torch.distributions.Normal(mean, log_std.exp()).rsample()
    _close(a, torch.tanh(x_t) * actor.action_scale + actor.action_bias)


def _run_updates(graph, n=6, autotune=True, B=256, od=17, D=6):
    from cleanrl_b200 import ops
    from cleanrl_b200.agents import (SACContinuousActor, SACContinuousState, SoftQNetworkMLP, _sacc_update_body,
                                     sac_continuous_update)
    from cleanrl_b200.replay import DeviceReplayRing
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    env = SyntheticGymnasiumVec(2, kind="continuous", obs_dim=od, act_dim=D)
    torch.manual_seed(1)
    nets = [n.to(DEV) for n in (SACContinuousActor(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env),
                                 SoftQNetworkMLP(env), SoftQNetworkMLP(env))]
    nets[3].load_state_dict(nets[1].state_dict())
    nets[4].load_state_dict(nets[2].state_dict())
    st = SACContinuousState(*nets, DEV, autotune=autotune)
    rb = DeviceReplayRing(4096, (od,), 2, DEV, optimize_memory_usage=False, obs_dtype=torch.float32, action_shape=(D,))
    g = np.random.default_rng(3)
    for _ in range(600):
        rb.add(g.standard_normal((2, od)), g.standard_normal((2, od)), g.uniform(-1, 1, (2, D)), g.standard_normal(2),
               (g.random(2) < 0.05).astype(np.float32))
    args = types.SimpleNamespace(policy_frequency=2, target_network_frequency=1, q_lr=1e-3, policy_lr=3e-4, gamma=0.99,
                                 tau=0.005)
    np.random.seed(5)
    torch.manual_seed(6)
    counts = []
    for step in range(1, n + 1):
        batch = rb.sample(B)
        c0 = ops._lib.load().b200rl_launch_count()
        sac_continuous_update(st, rb, batch, step, args, graph=graph)
        counts.append(ops._lib.load().b200rl_launch_count() - c0)
    torch.cuda.synchronize()
    return st, nets, counts


def test_graph_replay_is_bitwise_eager_and_repeatable():
    st_e, nets_e, counts = _run_updates(graph=False)
    st_e2, _, _ = _run_updates(graph=False)
    st_g, nets_g, _ = _run_updates(graph=True)
    for a, b, c in ((st_e.q.flat, st_e2.q.flat, st_g.q.flat), (st_e.qt.flat, st_e2.qt.flat, st_g.qt.flat),
                    (nets_e[0].flat.flat, st_e2.actor.flat.flat, nets_g[0].flat.flat),
                    (st_e.astats, st_e2.astats, st_g.astats), (st_e.qstats, st_e2.qstats, st_g.qstats),
                    (st_e.log_alpha, st_e2.log_alpha, st_g.log_alpha)):
        assert torch.equal(a, b) and torch.equal(a, c)
    assert bool(torch.isfinite(st_e.q.flat).all()) and float(st_e.log_alpha) != 0.0
    # launch budget: critic-only steps (odd) and steps with two actor + temperature steps (even)
    assert max(counts[0::2]) <= 12 and max(counts[1::2]) <= 32, counts


def test_graph_replay_at_the_column_limit():
    st_e, _, _ = _run_updates(graph=False, n=2, B=64, od=1000, D=24)
    st_g, _, _ = _run_updates(graph=True, n=2, B=64, od=1000, D=24)
    assert torch.equal(st_e.q.flat, st_g.q.flat) and torch.equal(st_e.actor.flat.flat, st_g.actor.flat.flat)
    assert bool(torch.isfinite(st_e.q.flat).all())


def test_min_propagates_nan_like_torch_min():
    from cleanrl_b200 import ops
    q = torch.tensor([[1.0, float("nan")], [2.0, 0.5]], device=DEV)
    qn = torch.tensor([[float("nan"), 1.0], [0.0, 1.0]], device=DEV)
    z = torch.zeros(2, device=DEV)
    ops.sacc_critic_loss(qn, z, q, z, z, torch.zeros(1, device=DEV), 0.99, y=(y := torch.empty(2, device=DEV)))
    assert bool(torch.isnan(y[0])) and not bool(torch.isnan(y[1]))


def test_update_matches_the_eager_reference_update():
    """The first update against the oracle's autograd / torch.optim update on the same batch and noise."""
    from cleanrl_b200.agents import (SACContinuousActor, SACContinuousState, SoftQNetworkMLP, sac_continuous_update)
    from cleanrl_b200.replay import DeviceReplayRing
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    od, D, B = 17, 6, 256
    env = SyntheticGymnasiumVec(1, kind="continuous")
    torch.manual_seed(2)
    nets = [n.to(DEV) for n in (SACContinuousActor(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env),
                                 SoftQNetworkMLP(env), SoftQNetworkMLP(env))]
    nets[3].load_state_dict(nets[1].state_dict())
    nets[4].load_state_dict(nets[2].state_dict())
    st = SACContinuousState(*nets, DEV)
    ref = O.EagerSAC(st.actor.flat.flat[:st.actor.flat.numel].clone(), st.q.flat[:st.q.numel].clone(),
                     st.qt.flat[:st.qt.numel].clone(), od, D, nets[0].action_scale, nets[0].action_bias, DEV)
    rb = DeviceReplayRing(1000, (od,), 1, DEV, optimize_memory_usage=False, obs_dtype=torch.float32, action_shape=(D,))
    g = np.random.default_rng(0)
    for _ in range(500):
        rb.add(g.standard_normal((1, od)), g.standard_normal((1, od)), g.uniform(-1, 1, (1, D)), g.standard_normal(1),
               (g.random(1) < 0.05).astype(np.float32))
    args = types.SimpleNamespace(policy_frequency=2, target_network_frequency=1, q_lr=1e-3, policy_lr=3e-4, gamma=0.99,
                                 tau=0.005)
    np.random.seed(1)
    batch = rb.sample(B)
    torch.manual_seed(11)
    sac_continuous_update(st, rb, batch, 2, args)
    torch.manual_seed(11)
    noise = lambda shape: torch.empty(shape, device=DEV).normal_()   # noqa: E731
    ref.update(2, rb.frames[batch["rows"]], rb.action_rows[batch["rows"]], rb.next_frames[batch["rows"]], rb.reward_rows[batch["rows"]],
               rb.done_rows[batch["rows"]], noise)
    torch.cuda.synchronize()
    _close(st.qstats, torch.tensor([ref.stats[k]() for k in ("qf1_values", "qf2_values", "qf1_loss", "qf2_loss")]))
    _close(st.astats[:3], torch.tensor([ref.stats["actor_loss"](), ref.stats["alpha_loss"](), ref.alpha]), rtol=1e-4)
    want_q = torch.cat([torch.nn.utils.parameters_to_vector(q.parameters()) for q in (ref.qf1, ref.qf2)])
    want_qt = torch.cat([torch.nn.utils.parameters_to_vector(q.parameters()) for q in (ref.qf1_target, ref.qf2_target)])
    _close(st.q.flat[:st.q.numel], want_q, rtol=1e-4)
    _close(st.qt.flat[:st.qt.numel], want_qt, rtol=1e-4)
    _close(st.actor.flat.flat[:st.actor.flat.numel], torch.nn.utils.parameters_to_vector(ref.actor.parameters()),
           rtol=1e-4)


def test_drop_in_runs_and_logs_the_reference_tags(tmp_path, monkeypatch):
    from cleanrl_b200 import sac_continuous_action as m
    monkeypatch.chdir(tmp_path)
    scalars = []

    class W:
        def __init__(self, *a, **k):
            pass

        def add_text(self, *a, **k):
            pass

        def add_scalar(self, tag, v, step):
            scalars.append((tag, step))

        def close(self):
            pass

    m.main(["--synthetic-env", "--total-timesteps", "420", "--learning-starts", "100", "--batch-size", "64",
            "--num-envs", "2", "--buffer-size", "300"], writer_factory=W)
    tags = {t for t, _ in scalars}
    for t in ("losses/qf1_values", "losses/qf2_values", "losses/qf1_loss", "losses/qf2_loss", "losses/qf_loss",
              "losses/actor_loss", "losses/alpha", "charts/SPS", "losses/alpha_loss"):
        assert t in tags, t
    assert sorted({s for t, s in scalars if t == "losses/alpha"}) == [200, 300, 400]


# ------------------------------------------------------------ the drop-in against runs of the unmodified reference
from pathlib import Path  # noqa: E402

GOLDEN = Path(__file__).resolve().parent / "golden"
FIXTURES = ["sac_continuous_n2_seed1.npz", "sac_continuous_seed2_alpha01.npz"]
LATER_UPDATES_RTOL = 1e-2        # fp32 updates after the first: bound on the relative deviation from the reference


def _cpu_normal(n, D, device):
    # the reference ran on the CPU: Normal.rsample drew torch.empty(n, D).normal_() from the CPU generator
    return torch.empty(n, D, dtype=torch.float32).normal_().to(device)


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)) / np.maximum(1.0, np.abs(np.asarray(b)))


@pytest.mark.parametrize("name", FIXTURES)
def test_drop_in_vs_reference_run(name, monkeypatch, tmp_path):
    from cleanrl_b200 import agents, sac_continuous_action as m
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    z = np.load(GOLDEN / name)
    argv = [a for a in z["argv"].tolist() if a != "--no-cuda"] + ["--synthetic-env"]
    autotune = "--no-autotune" not in argv
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(agents, "_normal_noise", _cpu_normal)
    stream, recs, scalars = [], [], []
    orig = SyntheticGymnasiumVec.step

    def step(self_, act):
        stream.append(np.asarray(act, dtype=np.float32).copy())
        return orig(self_, act)
    monkeypatch.setattr(SyntheticGymnasiumVec, "step", step)

    def sums(params):
        return np.array([p.detach().double().sum().item() for p in params])

    def on_update(step_, st):
        recs.append({"q": st.qstats.cpu().numpy().copy(), "a": st.astats.cpu().numpy().copy(),
                     "q_sums": sums(st.q.params), "actor_sums": sums(st.actor.parameters())})

    class W:
        def __init__(self, *a, **k):
            pass

        def add_text(self, *a, **k):
            pass

        def add_scalar(self, tag, v, s_):
            scalars.append((tag, s_))

        def close(self):
            pass

    actor, qf1, _, _ = m.main(argv, writer_factory=W, on_update=on_update)
    assert list(actor.state_dict()) == z["actor_keys"].tolist() and list(qf1.state_dict()) == z["qf_keys"].tolist()
    assert len(recs) == len(z["qf1_loss"])
    ls = int(argv[argv.index("--learning-starts") + 1])
    got = np.stack(stream)
    assert np.array_equal(got[:ls], z["action_stream"][:ls])          # random actions: the same Box draws
    assert (_rel(got, z["action_stream"]) <= LATER_UPDATES_RTOL).all()
    for k, rec in enumerate(recs):
        tol = 1e-5 if k == 0 else LATER_UPDATES_RTOL
        for i, key in enumerate(("qf1_values", "qf2_values", "qf1_loss", "qf2_loss")):
            assert _rel(rec["q"][i], z[key][k]) <= tol, (k, key, rec["q"][i], z[key][k])
        assert (_rel(rec["q_sums"], z["q_sums"][k]) <= tol).all(), k
        if not np.isnan(z["actor_loss"][k]):                            # an update with actor steps
            assert _rel(rec["a"][0], z["actor_loss"][k]) <= tol, (k, rec["a"][0], z["actor_loss"][k])
            assert (_rel(rec["actor_sums"], z["actor_sums"][k]) <= tol).all(), k
            if autotune:
                assert _rel(rec["a"][1], z["alpha_loss"][k]) <= tol, k
                assert _rel(rec["a"][3], z["log_alpha"][k]) <= tol, k
        if autotune and k + 1 < len(recs):
            assert _rel(rec["a"][2], z["alpha"][k + 1]) <= tol, k              # alpha the next update uses
    ref_tags = {k[3:]: z[k] for k in z.files if k.startswith("tb/")}
    tags = {}
    for t, s_ in scalars:
        tags.setdefault(t, []).append(s_)
    assert set(tags) == set(ref_tags)
    for t in ref_tags:
        assert tags[t] == ref_tags[t][:, 0].astype(int).tolist(), t
