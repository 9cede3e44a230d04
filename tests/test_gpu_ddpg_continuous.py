"""DDPG on the continuous-control kernels (csrc/sac_continuous.cu) on the GPU: the fused one-critic loss and data
backward and the one-critic weight gradient against the fp32 oracle over batch sizes and (obs, act) shapes, and bit for
bit against network 0 of the twin-critic kernels; NaN propagation; graph replay against eager launches and the launch
budget; an update against the eager reference update; and the drop-in end to end, against both reference runs and
through --save-model under a batched action space."""
from __future__ import annotations

import types
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import ddpg_continuous_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
SHAPES = [(17, 6), (3, 1), (376, 17), (1000, 24), (1023, 1)]     # the last two at the 1024-column limit
BATCHES = [1, 7, 256, 1000, 8192]


def _close(got, want, rtol=1e-5):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    err = float((got - want).abs().max()) if got.numel() else 0.0
    assert err <= rtol * max(1.0, float(want.abs().max())), (err, float(want.abs().max()), got.shape)


def _critic(od, D, seed=0):
    torch.manual_seed(seed)
    return torch.nn.utils.parameters_to_vector(O._Q(od, D).parameters()).detach().to(DEV)


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("od,D", SHAPES)
def test_kernels_match_the_oracle_and_the_twin_path(B, od, D):
    from cleanrl_b200 import ops
    g = torch.Generator().manual_seed(B + od)
    qf = _critic(od, D)
    S = qf.numel()
    assert S == ops.sacc_param_count(od, D, True)
    N = B + 5
    obs = torch.randn(N, od, generator=g).to(DEV)
    act = (torch.rand(N, D, generator=g) * 2 - 1).to(DEV)
    rows = torch.randint(0, N, (B,), generator=g).to(DEV)
    rew, done = torch.randn(N, generator=g).to(DEV), (torch.rand(N, generator=g) < 0.1).float().to(DEV)
    qn = torch.randn(1, B, generator=g).to(DEV)
    x, a = obs[rows], act[rows]
    keep = dict(keep_x=torch.empty(B, od + D, device=DEV), keep_h1=torch.empty(1, B, 256, device=DEV),
                keep_h2=torch.empty(1, B, 256, device=DEV))
    q = ops.sacc_critic_fwd(qf, 0, obs, act, B, od, D, obs_rows=rows, act_rows=rows, q=torch.empty(1, B, device=DEV),
                            **keep)
    y = torch.empty(B, device=DEV)
    stats, dq, dz1, dz2 = ops.ddpg_critic_loss_bwd(qf, B, od, D, qn, q, rew, done, 0.99, keep["keep_h1"],
                                                   keep["keep_h2"], rows=rows, y=y)
    grad = torch.full_like(qf, float("nan"))
    ops.sacc_wgrad(True, B, od, D, keep["keep_x"], keep["keep_h1"], keep["keep_h2"], dz1, dz2, dq, grad, 0)
    # the oracle: autograd through the critic of F.mse_loss(q, y) with the target held fixed
    leaf = qf.clone().requires_grad_(True)
    p, _ = O.mlp_params(leaf, od + D, 1)
    w1, b1, w2, b2, w3, b3 = p
    h1 = torch.relu(torch.nn.functional.linear(torch.cat([x, a], 1), w1, b1))
    h2 = torch.relu(torch.nn.functional.linear(h1, w2, b2))
    q_o = torch.nn.functional.linear(h2, w3, b3).view(-1)
    y_o, loss_o, dq_o = O.critic_loss(q_o.detach(), qn[0], rew[rows], done[rows], 0.99)
    torch.nn.functional.mse_loss(q_o, y_o).backward()
    with torch.no_grad():
        dz2_o = (h2 > 0).float() * (dq_o[:, None] * w3)
        dz1_o = (h1 > 0).float() * (dz2_o @ w2)
    assert torch.equal(keep["keep_x"], torch.cat([x, a], 1))
    _close(q[0], q_o)
    _close(y, y_o)
    _close(dq, dq_o)
    _close(dz2, dz2_o)
    _close(dz1, dz1_o)
    _close(stats, torch.stack([q_o.mean(), loss_o]))
    _close(grad, leaf.grad)
    # bit for bit against network 0 of the twin kernels on the same inputs
    twin = torch.cat([qf, _critic(od, D, seed=1)])
    th1, th2 = torch.cat([keep["keep_h1"], keep["keep_h1"]]), torch.cat([keep["keep_h2"], keep["keep_h2"]])
    tdq = torch.stack([dq, dq])
    tz1, tz2 = torch.empty(2, B, 256, device=DEV), torch.empty(2, B, 256, device=DEV)
    ops.sacc_critic_bwd(twin, S, B, od, D, th1, th2, dq=tdq, dz1=tz1, dz2=tz2)
    tgrad = torch.empty_like(twin)
    ops.sacc_wgrad(True, B, od, D, keep["keep_x"], th1, th2, tz1, tz2, tdq, tgrad, S)
    assert torch.equal(dz1, tz1[0]) and torch.equal(dz2, tz2[0])
    assert torch.equal(grad, tgrad[:S])


def test_nan_propagates_to_y_dq_and_the_loss():
    from cleanrl_b200 import ops
    od, D, B = 17, 6, 3
    qf = _critic(od, D)
    h = torch.ones(1, B, 256, device=DEV)
    q = torch.tensor([[1.0, float("nan"), 2.0]], device=DEV)
    qn = torch.tensor([[float("nan"), 1.0, 0.5]], device=DEV)
    z = torch.zeros(B, device=DEV)
    y = torch.empty(B, device=DEV)
    stats, dq, dz1, dz2 = ops.ddpg_critic_loss_bwd(qf, B, od, D, qn, q, z, z, 0.99, h, h, y=y)
    y_o, loss_o, dq_o = O.critic_loss(q[0].cpu(), qn[0].cpu(), z.cpu(), z.cpu(), 0.99)
    assert torch.equal(torch.isnan(y).cpu(), torch.isnan(y_o)) and torch.equal(torch.isnan(dq).cpu(), torch.isnan(dq_o))
    assert bool(torch.isnan(y[0])) and not bool(torch.isnan(y[1])) and bool(torch.isnan(dq[1]))
    assert float(y[2]) == pytest.approx(0.495) and float(dq[2]) == pytest.approx(2.0 / 3 * (2.0 - 0.495))
    assert bool(torch.isnan(stats).all()) and bool(torch.isnan(loss_o))
    assert bool(torch.isnan(dz2[0]).all()) and bool(torch.isfinite(dz2[2]).all())


def _env(batched=False, od=17, D=6):
    from cleanrl_b200.synthetic_envs import Box, SyntheticGymnasiumVec
    env = SyntheticGymnasiumVec(1, kind="continuous", obs_dim=od, act_dim=D)
    if batched:
        env.action_space = Box(-1.0, 1.0, (1, D), np.float32)
    return env


def _nets(env, seed):
    from cleanrl_b200.agents import DDPGActor, SoftQNetworkMLP
    torch.manual_seed(seed)
    nets = [n.to(DEV) for n in (DDPGActor(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env), DDPGActor(env))]
    nets[3].load_state_dict(nets[0].state_dict())
    nets[2].load_state_dict(nets[1].state_dict())
    return nets


ARGS = types.SimpleNamespace(policy_frequency=2, learning_rate=3e-4, gamma=0.99, tau=0.005)


def _ring(od, D, fill, seed):
    from cleanrl_b200.replay import DeviceReplayRing
    rb = DeviceReplayRing(4096, (od,), 1, DEV, optimize_memory_usage=False, obs_dtype=torch.float32, action_shape=(D,))
    g = np.random.default_rng(seed)
    for _ in range(fill):
        rb.add(g.standard_normal((1, od)), g.standard_normal((1, od)), g.uniform(-1, 1, (1, D)), g.standard_normal(1),
               (g.random(1) < 0.05).astype(np.float32))
    return rb


def _run_updates(graph, n=6, B=256, od=17, D=6):
    from cleanrl_b200 import ops
    from cleanrl_b200.agents import DDPGState, ddpg_update
    st = DDPGState(*_nets(_env(True, od, D), 1), DEV)
    rb = _ring(od, D, 600, 3)
    np.random.seed(5)
    counts = []
    for step in range(1, n + 1):
        batch = rb.sample(B)
        c0 = ops._lib.load().b200rl_launch_count()
        ddpg_update(st, rb, batch, step, ARGS, graph=graph)
        counts.append(ops._lib.load().b200rl_launch_count() - c0)
    torch.cuda.synchronize()
    return st, counts


def _state_tensors(st):
    return (st.q.flat, st.qt.flat, st.actor.flat.flat, st.target_actor.flat.flat, st.qstats, st.astats)


def test_graph_replay_is_bitwise_eager_and_repeatable():
    st_e, counts = _run_updates(graph=False)
    st_e2, _ = _run_updates(graph=False)
    st_g, counts_g = _run_updates(graph=True)
    st_g2, _ = _run_updates(graph=True)
    for a, b, c, d in zip(_state_tensors(st_e), _state_tensors(st_e2), _state_tensors(st_g), _state_tensors(st_g2)):
        assert torch.equal(a, b) and torch.equal(a, c) and torch.equal(a, d)
    assert bool(torch.isfinite(st_e.q.flat).all()) and float(st_e.astats[0]) != 0.0
    assert not torch.equal(st_e.target_actor.flat.flat, st_e.actor.flat.flat)
    assert not torch.equal(st_e.qt.flat, st_e.q.flat)
    # launch budget: critic-only updates (odd steps) and updates with the actor step and both soft updates (even)
    assert counts[0::2] == [6, 6, 6] and counts[1::2] == [14, 14, 14], counts
    assert len(st_g._graphs) == 2


def test_graph_replay_at_the_column_limit():
    st_e, _ = _run_updates(graph=False, n=2, B=64, od=1000, D=24)
    st_g, _ = _run_updates(graph=True, n=2, B=64, od=1000, D=24)
    for a, b in zip(_state_tensors(st_e), _state_tensors(st_g)):
        assert torch.equal(a, b)
    assert bool(torch.isfinite(st_e.q.flat).all())


def test_updates_match_the_eager_reference_update():
    """Four updates (two with the actor step) against the oracle's autograd / torch.optim updates on the same batches."""
    from cleanrl_b200.agents import DDPGState, ddpg_update
    od, D, B = 17, 6, 256
    nets = _nets(_env(), 2)
    st = DDPGState(*nets, DEV)
    flat = lambda f: f.flat[:f.numel].clone()   # noqa: E731
    ref = O.EagerDDPG(flat(st.actor.flat), flat(st.q), flat(st.qt), flat(st.target_actor.flat), od, D,
                      nets[0].action_scale, nets[0].action_bias, DEV)
    rb = _ring(od, D, 500, 0)
    np.random.seed(1)
    for step in (1, 2, 3, 4):
        batch = rb.sample(B)
        ddpg_update(st, rb, batch, step, ARGS)
        r = batch["rows"]
        ref.update(step, rb.frames[r], rb.action_rows[r], rb.next_frames[r], rb.reward_rows[r], rb.done_rows[r])
    torch.cuda.synchronize()
    _close(st.qstats, torch.tensor([ref.stats[k]() for k in ("qf1_values", "qf1_loss")]), rtol=1e-4)
    _close(st.astats, torch.tensor([ref.stats["actor_loss"]()]), rtol=1e-4)
    vec = lambda *ns: torch.cat([torch.nn.utils.parameters_to_vector(n.parameters()) for n in ns])   # noqa: E731
    _close(flat(st.q), vec(ref.qf1), rtol=1e-4)
    _close(flat(st.qt), vec(ref.qf1_target), rtol=1e-4)
    _close(flat(st.actor.flat), vec(ref.actor), rtol=1e-4)
    _close(flat(st.target_actor.flat), vec(ref.target_actor), rtol=1e-4)


class _Writer:
    def __init__(self, out):
        self.out = out

    def __call__(self, *a, **k):
        return self

    def add_text(self, *a, **k):
        pass

    def add_scalar(self, tag, v, step):
        self.out.append((tag, step))

    def close(self):
        pass


def test_save_model_loads_in_stock_torch_modules_and_evaluates(tmp_path, monkeypatch):
    """Under gymnasium's batched (1, D) action_space: the saved file holds [1, D] buffers and loads into stock
    restatements of the reference's Actor / QNetwork; the evaluation runs 10 episodes."""
    from cleanrl_b200 import ddpg_continuous_action as m
    monkeypatch.chdir(tmp_path)
    scalars = []
    m.main(["--total-timesteps", "150", "--learning-starts", "100", "--batch-size", "32", "--save-model",
            "--exp-name", "ddpg_save", "--upload-model"], writer_factory=_Writer(scalars),
           env_factory=lambda args: _env(True))
    (path,) = list((tmp_path / "runs").glob("*/ddpg_save.cleanrl_model"))
    actor_sd, qf1_sd = torch.load(path, map_location="cpu")
    assert actor_sd["action_scale"].shape == (1, 6) and actor_sd["action_bias"].shape == (1, 6)
    stock = O._Actor(17, 6, torch.ones(1, 6), torch.zeros(1, 6))
    stock.load_state_dict(actor_sd)
    O._Q(17, 6).load_state_dict(qf1_sd)
    assert sorted(s for t, s in scalars if t == "eval/episodic_return") == list(range(10))


# ------------------------------------------------------------ the drop-in against runs of the unmodified reference
GOLDEN = Path(__file__).resolve().parent / "golden"
FIXTURES = ["ddpg_continuous_seed1.npz", "ddpg_continuous_seed2_pf3.npz"]
LATER_UPDATES_RTOL = 1e-2        # fp32 updates after the first: bound on the relative deviation from the reference


def _cpu_exploration(std):
    # the reference ran on the CPU: torch.normal(0, std) drew from the CPU generator
    return torch.normal(0, std.cpu()).to(std.device)


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)) / np.maximum(1.0, np.abs(np.asarray(b)))


@pytest.mark.parametrize("name", FIXTURES)
def test_drop_in_vs_reference_run(name, monkeypatch, tmp_path):
    from cleanrl_b200 import agents, ddpg_continuous_action as m
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    z = np.load(GOLDEN / name)
    argv = [a for a in z["argv"].tolist() if a != "--no-cuda"]
    batched = z["action_scale"].ndim == 2
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(agents, "_exploration_noise", _cpu_exploration)
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
                     "q_sums": sums(st.q.params), "actor_sums": sums(st.actor.parameters()),
                     "target_sums": sums(list(st.target_actor.parameters()) + st.qt.params)})

    actor, qf1, _ = m.main(argv, writer_factory=_Writer(scalars), env_factory=lambda args: _env(batched),
                           on_update=on_update)
    assert list(actor.state_dict()) == z["actor_keys"].tolist() and list(qf1.state_dict()) == z["qf_keys"].tolist()
    assert [str(tuple(v.shape)) for v in actor.state_dict().values()] == z["actor_shapes"].tolist()
    assert len(recs) == len(z["qf1_loss"])
    ls = int(argv[argv.index("--learning-starts") + 1])
    got = np.stack(stream)
    assert np.array_equal(got[:ls], z["action_stream"][:ls])          # random actions: the same Box draws
    assert (_rel(got, z["action_stream"]) <= LATER_UPDATES_RTOL).all()
    for k, rec in enumerate(recs):
        tol = 1e-5 if k == 0 else LATER_UPDATES_RTOL
        for i, key in enumerate(("qf1_values", "qf1_loss")):
            assert _rel(rec["q"][i], z[key][k]) <= tol, (k, key, rec["q"][i], z[key][k])
        assert (_rel(rec["q_sums"], z["q_sums"][k]) <= tol).all(), k
        assert (_rel(rec["target_sums"], z["target_sums"][k]) <= tol).all(), k
        if not np.isnan(z["actor_loss"][k]):                            # an update with the actor step
            assert _rel(rec["a"][0], z["actor_loss"][k]) <= tol, (k, rec["a"][0], z["actor_loss"][k])
            assert (_rel(rec["actor_sums"], z["actor_sums"][k]) <= tol).all(), k
    ref_tags = {k[3:]: z[k] for k in z.files if k.startswith("tb/")}
    tags = {}
    for t, s_ in scalars:
        tags.setdefault(t, []).append(s_)
    assert set(tags) == set(ref_tags)
    for t in ref_tags:
        assert tags[t] == ref_tags[t][:, 0].astype(int).tolist(), t
