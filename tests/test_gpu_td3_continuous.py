"""TD3 on the continuous-control kernels (csrc/sac_continuous.cu) on the GPU: the deterministic actor's forward with the
target policy smoothing, the critic loss without an entropy term, the single-network critic backward, the
deterministic actor's backward and weight gradient against the fp32 oracle over batch sizes and (obs, act) shapes;
graph replay against eager launches, the launch budget, NaN in the min, the first update against the eager reference
update, and the drop-in end to end, against both reference runs and through --save-model."""
from __future__ import annotations

import types

import numpy as np
import pytest
import torch

from oracle import td3_continuous_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
SHAPES = [(17, 6), (3, 1), (376, 17), (1000, 24), (1023, 1)]     # the last two at the 1024-column limit
BATCHES = [1, 7, 256, 1000, 8192]


def _close(got, want, rtol=1e-5):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    err = float((got - want).abs().max()) if got.numel() else 0.0
    assert err <= rtol * max(1.0, float(want.abs().max())), (err, float(want.abs().max()), got.shape)


def _setup(od, D, seed=0):
    """Flat actor and twin-critic parameters with the reference's default nn.Linear initialisation."""
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
    assert af.numel() == ops.sacc_param_count(od, D, ops.SACC_TD3_ACTOR)
    N = B + 5
    obs = torch.randn(N, od, generator=g).to(DEV)
    act = torch.rand(N, D, generator=g).to(DEV) * 2 - 1
    rows = torch.randint(0, N, (B,), generator=g).to(DEV)
    eps = torch.randn(B, D, generator=g).to(DEV)
    scale = torch.linspace(0.5, 1.5, D, device=DEV)
    bias = torch.linspace(-0.2, 0.2, D, device=DEV)
    x, xa = obs[rows], act[rows]
    # deterministic actor forward with the smoothed target action (tight bounds and a small noise_clip make both clamps bind)
    mu, ya, sm = (torch.empty(B, D, device=DEV) for _ in range(3))
    kh = dict(keep_x=torch.empty(B, od, device=DEV), keep_h1=torch.empty(B, 256, device=DEV),
              keep_h2=torch.empty(B, 256, device=DEV))
    smoothing = dict(eps=eps, policy_noise=0.5, noise_clip=0.3, low=-0.5, high=0.6, out=sm)
    ops.td3_actor_fwd(af, obs, B, od, D, scale, bias, rows=rows, mu=mu, keep_y=ya, smoothing=smoothing, **kh)
    pa, n_a = O.mlp_params(af, od, D)
    assert n_a == af.numel()
    mu_o, y_o = O.head_forward(O.actor_trunk(pa, x), scale, bias)
    _close(mu, mu_o)
    _close(ya, y_o)
    assert torch.equal(kh["keep_x"], x)
    _close(sm, O.smooth(mu_o, eps, scale, 0.5, 0.3, -0.5, 0.6))
    assert float(sm.min()) >= float(np.float32(-0.5)) and float(sm.max()) <= float(np.float32(0.6))
    # critic loss without the entropy term
    keep = dict(keep_x=torch.empty(B, od + D, device=DEV), keep_h1=torch.empty(2, B, 256, device=DEV),
                keep_h2=torch.empty(2, B, 256, device=DEV))
    q = ops.sacc_critic_fwd(qf, S, obs, act, B, od, D, obs_rows=rows, act_rows=rows, **keep)
    rew, done = torch.randn(N, generator=g).to(DEV), (torch.rand(N, generator=g) < 0.1).float().to(DEV)
    qn = torch.randn(2, B, generator=g).to(DEV)
    y = torch.empty(B, device=DEV)
    stats, dq = ops.sacc_critic_loss(qn, None, q, rew, done, None, 0.99, rows=rows, y=y)
    y_o, l1, l2, d1, d2 = O.critic_loss(q[0], q[1], qn[0], qn[1], rew[rows], done[rows], 0.99)
    _close(y, y_o)
    _close(dq, torch.stack([d1, d2]))
    _close(stats, torch.stack([q[0].mean(), q[1].mean(), l1, l2]))
    # actor step: qf1 alone on the actor's action, its single-network backward, the actor backward and weight gradient
    qpi = torch.empty(1, B, device=DEV)
    ops.sacc_critic_fwd(qf, 0, obs, mu, B, od, D, obs_rows=rows, q=qpi, keep_h1=keep["keep_h1"], keep_h2=keep["keep_h2"])
    dact = torch.empty(B, D, device=DEV)
    ops.sacc_critic_bwd(qf, 0, B, od, D, keep["keep_h1"], keep["keep_h2"], dact=dact)
    dhead, dz1a, dz2a = torch.empty(B, D, device=DEV), torch.empty(B, 256, device=DEV), torch.empty(B, 256, device=DEV)
    ast = torch.zeros(1, device=DEV)
    ops.td3_actor_bwd(af, B, od, D, ya, scale, dact, qpi[0], kh["keep_h1"], kh["keep_h2"], dhead, dz1a, dz2a, ast,
                      ops.sacc_workspace(B, DEV))
    agrad = torch.full_like(af, float("nan"))
    ops.sacc_wgrad(ops.SACC_TD3_ACTOR, B, od, D, kh["keep_x"], kh["keep_h1"], kh["keep_h2"], dz1a, dz2a, dhead, agrad)
    aleaf = af.clone().requires_grad_(True)
    pa2, _ = O.mlp_params(aleaf, od, D)
    pi, _ = O.head_forward(O.actor_trunk(pa2, x), scale, bias)
    p1, _ = O.mlp_params(qf[:S], od + D, 1)
    q1_pi = O.critic_forward(p1, x, pi).view(-1)
    al = O.actor_loss(q1_pi)
    al.backward()
    _close(qpi[0], q1_pi)
    _close(ast, al.detach().view(1))
    _close(agrad, aleaf.grad)


def test_min_propagates_nan_like_torch_min():
    from cleanrl_b200 import ops
    q = torch.tensor([[1.0, float("nan")], [2.0, 0.5]], device=DEV)
    qn = torch.tensor([[float("nan"), 1.0], [0.0, 1.0]], device=DEV)
    z = torch.zeros(2, device=DEV)
    y = torch.empty(2, device=DEV)
    ops.sacc_critic_loss(qn, None, q, z, z, None, 0.99, y=y)
    assert bool(torch.isnan(y[0])) and float(y[1]) == pytest.approx(0.99)


def _nets(env, seed):
    from cleanrl_b200.agents import SoftQNetworkMLP, TD3Actor
    torch.manual_seed(seed)
    nets = [n.to(DEV) for n in (TD3Actor(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env), SoftQNetworkMLP(env),
                                 SoftQNetworkMLP(env), TD3Actor(env))]
    nets[5].load_state_dict(nets[0].state_dict())
    nets[3].load_state_dict(nets[1].state_dict())
    nets[4].load_state_dict(nets[2].state_dict())
    return nets


ARGS = types.SimpleNamespace(policy_frequency=2, learning_rate=3e-4, gamma=0.99, tau=0.005, policy_noise=0.2,
                             noise_clip=0.5)


def _ring(od, D, n_envs, fill, seed):
    from cleanrl_b200.replay import DeviceReplayRing
    rb = DeviceReplayRing(4096, (od,), n_envs, DEV, optimize_memory_usage=False, obs_dtype=torch.float32,
                          action_shape=(D,))
    g = np.random.default_rng(seed)
    for _ in range(fill):
        rb.add(g.standard_normal((n_envs, od)), g.standard_normal((n_envs, od)), g.uniform(-1, 1, (n_envs, D)),
               g.standard_normal(n_envs), (g.random(n_envs) < 0.05).astype(np.float32))
    return rb


def _run_updates(graph, n=6, B=256, od=17, D=6):
    from cleanrl_b200 import ops
    from cleanrl_b200.agents import TD3State, td3_update
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    env = SyntheticGymnasiumVec(2, kind="continuous", obs_dim=od, act_dim=D)
    nets = _nets(env, 1)
    st = TD3State(*nets, DEV)
    rb = _ring(od, D, 2, 600, 3)
    np.random.seed(5)
    torch.manual_seed(6)
    counts = []
    for step in range(1, n + 1):
        batch = rb.sample(B)
        c0 = ops._lib.load().b200rl_launch_count()
        td3_update(st, rb, batch, step, ARGS, graph=graph)
        counts.append(ops._lib.load().b200rl_launch_count() - c0)
    torch.cuda.synchronize()
    return st, counts


def _state_tensors(st):
    return (st.q.flat, st.qt.flat, st.actor.flat.flat, st.target_actor.flat.flat, st.qstats, st.astats)


def test_graph_replay_is_bitwise_eager_and_repeatable():
    st_e, counts = _run_updates(graph=False)
    st_e2, _ = _run_updates(graph=False)
    st_g, counts_g = _run_updates(graph=True)
    for a, b, c in zip(_state_tensors(st_e), _state_tensors(st_e2), _state_tensors(st_g)):
        assert torch.equal(a, b) and torch.equal(a, c)
    assert bool(torch.isfinite(st_e.q.flat).all()) and float(st_e.astats[0]) != 0.0
    assert not torch.equal(st_e.target_actor.flat.flat, st_e.actor.flat.flat)
    # launch budget: critic-only updates (odd steps) and updates with the actor step and the target updates (even)
    assert counts[0::2] == [7, 7, 7] and counts[1::2] == [15, 15, 15], counts
    assert len(st_g._graphs) == 2


def test_graph_replay_at_the_column_limit():
    st_e, _ = _run_updates(graph=False, n=2, B=64, od=1000, D=24)
    st_g, _ = _run_updates(graph=True, n=2, B=64, od=1000, D=24)
    for a, b in zip(_state_tensors(st_e), _state_tensors(st_g)):
        assert torch.equal(a, b)
    assert bool(torch.isfinite(st_e.q.flat).all())


def test_update_matches_the_eager_reference_update():
    """An update with the actor step against the oracle's autograd / torch.optim update on the same batch and noise."""
    from cleanrl_b200.agents import TD3State, td3_update
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    od, D, B = 17, 6, 256
    nets = _nets(SyntheticGymnasiumVec(1, kind="continuous"), 2)
    st = TD3State(*nets, DEV)
    flat = lambda f: f.flat[:f.numel].clone()   # noqa: E731
    ref = O.EagerTD3(flat(st.actor.flat), flat(st.q), flat(st.qt), flat(st.target_actor.flat), od, D,
                     nets[0].action_scale, nets[0].action_bias, DEV)
    rb = _ring(od, D, 1, 500, 0)
    np.random.seed(1)
    batch = rb.sample(B)
    torch.manual_seed(11)
    td3_update(st, rb, batch, 2, ARGS)
    torch.manual_seed(11)
    noise = lambda shape: torch.empty(shape, device=DEV).normal_()   # noqa: E731
    r = batch["rows"]
    ref.update(2, rb.frames[r], rb.action_rows[r], rb.next_frames[r], rb.reward_rows[r], rb.done_rows[r], noise)
    torch.cuda.synchronize()
    _close(st.qstats, torch.tensor([ref.stats[k]() for k in ("qf1_values", "qf2_values", "qf1_loss", "qf2_loss")]))
    _close(st.astats, torch.tensor([ref.stats["actor_loss"]()]), rtol=1e-4)
    vec = lambda *ns: torch.cat([torch.nn.utils.parameters_to_vector(n.parameters()) for n in ns])   # noqa: E731
    _close(flat(st.q), vec(ref.qf1, ref.qf2), rtol=1e-4)
    _close(flat(st.qt), vec(ref.qf1_target, ref.qf2_target), rtol=1e-4)
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


def test_drop_in_runs_and_logs_the_reference_tags(tmp_path, monkeypatch):
    from cleanrl_b200 import td3_continuous_action as m
    monkeypatch.chdir(tmp_path)
    scalars = []
    m.main(["--synthetic-env", "--total-timesteps", "420", "--learning-starts", "100", "--batch-size", "64",
            "--num-envs", "2", "--buffer-size", "300"], writer_factory=_Writer(scalars))
    tags = {t for t, _ in scalars}
    for t in ("losses/qf1_values", "losses/qf2_values", "losses/qf1_loss", "losses/qf2_loss", "losses/qf_loss",
              "losses/actor_loss", "charts/SPS"):
        assert t in tags, t
        assert sorted({s for tt, s in scalars if tt == t}) == [200, 300, 400], t


def test_save_model_loads_in_stock_torch_modules_and_evaluates(tmp_path, monkeypatch):
    from cleanrl_b200 import td3_continuous_action as m
    monkeypatch.chdir(tmp_path)
    scalars = []
    m.main(["--synthetic-env", "--total-timesteps", "150", "--learning-starts", "100", "--batch-size", "32",
            "--save-model", "--exp-name", "td3_save"], writer_factory=_Writer(scalars))
    (path,) = list((tmp_path / "runs").glob("*/td3_save.cleanrl_model"))
    actor_sd, qf1_sd, qf2_sd = torch.load(path, map_location="cpu")
    stock = O._Actor(17, 6, torch.ones(6), torch.zeros(6))
    stock.load_state_dict(actor_sd)
    for sd in (qf1_sd, qf2_sd):
        O._Q(17, 6).load_state_dict(sd)
    assert sorted(s for t, s in scalars if t == "eval/episodic_return") == list(range(10))


# ------------------------------------------------------------ the drop-in against runs of the unmodified reference
from pathlib import Path  # noqa: E402

GOLDEN = Path(__file__).resolve().parent / "golden"
FIXTURES = ["td3_continuous_n2_seed1.npz", "td3_continuous_seed2_pf3.npz"]
LATER_UPDATES_RTOL = 1e-2        # fp32 updates after the first: bound on the relative deviation from the reference


def _cpu_normal(n, D, device):
    # the reference ran on the CPU: randn_like(actions) drew torch.empty(n, D).normal_() from the CPU generator
    return torch.empty(n, D, dtype=torch.float32).normal_().to(device)


def _cpu_exploration(std):
    return torch.normal(0, std.cpu()).to(std.device)


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)) / np.maximum(1.0, np.abs(np.asarray(b)))


@pytest.mark.parametrize("name", FIXTURES)
def test_drop_in_vs_reference_run(name, monkeypatch, tmp_path):
    from cleanrl_b200 import agents, td3_continuous_action as m
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    z = np.load(GOLDEN / name)
    argv = [a for a in z["argv"].tolist() if a != "--no-cuda"] + ["--synthetic-env"]
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(agents, "_normal_noise", _cpu_normal)
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

    actor, qf1, _, _ = m.main(argv, writer_factory=_Writer(scalars), on_update=on_update)
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
