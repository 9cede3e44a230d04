"""-m gpu: the SAC kernels against the numpy oracle, get_action's sampler, the graph-replayed bf16 update against eager
launches, and the sac_atari drop-in against the unmodified reference runs (tests/golden/sac_atari_*.npz)."""
import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import sac_oracle as O

pytestmark = pytest.mark.gpu

FIXTURES = ["sac_atari_b8_seed1.npz", "sac_atari_b8_seed2_alpha01.npz"]
LATER_UPDATES_RTOL = 1e-2        # fp32 updates after the first: bound on the relative deviation from the reference


class _Envs:
    def __init__(self, A):
        from cleanrl_b200.synthetic_envs import Box, Discrete
        self.single_observation_space = Box(0, 255, (4, 84, 84), np.uint8)
        self.single_action_space = Discrete(A)


def _cpu_noise(n, A, device):
    return torch.empty(n, A, dtype=torch.float32).exponential_(1).to(device)


def _case(B, A, seed):
    g = torch.Generator().manual_seed(seed)
    t = [torch.randn(B, A, generator=g) * 3 for _ in range(6)]
    a = torch.randint(0, A, (B,), generator=g)
    r = torch.randint(-1, 2, (B,), generator=g).float()
    d = (torch.rand(B, generator=g) < 0.2).float()
    return t, a, r, d


@pytest.mark.parametrize("B", [1, 64, 1000, 8192])
@pytest.mark.parametrize("A", [4, 18])
def test_sac_kernels_vs_oracle(lib, B, A):
    from cleanrl_b200 import ops
    (nl, q1t, q2t, q1, q2, lo), a, r, d = _case(B, A, B * 31 + A)
    c = lambda t: t.cuda()      # noqa: E731
    alpha = torch.tensor([0.37], device="cuda")
    st_o, y_o, dq1_o, dq2_o = O.critic_loss(nl.numpy(), q1t.numpy(), q2t.numpy(), q1.numpy(), q2.numpy(), a.numpy(),
                                            r.numpy(), d.numpy(), 0.99, 0.37)
    outs = [ops.sac_critic_loss(c(nl), c(q1t), c(q2t), c(q1), c(q2), c(a), c(r), c(d), 0.99, alpha) for _ in range(2)]
    st, y, dq1, dq2 = [t.cpu().numpy() for t in outs[0]]
    assert np.allclose(st, st_o, rtol=1e-5, atol=1e-5)
    assert np.abs(y - y_o).max() <= 1e-5 * max(1.0, np.abs(y_o).max())
    for g, g_o in ((dq1, dq1_o), (dq2, dq2_o)):
        assert np.abs(g - g_o).max() <= 1e-5 * max(np.abs(g_o).max(), 1e-12)
        off = np.ones_like(g, dtype=bool)
        off[np.arange(B), a.numpy()] = False
        assert (g[off] == 0).all()
    assert all(torch.equal(u, v) for u, v in zip(outs[0], outs[1]))
    # actor loss without and with the temperature step
    o = O.actor_loss(lo.numpy(), q1.numpy(), q2.numpy(), 0.37)
    st, dl = ops.sac_actor_loss(c(lo), c(q1), c(q2), alpha)
    assert abs(st[0].item() - o[0]) <= 1e-5 * max(1.0, abs(o[0])) and st[2].item() == np.float32(0.37)
    assert np.abs(dl.cpu().numpy() - o[1]).max() <= 1e-5 * np.abs(o[1]).max()
    te = O.target_entropy(A)
    runs = []
    for _ in range(2):
        la = torch.tensor([np.log(np.float32(0.37))], dtype=torch.float32, device="cuda")
        al = torch.exp(la)
        m, v = torch.full((1,), 0.01, device="cuda"), torch.full((1,), 1e-4, device="cuda")
        dyn = torch.tensor(ops.adam_step_scalars(3, 3e-4), device="cuda")
        st, dl = ops.sac_actor_loss(c(lo), c(q1), c(q2), al, te, la, m, v, dyn)
        runs.append([t.clone() for t in (st, dl, la, m, v, al)])
    la0 = np.float32(np.log(np.float32(0.37)))
    o = O.actor_loss(lo.numpy(), q1.numpy(), q2.numpy(), np.exp(la0), te, la0, 0.01, 1e-4, step=3)
    st = runs[0][0].cpu().numpy()
    assert abs(st[1] - o[2]) <= 1e-5 * max(1.0, abs(o[2]))
    assert abs(runs[0][2].item() - o[4][0]) <= 1e-7 and abs(st[3] - o[4][0]) <= 1e-7
    assert abs(st[2] - o[5]) <= 1e-6
    assert all(torch.equal(u, w) for u, w in zip(runs[0], runs[1]))


def test_get_action_samples_like_categorical_sample(lib):
    from cleanrl_b200 import ops
    from cleanrl_b200.agents import SACActor
    torch.manual_seed(0)
    actor = SACActor(_Envs(6)).cuda()
    obs = torch.randint(0, 256, (33, 4, 84, 84), dtype=torch.uint8).cuda()
    noise = torch.empty(33, 6, device="cuda").exponential_(1)
    actor.noise_fn = lambda n, A, dev: noise
    act, logp, probs = actor.get_action(obs.float())
    logits = actor(obs.float() / 255.0)
    ref, _, _, _ = ops.categorical_sample(logits, noise)
    assert torch.equal(act, ref)
    lp_o, p_o = O.policy(logits.cpu().numpy())
    assert np.abs(logp.cpu().numpy() - lp_o).max() <= 1e-5 and np.abs(probs.cpu().numpy() - p_o).max() <= 1e-6
    sd = {k: v.detach().cpu().double() for k, v in actor.state_dict().items()}
    x = obs.cpu().double() / 255.0
    for i in (0, 2, 4):
        x = torch.relu(torch.nn.functional.conv2d(x, sd[f"conv.{i}.weight"], sd[f"conv.{i}.bias"], stride=(4, 2, 1)[i // 2]))
    x = torch.relu(x.flatten(1) @ sd["fc1.weight"].t() + sd["fc1.bias"])
    want = x @ sd["fc_logits.weight"].t() + sd["fc_logits.bias"]
    assert (logits.cpu().double() - want).abs().max() <= 1e-4 * max(1.0, want.abs().max().item())


def _nets(A, precision, seed=1):
    from cleanrl_b200.agents import SACActor, SoftQNetwork
    torch.manual_seed(seed)
    nets = [SACActor(_Envs(A)), SoftQNetwork(_Envs(A)), SoftQNetwork(_Envs(A)), SoftQNetwork(_Envs(A)),
            SoftQNetwork(_Envs(A))]
    nets = [n.cuda() for n in nets]
    nets[3].load_state_dict(nets[1].state_dict())
    nets[4].load_state_dict(nets[2].state_dict())
    for n in nets:
        n.precision = precision
        n.flat
    return nets


@pytest.mark.parametrize("autotune", [True, False])
def test_graph_replay_equals_eager_bf16(lib, autotune):
    """Eight bf16 updates with a hard target sync after the fourth: the graph-replayed update and eager launches give the
    same bits in every parameter, Adam moment, the temperature and the statistics."""
    from cleanrl_b200.agents import SACState, dqn_sync_target, sac_update
    from cleanrl_b200.replay import DeviceReplayRing
    dev = torch.device("cuda")
    A, B = 6, 64
    ring = DeviceReplayRing(256, (4, 84, 84), 1, dev, optimize_memory_usage=False)
    g = torch.Generator(device="cuda").manual_seed(2)
    ring.observations.random_(0, 256, generator=g); ring.next_observations.random_(0, 256, generator=g)
    ring.actions.random_(0, A, generator=g); ring.rewards.normal_(generator=g); ring.dones.bernoulli_(0.1, generator=g)
    ring.pos, ring.full = 0, True
    results = []
    for graph in (False, True):
        nets = _nets(A, "bf16")
        st = SACState(A, dev, autotune=autotune, alpha=0.1)
        st.use_graph = graph
        np.random.seed(7)
        trace = []
        for k in range(8):
            sac_update(*nets, ring, ring.sample(B), st, 0.99, 3e-4, 3e-4)
            if k == 3:
                dqn_sync_target(nets[1], nets[3]); dqn_sync_target(nets[2], nets[4])
            trace.append([t.clone() for t in (st.qstats, st.astats, st.alpha, st.log_alpha, st.exp_avg, st.exp_avg_sq)])
        flats = [torch.cat([n.flat.flat, n.flat.exp_avg, n.flat.exp_avg_sq]) for n in nets]
        results.append((trace, flats))
        assert bool(st._graphs) == graph
    (te, fe), (tg, fg) = results
    for a, b in zip(te, tg):
        assert all(torch.equal(u, v) for u, v in zip(a, b))
    assert all(torch.equal(u, v) for u, v in zip(fe, fg))
    assert all(torch.isfinite(f).all() for f in fe)


class _Writer:
    def __init__(self, *a, **k): self.scalars = []
    def add_text(self, *a, **k): pass
    def add_scalar(self, tag, v, step): self.scalars.append((tag, float(np.asarray(v).reshape(-1)[0]), int(step)))
    def close(self): pass


def _sums(net):
    return np.array([p.detach().double().sum().item() for p in net.parameters()])


def _run_script(z, precision, monkeypatch):
    from cleanrl_b200 import agents, sac_atari as S
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    argv = [a for a in z["argv"].tolist() if a != "--no-cuda"] + ["--synthetic-env", "--precision", precision]
    stream, recs, writers = [], [], []
    orig = SyntheticGymnasiumVec.step

    def step(self_, act):
        stream.append(int(np.asarray(act).reshape(-1)[0]))
        return orig(self_, act)
    monkeypatch.setattr(SyntheticGymnasiumVec, "step", step)
    # the reference ran on the CPU: its samples came from torch's CPU generator
    monkeypatch.setattr(agents, "_exp_noise", _cpu_noise)

    def on_update(step_, st, nets):
        recs.append({"q": st.qstats.cpu().numpy().copy(), "a": st.astats.cpu().numpy().copy(),
                     "actor": _sums(nets[0]), "qf1": _sums(nets[1]), "qf2": _sums(nets[2])})

    def wf(p):
        w = _Writer(); writers.append(w); return w

    actor, qf1, _, _ = S.main(argv, writer_factory=wf, on_update=on_update)
    return argv, stream, recs, writers[0], actor, qf1


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)) / np.maximum(1.0, np.abs(np.asarray(b)))


@pytest.mark.parametrize("name", FIXTURES)
def test_sac_script_fp32_vs_reference_run(lib, name, monkeypatch):
    z = np.load(GOLDEN / name)
    autotune = "--no-autotune" not in z["argv"].tolist()
    _, stream, recs, w, actor, qf1 = _run_script(z, "fp32", monkeypatch)
    assert list(actor.state_dict().keys()) == z["actor_keys"].tolist()
    assert list(qf1.state_dict().keys()) == z["qf_keys"].tolist()
    assert len(recs) == len(z["qf1_loss"])
    assert stream == z["action_stream"].tolist()
    cols = [("q", 0, "qf1_values"), ("q", 1, "qf2_values"), ("q", 2, "qf1_loss"), ("q", 3, "qf2_loss"),
            ("a", 0, "actor_loss")] + ([("a", 1, "alpha_loss"), ("a", 3, "log_alpha")] if autotune else [])
    worst = 0.0
    for k, rec in enumerate(recs):
        tol = 1e-5 if k == 0 else LATER_UPDATES_RTOL
        for src, i, key in cols:
            dev_ = _rel(rec[src][i], z[key][k]).max()
            worst = max(worst, dev_ if k else 0.0)
            assert dev_ <= tol, (k, key, rec[src][i], z[key][k])
        if autotune and k + 1 < len(recs):
            assert _rel(rec["a"][2], z["alpha"][k + 1]).max() <= tol
        for net in ("actor", "qf1", "qf2"):
            ref = z[f"{net}_sums"][k]
            assert (np.abs(rec[net] - ref) <= tol * np.maximum(1.0, np.abs(ref))).all(), (k, net)
    print(f"{name}: largest relative deviation of updates 2..{len(recs)} from the reference: {worst:.3g}")
    ref_tags = {k[3:]: z[k] for k in z.files if k.startswith("tb/")}
    got = {}
    for t, v, s in w.scalars:
        got.setdefault(t, []).append((s, v))
    assert set(got) == set(ref_tags)
    for t in ref_tags:
        assert [s for s, _ in got[t]] == ref_tags[t][:, 0].astype(int).tolist(), t


@pytest.mark.parametrize("name", FIXTURES)
def test_sac_script_bf16_vs_reference_run(lib, name, monkeypatch):
    z = np.load(GOLDEN / name)
    _, stream, recs, w, _, _ = _run_script(z, "bf16", monkeypatch)
    assert len(recs) == len(z["qf1_loss"])
    for src, i, key in [("q", 0, "qf1_values"), ("q", 1, "qf2_values"), ("q", 2, "qf1_loss"), ("q", 3, "qf2_loss"),
                        ("a", 0, "actor_loss")]:
        assert _rel(recs[0][src][i], z[key][0]).max() <= 2e-2, key
    assert all(np.isfinite(r["q"]).all() and np.isfinite(r["a"]).all() for r in recs)
    ref_tags = {k[3:]: z[k] for k in z.files if k.startswith("tb/")}
    got = {}
    for t, v, s in w.scalars:
        got.setdefault(t, []).append(s)
    losses = {t for t in ref_tags if t.startswith("losses/") or t == "charts/SPS"}
    assert losses <= set(got)
    for t in losses:
        assert got[t] == ref_tags[t][:, 0].astype(int).tolist(), t
