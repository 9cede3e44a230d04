"""PQN (cleanrl/pqn.py) on the GPU: the LayerNorm Q-network kernels against the fp64 oracle, argmax and epsilon rules,
repeatability, Q(lambda) and clip + RAdam against CPU torch bit for bit, graph replay against eager launches, and the
drop-in against the reference runs."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import pqn_oracle as O

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden"
SHAPES = [(4, 2), (2, 3), (6, 3), (8, 4), (128, 18), (512, 64)]


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from cleanrl_b200 import _lib, build
    build.build()
    return _lib.load()


def _params(d, A, seed=0):
    rng = np.random.default_rng(seed + 1000 * d + A)
    ps = [rng.standard_normal(s) * ((2.0 / s[1]) ** 0.5 if len(s) == 2 else 0.1) for s in O.shapes(d, A)]
    ps[2] += 1.0
    ps[6] += 1.0
    flat = torch.tensor(np.concatenate([p.reshape(-1) for p in ps]), dtype=torch.float32, device="cuda")
    return [p.astype(np.float32).astype(np.float64) for p in ps], flat


def _close(got, want, tol):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = max(1.0, float(np.abs(want).max()))
    assert float(np.abs(got - want).max()) <= tol * scale, float(np.abs(got - want).max()) / scale


@pytest.mark.parametrize("d,A", SHAPES)
@pytest.mark.parametrize("n", [1, 3, 4, 128, 1000, 32768])
def test_forward_and_act_match_the_fp64_oracle(lib, d, A, n):
    from cleanrl_b200 import ops
    ps, flat = _params(d, A)
    rng = np.random.default_rng(n)
    x = torch.tensor(rng.standard_normal((n, d)), dtype=torch.float32, device="cuda")
    q = ops.pqn_forward(flat, x, d, A)
    want = O.forward(ps, x.double().cpu().numpy())
    _close(q.cpu().numpy(), want, 2e-5)
    values = torch.empty(n, device="cuda")
    acts = torch.empty(n, dtype=torch.int64, device="cuda")
    ops.pqn_act(flat, x, d, A, values, actions=acts)
    assert torch.equal(acts, torch.argmax(q, dim=1)) and torch.equal(values, q.max(1).values)
    # epsilon-greedy: u < fl32(eps) takes the random action
    ra = torch.randint(0, A, (n,), device="cuda")
    u = torch.rand(n, device="cuda")
    slot = torch.empty(n, d, device="cuda")
    ops.pqn_act(flat, x, d, A, values, random_actions=ra, u=u, eps=0.3, actions=acts, obs_slot=slot)
    assert torch.equal(acts, torch.where(u < 0.3, ra, torch.argmax(q, dim=1))) and torch.equal(slot, x)


@pytest.mark.parametrize("d,A", SHAPES)
@pytest.mark.parametrize("M", [2, 7, 16, 128, 1000, 32768])
def test_loss_bwd_and_wgrad_match_the_fp64_oracle(lib, d, A, M):
    from cleanrl_b200 import ops
    ps, flat = _params(d, A, seed=1)
    rng = np.random.default_rng(M + d)
    B = M + 5
    obs = torch.tensor(rng.standard_normal((B, d)), dtype=torch.float32, device="cuda")
    acts = torch.tensor(rng.integers(0, A, B), device="cuda")
    R = torch.tensor(rng.standard_normal(B), dtype=torch.float32, device="cuda")
    inds = torch.tensor(rng.permutation(B)[:M], device="cuda")
    ws = ops.pqn_workspace(M, "cuda")
    stats = torch.zeros(2, device="cuda")
    grad = torch.zeros(flat.numel(), device="cuda")
    ops.pqn_loss_bwd(flat, obs, d, A, inds, acts, R, stats, ws)
    ops.pqn_wgrad(obs, d, A, inds, acts, ws, grad)
    i = inds.cpu().numpy()
    loss, qmean, grads = O.loss_and_grads(ps, obs.double().cpu().numpy()[i], acts.cpu().numpy()[i], R.double().cpu().numpy()[i])
    s = stats.cpu().numpy()
    assert abs(s[0] - loss) <= 1e-4 * max(1.0, loss) and abs(s[1] - qmean) <= 1e-4 * max(1.0, abs(qmean))
    got = O.unflatten(grad.cpu().numpy(), d, A)
    for name, g, w in zip(O.PARAM_NAMES, got, grads):
        _close(g, w, 1e-3 if M >= 1000 else 2e-4)
    # bitwise repeatable
    stats2, grad2 = torch.zeros(2, device="cuda"), torch.zeros_like(grad)
    ops.pqn_loss_bwd(flat, obs, d, A, inds, acts, R, stats2, ws)
    ops.pqn_wgrad(obs, d, A, inds, acts, ws, grad2)
    assert torch.equal(stats, stats2) and torch.equal(grad, grad2)


def test_argmax_ties_nan_rows_and_the_epsilon_boundary(lib):
    from cleanrl_b200 import ops
    d, A = 4, 5
    ps, flat = _params(d, A)
    o = [int(np.prod(s)) for s in O.shapes(d, A)]
    w3 = sum(o[:8])
    f = flat.clone()
    f[w3 + 3 * 84:w3 + 4 * 84] = f[w3 + 1 * 84:w3 + 2 * 84]          # head rows 1 and 3 equal, biases equal
    f[w3 + 5 * 84 + 3] = f[w3 + 5 * 84 + 1]
    f[w3 + 1 * 84:w3 + 2 * 84] += 5.0                                    # make action 1 (and its twin 3) the maximum
    f[w3 + 3 * 84:w3 + 4 * 84] += 5.0
    x = torch.rand(64, d, device="cuda")
    x[5, 2] = float("nan")                                               # a NaN row: every Q is NaN
    q = ops.pqn_forward(f, x, d, A)
    values, acts = torch.empty(64, device="cuda"), torch.empty(64, dtype=torch.int64, device="cuda")
    ops.pqn_act(f, x, d, A, values, actions=acts)
    ref = torch.argmax(q.cpu(), dim=1)
    assert torch.equal(acts.cpu(), ref) and int(acts[0]) == 1 and int(acts[5]) == 0
    assert torch.isnan(values[5]) and torch.equal(values[:5].cpu(), q.cpu()[:5, 1])
    g = flat.clone()
    g[w3 + 2 * 84:w3 + 3 * 84] = float("nan")                           # column 2 NaN in every row: argmax is 2
    ops.pqn_act(g, x, d, A, values, actions=acts)
    assert int(acts[5]) == 0 and (acts[torch.arange(64, device="cuda") != 5] == 2).all()
    assert torch.equal(acts.cpu(), torch.argmax(ops.pqn_forward(g, x, d, A).cpu(), dim=1))
    for eps in (0.05, 1 / 3, 0.525):
        e32 = np.float32(eps)
        us = np.array([e32, np.nextafter(e32, np.float32(0)), np.nextafter(e32, np.float32(2))] * 2, np.float32)
        u = torch.tensor(us, device="cuda")
        ra = torch.full((6,), 4, dtype=torch.int64, device="cuda")
        ops.pqn_act(flat, x[:6].clone(), d, A, values[:6], random_actions=ra, u=u, eps=eps, actions=acts[:6])
        greedy = torch.argmax(ops.pqn_forward(flat, x[:6].clone(), d, A), 1)
        assert torch.equal(acts[:6], torch.where(torch.tensor(us) < eps, ra.cpu(), greedy.cpu()).cuda())


def _ref_qlambda(r, v, d, nv, nd, gamma, ql):
    returns = torch.zeros_like(r)
    T = r.shape[0]
    for t in reversed(range(T)):
        if t == T - 1:
            returns[t] = r[t] + gamma * nv * (1.0 - nd)
        else:
            returns[t] = r[t] + gamma * (ql * returns[t + 1] + (1 - ql) * v[t + 1]) * (1.0 - d[t + 1])
    return returns


@pytest.mark.parametrize("T", [1, 16, 128])
@pytest.mark.parametrize("N", [1, 4, 1024])
@pytest.mark.parametrize("ql", [0.0, 0.65, 1.0])
def test_qlambda_is_the_reference_loop_bit_for_bit(lib, T, N, ql):
    from cleanrl_b200 import ops
    g = torch.Generator().manual_seed(T * N)
    r = torch.randn(T, N, generator=g)
    v = torch.randn(T, N, generator=g) * 10
    d = (torch.rand(T, N, generator=g) < 0.1).float()
    nv, nd = torch.randn(N, generator=g), (torch.rand(N, generator=g) < 0.2).float()
    want = _ref_qlambda(r, v, d, nv, nd, 0.99, ql)
    got = ops.qlambda(r.cuda(), v.cuda(), d.cuda(), nv.cuda(), nd.cuda(), 0.99, ql)
    assert torch.equal(got.cpu(), want)


@pytest.mark.parametrize("max_norm", [1e6, 0.5])
def test_clip_radam_matches_torch_radam(lib, max_norm):
    """Steps 1-12 (both sides of rho_t > 5): bit for bit when the clip does not bind; within 1e-6 relative when it binds
    (the kernels fold the squares in double, clip_grad_norm_ in float32)."""
    from cleanrl_b200 import ops
    g = torch.Generator().manual_seed(5)
    P = 11342
    p0 = torch.randn(P, generator=g)
    t = torch.nn.Parameter(p0.clone())
    opt = torch.optim.RAdam([t], lr=2.5e-4, foreach=False)
    p, m, v = p0.cuda(), torch.zeros(P, device="cuda"), torch.zeros(P, device="cuda")
    p2, m2, v2 = p.clone(), m.clone(), v.clone()
    table = torch.zeros(4, device="cuda")
    for step in range(1, 13):
        grad = torch.randn(P, generator=g) * 0.1
        t.grad = grad.clone()
        torch.nn.utils.clip_grad_norm_([t], max_norm)
        opt.step()
        ops.clip_radam(p, grad.cuda(), m, v, step, 2.5e-4, max_norm=max_norm)
        table.copy_(torch.tensor(ops.radam_step_scalars(step, 2.5e-4)))
        ops.clip_radam_dyn(p2, grad.cuda(), m2, v2, table, max_norm=max_norm)
        assert torch.equal(p, p2) and torch.equal(m, m2) and torch.equal(v, v2), step
        if max_norm > 1e5:
            st = opt.state[t]
            assert torch.equal(m.cpu(), st["exp_avg"]) and torch.equal(v.cpu(), st["exp_avg_sq"]), step
            assert torch.equal(p.cpu(), t.detach()), step
        else:
            _close(p.cpu().numpy(), t.detach().numpy(), 1e-6)


def _engine(name, use_graph=True):
    from cleanrl_b200 import cli
    from cleanrl_b200.agents import PQNQNetwork
    from cleanrl_b200.pqn_engine import PQNEngine
    from cleanrl_b200.synthetic_envs import CartPoleVec
    z = np.load(GOLDEN / name)
    args = cli.parse(cli.pqn_args(), [str(a) for a in z["argv"] if a != "--no-cuda"])
    net = PQNQNetwork(CartPoleVec(args.num_envs))
    with torch.no_grad():
        for p, w in zip(net.parameters(), O.unflatten(z["init_flat"], 4, 2)):
            p.copy_(torch.as_tensor(w))
    net = net.cuda()
    eng = PQNEngine(net, args, args.num_envs, torch.device("cuda"))
    eng.use_graph = use_graph
    eng.obs.copy_(torch.as_tensor(z["it_obs"][0]).reshape(-1, 4))
    eng.actions.copy_(torch.as_tensor(z["it_actions"][0]).reshape(-1).long())
    eng.returns.copy_(torch.as_tensor(z["it_returns"][0]))
    return z, args, eng


@pytest.mark.parametrize("name", ["pqn_seed1.npz", "pqn_seed2_mb.npz"])
def test_update_replays_the_reference_first_iteration(lib, name):
    """Fed iteration 1's recorded rollout and the initial parameters, with numpy's generator seeded as the script
    seeds it: every RAdam step's loss, mean q and parameter sums (the first to 1e-5, later ones within 1e-2)."""
    from cleanrl_b200 import ops
    z, args, eng = _engine(name, use_graph=False)
    np.random.seed(args.seed)
    lr = float(z["lr"][0])
    E, nmb = eng.epochs, eng.nmb
    for k in range(E * nmb):
        eng.host_table[k] = torch.tensor(ops.radam_step_scalars(k + 1, lr))
    eng.table.copy_(eng.host_table)
    b_inds = np.arange(eng.B)
    for e in range(E):
        ops.numpy_global_shuffle(b_inds)
        eng.inds[e].copy_(torch.as_tensor(b_inds))
        for i in range(nmb):
            k = e * nmb + i
            assert np.array_equal(b_inds[eng.starts[i]:eng.starts[i] + z["mb_len"][k]], z["mb_inds"][k][:z["mb_len"][k]])
            eng._minibatch(e, i)
            s = eng.stats.cpu().numpy()
            sums = [float(p.double().sum()) for p in eng.q.parameters()]
            tol = 1e-5 if k == 0 else 1e-2
            assert abs(s[0] - z["loss"][k]) <= tol * max(1.0, abs(z["loss"][k])), k
            assert abs(s[1] - z["qmean"][k]) <= tol * max(1.0, abs(z["qmean"][k])), k
            np.testing.assert_allclose(sums, z["param_sums"][k], rtol=tol, atol=tol)


def test_graph_replay_is_eager_bit_for_bit_with_four_launches_per_minibatch(lib):
    from cleanrl_b200 import _lib
    out = []
    for graph in (False, True):
        z, args, eng = _engine("pqn_seed2_mb.npz", use_graph=graph)
        np.random.seed(3)
        for it in range(3):
            l0 = _lib.load().b200rl_launch_count()
            eng.update(1e-3 / (it + 1))
            n = _lib.load().b200rl_launch_count() - l0
            if not graph:
                assert n == 4 * eng.epochs * eng.nmb
        out.append((eng.flat.flat.clone(), eng.flat.exp_avg.clone(), eng.stats.clone()))
    assert all(torch.equal(a, b) for a, b in zip(*out))


class _Writer:
    def __init__(self, *a, **k):
        self.scalars = []

    def add_text(self, *a, **k):
        pass

    def add_scalar(self, tag, value, step=None):
        self.scalars.append((tag, float(np.asarray(value).reshape(-1)[0]), int(step)))

    def close(self):
        pass


@pytest.mark.parametrize("name", ["pqn_seed1.npz", "pqn_seed2_mb.npz"])
def test_drop_in_reproduces_the_reference_runs(lib, name):
    """pqn.main on CartPoleVec: the action stream exactly, values and returns (1e-5 in iteration 1, 1e-2 after), and
    every logged tag and step."""
    from cleanrl_b200 import pqn
    from cleanrl_b200.synthetic_envs import CartPoleVec
    z = np.load(GOLDEN / name)
    writers, seen = [], []

    def wf(*a, **k):
        writers.append(_Writer())
        return writers[-1]

    def on_it(it, eng, st):
        seen.append({k: getattr(eng, k).cpu().numpy().copy() for k in ("actions", "values", "returns")})

    pqn.main([str(a) for a in z["argv"] if a != "--no-cuda"], writer_factory=wf,
             env_factory=lambda a: CartPoleVec(a.num_envs), on_iteration=on_it)
    assert len(seen) == z["it_actions"].shape[0]
    for i, s in enumerate(seen):
        assert np.array_equal(s["actions"].reshape(z["it_actions"][i].shape), z["it_actions"][i].astype(np.int64)), i
        tol = 1e-5 if i == 0 else 1e-2
        np.testing.assert_allclose(s["values"], z["it_values"][i], rtol=tol, atol=tol)
        np.testing.assert_allclose(s["returns"], z["it_returns"][i], rtol=tol, atol=tol)
    w = writers[0].scalars
    for key in [k for k in z.files if k.startswith("tb/")]:
        tag = key[3:]
        mine = [(s, v) for t, v, s in w if t == tag]
        ref = z[key]
        assert [s for s, _ in mine] == [int(s) for s in ref[:, 0]], tag
        if tag != "charts/SPS":
            np.testing.assert_allclose([v for _, v in mine], ref[:, 1], rtol=1e-2, atol=1e-2)
    assert {t for t, _, _ in w} == {k[3:] for k in z.files if k.startswith("tb/")}


def test_drop_in_learns_cartpole(lib):
    """Seed 1 on CartPoleVec with the schedules of a 300 k-step run (epsilon reaches end_e at 150 k): the episodes that
    end in (175 k, 200 k] average >= 300.  The unmodified reference on the CPU gives 451 there (seeds 2 / 3: 481 / 455)
    and 184 in (75 k, 100 k]."""
    from cleanrl_b200 import pqn
    from cleanrl_b200.synthetic_envs import CartPoleVec
    ws = []

    def wf(*a, **k):
        ws.append(_Writer())
        return ws[-1]

    pqn.main(["--seed", "1", "--total-timesteps", "300000"], writer_factory=wf, env_factory=lambda a: CartPoleVec(a.num_envs))
    rets = [v for t, v, s in ws[0].scalars if t == "charts/episodic_return" and 175_000 < s <= 200_000]
    print(f"PQN CartPole: {len(rets)} episodes in (175k, 200k], mean return {np.mean(rets):.1f}")
    assert len(rets) > 0 and np.mean(rets) >= 300
