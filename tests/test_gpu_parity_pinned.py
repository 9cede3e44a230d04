"""-m gpu: the BENCHMARKED path (bf16 tensor cores, scan GAE, sorted minibatches, CUDA graphs) and the exact fp32 path,
pinned to the reference at the benchmarked size and update by update.

1. ``test_full_size_fixture_*``: cleanrl_b200/ppo_atari_envpool.py at BASELINE.json configs[1] (num_envs=1024,
   num_steps=128, minibatch 32 768) against tests/golden/ppo_atari_envpool_n1024_t128_seed1.npz, which the UNMODIFIED
   cleanrl/ppo_atari_envpool.py produced on CPU (oracle/make_golden.py ppo_atari_full).
2. ``test_bf16_script_vs_reference_fixtures``: the tensor-core path against every Atari fixture, tolerances stated.
3. ``test_updates_step_by_step_on_identical_inputs``: every one of the 16 minibatch updates of an iteration is
   replayed through PPOEngine.minibatch_update from the oracle's own pre-step parameters, Adam state and minibatch
   rows (the oracle port, itself pinned to the unmodified reference by the fixtures), so losses, gradients and the
   Adam step of updates 2..16 are compared on IDENTICAL inputs -- no chaotic drift to hide behind.
"""
import numpy as np
import pytest
import torch

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

FULL = "ppo_atari_envpool_n1024_t128_seed1.npz"
ATARI = ["ppo_atari_envpool_n8_t32_seed1.npz", "ppo_atari_envpool_n16_t16_seed3_noclipv.npz",
         "ppo_atari_gym_n8_t32_seed2.npz", "ppo_atari_envpool_n8_t16_seed5_flags.npz"]


class _Writer:
    def __init__(self, *a, **k):
        self.scalars = []
    def add_text(self, *a, **k): pass
    def add_scalar(self, tag, v, step): self.scalars.append((tag, float(v), int(step)))
    def close(self): pass


def _cpu_noise(n, A, device):
    return torch.empty(n, A, dtype=torch.float32).exponential_(1).to(device)


def _run(name, extra=()):
    import importlib
    S = importlib.import_module("cleanrl_b200.ppo_atari" if name.startswith("ppo_atari_gym") else
                                "cleanrl_b200.ppo_atari_envpool")
    from cleanrl_b200.agents import NatureCNNAgent
    z = np.load(GOLDEN / name)
    argv = [a for a in z["argv"].tolist() if a != "--no-cuda"] + list(extra) + ["--synthetic-env"]
    snaps, writers, engines = [], [], []

    def on_it(it, eng, st):
        engines.append(eng)
        snaps.append({k: getattr(eng, k).cpu().numpy().copy() for k in
                      ("actions", "logprobs", "values", "rewards", "dones", "advantages", "returns")} | {"st": st})

    orig = NatureCNNAgent.__init__

    def patched(self, envs):
        orig(self, envs)
        self.noise_fn = _cpu_noise          # the CPU reference run drew its noise from torch's CPU generator
    NatureCNNAgent.__init__ = patched
    try:
        def wf(path):
            w = _Writer(); writers.append(w); return w
        S.main(argv, writer_factory=wf, on_iteration=on_it)
    finally:
        NatureCNNAgent.__init__ = orig
    return z, snaps, writers[0], engines[0]


def _ref(z, k):
    """Array `k` of a fixture; the full-size fixture stores no returns: the reference computed them as advantages + values
    (float32), which reproduces them bit for bit."""
    if k == "returns" and k not in z:
        return (z["advantages"] + z["values"]).astype(np.float32)
    return z[k]


def _rel(a, b, where=None):
    d = np.abs(a.astype(np.float64) - b.astype(np.float64))
    if where is not None:
        d = d[where]
    return (d.max() if d.size else 0.0) / max(1.0, np.abs(b).max())


def _common_prefix(ours, ref):
    """[T, N] mask of the steps at which an env has received the reference's actions at EVERY earlier step (the
    synthetic env's next frame depends on the action, so one flipped action changes that env's later observations;
    rows after the first flip of an env are different inputs, not a numerics question), and the mask of steps whose
    own action also agrees."""
    same = ours == ref
    before = np.ones_like(same)
    before[1:] = np.cumprod(same, axis=0)[:-1].astype(bool)
    return before, before & same


COLS = ((0, "upd_pg_loss"), (1, "upd_v_loss"), (2, "upd_entropy_loss"), (3, "upd_old_approx_kl"), (4, "upd_approx_kl"),
        (6, "upd_loss"))


def test_full_size_fixture_fp32(lib):
    """Exact path at the headline size: 131 072 sampled actions bit-identical to the unmodified reference's,
    logprobs / values / advantages / returns <= 1e-5, the first update's losses <= 1e-5 (identical inputs), the
    other 15 updates of the iteration <= 1e-4 (each starts from parameters that already carry rounding-level
    differences; test 3 checks those updates on identical inputs)."""
    z, snaps, w, eng = _run(FULL, ["--gae-kernel", "sequential"])
    s = snaps[0]
    assert np.array_equal(s["actions"], z["actions"][0].astype(np.int64)), "actions differ at N=1024,T=128"
    assert np.array_equal(s["rewards"], z["rewards"][0].astype(np.float32))
    assert np.array_equal(s["dones"], z["dones"][0].astype(np.float32))
    for k in ("logprobs", "values", "advantages", "returns"):
        assert _rel(s[k], _ref(z, k)[0]) <= 1e-5, (k, _rel(s[k], _ref(z, k)[0]))
    per = s["st"]["per_update"]
    assert per.shape[0] == 16
    M = 32768
    worst = 0.0
    for u in range(16):
        for col, key in COLS:
            ref = float(z[key][u])
            err = abs(per[u, col] - ref) / max(1.0, abs(ref))
            worst = max(worst, err)
            assert err <= (1e-5 if u == 0 else 1e-4), (u, key, per[u, col], ref)
        assert abs(per[u, 5] - float(z["upd_clipfrac"][u])) <= (1.01 / M if u == 0 else 2e-3), (u, per[u, 5])
    print(f"full-size fp32: worst loss deviation over 16 updates {worst:.2e}")


def test_full_size_fixture_bf16_benchmarked_path(lib):
    """The path bench.py times (--precision bf16 --gae-kernel scan, sorted minibatches, per-slot CUDA graphs) at the
    headline size against the unmodified reference.  bf16 tolerances: sampled actions agree on >= 99.5 % of the
    131 072 samples (same noise; a flip needs two logits within the bf16 error of each other), logprobs / values /
    advantages / returns <= 2e-2 of the tensor's scale, first-update losses <= 1e-2, all 16 updates <= 3e-2."""
    z, snaps, w, eng = _run(FULL, ["--precision", "bf16", "--gae-kernel", "scan"])
    assert eng.s2d and eng.sort_minibatch and len(eng._graphs) > 0, "not the benchmarked configuration"
    s = snaps[0]
    ref_a = z["actions"][0].astype(np.int64)
    agree = (s["actions"] == ref_a).mean()
    assert agree >= 0.995, agree
    same_obs, same = _common_prefix(s["actions"], ref_a)     # steps whose observation is the reference's
    flips = int((same_obs & ~same).sum())
    assert flips <= 1024 * 0.05, flips                        # envs that ever left the reference trajectory
    assert _rel(s["values"], z["values"][0], same_obs) <= 2e-2
    assert np.abs(s["logprobs"] - z["logprobs"][0])[same].max() <= 2e-2
    # GAE mixes later steps of the env: compare it on envs that followed the reference trajectory to the end
    whole = same.all(axis=0)
    assert whole.mean() >= 0.9, whole.mean()
    for k in ("advantages", "returns"):
        assert _rel(s[k][:, whole], _ref(z, k)[0][:, whole]) <= 2e-2, (k, _rel(s[k][:, whole], _ref(z, k)[0][:, whole]))
    per = s["st"]["per_update"]
    for u in range(16):
        for col, key in COLS:
            ref = float(z[key][u])
            assert abs(per[u, col] - ref) <= (1e-2 if u == 0 else 3e-2) * max(1.0, abs(ref)), (u, key, per[u, col], ref)
    print(f"full-size bf16: action agreement {agree:.5f}, first flips {flips}, values {_rel(s['values'], z['values'][0], same_obs):.2e}")


@pytest.mark.parametrize("name", ATARI)
def test_bf16_script_vs_reference_fixtures(lib, name):
    """Every Atari fixture through the tensor-core path (scan GAE, sorted minibatches, graphs).  Iteration 1 (identical
    weights): action agreement >= 99 %, logprob / value <= 2e-2, update-1 losses <= 1e-2, the iteration's other
    updates <= 5e-2; later iterations: finite, same number of updates (incl. target-kl early stops within one
    epoch), action agreement >= 50 %."""
    z, snaps, w, eng = _run(name, ["--precision", "bf16", "--gae-kernel", "scan"])
    n_it = z["actions"].shape[0]
    assert len(snaps) == n_it
    upd = 0
    for it in range(n_it):
        s = snaps[it]
        ref_a = z["actions"][it].astype(np.int64)
        agree = (s["actions"] == ref_a).mean()
        per = s["st"]["per_update"]
        assert np.isfinite(per[:, :7]).all()
        if it == 0:
            assert agree >= 0.99, agree
            same_obs, same = _common_prefix(s["actions"], ref_a)
            assert np.abs(s["logprobs"] - z["logprobs"][it])[same].max() <= 2e-2
            assert _rel(s["values"], z["values"][it], same_obs) <= 2e-2
            for u in range(per.shape[0]):
                for col, key in COLS:
                    ref = float(z[key][upd + u])
                    assert abs(per[u, col] - ref) <= (1e-2 if u == 0 else 5e-2) * max(1.0, abs(ref)), (u, key, per[u, col], ref)
        else:
            assert agree >= 0.5, (it, agree)
        upd += per.shape[0]
    if "target-kl" not in " ".join(z["argv"].tolist()):
        assert upd == len(z["upd_loss"])


# ------------------------------------------------------------------ updates 1..16 on identical inputs
def _oracle_iteration(N, T, seed):
    """One PPO iteration of the oracle port on CPU with a snapshot of everything each update consumes."""
    from oracle import ppo_port
    snaps, roll = [], {}

    def hook(c):
        if not roll:
            for k in ("obs", "actions", "logprobs", "advantages", "returns", "values"):
                roll[k] = c[k].detach().clone()
        st = c["opt"].state
        ps = list(c["agent"].parameters())
        snaps.append(dict(
            params=[p.detach().clone() for p in ps], grads=[p.grad.detach().clone() for p in ps],
            exp_avg=[st[p]["exp_avg"].clone() if p in st and "exp_avg" in st[p] else torch.zeros_like(p) for p in ps],
            exp_avg_sq=[st[p]["exp_avg_sq"].clone() if p in st and "exp_avg_sq" in st[p] else torch.zeros_like(p) for p in ps],
            mb=np.array(c["mb"]).copy(), losses=dict(c["losses"]), lr=c["lr"]))

    state = np.random.get_state()
    try:
        out = ppo_port.run(num_envs=N, num_steps=T, num_iterations=1, total_iterations=3, seed=seed, threads=8, on_update=hook)
    finally:
        np.random.set_state(state)
    return snaps, roll, out


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_updates_step_by_step_on_identical_inputs(lib, precision):
    from bench import ppo_args
    from cleanrl_b200.agents import NatureCNNAgent
    from cleanrl_b200.ppo_engine import PPOEngine
    from cleanrl_b200.synthetic_envs import SyntheticAtariVec
    from oracle import ppo_port
    N, T, seed = 8, 32, 1
    snaps, roll, out = _oracle_iteration(N, T, seed)
    assert len(snaps) == 16
    # the oracle port itself is pinned to the unmodified reference: same first-update losses as the committed fixture
    z = np.load(GOLDEN / "ppo_atari_envpool_n8_t32_seed1.npz")
    for key, name in (("upd_pg_loss", "pg_loss"), ("upd_v_loss", "v_loss"), ("upd_loss", "loss")):
        for u in range(16):
            assert abs(snaps[u]["losses"][name] - float(z[key][u])) <= 1e-4 * max(1.0, abs(float(z[key][u]))), (key, u)
    # the final parameters of the oracle run = what the 16th Adam step produced
    dev = torch.device("cuda")
    envs = SyntheticAtariVec(N, seed=seed, mode="fresh")
    envs.single_observation_space, envs.single_action_space = envs.observation_space, envs.action_space
    agent = NatureCNNAgent(envs).to(dev)
    agent.precision = precision
    args = ppo_args(N, T, 3, precision)
    eng = PPOEngine(agent, args, (4, 84, 84), np.uint8, N, dev, gae_mode=0)
    for t in range(T):
        eng._upload_obs(t, roll["obs"][t].to(torch.uint8).numpy())
    eng.actions.copy_(roll["actions"].long())
    for k in ("logprobs", "advantages", "returns", "values"):
        getattr(eng, k).copy_(roll[k])
    flat = agent.flat
    ours = list(agent.parameters())                  # module order == the oracle agent's order
    off = [(p.data_ptr() - flat.flat.data_ptr()) // 4 for p in ours]
    B, M = N * T, N * T // 4
    # bf16 gradients vs the TRUE fp32 oracle (no operand-rounding emulation): a ReLU whose pre-activation is within the
    # bf16 error of zero flips its mask; a fraction f of flipped units moves a gradient by ~sqrt(f) in relative L2
    # (measured 2-12 % per tensor over the 16 updates, largest for conv1 whose gradient sees every mask downstream;
    # tests/test_gpu_network_bf16.py checks the same kernels at <= 1.5 % with the operand rounding emulated in the
    # reference).  The direction is pinned separately: cosine similarity >= 0.99 per tensor.
    ltol, gtol = (1e-5, 1e-5) if precision == "fp32" else (1e-2, 0.15)
    worst_l = worst_g = worst_p = 0.0
    for u, sn in enumerate(snaps):
        with torch.no_grad():
            for p, q, o, m, v in zip(ours, sn["params"], off, sn["exp_avg"], sn["exp_avg_sq"]):
                p.data.copy_(q)
                flat.exp_avg[o:o + q.numel()].copy_(m.reshape(-1))
                flat.exp_avg_sq[o:o + q.numel()].copy_(v.reshape(-1))
        agent.params_updated()
        flat.step = u
        mb = torch.from_numpy(sn["mb"]).to(dev)
        if eng.s2d and eng.sort_minibatch:
            mb = torch.sort(mb).values
        # (a) forward + loss + backward on the oracle's parameters and rows: losses and PRE-clip gradients
        aux = dict(aux=eng.obs_t.view(B, 64, 448)) if eng.u8_rollout else {}
        pol, val = agent.forward_train(eng.obs.view((B,) + tuple(eng.obs.shape[2:])), mb, **aux)
        b = {"actions": eng.actions.view(B), "logprobs": eng.logprobs.view(B), "advantages": eng.advantages.view(B),
             "returns": eng.returns.view(B), "values": eng.values.view(B)}
        stats = torch.zeros(16, device=dev)
        agent.loss_backward(pol, val, mb, b, args, stats, {})
        st = stats.cpu().numpy()
        for col, name in ((0, "pg_loss"), (1, "v_loss"), (2, "entropy"), (3, "old_approx_kl"), (4, "approx_kl"), (6, "loss")):
            ref = sn["losses"][name]
            err = abs(st[col] - ref) / max(1.0, abs(ref))
            worst_l = max(worst_l, err)
            assert err <= ltol, (u, name, st[col], ref)
        assert abs(st[5] - sn["losses"]["clipfrac"]) <= 1.01 / M + (0 if precision == "fp32" else 2.0 / M)
        for p, o, g in zip(ours, off, sn["grads"]):
            got = flat.grad[o:o + g.numel()].cpu().view(g.shape)
            if precision == "fp32":
                err = float((got - g).abs().max() / g.abs().max().clamp_min(1e-30))
            else:
                err = float((got - g).norm() / g.norm().clamp_min(1e-30))
            worst_g = max(worst_g, err)
            assert err <= gtol, (u, tuple(g.shape), err)
        # (b) the engine's own update (same forward/backward + clip + Adam) from the same state: parameters after
        flat.step = u
        eng.minibatch_update(mb, sn["lr"], k=u)
        nxt = snaps[u + 1]["params"] if u + 1 < len(snaps) else None
        if nxt is not None:
            for p, q in zip(ours, nxt):
                err = float((p.data.cpu() - q).abs().max())
                worst_p = max(worst_p, err)
                # fp32: rounding-level agreement of the Adam step.  bf16: an Adam step moves a parameter by at most
                # lr (early steps are sign-like, g / (|g| + eps)); a near-zero gradient whose sign differs at bf16
                # precision lands on the other side: <= 2 lr
                assert err <= (2e-6 if precision == "fp32" else 2 * sn["lr"] * 1.01), (u, tuple(q.shape), err)
    print(f"[{precision}] 16 updates on identical inputs: worst loss dev {worst_l:.2e}, gradient dev {worst_g:.2e}, "
          f"post-step parameter dev {worst_p:.2e}")


def test_workspaces_survive_many_batch_shapes_with_graphs(lib):
    """Captured step graphs bake raw pointers of the activation workspaces; touching many other batch shapes afterwards
    (evaluation batches, other minibatch sizes) must not free or move them: graph replays stay bit-identical."""
    from bench import ppo_args
    from cleanrl_b200.agents import NatureCNNAgent
    from cleanrl_b200.ppo_engine import PPOEngine
    from cleanrl_b200.synthetic_envs import SyntheticAtariVec
    dev = torch.device("cuda")
    N, T = 32, 3
    envs = SyntheticAtariVec(N, seed=3, mode="fresh")
    envs.single_observation_space, envs.single_action_space = envs.observation_space, envs.action_space
    torch.manual_seed(3)
    agent = NatureCNNAgent(envs).to(dev); agent.precision = "bf16"
    eng = PPOEngine(agent, ppo_args(N, T, 4, "bf16"), (4, 84, 84), np.uint8, N, dev)
    g = torch.Generator().manual_seed(5)
    frames = torch.randint(0, 256, (T, N, 4, 84, 84), dtype=torch.uint8, generator=g)
    done = np.zeros(N, dtype=np.float32)

    def rollout():
        torch.manual_seed(11)
        for t in range(T):
            eng.policy_step(t, frames[t].numpy(), done)
        torch.cuda.synchronize()
        return eng.actions.clone(), eng.logprobs.clone(), eng.values.clone()

    first = rollout()                        # captures one graph per slot
    assert len(eng._graphs) == T
    keys_before = {k: v.data_ptr() for k, v in agent._tc._acts.items()}
    for n in (1, 2, 3, 5, 7, 9, 11, 13):     # eight more shapes: far past the LRU capacity of unpinned workspaces
        x = torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8, generator=g).to(dev)
        agent.get_action_and_value(x)
    for k, ptr in keys_before.items():
        assert agent._tc._acts[k].data_ptr() == ptr, "a workspace referenced by a captured graph was evicted"
    again = rollout()                        # pure graph replays
    for a, b in zip(first, again):
        assert torch.equal(a, b)
