"""-m gpu: the mean-shifted Gaussian PPO loss (b200rl_ppo_loss_gaussian_shift_f32) against the unshifted kernel and the
oracle, its launches, and cleanrl_b200/rpo_continuous_action.py against the unmodified reference runs
(tests/golden/rpo_continuous_*.npz, HalfCheetah-shaped synthetic env: obs 17, act 6)."""
import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import rpo_continuous_oracle as R

pytestmark = pytest.mark.gpu
TOL = 1e-5
SHAPES = [(32768, 6, 131072), (128, 6, 512), (2, 1, 4), (1000, 17, 3000), (33, 32, 100)]
FLAGS = [(True, True), (False, False)]


def _case(M, D, B):
    g = torch.Generator().manual_seed(M + D)
    mean = torch.randn(M, D, generator=g)
    z = torch.empty(M, D).uniform_(-0.5, 0.5, generator=g)
    logstd = torch.randn(D, generator=g) * 0.2
    nv = torch.randn(M, generator=g)
    b_act = torch.randn(B, D, generator=g)
    b_lp = torch.randn(B, generator=g) * 0.2 - 1.4 * D
    b_adv = torch.randn(B, generator=g); b_ret = torch.randn(B, generator=g); b_val = b_ret + 0.3 * torch.randn(B, generator=g)
    inds = torch.randperm(B, generator=g)[:M]
    return mean, z, logstd, nv, inds, b_act, b_lp, b_adv, b_ret, b_val


def _loss(c, norm_adv, clip_vloss, mean=None, shift=None):
    from cleanrl_b200 import ops
    m, z, logstd, nv, inds, b_act, b_lp, b_adv, b_ret, b_val = [t.cuda() for t in c]
    out = ops.ppo_loss_gaussian(m if mean is None else mean, logstd, nv, inds, b_act, b_lp, b_adv, b_ret, b_val, 0.2, 0.01,
                                0.5, norm_adv, clip_vloss, mean_shift=shift)
    return [t.cpu() for t in out]


@pytest.mark.parametrize("M,D,B", SHAPES)
@pytest.mark.parametrize("norm_adv,clip_vloss", FLAGS)
def test_shift_is_bit_identical_to_the_unshifted_kernel_on_the_shifted_mean(lib, M, D, B, norm_adv, clip_vloss):
    c = _case(M, D, B)
    mean, z = c[0].cuda(), c[1].cuda()
    shifted = _loss(c, norm_adv, clip_vloss, mean=mean, shift=z)
    plain = _loss(c, norm_adv, clip_vloss, mean=mean + z)          # torch's fp32 add, as the reference's mean + z
    for a, b, name in zip(shifted, plain, ("stats", "dmean", "dlogstd", "dvalue")):
        assert torch.equal(a, b), name
    zero = _loss(c, norm_adv, clip_vloss, mean=mean, shift=torch.zeros_like(z))
    unshifted = _loss(c, norm_adv, clip_vloss, mean=mean)
    for a, b, name in zip(zero, unshifted, ("stats", "dmean", "dlogstd", "dvalue")):
        assert torch.equal(a, b), name


@pytest.mark.parametrize("M,D,B", SHAPES)
@pytest.mark.parametrize("norm_adv,clip_vloss", FLAGS)
def test_shift_vs_oracle(lib, M, D, B, norm_adv, clip_vloss):
    from cleanrl_b200 import ops
    c = _case(M, D, B)
    mean, z, logstd, nv, inds, b_act, b_lp, b_adv, b_ret, b_val = [t.numpy() for t in c]
    st_o, dm_o, dls_o, dv_o = R.ppo_loss_gaussian_shift(mean, z, logstd, nv, inds, b_act, b_lp, b_adv, b_ret, b_val, 0.2,
                                                        0.01, 0.5, norm_adv, clip_vloss)
    # a strided shift: rows of a wider buffer (ld_shift > D)
    wide = torch.zeros(M, D + 3, device="cuda")
    wide[:, 1:D + 1] = c[1].cuda()
    st, dm, dls, dv = _loss(c, norm_adv, clip_vloss, shift=wide[:, 1:D + 1])
    st = st.numpy()
    for i, k in enumerate(ops.STAT_NAMES):
        assert abs(st[i] - float(st_o[k])) <= 3 * TOL * max(1.0, abs(float(st_o[k]))), (k, st[i], st_o[k])
    assert np.abs(dm.numpy() - dm_o).max() <= 1e-4 * np.abs(dm_o).max() + 1e-12
    assert np.abs(dls.numpy() - dls_o).max() <= 1e-4 * max(1.0, np.abs(dls_o).max())
    assert np.abs(dv.numpy() - dv_o).max() <= TOL * np.abs(dv_o).max() + 1e-12


def test_shift_refuses_null_and_narrow_shifts_without_launching(lib):
    from cleanrl_b200 import ops
    M, D = 64, 6
    c = [t.cuda() for t in _case(M, D, 256)]
    mean, z, logstd, nv, inds, b_act, b_lp, b_adv, b_ret, b_val = c
    dmean, dls, dv, stats = (torch.empty(M, D, device="cuda"), torch.empty(D, device="cuda"),
                             torch.empty(M, device="cuda"), torch.zeros(16, device="cuda"))
    ws = torch.empty(lib.b200rl_ppo_loss_gaussian_workspace_bytes(M), dtype=torch.uint8, device="cuda")
    p = lambda t: t.data_ptr()
    for shift, ld in ((None, D), (p(z), D - 1)):
        before = lib.b200rl_launch_count()
        rc = lib.b200rl_ppo_loss_gaussian_shift_f32(
            p(mean), D, p(logstd), p(nv), 1, p(inds), p(b_act), p(b_lp), p(b_adv), p(b_ret), p(b_val), shift, ld, M, D,
            0.2, 0.01, 0.5, 1, 1, p(dmean), D, p(dls), p(dv), 1, p(stats), p(ws), ws.numel(), None)
        assert rc == -1 and "ppo_loss_gaussian_shift" in lib.b200rl_last_error().decode()
        assert lib.b200rl_launch_count() == before
    with pytest.raises(ValueError, match="mean_shift"):
        ops.ppo_loss_gaussian(mean, logstd, nv, inds, b_act, b_lp, b_adv, b_ret, b_val, 0.2, 0.01, 0.5,
                              mean_shift=z[:, :D - 1])


class _Args:
    num_steps, num_minibatches, update_epochs = 64, 4, 3
    gamma, gae_lambda, clip_coef, ent_coef, vf_coef, max_grad_norm = 0.99, 0.95, 0.2, 0.0, 0.5, 0.5
    norm_adv, clip_vloss, target_kl = True, True, None


def _engine(agent_cls, *extra):
    from cleanrl_b200.ppo_engine import PPOEngine
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    env = SyntheticGymnasiumVec(4, kind="continuous")
    torch.manual_seed(3)
    agent = agent_cls(env, *extra).cuda()
    eng = PPOEngine(agent, _Args, env.single_observation_space.shape, np.float32, 4, torch.device("cuda"))
    g = torch.Generator(device="cuda").manual_seed(5)
    for t in (eng.actions, eng.logprobs, eng.values, eng.advantages, eng.returns):
        t.copy_(torch.randn(t.shape, generator=g, device="cuda"))
    eng.obs.copy_(torch.randn(eng.obs.shape, generator=g, device="cuda"))
    return agent, eng


def test_rpo_update_makes_the_launches_of_a_ppo_update_and_one_upload_per_epoch(lib):
    from cleanrl_b200.agents import ContinuousMLPAgent, RPOAgent
    counts = {}
    for name, cls, extra in (("ppo", ContinuousMLPAgent, ()), ("rpo", RPOAgent, (0.5,))):
        agent, eng = _engine(cls, *extra)
        calls = []
        if name == "rpo":
            orig = agent.begin_update_epoch
            agent.begin_update_epoch = lambda *a: (calls.append(a), orig(*a))
        eng.update(1e-4)                       # first update allocates workspaces
        calls.clear()
        l0 = lib.b200rl_launch_count()
        st = eng.update(1e-4)
        torch.cuda.synchronize()
        counts[name] = (lib.b200rl_launch_count() - l0, st["num_updates"])
        if name == "rpo":
            B = eng.B
            assert calls == [(e, _Args.update_epochs, B) for e in range(_Args.update_epochs)]
            assert tuple(agent._z_h.shape) == (_Args.update_epochs, B, 6) and agent._z_h.is_pinned()
            assert tuple(agent._z.shape) == (B, 6) and agent._z.is_cuda
            assert torch.equal(agent._z.cpu(), agent._z_h[-1])          # the last epoch's draws are on the device
            assert np.isfinite(st["loss"])
    assert counts["rpo"] == counts["ppo"], counts
    assert counts["rpo"][1] == _Args.update_epochs * _Args.num_minibatches


def test_get_action_and_value_matches_the_reference_agent(lib):
    from torch.distributions.normal import Normal
    from cleanrl_b200.agents import RPOAgent
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    env = SyntheticGymnasiumVec(4, kind="continuous")
    torch.manual_seed(7)
    ref = RPOAgent(env, 0.5)                    # CPU copy of the same weights, evaluated with torch as the reference
    with torch.no_grad():
        ref.actor_logstd.add_(torch.randn(1, 6) * 0.2)
    agent = RPOAgent(env, 0.5).cuda()
    agent.load_state_dict(ref.state_dict())
    x, a = torch.randn(300, 17), torch.randn(300, 6)
    torch.manual_seed(99)
    with torch.no_grad():
        mean = ref.actor_mean(x)
        z = torch.empty(mean.shape).uniform_(-0.5, 0.5)
        probs = Normal(mean + z, torch.exp(ref.actor_logstd.expand_as(mean)))
        lp_r, ent_r, v_r = probs.log_prob(a).sum(1), probs.entropy().sum(1), ref.critic(x)
    torch.manual_seed(99)
    act, lp, ent, v = agent.get_action_and_value(x.cuda(), a.cuda())
    assert torch.equal(act.cpu(), a)
    assert (lp.cpu() - lp_r).abs().max() <= 1e-5 * lp_r.abs().max()
    assert (ent.cpu() - ent_r).abs().max() <= 1e-6 * max(1.0, ent_r.abs().max().item())
    assert (v.cpu() - v_r).abs().max() <= 1e-5 * max(1.0, v_r.abs().max().item())
    after = torch.get_rng_state()
    torch.manual_seed(99)
    torch.empty(300, 6).uniform_()
    assert torch.equal(torch.get_rng_state(), after)                 # exactly one [n, D] draw, as the reference
    torch.manual_seed(5)
    a1, _, _, _ = agent.get_action_and_value(x.cuda())                # action=None: the PPO agent's sampling path
    assert a1.shape == (300, 6)


class _Writer:
    def __init__(self, *a, **k): self.scalars = []
    def add_text(self, *a, **k): pass
    def add_scalar(self, tag, v, step): self.scalars.append((tag, float(v), int(step)))
    def close(self): pass


@pytest.mark.parametrize("name", ["rpo_continuous_n4_t64_seed2.npz", "rpo_continuous_n4_t64_seed5_kl.npz"])
def test_rpo_script_reproduces_reference_run(lib, tmp_path, monkeypatch, name):
    from cleanrl_b200 import rpo_continuous_action as S
    z = np.load(GOLDEN / name)
    argv = [a for a in z["argv"].tolist() if a != "--no-cuda"] + ["--synthetic-env"]
    snaps, writers, agents = [], [], []

    def on_it(it, eng, st):
        snaps.append({k: getattr(eng, k).cpu().numpy().copy() for k in
                      ("actions", "logprobs", "values", "rewards", "dones", "advantages", "returns")} | {"st": st})

    def hook(agent):
        agent.noise_fn = lambda n, D, dev: torch.randn(n, D).to(dev)    # CPU generator, as the CPU reference run
        agents.append(agent)

    def wf(p):
        w = _Writer(); writers.append(w); return w

    monkeypatch.chdir(tmp_path)
    S.main(argv, writer_factory=wf, on_iteration=on_it, agent_hook=hook)
    assert list(agents[0].state_dict().keys()) == z["state_dict_keys"].tolist()
    alpha = float(argv[argv.index("--rpo-alpha") + 1]) if "--rpo-alpha" in argv else 0.5
    assert agents[0].rpo_alpha == alpha
    s0 = snaps[0]
    assert np.abs(s0["actions"] - z["actions"][0]).max() <= 2e-6 * np.abs(z["actions"][0]).max()
    assert np.array_equal(s0["dones"], z["dones"][0])
    for k in ("rewards", "logprobs", "values", "advantages", "returns"):
        d = np.abs(s0[k].astype(np.float64) - z[k][0]).max() / max(1.0, np.abs(z[k][0]).max())
        assert d <= 2 * TOL, (k, d)
    assert [s["st"]["num_updates"] for s in snaps] == z["updates_per_iteration"].tolist()
    per = np.concatenate([s["st"]["per_update"] for s in snaps])
    assert len(per) == len(z["upd_loss"])
    for col, key in ((0, "upd_pg_loss"), (1, "upd_v_loss"), (4, "upd_approx_kl"), (6, "upd_loss")):
        ref = z[key]
        err = np.abs(per[:, col] - ref) / np.maximum(1.0, np.abs(ref))
        assert err.max() <= 2 * TOL, (key, int(err.argmax()), err.max())
    sums = np.array([p.detach().double().sum().item() for p in agents[0].parameters()])
    ref = z["final_param_sums"]
    assert np.abs(sums - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max()), (sums, ref)
    assert {t for t, _, _ in writers[0].scalars} == {k[3:] for k in z.files if k.startswith("tb/")}
