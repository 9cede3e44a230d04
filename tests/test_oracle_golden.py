"""CPU tests: pin the oracle (oracle/ppo_oracle.py) against fixtures produced by the
UNMODIFIED reference scripts (oracle/make_golden.py -> tests/golden/*.npz).

The reference's own tests hold no golden vectors for this path (SURVEY.md 8c:
only a JAX GAE scan-vs-loop equality test, tests/test_jax_compute_gae.py:66-91);
the pin is therefore the reference script itself, executed in the build
container on the synthetic envs.
"""
import numpy as np
import pytest

from conftest import GOLDEN
from oracle import ppo_oracle as O

ATARI = ["ppo_atari_envpool_n8_t32_seed1.npz", "ppo_atari_envpool_n16_t16_seed3_noclipv.npz",
         "ppo_atari_gym_n8_t32_seed2.npz", "ppo_atari_envpool_n8_t16_seed5_flags.npz"]


def _args(z):
    argv = [str(x) for x in z["argv"]]
    def get(flag, default, cast=float):
        return cast(argv[argv.index(flag) + 1]) if flag in argv else default
    return dict(gamma=get("--gamma", 0.99), lam=get("--gae-lambda", 0.95), seed=get("--seed", 1, int),
                num_envs=get("--num-envs", 8, int), num_steps=get("--num-steps", 128, int),
                clip_vloss="--no-clip-vloss" not in argv, ent_coef=get("--ent-coef", 0.01),
                update_epochs=get("--update-epochs", 4, int), num_minibatches=get("--num-minibatches", 4, int),
                target_kl=get("--target-kl", None), anneal_lr="--no-anneal-lr" not in argv)


@pytest.mark.parametrize("name", ATARI + ["ppo_mlp_n4_t128_seed1.npz", "ppo_atari_lstm_n8_t16_seed4.npz",
                                          "ppo_atari_envpool_n1024_t128_seed1.npz"])
def test_gae_oracle_bit_exact_vs_reference_run(name):
    z = np.load(GOLDEN / name)
    a = _args(z)
    for it in range(z["rewards"].shape[0]):
        adv, ret = O.gae(z["rewards"][it].astype(np.float32), z["values"][it], z["dones"][it].astype(np.float32),
                         z["next_value"][it].reshape(-1), z["next_done"][it], a["gamma"], a["lam"])
        assert np.array_equal(adv, z["advantages"][it])
        # the full-size fixture stores no returns: the reference computed them as advantages + values (float32)
        ref_ret = z["returns"][it] if "returns" in z else (z["advantages"][it] + z["values"][it]).astype(np.float32)
        assert np.array_equal(ret, ref_ret)


def test_gae_oracle_scan_equals_loop_at_reference_test_shape():
    """Property of the reference's only numeric test (tests/test_jax_compute_gae.py: T=123, N=7,
    gamma=.99, lambda=.95): a scan formulation equals the python loop.  Here: oracle loop vs an
    independent float64 closed-form evaluation, 1e-5."""
    rng = np.random.default_rng(42)
    T, N = 123, 7
    r = rng.standard_normal((T, N)).astype(np.float32)
    v = rng.standard_normal((T, N)).astype(np.float32)
    d = (rng.random((T, N)) < 0.1).astype(np.float32)
    nv = rng.standard_normal(N).astype(np.float32)
    nd = (rng.random(N) < 0.1).astype(np.float32)
    adv, ret = O.gae(r, v, d, nv, nd, 0.99, 0.95)
    vv = np.concatenate([v, nv[None]], 0).astype(np.float64)
    dd = np.concatenate([d, nd[None]], 0).astype(np.float64)
    delta = r + 0.99 * vv[1:] * (1 - dd[1:]) - vv[:-1]
    ref = np.zeros((T + 1, N))
    for t in reversed(range(T)):
        ref[t] = delta[t] + 0.99 * 0.95 * (1 - dd[t + 1]) * ref[t + 1]
    assert np.abs(adv - ref[:-1]).max() < 1e-5


def test_loss_oracle_vs_reference_minibatches():
    z = np.load(GOLDEN / "ppo_mlp_n4_t128_seed1.npz")
    for u in range(z["mb_logits"].shape[0]):
        st, dl, dv = O.ppo_loss(z["mb_logits"][u], z["mb_newvalue"][u].reshape(-1), z["mb_mb_inds"][u],
                                z["b_actions"], z["b_logprobs"], z["b_advantages"], z["b_returns"], z["b_values"],
                                clip_coef=0.2, ent_coef=0.01, vf_coef=0.5)
        for ok, rk in (("pg_loss", "upd_pg_loss"), ("v_loss", "upd_v_loss"), ("entropy", "upd_entropy_loss"),
                       ("old_approx_kl", "upd_old_approx_kl"), ("approx_kl", "upd_approx_kl"),
                       ("clipfrac", "upd_clipfrac"), ("loss", "upd_loss")):
            assert abs(float(st[ok]) - float(z[rk][u])) <= 1e-6 * max(1.0, abs(float(z[rk][u]))), (u, ok)
        # normalised advantages and logprob/entropy of the gathered rows
        lp, ent = O.categorical_eval(z["mb_logits"][u], z["b_actions"][z["mb_mb_inds"][u]].astype(np.int64))
        assert np.abs(lp - z["mb_newlogprob"][u]).max() <= 1e-6
        assert np.abs(ent - z["mb_entropy"][u]).max() <= 1e-6
    # note: b_* tensors are the first iteration's; only the first 4 minibatches (epoch 1) index them
    # with the shuffles of iteration 1 -- all 6 recorded updates belong to iteration 1 (16 per iteration).


def test_adam_oracle_vs_reference_optimizer_steps():
    z = np.load(GOLDEN / "ppo_mlp_n4_t128_seed1.npz")
    P = z["params_before_flat"].shape[1]
    m = np.zeros(P, np.float32)
    v = np.zeros(P, np.float32)
    for u in range(z["grads_flat"].shape[0]):
        p, m, v, _ = O.clip_adam(z["params_before_flat"][u], z["grads_flat"][u], m, v, step=u + 1,
                                 lr=float(z["upd_lr"][u]), eps=1e-5, max_norm=None)
        assert np.abs(p - z["params_after_flat"][u]).max() <= 2e-7
        if u + 1 < z["grads_flat"].shape[0]:
            assert np.array_equal(z["params_after_flat"][u], z["params_before_flat"][u + 1])


def test_clip_coefficient_matches_reference_postclip_norm():
    """The recorded grads are post-clip: their norm must be min(norm, max_norm) (+1e-6 slack of torch)."""
    z = np.load(GOLDEN / "ppo_mlp_n4_t128_seed1.npz")
    for u in range(z["grads_flat"].shape[0]):
        n = np.sqrt((z["grads_flat"][u].astype(np.float64) ** 2).sum())
        assert n <= 0.5 + 1e-5


@pytest.mark.parametrize("name", ATARI)
def test_numpy_shuffle_stream_matches_reference(name):
    """np.random.seed(seed) + shuffle(arange(B)) per epoch is the minibatch order (ppo.py:155,242-245)."""
    z = np.load(GOLDEN / name)
    a = _args(z)
    B = a["num_envs"] * a["num_steps"]
    np_state = np.random.get_state()
    try:
        np.random.seed(a["seed"])
        k = 0
        # epochs actually run per iteration: all of them, unless --target-kl stopped the update early (ppo.py:292-293);
        # the reference logged one learning rate per update, constant within an iteration
        lrs = z["upd_lr"]
        n_it = z["rewards"].shape[0]
        if a.get("target_kl") is not None and a.get("anneal_lr", True):
            per_it = [int((lrs == v).sum()) // a["num_minibatches"] for v in sorted(set(lrs.tolist()), reverse=True)]
        else:
            per_it = [a["update_epochs"]] * n_it
        assert len(per_it) == n_it
        for it in range(n_it):
            inds = np.arange(B)
            for e in range(per_it[it]):
                np.random.shuffle(inds)
                assert np.array_equal(inds[:32], z["shuffles"][k])
                k += 1
        assert k == z["shuffles"].shape[0]
    finally:
        np.random.set_state(np_state)


def test_anneal_lr_matches_reference_log():
    z = np.load(GOLDEN / ATARI[0])
    lrs = z["tb/charts/learning_rate"][:, 1]
    n_it = len(lrs)
    for i in range(n_it):
        assert lrs[i] == O.anneal_lr(i + 1, n_it, 2.5e-4)


def test_categorical_sample_oracle_vs_torch_cpu():
    import torch
    from torch.distributions import Categorical
    g = torch.Generator().manual_seed(0)
    logits = torch.randn(4096, 6, generator=g) * 3
    torch.manual_seed(7)
    c = Categorical(logits=logits)
    act = c.sample()
    torch.manual_seed(7)
    q = torch.empty(4096, 6).exponential_(1)
    a, lp, ent = O.categorical_sample(logits.numpy(), q.numpy())
    assert np.array_equal(a, act.numpy())
    assert np.abs(lp - c.log_prob(act).numpy()).max() < 1e-6
    assert np.abs(ent - c.entropy().numpy()).max() < 1e-6


def test_loss_oracle_gradients_vs_torch_autograd():
    import torch
    from torch.distributions import Categorical
    torch.manual_seed(0)
    M, A, B = 512, 4, 2048
    logits = (torch.randn(M, A) * 2).requires_grad_(True)
    nv = torch.randn(M, requires_grad=True)
    b_act = torch.randint(0, A, (B,)); b_lp = torch.randn(B) * 0.1 - 1.3; b_adv = torch.randn(B)
    b_ret = torch.randn(B); b_val = b_ret + 0.3 * torch.randn(B)
    inds = torch.randperm(B)[:M]
    for clip_vloss in (True, False):
        logits.grad = None; nv.grad = None
        c = Categorical(logits=logits)
        ratio = (c.log_prob(b_act[inds]) - b_lp[inds]).exp()
        mb = b_adv[inds]; mb = (mb - mb.mean()) / (mb.std() + 1e-8)
        pg = torch.max(-mb * ratio, -mb * torch.clamp(ratio, 0.9, 1.1)).mean()
        if clip_vloss:
            vu = (nv - b_ret[inds]) ** 2
            vc = (b_val[inds] + torch.clamp(nv - b_val[inds], -0.1, 0.1) - b_ret[inds]) ** 2
            vl = 0.5 * torch.max(vu, vc).mean()
        else:
            vl = 0.5 * ((nv - b_ret[inds]) ** 2).mean()
        loss = pg - 0.01 * c.entropy().mean() + vl * 0.5
        loss.backward()
        st, dl, dv = O.ppo_loss(logits.detach().numpy(), nv.detach().numpy(), inds.numpy(), b_act.numpy(), b_lp.numpy(),
                                b_adv.numpy(), b_ret.numpy(), b_val.numpy(), 0.1, 0.01, 0.5, True, clip_vloss)
        assert abs(float(st["loss"]) - float(loss)) < 1e-6
        assert np.abs(dl - logits.grad.numpy()).max() < 1e-8
        assert np.abs(dv - nv.grad.numpy()).max() < 1e-8


def test_gaussian_oracle_vs_torch_normal_and_autograd():
    """Gaussian policy oracle vs torch.distributions.Normal (sample stream, log_prob, entropy) and autograd of
    the continuous PPO loss (cleanrl/ppo_continuous_action.py:134-141,262-300)."""
    import torch
    from torch.distributions.normal import Normal
    torch.manual_seed(0)
    M, D, B = 256, 6, 1024
    mean = torch.randn(M, D, requires_grad=True)
    logstd = (torch.randn(1, D) * 0.3).requires_grad_(True)
    nv = torch.randn(M, requires_grad=True)
    torch.manual_seed(9)
    act = Normal(mean, logstd.expand_as(mean).exp()).sample()
    torch.manual_seed(9)
    eps = torch.randn(M, D)
    a, lp, ent = O.gaussian_sample(mean.detach().numpy(), logstd.detach().numpy(), eps.numpy())
    # same N(0,1) stream; exp(logstd) differs by <= 1 ulp between numpy and torch => compare at 1e-6
    assert np.abs(a - act.numpy()).max() <= 1e-6 * np.abs(act.numpy()).max()
    a = act.numpy()
    lp, ent = O.gaussian_eval(mean.detach().numpy(), logstd.detach().numpy(), a)
    dist = Normal(mean, logstd.expand_as(mean).exp())
    assert np.abs(lp - dist.log_prob(act).sum(1).detach().numpy()).max() < 1e-5
    assert np.abs(ent - dist.entropy().sum(1).detach().numpy()).max() < 1e-5
    b_act = torch.randn(B, D); b_lp = torch.randn(B) * 0.2 - 5.0; b_adv = torch.randn(B)
    b_ret = torch.randn(B); b_val = b_ret + 0.3 * torch.randn(B)
    inds = torch.randperm(B)[:M]
    dist = Normal(mean, logstd.expand_as(mean).exp())
    ratio = (dist.log_prob(b_act[inds]).sum(1) - b_lp[inds]).exp()
    mb = b_adv[inds]; mb = (mb - mb.mean()) / (mb.std() + 1e-8)
    pg = torch.max(-mb * ratio, -mb * torch.clamp(ratio, 0.8, 1.2)).mean()
    vu = (nv - b_ret[inds]) ** 2
    vc = (b_val[inds] + torch.clamp(nv - b_val[inds], -0.2, 0.2) - b_ret[inds]) ** 2
    vl = 0.5 * torch.max(vu, vc).mean()
    loss = pg - 0.01 * dist.entropy().sum(1).mean() + vl * 0.5
    loss.backward()
    st, dm, dls, dv = O.ppo_loss_gaussian(mean.detach().numpy(), logstd.detach().numpy(), nv.detach().numpy(), inds.numpy(),
                                          b_act.numpy(), b_lp.numpy(), b_adv.numpy(), b_ret.numpy(), b_val.numpy(), 0.2, 0.01, 0.5)
    assert abs(float(st["loss"]) - float(loss.detach())) < 1e-5 * max(1.0, abs(float(loss.detach())))
    assert np.abs(dm - mean.grad.numpy()).max() <= 1e-5 * np.abs(mean.grad.numpy()).max()
    assert np.abs(dls - logstd.grad.numpy().reshape(-1)).max() <= 1e-5 * max(1.0, np.abs(logstd.grad.numpy()).max())
    assert np.abs(dv - nv.grad.numpy()).max() <= 1e-7


def test_lstm_env_shuffle_stream_matches_reference():
    """cleanrl/ppo_atari_lstm.py:297-303 shuffles ENV indices (not samples) per epoch: np.random.seed(seed) + shuffle(arange(N))."""
    z = np.load(GOLDEN / "ppo_atari_lstm_n8_t16_seed4.npz")
    a = _args(z)
    state = np.random.get_state()
    try:
        np.random.seed(a["seed"])
        k = 0
        for it in range(z["rewards"].shape[0]):
            env = np.arange(a["num_envs"])
            for e in range(a["update_epochs"]):
                np.random.shuffle(env)
                assert np.array_equal(env, z["shuffles"][k])
                k += 1
    finally:
        np.random.set_state(state)
