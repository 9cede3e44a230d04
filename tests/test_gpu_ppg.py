"""-m gpu: phasic policy gradient.  The fused auxiliary loss and the per-tensor clip + Adam against their references, the
three-headed IMPALA-CNN agent (fp32 against fp64 autograd, bf16 against the rounded-torch mirror of
tests/test_gpu_procgen_bf16.py) with its detached critic, and the drop-in script against runs of the UNMODIFIED
cleanrl/ppg_procgen.py (tests/golden/ppg_procgen_n4_t8_seed3*.npz)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN
from oracle import ppg_oracle
from test_gpu_procgen import _Envs, _Writer, _cpu_noise, _ref_forward
from test_gpu_procgen_bf16 import _mirror_forward, _no_tf32, _stored_forward  # noqa: F401  (_no_tf32: autouse fixture)

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------ fused auxiliary loss
@pytest.mark.parametrize("A", [4, 15, 22])
@pytest.mark.parametrize("n", [1, 33, 1024, 4096])
def test_aux_loss_kernel_vs_oracle(lib, A, n):
    from cleanrl_b200 import ops
    g = torch.Generator().manual_seed(n * 31 + A)
    B = 3 * n + 5
    head_buf = torch.randn(n, A + 7, generator=g)                  # strided head_out: a wider buffer's first A + 2 columns
    old = torch.randn(B, A, generator=g) * 2
    old[:, 1] = -float("inf")                                      # an old action of probability zero in every row
    old = old - old.logsumexp(-1, keepdim=True)
    ret = torch.randn(B, generator=g)
    rows = torch.randperm(B, generator=g)[:n]
    beta, accum = 0.7, 2
    head = head_buf.cuda()[:, :A + 2]
    st, dhead = ops.ppg_aux_loss(head, rows.cuda(), old.cuda(), ret.cuda(), beta, 1.0 / accum)
    st2, dhead2 = ops.ppg_aux_loss(head, rows.cuda(), old.cuda(), ret.cuda(), beta, 1.0 / accum)
    torch.cuda.synchronize()
    assert torch.equal(st, st2) and torch.equal(dhead, dhead2)
    ref, dref = ppg_oracle.aux_loss(head_buf[:, :A + 2].numpy(), old[rows].numpy(), ret[rows].numpy(), beta, accum)
    got = dhead.cpu().double().numpy()
    assert np.isfinite(got).all()
    assert np.abs(got - dref).max() <= 1e-5 * np.abs(dref).max()
    for i, k in enumerate(ops.PPG_AUX_STAT_NAMES):
        assert abs(float(st[i]) - ref[k]) <= 1e-5 * max(abs(ref[k]), 1e-3), (k, float(st[i]), ref[k])
    # rows = None reads the buffers in order
    st3, dhead3 = ops.ppg_aux_loss(head, None, old[rows].cuda(), ret[rows].cuda(), beta, 1.0 / accum)
    assert torch.equal(dhead3, dhead) and torch.equal(st3, st)


def test_aux_loss_kernel_infinite_when_the_new_policy_drops_an_action(lib):
    from cleanrl_b200 import ops
    head = torch.zeros(2, 5); head[0, 0] = -float("inf")
    st, _ = ops.ppg_aux_loss(head.cuda(), None, torch.zeros(2, 3).cuda(), torch.zeros(2).cuda(), 1.0)
    assert float(st[0]) == float("inf")


# ------------------------------------------------------------------ clip + Adam with per-tensor semantics
def test_clip_adam_ranges_vs_torch_with_a_gradless_tensor(lib):
    """torch.optim.Adam(eps=1e-8) + clip_grad_norm_ on three tensors, the middle one with ``grad = None`` for the first
    k steps and then stepping with its own count: frozen ranges bit-untouched, the rest at the tolerance of the existing
    clip_adam test."""
    from cleanrl_b200 import ops
    g = torch.Generator().manual_seed(0)
    sizes, k, steps, lr = (1001, 257, 33), 3, 8, 5e-4
    ps = [torch.nn.Parameter(torch.randn(s, generator=g)) for s in sizes]
    opt = torch.optim.Adam(ps, lr=lr, eps=1e-8)
    flat = torch.cat([p.detach() for p in ps]).cuda()
    m, v = torch.zeros_like(flat), torch.zeros_like(flat)
    lo = sizes[0]
    ranges = [(lo, lo + 100), (lo + 100, lo + sizes[1])]            # two adjacent ranges = the middle tensor
    norm = torch.zeros(1, device="cuda")
    for t in range(1, steps + 1):
        grads = [torch.randn(s, generator=g) * (3.0 if t % 2 else 0.01) for s in sizes]
        frozen = t <= k
        for i, p in enumerate(ps):
            p.grad = None if (frozen and i == 1) else grads[i].clone()
        ref_norm = torch.nn.utils.clip_grad_norm_(ps, 0.5)
        opt.step()
        gflat = torch.cat(grads).cuda()
        before = flat.clone(), m.clone(), v.clone()
        ops.clip_adam_ranges(flat, gflat, m, v, t, lr, ranges, 0 if frozen else t - k, lr, eps=1e-8, max_norm=0.5, norm_out=norm)
        torch.cuda.synchronize()
        assert abs(float(norm) - float(ref_norm)) <= 1e-5 * float(ref_norm)
        if frozen:
            for now, was in zip((flat, m, v), before):
                assert torch.equal(now[lo:lo + sizes[1]], was[lo:lo + sizes[1]])
        ref = torch.cat([p.detach() for p in ps])
        assert (flat.cpu() - ref).abs().max() <= 1e-6, t
    assert float(opt.state[ps[1]]["step"]) == steps - k


# ------------------------------------------------------------------ the agent
def _ppg_agent(A, precision, seed=2, head_gain=10.0, trunk_bias=0.0):
    from cleanrl_b200.agents import PPGAgent
    torch.manual_seed(seed)
    agent = PPGAgent(_Envs(A)).cuda()
    if trunk_bias:
        with torch.no_grad():
            for k, p in agent.named_parameters():
                if k.startswith("network.") and k.endswith(".bias"):
                    p.normal_(0, trunk_bias)
    with torch.no_grad():                      # non-zero biases (and, for bf16, heads of ordinary size): every path has signal
        for h in (agent.actor, agent.critic, agent.aux_critic):
            h.weight.mul_(head_gain); h.bias.normal_()
    agent.precision = precision
    agent.flat
    return agent


def _three_heads(sd, x, detach=True):
    """cleanrl/ppg_procgen.py:206-208 in fp64 on the trunk of tests/test_gpu_procgen.py."""
    hid = {}
    sd2 = dict(sd)
    sd2["actor.weight"] = torch.cat([sd["actor.weight"], sd["aux_critic.weight"]])
    sd2["actor.bias"] = torch.cat([sd["actor.bias"], sd["aux_critic.bias"]])
    orig = F.linear

    def linear(inp, w, b=None):                # the critic reads hidden.detach()
        if detach and w is sd["critic.weight"]:
            hid["h"] = inp
            inp = inp.detach()
        return orig(inp, w, b)
    F.linear = linear
    try:
        la, value = _ref_forward(sd2, x)
    finally:
        F.linear = orig
    A = sd["actor.weight"].shape[0]
    return la[:, :A], value, la[:, A], hid.get("h")


def _routing_mismatches(agent, sd, x):
    """ReLU masks and max-pool arg-maxes the fp32 forward kept, against those of the fp64 forward: how many differ."""
    sd = {k: v.detach() for k, v in sd.items()}
    h = x.permute(0, 3, 1, 2).double() / 255.0
    bad = 0
    for i, rec in enumerate(agent._saved["seqs"]):
        c = F.conv2d(h, sd[f"network.{i}.conv.weight"], sd[f"network.{i}.conv.bias"], padding=1)
        b, idx = F.max_pool2d(c, 3, 2, 1, return_indices=True)
        arg = rec["arg"].cpu().long()                          # position in the 3x3 window, row-major
        OH, OW = arg.shape[-2:]
        oy, ox = torch.arange(OH).view(1, 1, OH, 1), torch.arange(OW).view(1, 1, 1, OW)
        bad += int(((oy * 2 + arg // 3 - 1) * c.shape[-1] + (ox * 2 + arg % 3 - 1) != idx).sum())
        for bi, (r0, y0) in enumerate(rec["blocks"]):
            pre = f"network.{i}.res_block{bi}"
            y = F.relu(F.conv2d(F.relu(b), sd[f"{pre}.conv0.weight"], sd[f"{pre}.conv0.bias"], padding=1))
            bad += int(((r0.cpu() > 0) != (b > 0)).sum()) + int(((y0.cpu() > 0) != (y > 0)).sum())
            b = b + F.conv2d(y, sd[f"{pre}.conv1.weight"], sd[f"{pre}.conv1.bias"], padding=1)
        h = b
    return bad


@pytest.mark.parametrize("n,B,A", [(6, 20, 22), (1, 3, 4), (33, 33, 15), (33, 33, 22)])
def test_ppg_agent_fp32_vs_autograd(lib, n, B, A):
    # The trunk biases are drawn non-zero, as a trained network's are.  With the initial zero biases and n >= 12 one
    # max-pool window of sequence 1 holds a near-tie that the fp32 kernels and fp64 resolve differently; that one re-routed
    # gradient moves network.1.conv.weight's by 4e-3 of its maximum, with every mask, every other arg-max, d_hid, the fc and
    # the heads in agreement.  The routing is therefore asserted equal first, and the gradients compared on equal routing.
    agent = _ppg_agent(A, "fp32", head_gain=1.0, trunk_bias=0.1)
    g = torch.Generator().manual_seed(4)
    obs = torch.randint(0, 256, (B, 64, 64, 3), dtype=torch.uint8, generator=g)
    rows = torch.randperm(B, generator=g)[:n]
    ref = {k: v.detach().cpu().double().requires_grad_(True) for k, v in agent.state_dict().items()}
    logits, value, aux, hid = _three_heads(ref, obs[rows])
    hid.retain_grad()
    out = agent.forward_aux(obs.cuda(), rows.cuda())
    torch.cuda.synchronize()
    want = torch.cat([logits, value[:, None], aux[:, None]], 1)
    assert out.shape == (n, A + 2)
    assert (out.cpu().double() - want).abs().max() <= 1e-5 * max(1.0, want.abs().max().item())
    d = torch.randn(n, A + 2, generator=g)
    (want * d.double()).sum().backward()
    assert _routing_mismatches(agent, ref, obs[rows]) == 0
    # the hidden layer's gradient itself: (dhead without the critic column) . Wh under the ReLU mask
    hidk = agent._saved["hid"]
    dd = d.cuda().clone(); dd[:, A] = 0
    d_hid = agent.head.bwd_data(dd, hidk, "relu").cpu().double()
    Wh = torch.cat([ref["actor.weight"], ref["critic.weight"], ref["aux_critic.weight"]]).detach()
    want_dh = (dd.cpu().double() @ Wh) * (hidk.cpu() > 0)
    assert (d_hid - want_dh).abs().max() <= 1e-5 * want_dh.abs().max()
    agent.backward(d.cuda())
    torch.cuda.synchronize()
    errs = {k: (p.grad.cpu().double() - ref[k].grad).abs().max().item() / max(ref[k].grad.abs().max().item(), 1e-30)
            for k, p in agent.named_parameters()}
    assert max(errs.values()) <= 1e-4, errs
    # the critic's column must not reach the hidden layer: with it alone, only critic.* has a gradient
    d0 = torch.zeros(n, A + 2); d0[:, A] = d[:, A]
    agent.forward_aux(obs.cuda(), rows.cuda())
    agent.backward(d0.cuda())
    torch.cuda.synchronize()
    for k, p in agent.named_parameters():
        if k.startswith("critic."):
            assert p.grad.abs().max() > 0
        else:
            assert p.grad.abs().max() == 0, k
    # the reference API
    pi, v, av = agent.get_pi_value_and_aux_value(obs[rows].cuda())
    assert torch.equal(pi, agent.get_pi(obs[rows].cuda())) and v.shape == av.shape == (n, 1)
    assert (pi.exp().sum(-1) - 1).abs().max() <= 1e-5
    assert (agent.get_value(obs[rows].cuda()).cpu().double()[:, 0] - value).abs().max() <= 1e-5 * max(1.0, value.abs().max().item())


@pytest.mark.parametrize("n", [1, 33, 1024, 2049])
def test_ppg_agent_bf16_vs_rounded_torch(lib, n):
    A = 15
    agent = _ppg_agent(A, "bf16")
    g = torch.Generator().manual_seed(4)
    obs = torch.randint(0, 256, (n, 64, 64, 3), dtype=torch.uint8, generator=g).cuda()
    rows = torch.randperm(n, generator=g).cuda()
    d = (torch.randn(n, A + 2, generator=g) / n).cuda()
    out = agent.forward_aux(obs, rows).clone()
    agent.backward(d)
    grad = agent.flat.grad.clone()
    out2 = agent.forward_aux(obs, rows).clone()
    agent.backward(d)
    torch.cuda.synchronize()
    assert torch.equal(out, out2) and torch.equal(grad, agent.flat.grad)            # deterministic
    p = {k: v.detach().clone() for k, v in agent.state_dict().items()}
    join = lambda q: dict(q, **{"actor.weight": torch.cat([q["actor.weight"], q["aux_critic.weight"]]),
                                "actor.bias": torch.cat([q["actor.bias"], q["aux_critic.bias"]])})
    with torch.no_grad():
        la, value = _mirror_forward(join(p), obs[rows])
    want = torch.cat([la[:, :A], value[:, None], la[:, A:]], 1)
    assert (out - want).abs().max() <= 1e-2 * max(want.abs().max().item(), 1e-6)
    # backward on the kernels' stored tensors; the critic column is left out of the loss that reaches the trunk
    T = agent._tc.act_tensors(n)
    p = {k: v.detach().clone().requires_grad_(True) for k, v in agent.state_dict().items()}
    l2, _ = _stored_forward(join(p), obs[rows], T)
    (l2 * torch.cat([d[:, :A], d[:, A + 1:]], 1)).sum().backward()
    for k, prm in agent.named_parameters():
        if k.startswith("critic."):
            continue
        err = ((prm.grad - p[k].grad).norm() / max(p[k].grad.norm().item(), 1e-30)).item()
        assert err <= 2e-2, (k, err)
    hid = T["hid"].float()
    assert (agent.critic.weight.grad[0] - d[:, A] @ hid).abs().max() <= 1e-4 * max((d[:, A] @ hid).abs().max().item(), 1e-6)
    assert abs(float(agent.critic.bias.grad[0]) - float(d[:, A].sum())) <= 1e-5


def test_ppg_agent_bf16_rows_do_not_depend_on_the_batch_and_match_the_impala_plan(lib):
    from cleanrl_b200.agents import ImpalaAgent
    A = 15
    agent = _ppg_agent(A, "bf16")
    g = torch.Generator().manual_seed(9)
    obs = torch.randint(0, 256, (8192, 64, 64, 3), dtype=torch.uint8, generator=g).cuda()
    big = agent._head_out(obs).clone()
    small = agent._head_out(obs[1024:2048]).clone()
    assert torch.equal(big[1024:2048], small)
    # the two-headed plan on the same trunk, actor and critic: its A + 1 outputs bit for bit
    torch.manual_seed(0)
    imp = ImpalaAgent(_Envs(A)).cuda()
    imp.precision = "bf16"
    sd = {k: v for k, v in agent.state_dict().items() if not k.startswith("aux_critic.")}
    imp.load_state_dict(sd)
    imp.flat
    lg, val = imp._forward_heads(obs[:2048])
    assert torch.equal(lg, big[:2048, :A]) and torch.equal(val, big[:2048, A])


# ------------------------------------------------------------------ the script against the reference's run
def _run_script(name, extra):
    from cleanrl_b200 import ppg_procgen as S
    z = np.load(GOLDEN / name)
    argv = [a for a in z["argv"].tolist() if a != "--no-cuda"] + ["--synthetic-env"] + extra
    its, phases, writers = [], [], []

    def on_it(phase, update, eng, st):
        its.append({k: getattr(eng, k).cpu().numpy().copy() for k in
                    ("actions", "logprobs", "values", "rewards", "dones", "advantages", "returns")} |
                   {"st": st, "sums": _param_sums(eng), "aux_critic": _aux_critic(eng), "heads": _heads(eng, list(z["head_names"]))})

    def on_aux(phase, eng, aux):
        phases.append({"aux": aux, "aux_pi": eng.aux_pi.cpu().numpy().copy(), "aux_returns": eng.aux_returns.cpu().numpy().copy(),
                       "sums": _param_sums(eng), "aux_critic": _aux_critic(eng), "aux_step": eng.aux_step,
                       "heads": _heads(eng, list(z["head_names"])),
                       "step": eng.flat.step})

    def hook(agent):
        agent.noise_fn = _cpu_noise

    def wf(path):
        w = _Writer(); writers.append(w); return w

    S.main(argv, writer_factory=wf, on_iteration=on_it, on_aux_phase=on_aux, agent_hook=hook)
    return z, its, phases, writers[0]


def _param_sums(eng):
    return np.array([p.detach().double().sum().item() for p in eng.agent.parameters()])


def _heads(eng, names):
    sd = dict(eng.agent.named_parameters())
    return torch.cat([sd[k].detach().reshape(-1) for k in names]).cpu().numpy().copy()


def _aux_critic(eng):
    return torch.cat([eng.agent.aux_critic.weight.detach().reshape(-1), eng.agent.aux_critic.bias.detach()]).cpu().numpy().copy()


def _check_tags(z, writer):
    ours = {}
    for tag, v, step in writer.scalars:
        ours.setdefault(tag, []).append((step, v))
    for key in z.files:
        if key.startswith("tb/") and key != "tb/charts/SPS":
            tag, ref = key[3:], z[key]
            assert tag in ours, tag
            if not tag.startswith("charts/episodic"):
                assert np.array_equal(np.array(ours[tag])[:, 0], ref[:, 0]), tag
    return ours


@pytest.mark.parametrize("name", ["ppg_procgen_n4_t8_seed3.npz", "ppg_procgen_n4_t8_seed3_accum2.npz"])
def test_ppg_script_fp32_reproduces_reference_run(lib, name):
    """Two phases of 2 policy iterations x 2 minibatches and 2 auxiliary epochs x 4 minibatches.  Phase 1 at the
    tolerances of the ppo_procgen script test (first policy iteration's rollout <= 1e-5, actions bit-exact, losses <= 1e-5
    for the first update and <= 1e-4 after); parameters after every policy iteration and every phase, ``aux_pi``, every
    auxiliary minibatch's losses and the logged scalars; Adam's two step counts."""
    z, its, phases, writer = _run_script(name, [])
    rel = lambda a, b: np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max() / max(1.0, np.abs(b).max())
    s = its[0]
    assert np.array_equal(s["actions"], z["actions"][0].astype(np.int64))
    assert np.array_equal(s["rewards"], z["rewards"][0]) and np.array_equal(s["dones"], z["dones"][0])
    for k in ("logprobs", "values", "advantages", "returns"):
        assert rel(s[k], z[k][0]) <= 1e-5, (k, rel(s[k], z[k][0]))
    assert len(its) == 4 and len(phases) == 2
    aux_steps = z["step_aux"]
    names = list(z["param_names"])
    from cleanrl_b200.agents import PPGAgent
    assert [n for n, _ in PPGAgent(_Envs(15)).named_parameters()] == names
    # parameter sums after every policy iteration (2 Adam steps each) and after every auxiliary phase
    n_aux = int(aux_steps.sum()) // 2
    step = 0
    # a sampled action can fall on the other side of a rounding difference once the weights have moved; from that rollout
    # on the two runs see different data, so the trajectory is compared for as long as the actions are the reference's
    same = [all(np.array_equal(its[j]["actions"], z["actions"][j].astype(np.int64)) for j in range(i + 1)) for i in range(4)]
    assert same[0] and same[1], "phase 1 is always compared"
    print("iterations whose actions are the reference's:", same)
    for ph in range(2):
        for u in range(2):
            step += 2
            ref = z["step_sums_after"][step - 1]
            tol = 1e-4 if (ph, u) == (0, 0) else 1e-2
            if same[ph * 2 + u]:
                assert np.abs(its[ph * 2 + u]["sums"] - ref).max() <= tol * max(1.0, np.abs(ref).max()), (ph, u)
        step += n_aux
        assert phases[ph]["step"] == step and phases[ph]["aux_step"] == n_aux * (ph + 1)
        assert np.isfinite(phases[ph]["sums"]).all() and phases[ph]["aux"]["per_minibatch"].shape[0] == 8
        if not same[ph * 2 + 1]:
            continue
        ref = z["step_sums_after"][step - 1]
        assert np.abs(phases[ph]["sums"] - ref).max() <= 2e-2 * max(1.0, np.abs(ref).max()), ph
        assert rel(phases[ph]["aux_pi"], z["aux_pi"][ph]) <= (1e-4 if ph == 0 else 5e-3)
        assert rel(phases[ph]["aux_returns"], z["aux_returns"][ph]) <= (1e-5 if ph == 0 else 5e-2)
        per = phases[ph]["aux"]["per_minibatch"]
        for j, key in enumerate(("aux_kl_loss", "aux_aux_value_loss", "aux_real_value_loss")):
            ref = z[key][ph * 8:(ph + 1) * 8]
            tol = 1e-4 if ph == 0 else 2e-2
            assert np.abs(per[:, j] - ref).max() <= tol * max(1.0, np.abs(ref).max()), (ph, key, per[:, j], ref)
    # the recorded head tensors themselves (actor.bias, critic.*, aux_critic.*) at every checkpoint of phase 1: a wrong step
    # count or learning rate for aux_critic moves them by a fraction of lr = 5e-4 per step
    for got, s_ in ((its[0]["heads"], 1), (its[1]["heads"], 3), (phases[0]["heads"], 3 + n_aux)):
        assert np.abs(got - z["step_after"][s_]).max() <= 5e-5, (s_, np.abs(got - z["step_after"][s_]).max())
    # aux_critic: bit-untouched across a policy phase, moved by the auxiliary phase
    assert np.array_equal(its[0]["aux_critic"], its[1]["aux_critic"])
    assert np.array_equal(phases[0]["aux_critic"], its[2]["aux_critic"]) and np.array_equal(its[2]["aux_critic"], its[3]["aux_critic"])
    assert not np.array_equal(phases[0]["aux_critic"], its[1]["aux_critic"])
    ours = _check_tags(z, writer)
    for tag in ("losses/aux/kl_loss", "losses/aux/aux_value_loss", "losses/aux/real_value_loss"):
        ref = z["tb/" + tag]
        if same[1]:
            assert abs(ours[tag][0][1] - ref[0, 1]) <= 1e-4 * max(1.0, abs(ref[0, 1])), tag
    per = its[0]["st"]["per_update"]
    for col, tag in ((1, "losses/value_loss"), (0, "losses/policy_loss"), (2, "losses/entropy")):
        ref = z["tb/" + tag][0, 1]
        assert abs(per[-1, col] - ref) <= 1e-4 * max(1.0, abs(ref)), tag


def test_ppg_script_bf16_vs_reference_run(lib):
    z, its, phases, writer = _run_script("ppg_procgen_n4_t8_seed3.npz", ["--precision", "bf16"])
    rel = lambda a, b: np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max() / max(1.0, np.abs(b).max())
    s = its[0]
    assert (s["actions"] == z["actions"][0].astype(np.int64)).mean() >= 0.9
    for k in ("logprobs", "values"):
        assert rel(s[k], z[k][0]) <= 2e-2, (k, rel(s[k], z[k][0]))
    assert rel(phases[0]["aux_pi"], z["aux_pi"][0]) <= 5e-2
    per = phases[0]["aux"]["per_minibatch"]
    assert np.isfinite(per).all() and per.shape[0] == 8
    for j, key in enumerate(("aux_kl_loss", "aux_aux_value_loss", "aux_real_value_loss")):
        ref = z[key][:8]
        assert np.abs(per[:, j] - ref).max() <= 5e-2 * max(1.0, np.abs(ref).max()), (key, per[:, j], ref)
    assert np.array_equal(its[0]["aux_critic"], its[1]["aux_critic"])
    assert np.array_equal(phases[0]["aux_critic"], its[2]["aux_critic"]) and np.array_equal(its[2]["aux_critic"], its[3]["aux_critic"])
    assert not np.array_equal(phases[0]["aux_critic"], its[1]["aux_critic"])
    for ph in phases:
        assert np.isfinite(ph["sums"]).all()
    _check_tags(z, writer)


# ------------------------------------------------------------------ graph replay of the auxiliary update
def test_aux_graph_replay_equals_eager_bit_for_bit(lib, monkeypatch):
    """One auxiliary phase (2 epochs x 4 minibatches, after a policy update that leaves a gradient behind) with the update
    replayed as a CUDA graph and launched eagerly: parameters, Adam moments, losses and step counts identical."""
    from cleanrl_b200 import cli
    from cleanrl_b200.ppg_engine import PPGEngine
    from cleanrl_b200.synthetic_envs import SyntheticProcgenVec
    runs = []
    for graph in ("0", "1"):
        monkeypatch.setenv("CLEANRL_B200_PPG_AUX_GRAPH", graph)
        torch.manual_seed(3); np.random.seed(3)
        a = cli.ppg_procgen_args()()
        a.num_envs, a.num_steps, a.n_iteration, a.num_aux_rollouts, a.e_auxiliary, a.num_minibatches = 4, 8, 2, 2, 2, 2
        a.precision = "bf16"
        agent = _ppg_agent(15, "bf16", head_gain=1.0)
        eng = PPGEngine(agent, a, (64, 64, 3), 4, torch.device("cuda"))
        assert eng.aux_graph == (graph == "1")
        g = torch.Generator().manual_seed(5)
        eng.aux_obs.copy_(torch.randint(0, 256, eng.aux_obs.shape, dtype=torch.uint8, generator=g))
        eng.aux_returns.copy_(torch.randn(eng.aux_returns.shape, generator=g))
        eng.flat.grad.copy_(torch.randn(eng.flat.grad.shape, generator=g) * 1e-3)      # what a policy update leaves behind
        eng.grad_norm.fill_(float(eng.flat.grad.norm()))
        out = [eng.aux_phase(5e-4), eng.aux_phase(5e-4)]
        torch.cuda.synchronize()
        assert (eng._aux_g is not None) == (graph == "1")
        runs.append((eng.flat.flat.clone(), eng.flat.exp_avg.clone(), eng.flat.exp_avg_sq.clone(),
                     np.concatenate([o["per_minibatch"] for o in out]), eng.flat.step, eng.aux_step))
    for x, y in zip(runs[0][:3], runs[1][:3]):
        assert torch.equal(x, y)
    assert np.array_equal(runs[0][3], runs[1][3]) and np.isfinite(runs[0][3]).all()
    assert runs[0][4:] == runs[1][4:] == (16, 16)
