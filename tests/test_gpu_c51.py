"""-m gpu: C51 kernels vs the numpy oracle, the wide (wgmma) bf16 head vs torch with the kernels' operand rounding,
and the c51_atari drop-in vs the unmodified reference run (tests/golden/c51_atari_b8_seed1.npz)."""
import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import c51_oracle as O

pytestmark = pytest.mark.gpu


class _Envs:
    def __init__(self, A):
        from cleanrl_b200.synthetic_envs import Box, Discrete
        self.single_observation_space = Box(0, 255, (4, 84, 84), np.uint8)
        self.single_action_space = Discrete(A)


def _case(B, A, Z, seed):
    g = torch.Generator().manual_seed(seed)
    atoms = torch.linspace(-10, 10, Z)
    logits = torch.randn(B, A * Z, generator=g) * 2
    nlogits = torch.randn(B, A * Z, generator=g) * 2
    a = torch.randint(0, A, (B,), generator=g)
    r = torch.randint(-1, 2, (B,), generator=g).float()
    d = (torch.rand(B, generator=g) < 0.2).float()
    return atoms, logits, nlogits, a, r, d


@pytest.mark.parametrize("B,A,Z", [(8192, 4, 51), (32, 18, 51), (1, 2, 101), (1000, 6, 51)])
def test_c51_kernels_vs_oracle(lib, B, A, Z):
    from cleanrl_b200 import ops
    atoms, logits, nlogits, a, r, d = _case(B, A, Z, B + A + Z)
    loss, qv, dl_o, _ = O.loss_and_grad(logits.numpy(), nlogits.numpy(), atoms.numpy(), a.numpy(), r.numpy(), d.numpy(),
                                        0.99, -10.0, 10.0)
    st, dl = ops.c51_loss(logits.cuda(), nlogits.cuda(), atoms.cuda(), a.cuda(), r.cuda(), d.cuda(), 0.99, -10.0, 10.0)
    st = st.cpu().numpy()
    assert abs(st[0] - loss) <= 1e-5 * max(1.0, abs(loss)) and abs(st[1] - qv) <= 1e-5 * max(1.0, abs(qv))
    assert np.abs(dl.cpu().numpy() - dl_o).max() <= 1e-5 * np.abs(dl_o).max()
    # bitwise reproducible
    st2, dl2 = ops.c51_loss(logits.cuda(), nlogits.cuda(), atoms.cuda(), a.cuda(), r.cuda(), d.cuda(), 0.99, -10.0, 10.0)
    assert torch.equal(dl2, dl) and np.array_equal(st2.cpu().numpy(), st)
    # get_action: greedy and given actions
    act_o, pmf_o, q_o = O.get_action(logits.numpy(), atoms.numpy())
    act, q, pmf = ops.c51_act(logits.cuda(), atoms.cuda(), want_q=True)
    act, q, pmf = act.cpu().numpy(), q.cpu().numpy(), pmf.cpu().numpy()
    assert np.abs(q - q_o).max() <= 1e-5 * max(1.0, np.abs(q_o).max())
    top2 = np.sort(q_o, 1)[:, -2:] if A > 1 else np.zeros((B, 2))
    tie = (top2[:, 1] - top2[:, 0]) <= 1e-6
    assert np.array_equal(act[~tie], act_o[~tie])
    _, pmf_sel_o, _ = O.get_action(logits.numpy(), atoms.numpy(), act)
    assert np.abs(pmf - pmf_sel_o).max() <= 1e-6
    act_g, _, pmf_g = ops.c51_act(logits.cuda(), atoms.cuda(), a.cuda())
    assert torch.equal(act_g.cpu(), a)
    _, pmf_a_o, _ = O.get_action(logits.numpy(), atoms.numpy(), a.numpy())
    assert np.abs(pmf_g.cpu().numpy() - pmf_a_o).max() <= 1e-6


def _rel(a, b):
    a = a.detach().double().cpu(); b = b.detach().double().cpu()
    return ((a - b).norm() / max(b.norm().item(), 1e-30)).item()


@pytest.mark.parametrize("A,Z", [(4, 51), (18, 51), (18, 101)])
def test_wide_bf16_head_layer(lib, A, Z):
    """Head widths 204, 918, 1818 on wgmma: fp32 output + bias from the kernel's own bf16 hidden, dWh / dbh / dhid
    against torch with bf16 operands (hidden, head weights, dhead), and bitwise-identical repeats."""
    from cleanrl_b200.agents import C51QNetwork
    torch.manual_seed(3)
    net = C51QNetwork(_Envs(A), n_atoms=Z, v_min=-10, v_max=10).cuda()
    net.precision = "bf16"
    f = net.flat
    W1 = A * Z
    g = torch.Generator().manual_seed(4)
    B, n = 300, 257
    obs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g).cuda()
    rows = torch.randperm(B, generator=g)[:n].cuda()
    out = net.logits(obs, rows=rows, keep=True)
    torch.cuda.synchronize()
    acts = net._tc.acts(n, 0).view(torch.bfloat16)
    o_hid = n * (28224 + 12800 + 5184 + 3136)
    hid = acts[o_hid:o_hid + n * 512].view(n, 512).float()
    Wh = net.network[9].weight.detach().float()
    bh = net.network[9].bias.detach().float()
    ref = hid.double() @ Wh.to(torch.bfloat16).double().t() + bh.double()
    assert out.shape == (n, W1)
    assert ((out.double() - ref).abs().max() / ref.abs().max()).item() <= 3e-3
    dhead = (torch.randn(n, W1, generator=g) * 1e-3).cuda()
    net.backward(dhead)
    torch.cuda.synchronize()
    dW1, db1 = net.network[9].weight.grad.clone(), net.network[9].bias.grad.clone()
    dhid = acts[o_hid + n * 512:o_hid + 2 * n * 512].view(n, 512).float()
    d16 = dhead.to(torch.bfloat16).double()
    assert _rel(dW1, d16.t() @ hid.double()) <= 1.5e-2
    assert _rel(db1, dhead.double().sum(0)) <= 1.5e-2
    assert _rel(dhid, (d16 @ Wh.to(torch.bfloat16).double()) * (hid > 0)) <= 1.5e-2
    grads1 = f.grad.clone()
    out2 = net.logits(obs, rows=rows, keep=True)
    net.backward(dhead)
    torch.cuda.synchronize()
    assert torch.equal(out2, out) and torch.equal(f.grad, grads1)


def test_wide_head_limit(lib):
    assert lib.b200rl_naturecnn_bf16_packed_bytes(2047) > 0 and lib.b200rl_naturecnn_bf16_packed_bytes(2048) == 0


class _Writer:
    def __init__(self, *a, **k): self.scalars = []
    def add_text(self, *a, **k): pass
    def add_scalar(self, tag, v, step): self.scalars.append((tag, float(np.asarray(v).reshape(-1)[0]), int(step)))
    def close(self): pass


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_c51_script_vs_reference_run(lib, precision, monkeypatch):
    from cleanrl_b200 import c51_atari as S
    from cleanrl_b200.synthetic_envs import SyntheticGymnasiumVec
    z = np.load(GOLDEN / "c51_atari_b8_seed1.npz")
    argv = [a for a in z["argv"].tolist() if a != "--no-cuda"] + ["--synthetic-env", "--precision", precision]
    stream, losses, writers = [], [], []
    orig = SyntheticGymnasiumVec.step

    def step(self_, act):
        stream.append(int(np.asarray(act).reshape(-1)[0]))
        return orig(self_, act)
    monkeypatch.setattr(SyntheticGymnasiumVec, "step", step)

    def on_update(step_, stats, qn):
        losses.append(stats.cpu().numpy().copy())

    def wf(p):
        w = _Writer(); writers.append(w); return w

    qn = S.main(argv, writer_factory=wf, on_update=on_update)
    assert list(qn.state_dict().keys()) == z["state_dict_keys"].tolist()
    ref = z["losses"]
    assert len(losses) == len(ref)
    got = np.array([l[0] for l in losses])
    assert np.isfinite(got).all()
    if precision == "fp32":
        assert abs(got[0] - ref[0]) <= 1e-5 * max(1.0, abs(ref[0]))
        assert abs(losses[0][1] - z["q_values"][0]) <= 1e-5 * max(1.0, abs(z["q_values"][0]))
        # every action chosen before the first update (its step is included) follows the reference's stream
        ls, tf = (int(argv[argv.index(k) + 1]) for k in ("--learning-starts", "--train-frequency"))
        n0 = (ls // tf + 1) * tf + 1
        assert stream[:n0] == z["action_stream"][:n0].tolist()
        assert np.abs(got[:10] - ref[:10]).max() <= 2e-2 * np.abs(ref[:10]).max()
    else:
        assert abs(got[0] - ref[0]) <= 2e-2 * max(1.0, abs(ref[0]))
    tags = {t for t, _, _ in writers[0].scalars}
    assert {"losses/loss", "losses/q_values", "charts/SPS"} <= tags


def test_c51_save_model_and_evaluate(lib, tmp_path, monkeypatch):
    """--save-model writes {"model_weights", "args"} that loads into a reference-shaped QNetwork, then evaluates it
    epsilon-greedily for 10 episodes (cleanrl_utils/evals/c51_eval.py), logging eval/episodic_return."""
    from cleanrl_b200 import c51_atari as S
    monkeypatch.chdir(tmp_path)
    writers = []

    def wf(p):
        w = _Writer(); writers.append(w); return w

    qn = S.main(["--total-timesteps", "120", "--learning-starts", "40", "--buffer-size", "64", "--batch-size", "8",
                 "--train-frequency", "4", "--seed", "1", "--n-atoms", "21", "--v-min", "-5", "--v-max", "5",
                 "--synthetic-env", "--save-model", "--precision", "bf16"], writer_factory=wf)
    files = list(tmp_path.glob("runs/*/c51_atari.cleanrl_model"))
    assert len(files) == 1
    data = torch.load(files[0])
    assert data["args"]["n_atoms"] == 21 and data["args"]["v_min"] == -5
    ref_shaped = S.QNetwork(_Envs(4), n_atoms=data["args"]["n_atoms"], v_min=data["args"]["v_min"],
                            v_max=data["args"]["v_max"])
    ref_shaped.load_state_dict(data["model_weights"])
    for k, v in qn.state_dict().items():
        assert torch.equal(data["model_weights"][k], v.detach().cpu()), k
    evals = [(step, v) for tag, v, step in writers[0].scalars if tag == "eval/episodic_return"]
    assert [s for s, _ in evals] == list(range(10)) and all(np.isfinite(v) for _, v in evals)
