"""DQN path (config 5): TD-loss oracle/kernels, device replay ring vs the reference's numpy ReplayBuffer,
and the dqn_atari drop-in vs the unmodified reference run (tests/golden/dqn_atari_b8_seed1.npz)."""
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import ppo_oracle as O


def test_td_loss_oracle_vs_torch():
    import torch.nn.functional as F
    torch.manual_seed(0)
    B, A = 257, 4
    q = torch.randn(B, A, requires_grad=True)
    qt = torch.randn(B, A)
    a = torch.randint(0, A, (B, 1)); r = torch.randn(B); d = (torch.rand(B) < 0.1).float()
    for huber in (False, True):
        q.grad = None
        td = r + 0.99 * qt.max(dim=1)[0] * (1 - d)
        old = q.gather(1, a).squeeze()
        loss = F.smooth_l1_loss(td, old) if huber else F.mse_loss(td, old)
        loss.backward()
        l, qm, dq = O.dqn_td_loss(q.detach().numpy(), qt.numpy(), a.numpy(), r.numpy(), d.numpy(), 0.99, huber)
        assert abs(float(l) - float(loss.detach())) < 1e-6 and abs(float(qm) - float(old.mean())) < 1e-6
        assert np.abs(dq - q.grad.numpy()).max() < 1e-8


def test_replay_ring_matches_reference_replay_buffer():
    """Same adds, same numpy seed => same sampled transitions as cleanrl_utils/buffers.py ReplayBuffer
    (optimize_memory_usage=True), before and after the ring wraps.  The reference's samples are stored in
    tests/golden/replay_buffer_samples.npz (observations as indices into the generated frame sequence)."""
    from cleanrl_b200.replay import DeviceReplayRing
    ref = np.load(GOLDEN / "replay_buffer_samples.npz")
    rng = np.random.default_rng(0)
    size = 50
    ring = DeviceReplayRing(size, (4, 84, 84), 1, torch.device("cpu"))
    frames = [rng.integers(0, 256, (1, 4, 84, 84), dtype=np.uint8)]
    for t in range(137):
        nxt = rng.integers(0, 256, (1, 4, 84, 84), dtype=np.uint8)
        a = rng.integers(0, 4, (1,)); r = rng.standard_normal(1).astype(np.float32); d = rng.random(1) < 0.1
        ring.add(frames[-1], nxt, a, r, d, [{}])
        frames.append(nxt)
        if t in (20, 49, 50, 77, 136):
            seq = torch.from_numpy(np.concatenate(frames))
            st = np.random.get_state()
            np.random.seed(t)
            b = ring.sample(16)
            np.random.set_state(st)
            assert torch.equal(ring.frames[b["rows"]], seq[torch.from_numpy(ref[f"t{t}_obs_frame"])])
            assert torch.equal(ring.frames[b["next_rows"]], seq[torch.from_numpy(ref[f"t{t}_next_obs_frame"])])
            assert torch.equal(b["actions"], torch.from_numpy(ref[f"t{t}_actions"]))
            assert torch.equal(b["rewards"], torch.from_numpy(ref[f"t{t}_rewards"]))
            assert torch.equal(b["dones"], torch.from_numpy(ref[f"t{t}_dones"]))


@pytest.mark.gpu
@pytest.mark.parametrize("B,A", [(8192, 4), (32, 6), (1, 2), (1000, 18)])
@pytest.mark.parametrize("huber", [False, True])
def test_td_loss_kernel_vs_oracle(lib, B, A, huber):
    from cleanrl_b200 import ops
    g = torch.Generator().manual_seed(B + A)
    q = torch.randn(B, A, generator=g); qt = torch.randn(B, A, generator=g)
    a = torch.randint(0, A, (B,), generator=g); r = torch.randn(B, generator=g); d = (torch.rand(B, generator=g) < 0.1).float()
    l, qm, dq_o = O.dqn_td_loss(q.numpy(), qt.numpy(), a.numpy(), r.numpy(), d.numpy(), 0.99, huber)
    st, dq = ops.dqn_td_loss(q.cuda(), qt.cuda(), a.cuda(), r.cuda(), d.cuda(), 0.99, huber)
    st = st.cpu().numpy()
    assert abs(st[0] - float(l)) <= 1e-5 * max(1.0, abs(float(l))) and abs(st[1] - float(qm)) <= 1e-5
    assert np.abs(dq.cpu().numpy() - dq_o).max() <= 1e-5 * np.abs(dq_o).max() + 1e-12
    assert torch.equal(ops.argmax(q.cuda()).cpu(), q.argmax(dim=1))


class _Writer:
    def __init__(self, *a, **k): self.scalars = []
    def add_text(self, *a, **k): pass
    def add_scalar(self, tag, v, step): self.scalars.append((tag, float(np.asarray(v).reshape(-1)[0]), int(step)))
    def close(self): pass


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_dqn_script_vs_reference_run(lib, precision):
    from cleanrl_b200 import dqn_atari as S
    z = np.load(GOLDEN / "dqn_atari_b8_seed1.npz")
    argv = [a for a in z["argv"].tolist() if a != "--no-cuda"] + ["--synthetic-env", "--precision", precision]
    losses, writers = [], []

    def on_update(step, stats, qn):
        losses.append(stats.cpu().numpy().copy())

    def wf(p):
        w = _Writer(); writers.append(w); return w

    qn = S.main(argv, writer_factory=wf, on_update=on_update)
    assert list(qn.state_dict().keys()) == z["state_dict_keys"].tolist()
    ref = z["td_losses"]
    assert len(losses) == len(ref)
    got = np.array([l[0] for l in losses])
    if precision == "fp32":
        # first update: identical inputs => 1e-5; afterwards two Adam chains with different fp32 summation
        # orders (see tests/test_gpu_ppo_loop.py) => 2e-2 while the epsilon-greedy action streams agree
        assert abs(got[0] - ref[0]) <= 1e-5 * max(1.0, abs(ref[0]))
        assert abs(losses[0][1] - z["q_means"][0]) <= 1e-5
        assert np.abs(got[:10] - ref[:10]).max() <= 2e-2 * np.abs(ref[:10]).max()
    else:
        assert abs(got[0] - ref[0]) <= 2e-2 * max(1.0, abs(ref[0]))
    assert np.isfinite(got).all()
    tags = {t for t, _, _ in writers[0].scalars}
    assert {"losses/td_loss", "losses/q_values", "charts/SPS"} <= tags


@pytest.mark.gpu
def test_dqn_save_model_and_evaluate(lib, tmp_path, monkeypatch):
    """--save-model writes a reference-compatible state_dict and evaluates it epsilon-greedily for 10 episodes
    (cleanrl/dqn_atari.py:244-261, cleanrl_utils/evals/dqn_eval.py), logging eval/episodic_return."""
    import torch
    from cleanrl_b200 import dqn_atari as S
    monkeypatch.chdir(tmp_path)
    writers = []

    def wf(p):
        w = _Writer(); writers.append(w); return w

    qn = S.main(["--total-timesteps", "120", "--learning-starts", "40", "--buffer-size", "64", "--batch-size", "8",
                 "--train-frequency", "4", "--seed", "1", "--synthetic-env", "--save-model"], writer_factory=wf)
    files = list(tmp_path.glob("runs/*/dqn_atari.cleanrl_model"))
    assert len(files) == 1
    sd = torch.load(files[0])
    assert list(sd.keys()) == list(qn.state_dict().keys())
    for k, v in qn.state_dict().items():
        assert torch.equal(sd[k], v.detach().cpu()), k
    evals = [(step, v) for tag, v, step in writers[0].scalars if tag == "eval/episodic_return"]
    assert [s for s, _ in evals] == list(range(10)) and all(np.isfinite(v) for _, v in evals)
