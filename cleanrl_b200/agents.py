"""Agent nn.Modules with the reference's surface, executed by libb200rl kernels.

Surface kept (SURVEY.md 8b): ctor ``Agent(envs)`` reading
``envs.single_observation_space`` / ``envs.single_action_space``; sub-module
names (=> identical ``state_dict`` keys); ``get_value(x)`` and
``get_action_and_value(x, action=None)`` returning
``(action i64 [n], logprob f32 [n], entropy f32 [n], value f32 [n,1])``.
Initialisation calls torch's ``orthogonal_`` in the reference's layer order so
a seed yields the reference's weights (cleanrl/ppo_atari_envpool.py:117-138,
cleanrl/ppo.py:94-116).

Forward/backward never touch autograd or cuDNN: they are explicit kernel
launches on CUDA tensors, and raise on CPU tensors (no fallback).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from . import nets, ops


def layer_init(layer, std=np.sqrt(2), bias_const=0.0):
    torch.nn.init.orthogonal_(layer.weight, std)
    torch.nn.init.constant_(layer.bias, bias_const)
    return layer


def _exp_noise(n, A, device):
    # what torch.multinomial consumes internally: empty_like(probs).exponential_(1)
    return torch.empty(n, A, dtype=torch.float32, device=device).exponential_(1)


_exp_noise.graph_safe = True      # device-generator draw: capturable in a CUDA graph
_exp_noise.inplace = lambda buf: buf.exponential_(1)     # same generator consumption as the out-of-place draw


class KernelAgent(nn.Module):
    """Shared plumbing: flat parameter binding + categorical head."""

    def __init__(self):
        super().__init__()
        self._flat = None
        self.noise_fn = _exp_noise   # tests may inject CPU-generator noise for cross-device parity

    # -- flat-buffer binding ------------------------------------------------
    def _param_order(self):
        return list(self.parameters())

    def bind(self):
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("cleanrl_b200 agents execute on CUDA only (libb200rl kernels); "
                               f"parameters are on {dev}. There is no CPU fallback.")
        self._flat = nets.FlatParams(self._param_order(), dev)
        self._build_plan()
        return self._flat

    @property
    def flat(self):
        p = next(self.parameters())
        if self._flat is None or self._flat.flat.device != p.device or \
                p.data_ptr() < self._flat.flat.data_ptr() or \
                p.data_ptr() >= self._flat.flat.data_ptr() + self._flat.flat.numel() * 4:
            self.bind()
        return self._flat

    # -- to be provided by subclasses --------------------------------------
    def _build_plan(self):
        raise NotImplementedError

    def _forward_heads(self, x, rows=None, keep=False):
        """returns (logits view [n,A] , value view [n] ) possibly strided"""
        raise NotImplementedError

    def backward(self, dlogits, dvalue):
        raise NotImplementedError

    # -- engine hooks (one policy step / one minibatch loss+backward) ---------------
    action_dim = 0          # 0 = discrete (int64 actions [n]); D > 0 = continuous (f32 actions [n, D])

    # may the engine capture the per-step device work (frame conversion, network, sampler) in CUDA graphs?
    graph_capturable = True

    def uses_tc_plan(self):
        """Do forward and backward run on a tensor-core plan (``TensorCoreAgent`` with ``precision = "bf16"``)?"""
        return False

    def params_updated(self):
        """Call after the optimiser changed the flat parameters."""

    def pin_workspaces(self):
        """Call after capturing a CUDA graph that runs this agent."""

    def grad_tail(self):
        """(offset, event) when ``flat.grad[offset:]`` is final before ``backward`` returns (NatureCNNAgent), else None."""
        return None

    @property
    def graph_friendly(self):
        """... and may the noise draw be captured too (device generator)?  Needed for whole-rollout graphs."""
        return getattr(self.noise_fn, "graph_safe", False) and self.graph_capturable

    def noise_shape(self, n):
        return (n, self.num_actions)

    def draw_noise_into(self, buf):
        """Fill ``buf`` [n, A] with this step's sampling noise (one draw for the whole env batch)."""
        if hasattr(self.noise_fn, "inplace"):
            self.noise_fn.inplace(buf)
        else:
            buf.copy_(self.noise_fn(buf.shape[0], buf.shape[1], buf.device))

    def sample_into(self, obs, actions_out, logprobs_out, values_out, noise=None):
        """Rollout step: forward + sample, writing straight into the rollout slots (ppo.py:197-202).
        ``noise``: pre-drawn rows of the step's noise tensor (chunked H2D/compute pipeline)."""
        logits, value = self._forward_heads(obs)
        n, A = logits.shape
        q = noise if noise is not None else self.noise_fn(n, A, logits.device)
        ops.categorical_sample(logits, q, value, out=(actions_out, logprobs_out, None, values_out))

    def loss_backward(self, policy_out, value, mb_inds, b, a, stats_row, scratch):
        """Minibatch loss (+ its gradient) and the network backward (ppo.py:251-288)."""
        M = policy_out.shape[0]
        if scratch.get("M") != M:
            scratch["M"] = M
            scratch["dhead"], scratch["dl"], scratch["dv"] = self.alloc_head_grad(M, policy_out.device)
        ops.ppo_loss(policy_out, value, mb_inds, b["actions"], b["logprobs"], b["advantages"], b["returns"], b["values"],
                     a.clip_coef, a.ent_coef, a.vf_coef, a.norm_adv, a.clip_vloss,
                     dlogits=scratch["dl"], dvalue=scratch["dv"], stats=stats_row)
        self.backward(scratch["dhead"])

    def alloc_head_grad(self, M, device):
        """(dhead [M, A+1], its dlogits view, its dvalue view): the gradient of the joint actor / critic head."""
        A = self.num_actions
        d = torch.empty(M, A + 1, dtype=torch.float32, device=device)
        return d, d[:, :A], d[:, A]

    # -- reference API ---------------------------------------------------------
    def get_value(self, x):
        self.flat
        _, value = self._forward_heads(x)
        return value.reshape(-1, 1).clone() if not value.is_contiguous() else value.reshape(-1, 1)

    def get_action_and_value(self, x, action=None):
        self.flat
        logits, value = self._forward_heads(x)
        n, A = logits.shape
        if action is None:
            q = self.noise_fn(n, A, logits.device)
            action, logprob, entropy, v = ops.categorical_sample(logits, q, value)
        else:
            logprob, entropy = ops.categorical_eval(logits, action)
            v = value.clone() if not value.is_contiguous() else value
        return action, logprob, entropy, v.reshape(-1, 1)


class TensorCoreAgent(KernelAgent):
    """An agent whose network ``precision = "bf16"`` runs on the tensor cores through an ``ops`` plan (``plan_class``,
    built on first use for ``_head_outputs()`` outputs); its packed bf16 weight copies are refreshed lazily after every
    change of the flat parameters."""

    precision = "fp32"
    plan_class = None
    _tc = None               # the plan
    _tc_dirty = True         # the plan's packed weights are stale

    def _head_outputs(self):
        return self.num_actions + 1          # actor + critic

    def _plan_actions(self):
        """The ``A`` the plan is built for: its head is A actions + the plan's value outputs."""
        return self._head_outputs() - 1

    def bind(self):
        self._tc, self._tc_dirty = None, True
        return super().bind()

    def uses_tc_plan(self):
        return self.precision == "bf16"

    @property
    def graph_capturable(self):
        """Only the bf16 plan is free of host work and allocations inside forward / backward."""
        return self.uses_tc_plan()

    def params_updated(self):
        """Call after the optimiser changed the flat parameters: the packed bf16 operands are stale."""
        self._tc_dirty = True

    def _tc_plan(self):
        f = self._flat
        if self._tc is None:
            self._tc = self.plan_class(self._plan_actions(), f.flat.device)
            assert f.flat.numel() >= self._tc.param_count
        if self._tc_dirty:
            self._tc.pack(f.flat)
            self._tc_dirty = False
        return self._tc

    def load_state_dict(self, *a, **k):
        out = super().load_state_dict(*a, **k)
        self._tc_dirty = True
        return out

    def pin_workspaces(self):
        """A CUDA graph captured by the engine holds raw pointers into the plan's workspaces: keep them all alive."""
        if self._tc is not None:
            self._tc.pin()

    def _joint_head(self):
        """``actor`` and the value heads as ONE layer over the flat buffer (adjacent in ``_param_order``): weight
        [_head_outputs(), hidden], bias [_head_outputs()]."""
        f, A1, H = self._flat, self._head_outputs(), self.actor.in_features
        ow = (f.view_of(self.actor.weight)[0].data_ptr() - f.flat.data_ptr()) // 4
        ob = (f.view_of(self.actor.bias)[0].data_ptr() - f.flat.data_ptr()) // 4
        return nets.Linear(None, None, f.flat[ow:ow + A1 * H].view(A1, H), f.flat[ob:ob + A1],
                           f.grad[ow:ow + A1 * H].view(A1, H), f.grad[ob:ob + A1])


class NatureCNNAgent(TensorCoreAgent):
    """NatureCNN actor-critic (reference: cleanrl/ppo_atari_envpool.py:123-149)."""

    plan_class = ops.NatureCNNBf16

    def __init__(self, envs):
        super().__init__()
        c, h, w = envs.single_observation_space.shape
        assert (c, h, w) == (4, 84, 84), "NatureCNN geometry is 4x84x84"
        trunk = []
        for cin, cout, k, s in ((4, 32, 8, 4), (32, 64, 4, 2), (64, 64, 3, 1)):
            trunk += [layer_init(nn.Conv2d(cin, cout, k, stride=s)), nn.ReLU()]
        trunk += [nn.Flatten(), layer_init(nn.Linear(64 * 7 * 7, 512)), nn.ReLU()]
        self.network = nn.Sequential(*trunk)
        self.actor = layer_init(nn.Linear(512, envs.single_action_space.n), std=0.01)
        self.critic = layer_init(nn.Linear(512, 1), std=1)
        self.num_actions = int(envs.single_action_space.n)

    def _param_order(self):
        net = [p for m in self.network for p in m.parameters()]
        # both heads adjacent => one [A+1, 512] GEMM operand and one [A+1] bias
        return net + [self.actor.weight, self.critic.weight, self.actor.bias, self.critic.bias]

    def _build_plan(self):
        n = self.network
        self.trunk = nets.Chain([
            nets.Conv(n[0], "relu", in_div=255.0), nets.Conv(n[2], "relu"), nets.Conv(n[4], "relu"),
            nets.Linear(n[7], "relu")])
        self.head = self._joint_head()

    def _forward_heads(self, x, rows=None, keep=False, aux=None):
        if self.precision == "bf16":
            if x.dtype not in (torch.uint8, torch.bfloat16):
                x = x.to(torch.uint8)       # frames are integers 0..255 (reference passes them as fp32)
            tc = self._tc_plan()
            out = tc.forward(x.contiguous(), rows, self._flat.flat)
            if keep:
                self._tc_obs, self._tc_rows, self._tc_aux = x, rows, aux
            A = self.num_actions
            return out[:, :A], out[:, A]
        if x.dtype not in (torch.uint8, torch.float32):
            x = x.float()
        hidden = self.trunk.fwd(x.contiguous(), rows=rows, keep=keep)
        out = self.head.fwd(hidden)
        if keep:
            self._hidden = hidden
        A = self.num_actions
        return out[:, :A], out[:, A]

    def forward_train(self, b_obs, mb_inds, aux=None):
        """Minibatch forward with fused row gather (b_obs[mb_inds] never materialised); keeps activations.
        ``aux``: channel-major copy of a uint8 space-to-depth rollout (consumed by the conv1 weight gradient)."""
        self.flat
        return self._forward_heads(b_obs, rows=mb_inds, keep=True, aux=aux)

    def grad_tail(self):
        """(offset, event): ``flat.grad[offset:]`` (fc + heads, 95 % of the vector) is final when ``event`` fires in the
        middle of ``backward`` -- lets the engine overlap the DP exchange of the tail with the conv backward.  None on
        the fp32 path (layer-by-layer backward finishes the first layers' gradients last anyway, but records no event)."""
        if self.precision != "bf16":
            return None
        if getattr(self, "_tail_event", None) is None:
            self._tail_event = torch.cuda.Event()
            self._tail_event.record()                      # materialise the cudaEvent_t handle
        return self._tc_plan().grad_tail_offset(), self._tail_event

    def backward(self, dhead):
        """dhead [M, A+1] = [dlogits | dvalue]; fills the flat gradient buffer."""
        if self.precision == "bf16":
            self._tc.backward(self._tc_obs, self._tc_rows, self._flat.flat, dhead, self._flat.grad,
                              tail_event=getattr(self, "_tail_event", None), obs_aux=getattr(self, "_tc_aux", None))
            self._tc_obs = self._tc_rows = self._tc_aux = None
            return
        hidden = self._hidden
        self.head.bwd_weight(hidden, dhead)
        dh = self.head.bwd_data(dhead, hidden, "relu")
        self.trunk.bwd(dh)
        self._hidden = None


class MLPAgent(KernelAgent):
    """Two 64-wide tanh MLPs, discrete actions (reference: cleanrl/ppo.py:100-126)."""

    def __init__(self, envs):
        super().__init__()
        d = int(np.array(envs.single_observation_space.shape).prod())
        A = int(envs.single_action_space.n)
        self.critic = nn.Sequential(layer_init(nn.Linear(d, 64)), nn.Tanh(), layer_init(nn.Linear(64, 64)), nn.Tanh(),
                                    layer_init(nn.Linear(64, 1), std=1.0))
        self.actor = nn.Sequential(layer_init(nn.Linear(d, 64)), nn.Tanh(), layer_init(nn.Linear(64, 64)), nn.Tanh(),
                                   layer_init(nn.Linear(64, A), std=0.01))
        self.num_actions = A

    def _build_plan(self):
        mk = lambda seq: nets.Chain([nets.Linear(seq[0], "tanh"), nets.Linear(seq[2], "tanh"), nets.Linear(seq[4], None)])
        self.c_chain, self.a_chain = mk(self.critic), mk(self.actor)

    def _forward_heads(self, x, rows=None, keep=False):
        x = x.float() if x.dtype != torch.float32 else x
        x = x.reshape(x.shape[0], -1).contiguous()
        logits = self.a_chain.fwd(x, rows=rows, keep=keep)
        value = self.c_chain.fwd(x, rows=rows, keep=keep)
        return logits, value[:, 0]

    def forward_train(self, b_obs, mb_inds):
        self.flat
        return self._forward_heads(b_obs, rows=mb_inds, keep=True)

    def alloc_head_grad(self, M, device):
        dl = torch.empty(M, self.num_actions, dtype=torch.float32, device=device)
        dv = torch.empty(M, 1, dtype=torch.float32, device=device)
        return (dl, dv), dl, dv[:, 0]

    def backward(self, dhead):
        dl, dv = dhead
        self.a_chain.bwd(dl)
        self.c_chain.bwd(dv)


class LSTMAgent(TensorCoreAgent):
    """Recurrent actor-critic (reference: cleanrl/ppo_atari_lstm.py:117-160): NatureCNN trunk over ONE grayscale frame,
    ``nn.LSTM(512, 128)`` with the state reset by ``(1 - done)`` before every step, ``actor`` / ``critic`` on the LSTM
    output.  Same module names / ``state_dict`` keys (``network.*``, ``lstm.weight_ih_l0`` ..., ``actor.*``, ``critic.*``),
    same initialisation order (orthogonal_ on the two LSTM weight matrices with gain 1, biases zero).

    Execution: fp32 kernels of libb200rl, no autograd.  The trunk and the input-gate GEMM ``x W_ih^T + b_ih`` run once over
    ALL steps of a sequence; per step there is one small GEMM ``h' W_hh^T + b_hh`` and one fused cell kernel.  The backward
    pass is explicit back-propagation through time (one cell-backward kernel + one ``dgates W_hh`` GEMM per step), after
    which the weight gradients of both LSTM matrices and of the trunk are single GEMMs over the whole sequence.
    ``precision = "bf16"`` runs the whole network on the tensor cores instead (ops.LSTMAgentBf16; uint8 frames
    [*, 1, 84, 84] only): one launch per sequence for the recurrence in each direction."""

    plan_class = ops.LSTMAgentBf16
    graph_capturable = False

    def __init__(self, envs):
        super().__init__()
        c, h, w = envs.single_observation_space.shape
        assert (h, w) == (84, 84), "NatureCNN trunk geometry is 84x84"
        trunk = []
        for cin, cout, k, s in ((c, 32, 8, 4), (32, 64, 4, 2), (64, 64, 3, 1)):
            trunk += [layer_init(nn.Conv2d(cin, cout, k, stride=s)), nn.ReLU()]
        trunk += [nn.Flatten(), layer_init(nn.Linear(64 * 7 * 7, 512)), nn.ReLU()]
        self.network = nn.Sequential(*trunk)
        self.lstm = nn.LSTM(512, 128)
        for name, param in self.lstm.named_parameters():
            if "bias" in name:
                nn.init.constant_(param, 0)
            elif "weight" in name:
                nn.init.orthogonal_(param, 1.0)
        self.actor = layer_init(nn.Linear(128, envs.single_action_space.n), std=0.01)
        self.critic = layer_init(nn.Linear(128, 1), std=1)
        self.num_actions = int(envs.single_action_space.n)
        self.hidden_size = 128

    def _param_order(self):
        net = [p for m in self.network for p in m.parameters()]
        return net + list(self.lstm.parameters()) + [self.actor.weight, self.critic.weight, self.actor.bias, self.critic.bias]

    def _build_plan(self):
        n = self.network
        self.trunk = nets.Chain([nets.Conv(n[0], "relu", in_div=255.0), nets.Conv(n[2], "relu"), nets.Conv(n[4], "relu"),
                                 nets.Linear(n[7], "relu")])
        self.head = self._joint_head()
        L = self.lstm
        self.l_ih = nets.Linear(None, None, L.weight_ih_l0.data, L.bias_ih_l0.data, L.weight_ih_l0.grad, L.bias_ih_l0.grad)
        self.l_hh = nets.Linear(None, None, L.weight_hh_l0.data, L.bias_hh_l0.data, L.weight_hh_l0.grad, L.bias_hh_l0.grad)

    def _tc_states(self, x, lstm_state, done, rows, keep):
        ops.LSTMAgentBf16.check_obs(x)
        H = self.hidden_size
        h0 = lstm_state[0].reshape(-1, H).to(torch.float32).contiguous()
        c0 = lstm_state[1].reshape(-1, H).to(torch.float32).contiguous()
        n = h0.shape[0]
        total = rows.numel() if rows is not None else x.shape[0]
        assert total % n == 0, "the sequence batch must be steps x envs"
        S = total // n
        done = done.reshape(-1).to(torch.float32).contiguous()
        x = x.contiguous()
        tc = self._tc_plan()
        self._tc_head, h, c = tc.forward(x, rows, S, n, self._flat.flat, h0, c0, done)
        if keep:
            self._tc_seq = (x, rows, S, n, done)
        return tc.act_tensors(S, n)["hseq"], (h.view(1, n, H), c.view(1, n, H))

    # ------------------------------------------------------------------ forward
    def get_states(self, x, lstm_state, done, rows=None, keep=False):
        """hidden [S*n, H], (h_S, c_S): ``x`` = S*n frames (or ``rows`` gathering them from a larger buffer), time-major."""
        self.flat
        if self.precision == "bf16":
            return self._tc_states(x, lstm_state, done, rows, keep)
        H = self.hidden_size
        h, c = lstm_state[0].reshape(-1, H).contiguous(), lstm_state[1].reshape(-1, H).contiguous()
        n = h.shape[0]
        if x.dtype not in (torch.uint8, torch.float32):
            x = x.float()
        feats = self.trunk.fwd(x.contiguous(), rows=rows, keep=keep)            # [S*n, 512], post-ReLU
        total = feats.shape[0]
        assert total % n == 0, "the sequence batch must be steps x envs"
        S = total // n
        dev = feats.device
        done = done.reshape(S, n).to(torch.float32).contiguous()
        gx = self.l_ih.fwd(feats)                                               # [S*n, 4H] for every step at once
        hidden = torch.empty(S, n, H, dtype=torch.float32, device=dev)
        hm = torch.empty(S, n, H, dtype=torch.float32, device=dev)
        cm = torch.empty(S, n, H, dtype=torch.float32, device=dev)
        save = torch.empty(S, n, 5 * H, dtype=torch.float32, device=dev) if keep else None
        c_cur = torch.empty(n, H, dtype=torch.float32, device=dev)
        for t in range(S):
            ops.lstm_mask_state(h, c, done[t], out=(hm[t], cm[t]))
            gh = self.l_hh.fwd(hm[t])
            ops.lstm_cell_fwd(gx[t * n:(t + 1) * n], gh, cm[t], hidden[t], c_cur, save[t] if keep else None)
            h, c = hidden[t], c_cur
            if t + 1 < S:
                c_cur = torch.empty(n, H, dtype=torch.float32, device=dev)
        if keep:
            self._seq = dict(feats=feats, hidden=hidden, hm=hm, cm=cm, save=save, done=done, S=S, n=n)
        return hidden.view(S * n, H), (h.reshape(1, n, H).clone(), c.reshape(1, n, H).clone())

    def _heads(self, hidden):
        # bf16: the forward that produced ``hidden`` computed the heads too
        out = self._tc_head if self.precision == "bf16" else self.head.fwd(hidden)
        A = self.num_actions
        return out[:, :A], out[:, A]

    def get_value(self, x, lstm_state, done):
        hidden, _ = self.get_states(x, lstm_state, done)
        _, value = self._heads(hidden)
        return value.reshape(-1, 1).clone()

    def get_action_and_value(self, x, lstm_state, done, action=None, rows=None, keep=False):
        hidden, lstm_state = self.get_states(x, lstm_state, done, rows=rows, keep=keep)
        logits, value = self._heads(hidden)
        if keep and self.precision != "bf16":
            self._seq["logits"], self._seq["value"] = logits, value
        m, A = logits.shape
        if action is None:
            q = self.noise_fn(m, A, logits.device)
            action, logprob, entropy, v = ops.categorical_sample(logits, q, value)
        else:
            logprob, entropy = ops.categorical_eval(logits, action)
            v = value.clone()
        return action, logprob, entropy, v.reshape(-1, 1), lstm_state

    def forward_train(self, b_obs, mb_inds, lstm_state, b_dones):
        """Minibatch forward over whole env sequences (mb_inds time-major: step t of every env of the minibatch, then
        step t+1, ... as cleanrl/ppo_atari_lstm.py:303), activations kept for ``backward``."""
        done = b_dones.reshape(-1)[mb_inds]
        hidden, _ = self.get_states(b_obs, lstm_state, done, rows=mb_inds, keep=True)
        return self._heads(hidden)

    # ----------------------------------------------------------------- backward
    def backward(self, dhead):
        if self.precision == "bf16":
            x, rows, S, n, done = self._tc_seq
            self._tc.backward(x, rows, S, n, self._flat.flat, done, dhead, self._flat.grad)
            self._tc_seq = None
            return
        q = self._seq
        S, n, H = q["S"], q["n"], self.hidden_size
        hidden = q["hidden"].view(S * n, H)
        self.head.bwd_weight(hidden, dhead)
        dh_heads = self.head.bwd_data(dhead, None, None).view(S, n, H)
        dev = dhead.device
        dgates = torch.empty(S, n, 4 * H, dtype=torch.float32, device=dev)
        dc_a = torch.empty(n, H, dtype=torch.float32, device=dev)
        dc_b = torch.empty(n, H, dtype=torch.float32, device=dev)
        dh_rec, dc_rec = None, None
        for t in reversed(range(S)):
            ops.lstm_cell_bwd(dh_heads[t], dh_rec, q["done"][t + 1] if t + 1 < S else None, dc_rec, q["save"][t], q["cm"][t],
                              q["done"][t], dgates[t], dc_a)
            dc_rec, dc_a, dc_b = dc_a, dc_b, dc_a
            if t > 0:
                dh_rec = self.l_hh.bwd_data(dgates[t], None, None)             # dgates_t W_hh -> d h'_{t-1} (masked at t-1's kernel)
        dg = dgates.view(S * n, 4 * H)
        self.l_hh.bwd_weight(q["hm"].view(S * n, H), dg)
        self.l_ih.bwd_weight(q["feats"], dg)
        dfeats = self.l_ih.bwd_data(dg, q["feats"], "relu")
        self.trunk.bwd(dfeats)
        self._seq = None


class ResidualBlock(nn.Module):
    """Parameter container with the reference's names (cleanrl/ppo_procgen.py:89-102); executed by ImpalaAgent."""

    def __init__(self, channels):
        super().__init__()
        self.conv0 = nn.Conv2d(in_channels=channels, out_channels=channels, kernel_size=3, padding=1)
        self.conv1 = nn.Conv2d(in_channels=channels, out_channels=channels, kernel_size=3, padding=1)


class ConvSequence(nn.Module):
    """cleanrl/ppo_procgen.py:105-124: conv3x3 -> max_pool(3, stride 2, padding 1) -> two residual blocks."""

    def __init__(self, input_shape, out_channels):
        super().__init__()
        self._input_shape = input_shape
        self._out_channels = out_channels
        self.conv = nn.Conv2d(in_channels=self._input_shape[0], out_channels=self._out_channels, kernel_size=3, padding=1)
        self.res_block0 = ResidualBlock(self._out_channels)
        self.res_block1 = ResidualBlock(self._out_channels)

    def get_output_shape(self):
        _c, h, w = self._input_shape
        return (self._out_channels, (h + 1) // 2, (w + 1) // 2)


class ImpalaAgent(TensorCoreAgent):
    """IMPALA-CNN actor-critic (reference: cleanrl/ppo_procgen.py:89-150): three ConvSequences (16, 32, 32 channels),
    Flatten, ReLU, Linear(2048 -> 256), ReLU, ``actor`` / ``critic``.  Same module tree (``network.{0,1,2}.conv``,
    ``network.{0,1,2}.res_block{0,1}.conv{0,1}``, ``network.5``), same construction order, torch's default initialisation
    for the trunk (the reference only ``layer_init``s the heads), so a seed yields the reference's weights and
    ``state_dict`` files interchange.  Frames arrive NHWC uint8 ([n, 64, 64, 3]) and are permuted on the device.

    Execution: fp32 kernels of libb200rl (padded 3x3 convolutions, max-pool with arg-max, ReLU / add glue), explicit
    backward in reverse order; no autograd, no cuDNN.  ``precision = "bf16"`` runs the whole network on the tensor
    cores instead (ops.ImpalaCNNBf16, csrc/net_impala_tc.cu; uint8 frames [*, 64, 64, 3] only)."""

    plan_class = ops.ImpalaCNNBf16

    def __init__(self, envs):
        super().__init__()
        h, w, c = envs.single_observation_space.shape
        shape = (c, h, w)
        conv_seqs = []
        for out_channels in [16, 32, 32]:
            conv_seq = ConvSequence(shape, out_channels)
            shape = conv_seq.get_output_shape()
            conv_seqs.append(conv_seq)
        conv_seqs += [nn.Flatten(), nn.ReLU(),
                      nn.Linear(in_features=shape[0] * shape[1] * shape[2], out_features=256), nn.ReLU()]
        self.network = nn.Sequential(*conv_seqs)
        self.actor = layer_init(nn.Linear(256, envs.single_action_space.n), std=0.01)
        self.critic = layer_init(nn.Linear(256, 1), std=1)
        self.num_actions = int(envs.single_action_space.n)
        self._feat_shape = shape

    def _param_order(self):
        net = [p for p in self.network.parameters()]
        return net + [self.actor.weight, self.critic.weight, self.actor.bias, self.critic.bias]

    def _build_plan(self):
        self.head = self._joint_head()
        self.fc = nets.Linear(self.network[5], "relu")
        self.seqs = []
        for i in range(3):
            q = self.network[i]
            self.seqs.append(dict(conv=nets.Conv(q.conv, None, in_div=255.0 if i == 0 else 1.0),
                                  blocks=[(nets.Conv(b.conv0, "relu"), nets.Conv(b.conv1, None))
                                          for b in (q.res_block0, q.res_block1)]))

    # ------------------------------------------------------------------ forward
    def _forward_heads(self, x, rows=None, keep=False):
        out = self._head_out(x, rows, keep)
        A = self.num_actions
        return out[:, :A], out[:, A]

    def _head_out(self, x, rows=None, keep=False):
        """The joint head's output [n, _head_outputs()] for frames ``x[rows]``."""
        if x.dtype != torch.uint8:
            x = x.to(torch.uint8)          # frames are integers 0..255 (the reference passes them as fp32)
        if self.precision == "bf16":
            ops.ImpalaCNNBf16.check_obs(x)
            out = self._tc_plan().forward(x.contiguous(), rows, self._flat.flat)
            if keep:
                self._tc_obs, self._tc_rows = x, rows
            return out
        x = ops.nhwc_to_nchw_u8(x.contiguous(), rows)          # [n, 3, 64, 64] uint8; /255 inside the first convolution
        saved = []
        h = x
        for s in self.seqs:
            c = s["conv"].fwd(h)                               # conv, no activation
            p, arg = ops.maxpool3s2_fwd(c)
            rec = dict(x=h, c_hw=tuple(c.shape[-2:]), arg=arg, blocks=[])
            b = p
            for conv0, conv1 in s["blocks"]:
                r0 = ops.relu(b)                               # x -> relu -> conv0 -> relu -> conv1 -> + x
                y0 = conv0.fwd(r0)                             # relu fused on the output (the next op is a relu)
                c1 = conv1.fwd(y0)
                out = ops.add(c1, b)
                rec["blocks"].append((r0, y0))
                b = out
            saved.append(rec)
            h = b
        flat = h.reshape(h.shape[0], -1)
        h0 = ops.relu(flat)                                    # Flatten, ReLU
        hid = self.fc.fwd(h0)                                  # Linear + ReLU
        out = self.head.fwd(hid)
        if keep:
            self._saved = dict(seqs=saved, h0=h0, hid=hid, last_shape=tuple(h.shape))
        return out

    def forward_train(self, b_obs, mb_inds):
        self.flat
        return self._forward_heads(b_obs, rows=mb_inds, keep=True)

    # ----------------------------------------------------------------- backward
    def backward(self, dhead):
        if self.precision == "bf16":
            self._tc.backward(self._tc_obs, self._tc_rows, self._flat.flat, dhead, self._flat.grad)
            self._tc_obs = self._tc_rows = None
            return
        q = self._saved
        self.head.bwd_weight(q["hid"], dhead)
        d_hid = self.head.bwd_data(self._dhead_into_hidden(dhead), q["hid"], "relu")   # through the ReLU after the Linear
        self.fc.bwd_weight(q["h0"], d_hid)
        d = self.fc.bwd_data(d_hid, q["h0"], "relu").view(q["last_shape"])     # through the ReLU after Flatten
        for si in (2, 1, 0):
            s, rec = self.seqs[si], q["seqs"][si]
            for (conv0, conv1), (r0, y0) in zip(reversed(s["blocks"]), reversed(rec["blocks"])):
                conv1.bwd_weight(y0, d)
                dy0 = conv1.bwd_data(d, y0, "relu")                            # * (y0 > 0)
                conv0.bwd_weight(r0, dy0)
                d_in = conv0.bwd_data(dy0, None, None, in_hw=tuple(r0.shape[-2:]))
                d = ops.relu_bwd(d_in, r0, extra=d)                            # * (x > 0) + skip connection
            d_c = ops.maxpool3s2_bwd(d, rec["arg"], rec["c_hw"])
            s["conv"].bwd_weight(rec["x"], d_c)
            if si > 0:
                d = s["conv"].bwd_data(d_c, None, None, in_hw=tuple(rec["x"].shape[-2:]))
        self._saved = None

    def _dhead_into_hidden(self, dhead):
        """The head gradient that flows on into the hidden layer (all of it: every head reads ``hidden``)."""
        return dhead


def layer_init_normed(layer, norm_dim, scale=1.0):
    """cleanrl/ppg_procgen.py:101-105: every output unit rescaled to L2 norm ``scale``, bias zeroed; consumes no RNG."""
    with torch.no_grad():
        layer.weight.data *= scale / layer.weight.norm(dim=norm_dim, p=2, keepdim=True)
        layer.bias *= 0
    return layer


class PPGResidualBlock(nn.Module):
    """Parameter container with the reference's names and initialisation (cleanrl/ppg_procgen.py:124-132)."""

    def __init__(self, channels, scale):
        super().__init__()
        scale = np.sqrt(scale)
        conv0 = nn.Conv2d(in_channels=channels, out_channels=channels, kernel_size=3, padding=1)
        self.conv0 = layer_init_normed(conv0, norm_dim=(1, 2, 3), scale=scale)
        conv1 = nn.Conv2d(in_channels=channels, out_channels=channels, kernel_size=3, padding=1)
        self.conv1 = layer_init_normed(conv1, norm_dim=(1, 2, 3), scale=scale)


class PPGConvSequence(nn.Module):
    """cleanrl/ppg_procgen.py:143-165: conv3x3 -> max_pool(3, stride 2, padding 1) -> two residual blocks."""

    def __init__(self, input_shape, out_channels, scale):
        super().__init__()
        self._input_shape = input_shape
        self._out_channels = out_channels
        conv = nn.Conv2d(in_channels=self._input_shape[0], out_channels=self._out_channels, kernel_size=3, padding=1)
        self.conv = layer_init_normed(conv, norm_dim=(1, 2, 3), scale=1.0)
        nblocks = 2
        scale = scale / np.sqrt(nblocks)
        self.res_block0 = PPGResidualBlock(self._out_channels, scale=scale)
        self.res_block1 = PPGResidualBlock(self._out_channels, scale=scale)

    def get_output_shape(self):
        _c, h, w = self._input_shape
        return (self._out_channels, (h + 1) // 2, (w + 1) // 2)


class PPGAgent(ImpalaAgent):
    """IMPALA-CNN agent of phasic policy gradient (reference: cleanrl/ppg_procgen.py:168-211): the ImpalaAgent trunk with
    ``layer_init_normed`` initialisation and three heads, ``actor``, ``critic`` and ``aux_critic``.  Same module tree and
    ``state_dict`` keys, same construction order, so a seed yields the reference's weights.

    The three heads run as ONE joint head of A + 2 outputs, [logits | value | aux_value].  ``critic`` reads
    ``hidden.detach()`` in every method of the reference: its column of the head gradient reaches ``critic.weight`` and
    ``critic.bias`` only and is left out of the hidden layer's gradient (fp32: a copy of ``dhead`` with that column zeroed;
    bf16: ops.ImpalaPPGBf16 skips the column)."""

    plan_class = ops.ImpalaPPGBf16

    def __init__(self, envs):
        TensorCoreAgent.__init__(self)
        h, w, c = envs.single_observation_space.shape
        shape = (c, h, w)
        conv_seqs = []
        chans = [16, 32, 32]
        scale = 1 / np.sqrt(len(chans))
        for out_channels in chans:
            conv_seq = PPGConvSequence(shape, out_channels, scale=scale)
            shape = conv_seq.get_output_shape()
            conv_seqs.append(conv_seq)
        encodertop = nn.Linear(in_features=shape[0] * shape[1] * shape[2], out_features=256)
        encodertop = layer_init_normed(encodertop, norm_dim=1, scale=1.4)
        conv_seqs += [nn.Flatten(), nn.ReLU(), encodertop, nn.ReLU()]
        self.network = nn.Sequential(*conv_seqs)
        self.actor = layer_init_normed(nn.Linear(256, envs.single_action_space.n), norm_dim=1, scale=0.1)
        self.critic = layer_init_normed(nn.Linear(256, 1), norm_dim=1, scale=0.1)
        self.aux_critic = layer_init_normed(nn.Linear(256, 1), norm_dim=1, scale=0.1)
        self.num_actions = int(envs.single_action_space.n)
        if self.num_actions + 2 > 24:
            raise ValueError(f"PPGAgent supports at most 22 actions (got {self.num_actions})")
        self._feat_shape = shape

    def _param_order(self):
        net = [p for p in self.network.parameters()]
        return net + [self.actor.weight, self.critic.weight, self.aux_critic.weight,
                      self.actor.bias, self.critic.bias, self.aux_critic.bias]

    def _head_outputs(self):
        return self.num_actions + 2          # actor + critic + aux_critic

    def _plan_actions(self):
        return self.num_actions

    def aux_critic_ranges(self):
        """Element ranges [(lo, hi), ...] of ``aux_critic.weight`` and ``aux_critic.bias`` in the flat parameter vector."""
        f = self.flat
        out = []
        for p in (self.aux_critic.weight, self.aux_critic.bias):
            lo = (f.view_of(p)[0].data_ptr() - f.flat.data_ptr()) // 4
            out.append((lo, lo + p.numel()))
        return out

    def alloc_head_grad(self, M, device):
        """(dhead [M, A+2], its dlogits view, its dvalue view); the ``aux_value`` column stays zero: the policy phase's
        loss does not read ``aux_critic``."""
        A = self.num_actions
        d = torch.zeros(M, A + 2, dtype=torch.float32, device=device)
        return d, d[:, :A], d[:, A]

    def _dhead_into_hidden(self, dhead):
        d = dhead.clone()
        d[:, self.num_actions] = 0           # critic(hidden.detach())
        return d

    def forward_aux(self, b_obs, rows):
        """Auxiliary-phase forward over ``b_obs[rows]`` (gather fused, activations kept): [n, A + 2]."""
        self.flat
        return self._head_out(b_obs, rows=rows, keep=True)

    # -- reference API (cleanrl/ppg_procgen.py:205-211)
    def get_pi_value_and_aux_value(self, x):
        """(normalised logits [n, A] as ``Categorical.logits``, value [n, 1], aux_value [n, 1])."""
        self.flat
        out = self._head_out(x)
        A = self.num_actions
        lg = out[:, :A]
        return lg - lg.logsumexp(dim=-1, keepdim=True), out[:, A:A + 1].clone(), out[:, A + 1:A + 2].clone()

    def get_pi(self, x, rows=None):
        """Normalised logits [n, A] of the policy for ``x`` (or ``x[rows]``, gathered by the network), as
        ``Categorical(logits=...).logits``."""
        self.flat
        out = self._head_out(x, rows=rows)
        lg = out[:, :self.num_actions]
        return lg - lg.logsumexp(dim=-1, keepdim=True)


def _normal_noise(n, D, device):
    # what Normal(mean, std).sample() == torch.normal(mean, std) consumes: one N(0,1) per element
    return torch.randn(n, D, dtype=torch.float32, device=device)


_normal_noise.graph_safe = True
_normal_noise.inplace = lambda buf: buf.normal_(0, 1)


class ContinuousMLPAgent(KernelAgent):
    """Gaussian-policy MLP agent (reference: cleanrl/ppo_continuous_action.py:112-141): ``critic`` and
    ``actor_mean`` Sequentials plus the state-independent ``actor_logstd`` parameter [1, D]."""

    def __init__(self, envs):
        super().__init__()
        d = int(np.array(envs.single_observation_space.shape).prod())
        D = int(np.prod(envs.single_action_space.shape))
        self.critic = nn.Sequential(layer_init(nn.Linear(d, 64)), nn.Tanh(), layer_init(nn.Linear(64, 64)), nn.Tanh(),
                                    layer_init(nn.Linear(64, 1), std=1.0))
        self.actor_mean = nn.Sequential(layer_init(nn.Linear(d, 64)), nn.Tanh(), layer_init(nn.Linear(64, 64)), nn.Tanh(),
                                        layer_init(nn.Linear(64, D), std=0.01))
        self.actor_logstd = nn.Parameter(torch.zeros(1, D))
        self.action_dim = D
        self.noise_fn = _normal_noise

    def _build_plan(self):
        mk = lambda seq: nets.Chain([nets.Linear(seq[0], "tanh"), nets.Linear(seq[2], "tanh"), nets.Linear(seq[4], None)])
        self.c_chain, self.a_chain = mk(self.critic), mk(self.actor_mean)

    def _forward_heads(self, x, rows=None, keep=False):
        x = x.float() if x.dtype != torch.float32 else x
        x = x.reshape(x.shape[0], -1).contiguous()
        mean = self.a_chain.fwd(x, rows=rows, keep=keep)
        value = self.c_chain.fwd(x, rows=rows, keep=keep)
        return mean, value[:, 0]

    def forward_train(self, b_obs, mb_inds):
        self.flat
        return self._forward_heads(b_obs, rows=mb_inds, keep=True)

    def _logstd(self):
        return self.actor_logstd.data.view(-1)

    def noise_shape(self, n):
        return (n, self.action_dim)

    def sample_into(self, obs, actions_out, logprobs_out, values_out, noise=None):
        mean, value = self._forward_heads(obs)
        n, D = mean.shape
        eps = noise if noise is not None else self.noise_fn(n, D, mean.device)
        ops.gaussian_sample(mean, self._logstd(), eps, value, out=(actions_out, logprobs_out, None, values_out))

    def loss_backward(self, policy_out, value, mb_inds, b, a, stats_row, scratch, mean_shift=None):
        M, D = policy_out.shape
        dev = policy_out.device
        if scratch.get("M") != M:
            scratch["M"] = M
            scratch["dmean"] = torch.empty(M, D, dtype=torch.float32, device=dev)
            scratch["dv"] = torch.empty(M, 1, dtype=torch.float32, device=dev)
        ops.ppo_loss_gaussian(policy_out, self._logstd(), value, mb_inds, b["actions"], b["logprobs"], b["advantages"],
                              b["returns"], b["values"], a.clip_coef, a.ent_coef, a.vf_coef, a.norm_adv, a.clip_vloss,
                              dmean=scratch["dmean"], dlogstd=self.actor_logstd.grad.view(-1), dvalue=scratch["dv"][:, 0],
                              stats=stats_row, mean_shift=mean_shift)
        self.a_chain.bwd(scratch["dmean"])
        self.c_chain.bwd(scratch["dv"])

    def get_action_and_value(self, x, action=None):
        self.flat
        mean, value = self._forward_heads(x)
        n, D = mean.shape
        if action is None:
            eps = self.noise_fn(n, D, mean.device)
            action, logprob, entropy, v = ops.gaussian_sample(mean, self._logstd(), eps, value)
        else:
            logprob, entropy = ops.gaussian_eval(mean, self._logstd(), action)
            v = value.clone() if not value.is_contiguous() else value
        return action, logprob, entropy, v.reshape(-1, 1)


class RPOAgent(ContinuousMLPAgent):
    """Robust policy optimization (reference: cleanrl/rpo_continuous_action.py:108-144): the continuous PPO agent (same
    modules, initialisation and state_dict keys) whose update evaluates the stored actions under
    ``Normal(mean + z, std)``, with z ~ U(-rpo_alpha, rpo_alpha) per row and action dimension from the CPU generator.

    The reference draws one [M, D] z per minibatch and copies it to the device.  ``begin_update_epoch`` draws the
    epoch's whole [B, D] instead, into the epoch's pinned slot, and uploads it with one asynchronous copy; minibatch
    ``mb_start`` reads rows [mb_start, mb_start + M).  CPU ``uniform_`` fills a tensor in order, so one [B, D] draw is
    the concatenation of the reference's per-minibatch draws, and the reference tests ``target_kl`` only after a whole
    epoch, so no draw is made that the reference would not make."""

    def __init__(self, envs, rpo_alpha):
        super().__init__(envs)
        self.rpo_alpha = rpo_alpha
        self._z_h = None       # pinned [update_epochs, B, D]: one slot per epoch, never rewritten while its copy is queued
        self._z = None         # device [B, D]: the current epoch's draws

    def begin_update_epoch(self, epoch, num_epochs, batch_size):
        """Draw and upload the mean shifts of update epoch ``epoch`` (PPOEngine calls it before the epoch's minibatches)."""
        D = self.action_dim
        if self._z_h is None or tuple(self._z_h.shape) != (num_epochs, batch_size, D):
            z_h = torch.empty(num_epochs, batch_size, D, dtype=torch.float32)
            self._z_h = z_h.pin_memory() if torch.cuda.is_available() else z_h
            self._z = torch.empty(batch_size, D, dtype=torch.float32, device=self.actor_logstd.device)
        self._z_h[epoch].uniform_(-self.rpo_alpha, self.rpo_alpha)
        self._z.copy_(self._z_h[epoch], non_blocking=True)

    def loss_backward(self, policy_out, value, mb_inds, b, a, stats_row, scratch, mb_start=0):
        if self._z is None:
            raise RuntimeError("RPOAgent.loss_backward: no mean shifts drawn; call begin_update_epoch first")
        M = policy_out.shape[0]
        super().loss_backward(policy_out, value, mb_inds, b, a, stats_row, scratch,
                              mean_shift=self._z[mb_start:mb_start + M])

    def get_action_and_value(self, x, action=None):
        if action is None:
            return super().get_action_and_value(x)
        self.flat
        mean, value = self._forward_heads(x)
        z = torch.empty(mean.shape, dtype=torch.float32).uniform_(-self.rpo_alpha, self.rpo_alpha).to(mean.device)
        logprob, entropy = ops.gaussian_eval(mean + z, self._logstd(), action)
        v = value.clone() if not value.is_contiguous() else value
        return action, logprob, entropy, v.reshape(-1, 1)


class QNetworkAgent(TensorCoreAgent):
    """DQN Q-network (reference: cleanrl/dqn_atari.py:108-125): NatureCNN trunk + Linear(512, A), default torch
    initialisation, ``forward(x)`` -> Q-values [n, A]; state_dict keys ``network.{0,2,4,7,9}.*``.  Its natural parameter
    order is libb200rl's NatureCNN order; the bf16 plan's W-wide head is the NatureCNN's (W-1) + 1 heads."""

    plan_class = ops.NatureCNNBf16

    def __init__(self, env):
        super().__init__()
        A = int(env.single_action_space.n)
        self.network = nn.Sequential(
            nn.Conv2d(4, 32, 8, stride=4), nn.ReLU(), nn.Conv2d(32, 64, 4, stride=2), nn.ReLU(),
            nn.Conv2d(64, 64, 3, stride=1), nn.ReLU(), nn.Flatten(), nn.Linear(3136, 512), nn.ReLU(), nn.Linear(512, A))
        self.num_actions = A

    def _build_plan(self):
        n = self.network
        self.chain = nets.Chain([nets.Conv(n[0], "relu", in_div=255.0), nets.Conv(n[2], "relu"), nets.Conv(n[4], "relu"),
                                 nets.Linear(n[7], "relu"), nets.Linear(n[9], None)])

    def _head_outputs(self):
        return self.num_actions

    def q_values(self, frames, rows=None, keep=False):
        """Q(s, .) for frames[rows] (uint8 [*,4,84,84]; rows gathers without materialising)."""
        self.flat
        if frames.dtype != torch.uint8:
            frames = frames.to(torch.uint8)
        if self.precision == "bf16":
            out = self._tc_plan().forward(frames.contiguous(), rows, self._flat.flat)
            if keep:
                self._saved = (frames, rows)
            return out
        return self.chain.fwd(frames.contiguous(), rows=rows, keep=keep)

    def forward(self, x):
        return self.q_values(x)

    def backward(self, dq):
        if self.precision == "bf16":
            frames, rows = self._saved
            self._tc.backward(frames, rows, self._flat.flat, dq, self._flat.grad)
            self._saved = None
        else:
            self.chain.bwd(dq)


def dqn_update(q_network, target_network, ring, batch, gamma, lr, huber=False, stats=None):
    """One TD update (reference: dqn_atari.py:219-235): target forward, online forward, fused TD loss + dL/dQ,
    hand-written backward, Adam (torch defaults eps=1e-8, no gradient clipping)."""
    frames = ring.frames
    with torch.no_grad():
        qt = target_network.q_values(frames, rows=batch["next_rows"])
        q = q_network.q_values(frames, rows=batch["rows"], keep=True)
        stats, dq = ops.dqn_td_loss(q, qt, batch["actions"], batch["rewards"], batch["dones"], gamma, huber=huber, stats=stats)
        q_network.backward(dq)
        f = q_network.flat
        f.step += 1
        ops.clip_adam(f.flat, f.grad, f.exp_avg, f.exp_avg_sq, f.step, lr, eps=1e-8, max_norm=None)
        q_network.params_updated()
    return stats


class C51QNetwork(QNetworkAgent):
    """C51 distributional Q-network (reference: cleanrl/c51_atari.py:111-138): NatureCNN trunk + Linear(512, A * n_atoms),
    default torch initialisation, the ``atoms`` buffer (linspace(v_min, v_max, n_atoms)); state_dict keys
    ``atoms, network.{0,2,4,7,9}.*``.  ``get_action(x, action=None)`` -> (action [n], pmf [n, n_atoms]) runs the head
    softmax / expectation / argmax in one kernel.  The bf16 path is the tensor-core NatureCNN with an A * n_atoms-wide
    head (wgmma); fp32 is the exact CUDA-core chain."""

    def __init__(self, env, n_atoms=101, v_min=-100, v_max=100):
        TensorCoreAgent.__init__(self)
        self.n_atoms = n_atoms
        self.register_buffer("atoms", torch.linspace(v_min, v_max, steps=n_atoms))
        self.n = int(env.single_action_space.n)
        self.network = nn.Sequential(
            nn.Conv2d(4, 32, 8, stride=4), nn.ReLU(), nn.Conv2d(32, 64, 4, stride=2), nn.ReLU(),
            nn.Conv2d(64, 64, 3, stride=1), nn.ReLU(), nn.Flatten(), nn.Linear(3136, 512), nn.ReLU(),
            nn.Linear(512, self.n * n_atoms))
        self.num_actions = self.n

    def _head_outputs(self):
        return self.n * self.n_atoms

    def logits(self, frames, rows=None, keep=False):
        """Head logits [n, A * n_atoms] for frames[rows]."""
        return self.q_values(frames, rows=rows, keep=keep)

    def forward(self, x):
        return self.logits(x)

    def get_action(self, x, action=None):
        self.flat
        act, _, pmf = ops.c51_act(self.logits(x), self.atoms, action)
        return act, pmf


def c51_update(q_network, target_network, ring, batch, gamma, lr, v_min, v_max, batch_size, stats=None):
    """One C51 update (reference: c51_atari.py:232-265): target forward on next_rows, online forward on rows (activations
    kept), fused projection + cross-entropy + dL/dlogits, hand-written backward, Adam with eps = 0.01 / batch_size and no
    gradient clipping."""
    frames = ring.frames
    with torch.no_grad():
        lt = target_network.logits(frames, rows=batch["next_rows"])
        lo = q_network.logits(frames, rows=batch["rows"], keep=True)
        stats, dl = ops.c51_loss(lo, lt, target_network.atoms, batch["actions"], batch["rewards"], batch["dones"],
                                 gamma, v_min, v_max, stats=stats)
        q_network.backward(dl)
        f = q_network.flat
        f.step += 1
        ops.clip_adam(f.flat, f.grad, f.exp_avg, f.exp_avg_sq, f.step, lr, eps=0.01 / batch_size, max_norm=None)
        q_network.params_updated()
    return stats


def dqn_sync_target(q_network, target_network, tau=1.0):
    """dqn_atari.py:238-242: target <- tau * online + (1 - tau) * target (flat buffers, one fused axpby)."""
    t, q = target_network.flat.flat, q_network.flat.flat
    if tau == 1.0:
        t.copy_(q)
    else:
        t.mul_(1.0 - tau).add_(q, alpha=tau)
    target_network.params_updated()


# ------------------------------------------------------------------------ discrete SAC (cleanrl/sac_atari.py)
def sac_layer_init(layer, bias_const=0.0):
    """sac_atari.py:102-105: kaiming-normal weight, constant bias."""
    nn.init.kaiming_normal_(layer.weight)
    torch.nn.init.constant_(layer.bias, bias_const)
    return layer


class _SACNet(QNetworkAgent):
    """NatureCNN with an A-wide head under the reference's SAC module names: ``conv`` (Conv2d 0/2/4, ReLU, Flatten),
    ``fc1`` and the head ``head_name``, initialised by ``sac_layer_init`` in the reference's construction order (each
    layer's default initialisation, then kaiming: the same generator consumption).  The parameter order is the NatureCNN
    plan's, so the bf16 plan and the fp32 chain of ``QNetworkAgent`` run it unchanged."""

    head_name = None

    def __init__(self, envs):
        TensorCoreAgent.__init__(self)
        obs_shape = tuple(envs.single_observation_space.shape)
        assert obs_shape == (4, 84, 84), "NatureCNN geometry is 4x84x84"
        self.conv = nn.Sequential(
            sac_layer_init(nn.Conv2d(obs_shape[0], 32, kernel_size=8, stride=4)), nn.ReLU(),
            sac_layer_init(nn.Conv2d(32, 64, kernel_size=4, stride=2)), nn.ReLU(),
            sac_layer_init(nn.Conv2d(64, 64, kernel_size=3, stride=1)), nn.Flatten())
        self.fc1 = sac_layer_init(nn.Linear(64 * 7 * 7, 512))
        setattr(self, self.head_name, sac_layer_init(nn.Linear(512, envs.single_action_space.n)))
        self.num_actions = int(envs.single_action_space.n)

    def _layers(self, in_div):
        c = self.conv
        return nets.Chain([nets.Conv(c[0], "relu", in_div=in_div), nets.Conv(c[2], "relu"), nets.Conv(c[4], "relu"),
                           nets.Linear(self.fc1, "relu"), nets.Linear(getattr(self, self.head_name), None)])

    def _build_plan(self):
        self.chain = self._layers(255.0)


class SoftQNetwork(_SACNet):
    """sac_atari.py:112-135: ``forward(x)`` takes frames (0..255) and returns Q-values [n, A]."""

    head_name = "fc_q"


class SACActor(_SACNet):
    """sac_atari.py:138-171.  ``forward(x)`` takes frames already divided by 255 and returns logits; ``get_action(x)``
    takes frames and returns (action, log_softmax, probs): the action is ``ops.categorical_sample`` on ``noise_fn``'s
    exponential noise (bit-identical to ``Categorical.sample()`` under the same generator state)."""

    head_name = "fc_logits"

    def _build_plan(self):
        super()._build_plan()
        self.chain_scaled = self._layers(1.0)

    def logits(self, frames, rows=None, keep=False):
        return self.q_values(frames, rows=rows, keep=keep)

    def forward(self, x):
        self.flat
        if self.precision == "bf16":
            # the tensor-core plan consumes frames: x * 255 restores them exactly for inputs that were frames / 255
            return self.q_values(torch.round(x.float() * 255.0).clamp_(0, 255).to(torch.uint8))
        return self.chain_scaled.fwd(x.float().contiguous())

    def get_action(self, x):
        logits = self.logits(x)
        n, A = logits.shape
        action, _, _, _ = ops.categorical_sample(logits, self.noise_fn(n, A, logits.device))
        log_prob, probs = ops.sac_policy(logits)
        return action, log_prob, probs


SAC_ADAM_EPS = 1e-4          # all three optimisers (sac_atari.py:215-223)


class SACState:
    """The device-resident part of a SAC update that is not a network: the temperature (``alpha`` f32[1], and with
    autotune ``log_alpha`` and its Adam moments), the update count, the logged statistics (``qstats`` =
    ``ops.SAC_CRITIC_STAT_NAMES``, ``astats`` = ``ops.SAC_ACTOR_STAT_NAMES``) and the scratch of the update.  A bf16
    update whose noise draw is graph-safe is replayed as one CUDA graph (``use_graph``) up to ``graph_max_batch`` rows:
    on an H100 the replay saved 0.1-0.6 ms of a 1.5-2 ms update at batch 64 (launch-bound) and was 0.15-0.2 ms slower
    than eager launches at batch 1024 (bench_sac.py)."""

    use_graph = True
    graph_max_batch = 256

    def __init__(self, num_actions, device, autotune=True, alpha=0.2, target_entropy_scale=0.89):
        f32 = torch.float32
        self.A, self.device, self.autotune = int(num_actions), device, bool(autotune)
        # -scale * log(1 / A) as the reference evaluates it: fp32 tensor arithmetic (sac_atari.py:226)
        self.target_entropy = float(-target_entropy_scale * torch.log(1 / torch.tensor(self.A)))
        self.log_alpha = torch.zeros(1, dtype=f32, device=device)
        self.alpha = torch.full((1,), 1.0 if autotune else float(alpha), dtype=f32, device=device)
        self.exp_avg = torch.zeros(1, dtype=f32, device=device)
        self.exp_avg_sq = torch.zeros(1, dtype=f32, device=device)
        self.qstats = torch.zeros(4, dtype=f32, device=device)
        self.astats = torch.zeros(4, dtype=f32, device=device)
        self.step = 0
        self._bufs = {}
        self._graphs = {}
        self._pool = None

    def buffers(self, B):
        """Fixed scratch of a batch size: dq1, dq2, dlogits, y, the two noise draws, the loss kernels' workspaces and the
        graph's input slots."""
        b = self._bufs.get(B)
        if b is None:
            f32, dev, A = torch.float32, self.device, self.A
            b = {k: torch.zeros(B, A, dtype=f32, device=dev) for k in ("dq1", "dq2", "dl", "noise1", "noise2")}
            b["y"] = torch.zeros(B, dtype=f32, device=dev)
            b["rows"] = torch.zeros(B, dtype=torch.int64, device=dev)
            b["actions"] = torch.zeros(B, dtype=torch.int64, device=dev)
            b["rewards"] = torch.zeros(B, dtype=f32, device=dev)
            b["dones"] = torch.zeros(B, dtype=f32, device=dev)
            b["dyn"] = torch.zeros(6, dtype=f32, device=dev)
            lib = ops._lib.load()
            b["ws_critic"] = torch.zeros(lib.b200rl_sac_critic_loss_workspace_bytes(B), dtype=torch.uint8, device=dev)
            b["ws_actor"] = torch.zeros(lib.b200rl_sac_actor_loss_workspace_bytes(B), dtype=torch.uint8, device=dev)
            self._bufs[B] = b
        return b

    def step_scalars(self, step, q_lr, policy_lr):
        """``adam_step_scalars`` of the q, actor and temperature optimisers (the last uses q_lr, sac_atari.py:223)."""
        return ops.adam_step_scalars(step, q_lr) + ops.adam_step_scalars(step, policy_lr) + ops.adam_step_scalars(step, q_lr)


def _sac_update_body(actor, qf1, qf2, qf1_target, qf2_target, frames, next_frames, rows, next_rows, actions, rewards, dones,
                     st, buf, dyn, gamma):
    """Steps 1-4 of sac_atari.py:271-314 on device buffers; every (step, lr) scalar comes from ``dyn`` (device f32[6])."""
    # 1. soft-Q target: the actor on next_obs (its sample is drawn and not used) and both target networks
    nl = actor.logits(next_frames, rows=next_rows)
    actor.draw_noise_into(buf["noise1"])
    q1t = qf1_target.q_values(next_frames, rows=next_rows)
    q2t = qf2_target.q_values(next_frames, rows=next_rows)
    # 2. critic loss, backward and the q optimiser (qf1 and qf2 are separate flat buffers; Adam is elementwise)
    q1 = qf1.q_values(frames, rows=rows, keep=True)
    q2 = qf2.q_values(frames, rows=rows, keep=True)
    ops.sac_critic_loss(nl, q1t, q2t, q1, q2, actions, rewards, dones, gamma, st.alpha, y=buf["y"], dq1=buf["dq1"],
                        dq2=buf["dq2"], stats=st.qstats, workspace=buf["ws_critic"])
    qf1.backward(buf["dq1"])
    qf2.backward(buf["dq2"])
    for q in (qf1, qf2):
        f = q.flat
        ops.clip_adam_dyn(f.flat, f.grad, f.exp_avg, f.exp_avg_sq, dyn[0:2], eps=SAC_ADAM_EPS, max_norm=None)
        q.params_updated()
    # 3. actor loss on the post-step Q values (the plans repack before these forwards), backward, actor optimiser;
    # 4. the temperature step inside the same kernel, after every row has used the old alpha
    lo = actor.logits(frames, rows=rows, keep=True)
    actor.draw_noise_into(buf["noise2"])
    q1 = qf1.q_values(frames, rows=rows)
    q2 = qf2.q_values(frames, rows=rows)
    if st.autotune:
        ops.sac_actor_loss(lo, q1, q2, st.alpha, st.target_entropy, st.log_alpha, st.exp_avg, st.exp_avg_sq, dyn[4:6],
                           eps=SAC_ADAM_EPS, dlogits=buf["dl"], stats=st.astats, workspace=buf["ws_actor"])
    else:
        ops.sac_actor_loss(lo, q1, q2, st.alpha, dlogits=buf["dl"], stats=st.astats, workspace=buf["ws_actor"])
    actor.backward(buf["dl"])
    f = actor.flat
    ops.clip_adam_dyn(f.flat, f.grad, f.exp_avg, f.exp_avg_sq, dyn[2:4], eps=SAC_ADAM_EPS, max_norm=None)
    actor.params_updated()


@torch.no_grad()
def sac_update(actor, qf1, qf2, qf1_target, qf2_target, ring, batch, state, gamma, q_lr, policy_lr):
    """One discrete-SAC update (reference: sac_atari.py:271-314) on a ``DeviceReplayRing`` batch: three actor / target
    forwards on next_obs, the fused soft-Q target + critic loss, both critic backwards and Adam steps, the actor forward
    and the post-step Q forwards, the fused actor loss + temperature step, the actor backward and Adam step.  Adam
    eps = 1e-4, no clipping.  Two [B, A] noise draws stand for the reference's two unused ``Categorical.sample()`` calls,
    so the rollout's actions stay on its generator stream.  Nothing is read back to the host; the statistics are in
    ``state.qstats`` / ``state.astats``.  bf16 with a graph-safe noise draw and at most ``state.graph_max_batch`` rows
    replays one CUDA graph per batch size."""
    B = int(batch["rows"].numel())
    buf = state.buffers(B)
    state.step += 1
    for net in (qf1, qf2, actor):
        net.flat.step = state.step
    buf["dyn"].copy_(torch.tensor(state.step_scalars(state.step, q_lr, policy_lr), dtype=torch.float32), non_blocking=True)
    nets_ = (actor, qf1, qf2, qf1_target, qf2_target)
    graph = state.use_graph and B <= state.graph_max_batch and all(n.uses_tc_plan() for n in nets_) and actor.graph_friendly
    args = (ring.frames, ring.next_frames)
    if not graph:
        _sac_update_body(actor, qf1, qf2, qf1_target, qf2_target, *args, batch["rows"], batch["next_rows"],
                         batch["actions"], batch["rewards"], batch["dones"], state, buf, buf["dyn"], gamma)
        return state
    same = batch["next_rows"] is batch["rows"]
    for k in ("rows", "actions", "rewards", "dones"):
        buf[k].copy_(batch[k].reshape(-1))
    if not same:
        buf.setdefault("next_rows", torch.zeros_like(buf["rows"])).copy_(batch["next_rows"])
    for t in (qf1_target, qf2_target):
        t._tc_plan()                          # the target repack stays outside the graph
    key = (B, same, args[0].data_ptr(), args[1].data_ptr())
    g = state._graphs.get(key)
    if g is None:
        for n in (actor, qf1, qf2):
            n.params_updated()                # the graph starts by packing the online networks' weights
        g = torch.cuda.CUDAGraph()
        if state._pool is None:
            state._pool = torch.cuda.graph_pool_handle()
        with torch.cuda.graph(g, pool=state._pool):
            _sac_update_body(actor, qf1, qf2, qf1_target, qf2_target, *args, buf["rows"],
                             buf["rows"] if same else buf["next_rows"], buf["actions"], buf["rewards"], buf["dones"],
                             state, buf, buf["dyn"], gamma)
        for n in nets_:
            n.pin_workspaces()
        state._graphs[key] = g
    g.replay()
    for n in (actor, qf1, qf2):
        n.params_updated()                    # no python ran inside the replay: the packed operand copies are stale
    return state


# ------------------------------------------------------- continuous SAC (cleanrl/sac_continuous_action.py)
SACC_LOG_STD_MAX = 2
SACC_LOG_STD_MIN = -5
SACC_ADAM_EPS = 1e-8        # torch.optim.Adam's default, all three optimisers (sac_continuous_action.py:199-207)


def _sacc_dims(env):
    return int(np.array(env.single_observation_space.shape).prod()), int(np.prod(env.single_action_space.shape))


class SoftQNetworkMLP(nn.Module):
    """sac_continuous_action.py:84-99: fc1 [obs + act -> 256], fc2, fc3 [-> 1], default nn.Linear initialisation.
    ``forward(x, a)`` runs the fp32 critic kernel on this one network (``net_stride`` 0)."""

    def __init__(self, env):
        super().__init__()
        self.obs_dim, self.act_dim = _sacc_dims(env)
        self.fc1 = nn.Linear(self.obs_dim + self.act_dim, 256)
        self.fc2 = nn.Linear(256, 256)
        self.fc3 = nn.Linear(256, 1)

    def flat_params(self):
        """The parameters as one flat f32 vector (a view when they already live in a flat buffer)."""
        ps = list(self.parameters())
        base = ps[0].data
        n = sum(p.numel() for p in ps)
        if base.is_contiguous() and all(p.data.data_ptr() == base.data_ptr() + 4 * sum(q.numel() for q in ps[:i])
                                        for i, p in enumerate(ps)):
            return torch.as_strided(base, (n,), (1,))
        return torch.cat([p.data.reshape(-1) for p in ps])

    @torch.no_grad()
    def forward(self, x, a):
        B = x.shape[0]
        q = ops.sacc_critic_fwd(self.flat_params(), 0, x.float().reshape(B, -1).contiguous(),
                                a.float().reshape(B, -1).contiguous(), B, self.obs_dim, self.act_dim)
        return q[0].reshape(B, 1)


class _FlatActor(nn.Module):
    """An actor whose parameters the kernels read from one ``nets.FlatParams`` buffer (``flat``, built on first use on
    the parameters' CUDA device), with the action noise drawn by ``noise_fn``."""

    @property
    def flat(self):
        p = next(self.parameters())
        f = self._flat
        if f is None or f.flat.device != p.device or p.data_ptr() != f.flat.data_ptr():
            if p.device.type != "cuda":
                raise RuntimeError("cleanrl_b200 agents execute on CUDA only (libb200rl kernels); there is no CPU fallback.")
            self._flat = nets.FlatParams(list(self.parameters()), p.device)
        return self._flat

    @property
    def graph_friendly(self):
        """May the noise draw be captured in a CUDA graph (a device-generator draw)?"""
        return getattr(self.noise_fn, "graph_safe", False)

    def draw_noise_into(self, buf):
        if hasattr(self.noise_fn, "inplace"):
            self.noise_fn.inplace(buf)
        else:
            buf.copy_(self.noise_fn(buf.shape[0], buf.shape[1], buf.device))

    def _obs(self, x):
        return x.float().reshape(x.shape[0], -1).contiguous()


class SACContinuousActor(_FlatActor):
    """sac_continuous_action.py:106-151: fc1, fc2, fc_mean, fc_logstd and the buffers action_scale / action_bias.
    ``forward(x)`` -> (mean, log_std); ``get_action(x)`` -> (action, log_prob [n, 1], squashed mean), drawing the
    [n, D] standard normals with ``noise_fn`` (``buf.normal_()`` on the default CUDA generator, what
    ``Normal.rsample`` consumes)."""

    def __init__(self, env):
        super().__init__()
        self.obs_dim, self.act_dim = _sacc_dims(env)
        self.fc1 = nn.Linear(self.obs_dim, 256)
        self.fc2 = nn.Linear(256, 256)
        self.fc_mean = nn.Linear(256, self.act_dim)
        self.fc_logstd = nn.Linear(256, self.act_dim)
        high, low = env.single_action_space.high, env.single_action_space.low
        self.register_buffer("action_scale", torch.tensor((high - low) / 2.0, dtype=torch.float32))
        self.register_buffer("action_bias", torch.tensor((high + low) / 2.0, dtype=torch.float32))
        self.noise_fn = _normal_noise
        self._flat = None

    @torch.no_grad()
    def forward(self, x):
        B, D = x.shape[0], self.act_dim
        ml = torch.empty(B, 2 * D, dtype=torch.float32, device=x.device)
        ops.sacc_actor_fwd(self.flat.flat, self._obs(x), B, self.obs_dim, D, None, self.action_scale, self.action_bias,
                           mean_logstd=ml)
        return ml[:, :D], ml[:, D:]

    @torch.no_grad()
    def get_action(self, x, eps=None):
        B, D = x.shape[0], self.act_dim
        dev = x.device
        eps = self.noise_fn(B, D, dev) if eps is None else eps
        action = torch.empty(B, D, dtype=torch.float32, device=dev)
        log_pi = torch.empty(B, 1, dtype=torch.float32, device=dev)
        mean = torch.empty(B, D, dtype=torch.float32, device=dev)
        ops.sacc_actor_fwd(self.flat.flat, self._obs(x), B, self.obs_dim, D, eps.contiguous(), self.action_scale,
                           self.action_bias, action=action, log_pi=log_pi, mean_out=mean)
        return action, log_pi, mean


class SACContinuousState:
    """Device-resident part of a continuous-SAC update that is not a network: the flat buffers of the twin critics
    (one parameter / gradient / Adam buffer, as ``q_optimizer`` covers both) and of the twin targets, the temperature
    (``alpha`` f32[1], with autotune ``log_alpha`` and its Adam moments), the Adam step counts of the q, actor and
    temperature optimisers with their device table of step scalars, the logged statistics (``qstats`` =
    ``ops.SACC_CRITIC_STAT_NAMES``, ``astats`` = ``ops.SACC_ACTOR_STAT_NAMES``) and the scratch of each batch size.
    With ``use_graph`` every update is replayed as one CUDA graph per (batch size, with actor steps, with target
    update)."""

    use_graph = True

    def __init__(self, actor, qf1, qf2, qf1_target, qf2_target, device, autotune=True, alpha=0.2, policy_frequency=2):
        f32 = torch.float32
        self.device, self.autotune, self.pf = device, bool(autotune), int(policy_frequency)
        self.actor, self.obs_dim, self.act_dim = actor, actor.obs_dim, actor.act_dim
        self.net_numel = ops.sacc_param_count(self.obs_dim, self.act_dim, True)
        self.q = nets.FlatParams(list(qf1.parameters()) + list(qf2.parameters()), device)
        self.qt = nets.FlatParams(list(qf1_target.parameters()) + list(qf2_target.parameters()), device)
        actor.flat
        # -torch.prod(torch.Tensor(envs.single_action_space.shape)).item()  (sac_continuous_action.py:204)
        self.target_entropy = -torch.prod(torch.Tensor((self.act_dim,))).item()
        self.log_alpha = torch.zeros(1, dtype=f32, device=device)
        self.alpha = torch.full((1,), 1.0 if autotune else float(alpha), dtype=f32, device=device)
        self.exp_avg = torch.zeros(1, dtype=f32, device=device)
        self.exp_avg_sq = torch.zeros(1, dtype=f32, device=device)
        self.qstats = torch.zeros(4, dtype=f32, device=device)
        self.astats = torch.zeros(4, dtype=f32, device=device)
        self.astats[2] = self.alpha[0]          # losses/alpha before the first temperature step
        self.steps = {"q": 0, "actor": 0, "alpha": 0}
        self._bufs, self._graphs, self._pool = {}, {}, None

    def buffers(self, B):
        b = self._bufs.get(B)
        if b is None:
            f32, dev, D, K = torch.float32, self.device, self.act_dim, self.obs_dim + self.act_dim
            z = lambda *s: torch.zeros(*s, dtype=f32, device=dev)   # noqa: E731
            b = {"rows": torch.zeros(B, dtype=torch.int64, device=dev), "dyn": z(2 + 4 * self.pf),
                 "x": z(B, K), "h1": z(2, B, 256), "h2": z(2, B, 256), "dz1": z(2, B, 256), "dz2": z(2, B, 256),
                 "q": z(2, B), "qn": z(2, B), "dq": z(2, B), "y": z(B), "pi_next": z(B, D), "logpi_next": z(B),
                 "eps_next": z(B, D), "eps_actor": z(self.pf, B, D), "eps_alpha": z(self.pf, B, D),
                 "xa": z(B, self.obs_dim), "h1a": z(B, 256), "h2a": z(B, 256), "head": z(B, 2 * D), "pi": z(B, D),
                 "logpi": z(B), "qpi": z(2, B), "dact": z(2, B, D), "dhead": z(B, 2 * D), "dz1a": z(B, 256),
                 "dz2a": z(B, 256), "logpi_alpha": z(B), "ws": ops.sacc_workspace(B, dev)}
            self._bufs[B] = b
        return b

    def step_table(self, actor_steps, q_lr, policy_lr):
        """Advance the optimisers' step counts and return their ``adam_step_scalars``: q, then per actor step the
        actor's and the temperature's (whose lr is q_lr, sac_continuous_action.py:207)."""
        self.steps["q"] += 1
        t = list(ops.adam_step_scalars(self.steps["q"], q_lr))
        for _ in range(self.pf):
            if actor_steps:
                self.steps["actor"] += 1
                t += ops.adam_step_scalars(self.steps["actor"], policy_lr)
                if self.autotune:
                    self.steps["alpha"] += 1
                    t += ops.adam_step_scalars(self.steps["alpha"], q_lr)
                else:
                    t += (1.0, 0.0)
            else:
                t += (1.0, 0.0, 1.0, 0.0)
        return t


def _sacc_update_body(st, obs, next_obs, actions, rewards, dones, rows, buf, actor_steps, target_update, gamma, tau):
    """sac_continuous_action.py:255-304 on device buffers; every (step, lr) scalar comes from ``buf["dyn"]``."""
    actor, B, od, D, S = st.actor, rows.numel(), st.obs_dim, st.act_dim, st.net_numel
    af, q, dyn, ws = actor.flat, st.q, buf["dyn"], buf["ws"]
    scale, bias = actor.action_scale, actor.action_bias
    # 1. soft-Q target on next_obs (the actor's sample, both targets) and the critic loss, backward and q optimiser
    actor.draw_noise_into(buf["eps_next"])
    ops.sacc_actor_fwd(af.flat, next_obs, B, od, D, buf["eps_next"], scale, bias, rows=rows, action=buf["pi_next"],
                       log_pi=buf["logpi_next"])
    ops.sacc_critic_fwd(st.qt.flat, S, next_obs, buf["pi_next"], B, od, D, obs_rows=rows, q=buf["qn"])
    ops.sacc_critic_fwd(q.flat, S, obs, actions, B, od, D, obs_rows=rows, act_rows=rows, q=buf["q"], keep_x=buf["x"],
                        keep_h1=buf["h1"], keep_h2=buf["h2"])
    ops.sacc_critic_loss(buf["qn"], buf["logpi_next"], buf["q"], rewards, dones, st.alpha, gamma, rows=rows, y=buf["y"],
                         dq=buf["dq"], stats=st.qstats, workspace=ws)
    ops.sacc_critic_bwd(q.flat, S, B, od, D, buf["h1"], buf["h2"], dq=buf["dq"], dz1=buf["dz1"], dz2=buf["dz2"])
    ops.sacc_wgrad(True, B, od, D, buf["x"], buf["h1"], buf["h2"], buf["dz1"], buf["dz2"], buf["dq"], q.grad, S)
    ops.clip_adam_dyn(q.flat, q.grad, q.exp_avg, q.exp_avg_sq, dyn[0:2], eps=SACC_ADAM_EPS, max_norm=None)
    # 2. policy_frequency actor steps, each followed by the temperature step on a fresh sample
    for k in range(st.pf if actor_steps else 0):
        eps = buf["eps_actor"][k]
        actor.draw_noise_into(eps)
        ops.sacc_actor_fwd(af.flat, obs, B, od, D, eps, scale, bias, rows=rows, action=buf["pi"], log_pi=buf["logpi"],
                           keep_x=buf["xa"], keep_h1=buf["h1a"], keep_h2=buf["h2a"], keep_head=buf["head"])
        ops.sacc_critic_fwd(q.flat, S, obs, buf["pi"], B, od, D, obs_rows=rows, q=buf["qpi"], keep_h1=buf["h1"],
                            keep_h2=buf["h2"])
        ops.sacc_critic_bwd(q.flat, S, B, od, D, buf["h1"], buf["h2"], q=buf["qpi"], dact=buf["dact"])
        ops.sacc_actor_bwd(af.flat, B, od, D, buf["head"], eps, scale, buf["dact"], buf["qpi"], buf["logpi"], st.alpha,
                           buf["h1a"], buf["h2a"], buf["dhead"], buf["dz1a"], buf["dz2a"], st.astats, ws)
        ops.sacc_wgrad(False, B, od, D, buf["xa"], buf["h1a"], buf["h2a"], buf["dz1a"], buf["dz2a"], buf["dhead"], af.grad)
        ops.clip_adam_dyn(af.flat, af.grad, af.exp_avg, af.exp_avg_sq, dyn[2 + 4 * k:4 + 4 * k], eps=SACC_ADAM_EPS,
                          max_norm=None)
        if st.autotune:
            e2 = buf["eps_alpha"][k]
            actor.draw_noise_into(e2)
            ops.sacc_actor_fwd(af.flat, obs, B, od, D, e2, scale, bias, rows=rows, log_pi=buf["logpi_alpha"],
                               temperature=dict(alpha=st.alpha, log_alpha=st.log_alpha, exp_avg=st.exp_avg,
                                                exp_avg_sq=st.exp_avg_sq, step_scalars=dyn[4 + 4 * k:6 + 4 * k],
                                                target_entropy=st.target_entropy, stats=st.astats),
                               workspace=ws)
    # 3. soft target update of both targets (one flat buffer)
    if target_update:
        ops.sacc_soft_update(q.flat, st.qt.flat, 2 * S, tau)


@torch.no_grad()
def sac_continuous_update(state, ring, batch, global_step, args, graph=None):
    """One update of sac_continuous_action.py:255-304 on a ``DeviceReplayRing`` batch: the critic step; on steps where
    ``global_step % policy_frequency == 0`` the ``policy_frequency`` actor and temperature steps on the same batch; the
    soft target update when ``global_step % target_network_frequency == 0``.  Nothing is read back to the host.  With
    ``graph`` (default ``state.use_graph``) the update replays one captured CUDA graph per (batch size, actor steps,
    target update) with the batch rows copied into a fixed slot."""
    st = state
    B = int(batch["rows"].numel())
    buf = st.buffers(B)
    actor_steps = global_step % args.policy_frequency == 0
    target_update = global_step % args.target_network_frequency == 0
    buf["dyn"].copy_(torch.tensor(st.step_table(actor_steps, args.q_lr, args.policy_lr), dtype=torch.float32),
                     non_blocking=True)
    views = (ring.frames, ring.next_frames, ring.action_rows, ring.reward_rows, ring.done_rows)
    use_graph = st.use_graph if graph is None else graph
    if not (use_graph and st.actor.graph_friendly):
        _sacc_update_body(st, *views, batch["rows"], buf, actor_steps, target_update, args.gamma, args.tau)
        return st
    buf["rows"].copy_(batch["rows"])
    key = (B, actor_steps, target_update, views[0].data_ptr(), float(args.gamma), float(args.tau))
    _replay_update_graph(st, key, lambda: _sacc_update_body(st, *views, buf["rows"], buf, actor_steps, target_update,
                                                            args.gamma, args.tau))
    return st


def _replay_update_graph(st, key, body):
    """Replay the update graph ``st`` captured under ``key``, capturing ``body()`` first if there is none (the graphs
    share one memory pool; the Adam workspace of the largest flat buffer, ``st.q``, is sized before any capture)."""
    g = st._graphs.get(key)
    if g is None:
        ops._workspace(st.device, "adam", ops._lib.load().b200rl_clip_adam_workspace_bytes(st.q.flat.numel()))
        g = torch.cuda.CUDAGraph()
        if st._pool is None:
            st._pool = torch.cuda.graph_pool_handle()
        with torch.cuda.graph(g, pool=st._pool):
            body()
        st._graphs[key] = g
    g.replay()


# ---------------------------------------------------------- TD3 (cleanrl/td3_continuous_action.py)
class TD3Actor(_FlatActor):
    """td3_continuous_action.py:106-132: fc1, fc2, fc_mu and the buffers action_scale / action_bias, default nn.Linear
    initialisation.  ``forward(x)`` = tanh(fc_mu(...)) * action_scale + action_bias on the deterministic-head kernel.
    ``noise_fn`` draws the [B, D] standard normals of the target policy smoothing (``randn_like(actions)`` on the
    default CUDA generator)."""

    def __init__(self, env):
        super().__init__()
        self.obs_dim, self.act_dim = _sacc_dims(env)
        self.fc1 = nn.Linear(self.obs_dim, 256)
        self.fc2 = nn.Linear(256, 256)
        self.fc_mu = nn.Linear(256, self.act_dim)
        high, low = env.single_action_space.high, env.single_action_space.low
        self.register_buffer("action_scale", torch.tensor((high - low) / 2.0, dtype=torch.float32))
        self.register_buffer("action_bias", torch.tensor((high + low) / 2.0, dtype=torch.float32))
        self.noise_fn = _normal_noise
        self._flat = None

    @torch.no_grad()
    def forward(self, x):
        B = x.shape[0]
        mu = torch.empty(B, self.act_dim, dtype=torch.float32, device=x.device)
        ops.td3_actor_fwd(self.flat.flat, self._obs(x), B, self.obs_dim, self.act_dim, self.action_scale,
                          self.action_bias, mu=mu)
        return mu


def _exploration_noise(std):
    """td3_continuous_action.py:203: ``torch.normal(0, std)``, one [D] draw that every env adds to its action."""
    return torch.normal(0, std)


class TD3State:
    """Device-resident part of a TD3 update that is not a network: the flat buffers of the twin critics (one parameter
    / gradient / Adam buffer, as ``q_optimizer`` covers both), of the twin targets and of the actor target, the Adam
    step counts of the q and actor optimisers with their device table of step scalars (``dyn``: q, then actor), the
    logged statistics (``qstats`` = ``ops.SACC_CRITIC_STAT_NAMES``, ``astats[0]`` = the latest actor_loss) and the
    scratch of each batch size.  With ``use_graph`` every update is replayed as one CUDA graph per (batch size, actor
    step, gamma, tau, policy_noise, noise_clip, bounds).  ``low`` / ``high``: the scalar bounds the smoothed target
    action is clamped to (the reference's ``single_action_space.low[0]`` / ``high[0]``; default: the actor's first
    dimension, action_bias -/+ action_scale)."""

    use_graph = True

    def __init__(self, actor, qf1, qf2, qf1_target, qf2_target, target_actor, device, low=None, high=None):
        f32 = torch.float32
        self.device = device
        b0, s0 = float(actor.action_bias[0]), float(actor.action_scale[0])
        self.low = float(b0 - s0 if low is None else low)
        self.high = float(b0 + s0 if high is None else high)
        self.actor, self.target_actor, self.obs_dim, self.act_dim = actor, target_actor, actor.obs_dim, actor.act_dim
        self.net_numel = ops.sacc_param_count(self.obs_dim, self.act_dim, True)
        self.q = nets.FlatParams(list(qf1.parameters()) + list(qf2.parameters()), device)
        self.qt = nets.FlatParams(list(qf1_target.parameters()) + list(qf2_target.parameters()), device)
        actor.flat
        target_actor.flat
        self.qstats = torch.zeros(4, dtype=f32, device=device)
        self.astats = torch.zeros(1, dtype=f32, device=device)
        self.steps = {"q": 0, "actor": 0}
        self._bufs, self._graphs, self._pool = {}, {}, None

    def buffers(self, B):
        b = self._bufs.get(B)
        if b is None:
            f32, dev, D, K = torch.float32, self.device, self.act_dim, self.obs_dim + self.act_dim
            z = lambda *s: torch.zeros(*s, dtype=f32, device=dev)   # noqa: E731
            b = {"rows": torch.zeros(B, dtype=torch.int64, device=dev), "dyn": z(4),
                 "x": z(B, K), "h1": z(2, B, 256), "h2": z(2, B, 256), "dz1": z(2, B, 256), "dz2": z(2, B, 256),
                 "q": z(2, B), "qn": z(2, B), "dq": z(2, B), "y": z(B), "eps_next": z(B, D), "a_next": z(B, D),
                 "xa": z(B, self.obs_dim), "h1a": z(B, 256), "h2a": z(B, 256), "ya": z(B, D), "pi": z(B, D),
                 "qpi": z(1, B), "dact": z(B, D), "dhead": z(B, D), "dz1a": z(B, 256), "dz2a": z(B, 256),
                 "ws": ops.sacc_workspace(B, dev)}
            self._bufs[B] = b
        return b

    def step_table(self, actor_step, lr):
        """Advance the optimisers' step counts and return their ``adam_step_scalars``: q, then the actor's (both at
        ``learning_rate``, td3_continuous_action.py:180-181)."""
        self.steps["q"] += 1
        t = list(ops.adam_step_scalars(self.steps["q"], lr))
        if actor_step:
            self.steps["actor"] += 1
            t += ops.adam_step_scalars(self.steps["actor"], lr)
        else:
            t += (1.0, 0.0)
        return t


def _td3_update_body(st, obs, next_obs, actions, rewards, dones, rows, buf, actor_step, gamma, tau, smoothing):
    """td3_continuous_action.py:231-267 on device buffers; the (step, lr) scalars come from ``buf["dyn"]``."""
    actor, ta, B, od, D, S = st.actor, st.target_actor, rows.numel(), st.obs_dim, st.act_dim, st.net_numel
    af, q, dyn, ws = actor.flat, st.q, buf["dyn"], buf["ws"]
    # 1. smoothed target action, the twin targets, the critic loss, its backward and the q optimiser
    actor.draw_noise_into(buf["eps_next"])
    ops.td3_actor_fwd(ta.flat.flat, next_obs, B, od, D, ta.action_scale, ta.action_bias, rows=rows,
                      smoothing=dict(smoothing, eps=buf["eps_next"], out=buf["a_next"]))
    ops.sacc_critic_fwd(st.qt.flat, S, next_obs, buf["a_next"], B, od, D, obs_rows=rows, q=buf["qn"])
    ops.sacc_critic_fwd(q.flat, S, obs, actions, B, od, D, obs_rows=rows, act_rows=rows, q=buf["q"], keep_x=buf["x"],
                        keep_h1=buf["h1"], keep_h2=buf["h2"])
    ops.sacc_critic_loss(buf["qn"], None, buf["q"], rewards, dones, None, gamma, rows=rows, y=buf["y"], dq=buf["dq"],
                         stats=st.qstats, workspace=ws)
    ops.sacc_critic_bwd(q.flat, S, B, od, D, buf["h1"], buf["h2"], dq=buf["dq"], dz1=buf["dz1"], dz2=buf["dz2"])
    ops.sacc_wgrad(True, B, od, D, buf["x"], buf["h1"], buf["h2"], buf["dz1"], buf["dz2"], buf["dq"], q.grad, S)
    ops.clip_adam_dyn(q.flat, q.grad, q.exp_avg, q.exp_avg_sq, dyn[0:2], eps=SACC_ADAM_EPS, max_norm=None)
    if not actor_step:
        return
    # 2. the delayed actor step on -qf1(obs, actor(obs)).mean(), then the soft update of all three targets
    ops.td3_actor_fwd(af.flat, obs, B, od, D, actor.action_scale, actor.action_bias, rows=rows, mu=buf["pi"],
                      keep_y=buf["ya"], keep_x=buf["xa"], keep_h1=buf["h1a"], keep_h2=buf["h2a"])
    ops.sacc_critic_fwd(q.flat, 0, obs, buf["pi"], B, od, D, obs_rows=rows, q=buf["qpi"], keep_h1=buf["h1"],
                        keep_h2=buf["h2"])
    ops.sacc_critic_bwd(q.flat, 0, B, od, D, buf["h1"], buf["h2"], dact=buf["dact"])
    ops.td3_actor_bwd(af.flat, B, od, D, buf["ya"], actor.action_scale, buf["dact"], buf["qpi"], buf["h1a"],
                      buf["h2a"], buf["dhead"], buf["dz1a"], buf["dz2a"], st.astats, ws)
    ops.sacc_wgrad(ops.SACC_TD3_ACTOR, B, od, D, buf["xa"], buf["h1a"], buf["h2a"], buf["dz1a"], buf["dz2a"],
                   buf["dhead"], af.grad)
    ops.clip_adam_dyn(af.flat, af.grad, af.exp_avg, af.exp_avg_sq, dyn[2:4], eps=SACC_ADAM_EPS, max_norm=None)
    ops.sacc_soft_update(af.flat, ta.flat.flat, af.numel, tau)
    ops.sacc_soft_update(q.flat, st.qt.flat, 2 * S, tau)


@torch.no_grad()
def td3_update(state, ring, batch, global_step, args, graph=None):
    """One update of td3_continuous_action.py:230-267 on a ``DeviceReplayRing`` batch: the critic step; on steps where
    ``global_step % policy_frequency == 0`` the actor step and the soft update of the actor target and both critic
    targets.  Nothing is read back to the host.  With ``graph`` (default ``state.use_graph``) the
    update replays one captured CUDA graph per (batch size, actor step, gamma, tau, policy_noise, noise_clip, bounds)
    with the batch rows copied into a fixed slot and the smoothing draw captured in it."""
    st = state
    B = int(batch["rows"].numel())
    buf = st.buffers(B)
    actor_step = global_step % args.policy_frequency == 0
    buf["dyn"].copy_(torch.tensor(st.step_table(actor_step, args.learning_rate), dtype=torch.float32),
                     non_blocking=True)
    smoothing = dict(policy_noise=float(args.policy_noise), noise_clip=float(args.noise_clip),
                     low=st.low, high=st.high)
    views = (ring.frames, ring.next_frames, ring.action_rows, ring.reward_rows, ring.done_rows)
    use_graph = st.use_graph if graph is None else graph
    if not (use_graph and st.actor.graph_friendly):
        _td3_update_body(st, *views, batch["rows"], buf, actor_step, args.gamma, args.tau, smoothing)
        return st
    buf["rows"].copy_(batch["rows"])
    key = (B, actor_step, views[0].data_ptr(), float(args.gamma), float(args.tau)) + tuple(smoothing.values())
    _replay_update_graph(st, key, lambda: _td3_update_body(st, *views, buf["rows"], buf, actor_step, args.gamma,
                                                           args.tau, smoothing))
    return st


# ---------------------------------------------------------- DDPG (cleanrl/ddpg_continuous_action.py)
class DDPGActor(TD3Actor):
    """ddpg_continuous_action.py:96-116: TD3's modules, initialisation and state_dict keys, with action_scale /
    action_bias taken from ``env.action_space`` -- the vector env's batched space, so [1, D] under gymnasium's
    ``SyncVectorEnv`` and [D] where ``action_space`` is unbatched.  The kernels read D contiguous floats either way."""

    def __init__(self, env):
        super().__init__(env)
        high, low = env.action_space.high, env.action_space.low
        self.action_scale = torch.tensor((high - low) / 2.0, dtype=torch.float32)
        self.action_bias = torch.tensor((high + low) / 2.0, dtype=torch.float32)


class DDPGState:
    """Device-resident part of a DDPG update that is not a network: the flat buffers of qf1 and of qf1_target (one
    network each), the actor target's (on the module), the Adam step counts of the q and actor optimisers with their
    device table of step scalars (``dyn``: q, then actor), the logged statistics (``qstats`` =
    ``ops.DDPG_CRITIC_STAT_NAMES``, ``astats[0]`` = the latest actor_loss) and the scratch of each batch size.  The
    update draws no random numbers; with ``use_graph`` it is replayed as one CUDA graph per (batch size, actor step,
    ring, gamma, tau)."""

    use_graph = True

    def __init__(self, actor, qf1, qf1_target, target_actor, device):
        f32 = torch.float32
        self.device = device
        self.actor, self.target_actor, self.obs_dim, self.act_dim = actor, target_actor, actor.obs_dim, actor.act_dim
        self.net_numel = ops.sacc_param_count(self.obs_dim, self.act_dim, True)
        self.q = nets.FlatParams(list(qf1.parameters()), device)
        self.qt = nets.FlatParams(list(qf1_target.parameters()), device)
        actor.flat
        target_actor.flat
        self.qstats = torch.zeros(2, dtype=f32, device=device)
        self.astats = torch.zeros(1, dtype=f32, device=device)
        self.steps = {"q": 0, "actor": 0}
        self._bufs, self._graphs, self._pool = {}, {}, None

    def buffers(self, B):
        b = self._bufs.get(B)
        if b is None:
            f32, dev, D, K = torch.float32, self.device, self.act_dim, self.obs_dim + self.act_dim
            z = lambda *s: torch.zeros(*s, dtype=f32, device=dev)   # noqa: E731
            b = {"rows": torch.zeros(B, dtype=torch.int64, device=dev), "dyn": z(4),
                 "x": z(B, K), "h1": z(1, B, 256), "h2": z(1, B, 256), "dz1": z(1, B, 256), "dz2": z(1, B, 256),
                 "q": z(1, B), "qn": z(1, B), "dq": z(B), "y": z(B), "a_next": z(B, D),
                 "xa": z(B, self.obs_dim), "h1a": z(B, 256), "h2a": z(B, 256), "ya": z(B, D), "pi": z(B, D),
                 "qpi": z(1, B), "dact": z(B, D), "dhead": z(B, D), "dz1a": z(B, 256), "dz2a": z(B, 256),
                 "ws": ops.sacc_workspace(B, dev)}
            self._bufs[B] = b
        return b

    step_table = TD3State.step_table      # both optimisers at learning_rate (ddpg_continuous_action.py:158-159)


def _ddpg_update_body(st, obs, next_obs, actions, rewards, dones, rows, buf, actor_step, gamma, tau):
    """ddpg_continuous_action.py:214-245 on device buffers; the (step, lr) scalars come from ``buf["dyn"]``."""
    actor, ta, B, od, D, S = st.actor, st.target_actor, rows.numel(), st.obs_dim, st.act_dim, st.net_numel
    af, q, dyn, ws = actor.flat, st.q, buf["dyn"], buf["ws"]
    # 1. target action (no smoothing), qf1_target, qf1, the fused loss + data backward, the weight gradient, q_optimizer
    ops.td3_actor_fwd(ta.flat.flat, next_obs, B, od, D, ta.action_scale, ta.action_bias, rows=rows, mu=buf["a_next"])
    ops.sacc_critic_fwd(st.qt.flat, 0, next_obs, buf["a_next"], B, od, D, obs_rows=rows, q=buf["qn"])
    ops.sacc_critic_fwd(q.flat, 0, obs, actions, B, od, D, obs_rows=rows, act_rows=rows, q=buf["q"], keep_x=buf["x"],
                        keep_h1=buf["h1"], keep_h2=buf["h2"])
    ops.ddpg_critic_loss_bwd(q.flat, B, od, D, buf["qn"], buf["q"], rewards, dones, gamma, buf["h1"], buf["h2"],
                             rows=rows, y=buf["y"], dq=buf["dq"], dz1=buf["dz1"], dz2=buf["dz2"], stats=st.qstats,
                             workspace=ws)
    ops.sacc_wgrad(True, B, od, D, buf["x"], buf["h1"], buf["h2"], buf["dz1"], buf["dz2"], buf["dq"], q.grad, 0)
    ops.clip_adam_dyn(q.flat, q.grad, q.exp_avg, q.exp_avg_sq, dyn[0:2], eps=SACC_ADAM_EPS, max_norm=None)
    if not actor_step:
        return
    # 2. the actor step on -qf1(obs, actor(obs)).mean() with the critic just updated (TD3's), then both soft updates
    ops.td3_actor_fwd(af.flat, obs, B, od, D, actor.action_scale, actor.action_bias, rows=rows, mu=buf["pi"],
                      keep_y=buf["ya"], keep_x=buf["xa"], keep_h1=buf["h1a"], keep_h2=buf["h2a"])
    ops.sacc_critic_fwd(q.flat, 0, obs, buf["pi"], B, od, D, obs_rows=rows, q=buf["qpi"], keep_h1=buf["h1"],
                        keep_h2=buf["h2"])
    ops.sacc_critic_bwd(q.flat, 0, B, od, D, buf["h1"], buf["h2"], dact=buf["dact"])
    ops.td3_actor_bwd(af.flat, B, od, D, buf["ya"], actor.action_scale, buf["dact"], buf["qpi"], buf["h1a"],
                      buf["h2a"], buf["dhead"], buf["dz1a"], buf["dz2a"], st.astats, ws)
    ops.sacc_wgrad(ops.SACC_TD3_ACTOR, B, od, D, buf["xa"], buf["h1a"], buf["h2a"], buf["dz1a"], buf["dz2a"],
                   buf["dhead"], af.grad)
    ops.clip_adam_dyn(af.flat, af.grad, af.exp_avg, af.exp_avg_sq, dyn[2:4], eps=SACC_ADAM_EPS, max_norm=None)
    ops.sacc_soft_update(af.flat, ta.flat.flat, af.numel, tau)
    ops.sacc_soft_update(q.flat, st.qt.flat, S, tau)


@torch.no_grad()
def ddpg_update(state, ring, batch, global_step, args, graph=None):
    """One update of ddpg_continuous_action.py:214-245 on a ``DeviceReplayRing`` batch: the critic step; on steps where
    ``global_step % policy_frequency == 0`` the actor step and the soft update of the actor target and qf1_target.
    Nothing is read back to the host and nothing is drawn.  With ``graph`` (default ``state.use_graph``) the update
    replays one captured CUDA graph per (batch size, actor step, ring, gamma, tau) with the batch rows copied into a
    fixed slot."""
    st = state
    B = int(batch["rows"].numel())
    buf = st.buffers(B)
    actor_step = global_step % args.policy_frequency == 0
    buf["dyn"].copy_(torch.tensor(st.step_table(actor_step, args.learning_rate), dtype=torch.float32),
                     non_blocking=True)
    views = (ring.frames, ring.next_frames, ring.action_rows, ring.reward_rows, ring.done_rows)
    if not (st.use_graph if graph is None else graph):
        _ddpg_update_body(st, *views, batch["rows"], buf, actor_step, args.gamma, args.tau)
        return st
    buf["rows"].copy_(batch["rows"])
    key = (B, actor_step, views[0].data_ptr(), float(args.gamma), float(args.tau))
    _replay_update_graph(st, key, lambda: _ddpg_update_body(st, *views, buf["rows"], buf, actor_step, args.gamma,
                                                            args.tau))
    return st
