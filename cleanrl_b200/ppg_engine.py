"""Phasic policy gradient on the PPO engine (reference: cleanrl/ppg_procgen.py:285-477).

The policy phase is ``PPOEngine``'s rollout, GAE and fused loss with three differences the reference makes: advantages are
normalised once over the whole batch (never per minibatch), Adam runs with ``eps = 1e-8``, and ``aux_critic`` has no
gradient, so torch's ``clip_grad_norm_`` and Adam skip it (``ops.clip_adam_ranges`` with the head's ranges frozen).

The auxiliary buffer lives on the device: after every policy iteration the rollout's uint8 frames and its returns are
copied device to device into their slice (the reference keeps them on the host and uploads every minibatch).  The
auxiliary phase runs without a host synchronisation inside an epoch: minibatch row vectors are built on the device from
the uploaded permutation, the network gathers its frames through them, the fused loss (``ops.ppg_aux_loss``) reads the
old logits and returns through the same rows, and the three losses of every minibatch are copied out once per phase.
"""
from __future__ import annotations

import os
import types

import numpy as np
import torch

from . import ops
from .ppo_engine import PPOEngine, _pin, _sync

ADAM_EPS = 1e-8                  # optim.Adam(agent.parameters(), lr=args.learning_rate, eps=1e-8), ppg_procgen.py:265
# bf16 without gradient accumulation: replay the auxiliary update as one CUDA graph (6.27 ms against 6.40 ms launched eagerly
# on an H100 at 700 W, DESIGN.md section 4); CLEANRL_B200_PPG_AUX_GRAPH=0 launches eagerly
AUX_GRAPH_DEFAULT = "1"
OLD_POLICY_ROWS = 8192           # rows per forward of the old-policy pass (a row's result does not depend on its batch)


class PPGEngine(PPOEngine):
    def __init__(self, agent, args, obs_shape, num_envs, device, gae_mode=0):
        ppo_args = types.SimpleNamespace(**vars(args))
        ppo_args.update_epochs, ppo_args.norm_adv = int(args.e_policy), False
        super().__init__(agent, ppo_args, obs_shape, np.uint8, num_envs, device, gae_mode=gae_mode)
        self.ppg = args
        self.update_graphs = False           # PPO's captured epoch steps every element with one flat Adam
        T, N, A = self.T, self.N, int(agent.num_actions)
        self.n_iteration = int(args.n_iteration)
        self.Na = N * self.n_iteration
        self.R = int(args.num_aux_rollouts)
        self.accum = int(args.n_aux_grad_accum)
        assert self.Na % self.R == 0, "num_envs * n_iteration must be divisible by num_aux_rollouts"
        frame = int(np.prod(obs_shape))
        need = T * self.Na * (frame + 4 + 4 * A)
        if device.type == "cuda":
            free, _ = torch.cuda.mem_get_info(device)
            if need > free:
                raise RuntimeError(f"the PPG auxiliary buffer ({T} steps x {self.Na} rollouts of {frame}-byte frames, returns "
                                   f"and old logits) needs {need / 2**30:.2f} GiB of device memory, {free / 2**30:.2f} GiB are "
                                   "free: lower --n-iteration or --num-envs (it is not spilled to the host)")
        f32 = torch.float32
        self.aux_obs = torch.zeros((T, self.Na) + tuple(obs_shape), dtype=torch.uint8, device=device)
        self.aux_returns = torch.zeros((T, self.Na), dtype=f32, device=device)
        self.aux_pi = torch.zeros((T, self.Na, A), dtype=f32, device=device)
        self.adv_norm = torch.zeros((T, N), dtype=f32, device=device)
        E = int(args.e_auxiliary)
        self.aux_inds_h = _pin(torch.zeros((max(E, 1), self.Na), dtype=torch.int64))
        self.aux_inds = torch.zeros((max(E, 1), self.Na), dtype=torch.int64, device=device)
        self.t_base = (torch.arange(T, device=device, dtype=torch.int64) * self.Na).view(T, 1)
        n_mb = max(E * (self.Na // self.R), 1)
        self.aux_stats = torch.zeros(n_mb, 4, dtype=f32, device=device)      # rows of 16 B; the kernel writes 3 values
        self.aux_stats_h = _pin(torch.zeros(n_mb, 4, dtype=f32))
        self.aux_hyper = torch.zeros(n_mb, 4, dtype=f32, device=device)
        self.aux_hyper_h = _pin(torch.zeros(n_mb, 4, dtype=f32))
        self.aux_dhead = torch.zeros(T * self.R, A + 2, dtype=f32, device=device)
        self.grad_acc = torch.zeros_like(self.flat.grad)
        self._acc_pending = False
        self.aux_step = 0                    # Adam's `step` of aux_critic: the auxiliary updates so far
        self.aux_ranges = agent.aux_critic_ranges()
        if agent.uses_tc_plan():
            # the plan's workspaces of the auxiliary phase's batch shapes, now: a run that does not fit fails here
            plan = agent._tc_plan()
            plan.acts(T * self.R)
            plan.acts(T * min(max(1, OLD_POLICY_ROWS // T), self.Na))
            plan.workspace(T * self.R)
        self.aux_graph = os.environ.get("CLEANRL_B200_PPG_AUX_GRAPH", AUX_GRAPH_DEFAULT) != "0"
        self._aux_g = None

    # ------------------------------------------------------------------ policy phase
    @torch.no_grad()
    def update(self, lr):
        adv = self.advantages
        if self.ppg.adv_norm_fullbatch:      # ppg_procgen.py:344-345 (torch.std: unbiased)
            torch.div(adv - adv.mean(), adv.std() + 1e-8, out=self.adv_norm)
        else:
            self.adv_norm.copy_(adv)
        self._acc_pending = False            # optimizer.zero_grad() before every policy backward drops leftovers
        return super().update(lr)

    @torch.no_grad()
    def minibatch_update(self, mb_inds, lr, k=0, dyn=None):
        """One policy-phase update: PPOEngine's with the full-batch-normalised advantages and PPG's optimiser semantics
        (``aux_critic`` frozen: the loss does not reach it)."""
        assert dyn is None
        a, agent, flat, B = self.args, self.agent, self.flat, self.B
        b = {"actions": self.actions.view(B), "logprobs": self.logprobs.view(B), "advantages": self.adv_norm.view(B),
             "returns": self.returns.view(B), "values": self.values.view(B)}
        if not hasattr(self, "_scratch"):
            self._scratch = {}
        policy_out, value = agent.forward_train(self.obs.view((B,) + tuple(self.obs.shape[2:])), mb_inds)
        agent.loss_backward(policy_out, value, mb_inds, b, a, self.stats[k], self._scratch)
        flat.step += 1
        ops.clip_adam_ranges(flat.flat, flat.grad, flat.exp_avg, flat.exp_avg_sq, flat.step, lr, self.aux_ranges, 0,
                             eps=ADAM_EPS, max_norm=a.max_grad_norm, norm_out=self.grad_norm)
        agent.params_updated()

    @torch.no_grad()
    def store_rollout(self, update):
        """ppg_procgen.py:415-418: the rollout of policy iteration ``update`` (1-based) into its slice of the buffer."""
        sl = slice(self.N * (update - 1), self.N * update)
        self.aux_obs[:, sl].copy_(self.obs)
        self.aux_returns[:, sl].copy_(self.returns)

    # --------------------------------------------------------------- auxiliary phase
    def _rows(self, cols):
        """Buffer rows of whole rollouts ``cols`` (device int64), step-major as ``flatten01`` orders them."""
        return (self.t_base + cols.view(1, -1)).reshape(-1)

    @torch.no_grad()
    def old_policy_pass(self):
        """ppg_procgen.py:423-434: the current policy's normalised logits over the whole buffer -> ``aux_pi``."""
        T, Na, A = self.T, self.Na, self.agent.num_actions
        obs = self.aux_obs.view((T * Na,) + tuple(self.aux_obs.shape[2:]))
        pi = self.aux_pi.view(T * Na, A)
        chunk = max(1, OLD_POLICY_ROWS // T)
        cols = torch.arange(Na, device=self.device, dtype=torch.int64)
        for start in range(0, Na, chunk):
            rows = self._rows(cols[start:start + chunk])
            pi.index_copy_(0, rows, self.agent.get_pi(obs, rows=rows))

    @torch.no_grad()
    def aux_minibatch(self, cols, lr, stats_row, step_now, dyn=None):
        """Forward, fused loss, backward on the rollouts ``cols``; clip + Adam when ``step_now``.  ``dyn``: the update is
        being captured, its (step, lr) scalars come from that device slot."""
        agent, flat, a = self.agent, self.flat, self.ppg
        T, Na, A = self.T, self.Na, agent.num_actions
        obs = self.aux_obs.view((T * Na,) + tuple(self.aux_obs.shape[2:]))
        rows = self._rows(cols)
        head = agent.forward_aux(obs, rows)
        ops.ppg_aux_loss(head, rows, self.aux_pi.view(T * Na, A), self.aux_returns.view(-1), a.beta_clone, 1.0 / self.accum,
                         dhead=self.aux_dhead, stats=stats_row)
        agent.backward(self.aux_dhead)
        grads = flat.grad
        if self._acc_pending:                # backward overwrites flat.grad: sum the minibatches in their order
            grads = self.grad_acc.add_(flat.grad)
        elif self.accum > 1:
            grads = self.grad_acc.copy_(flat.grad)
            self._acc_pending = True
        if dyn is not None:
            ops.clip_adam_ranges_dyn(flat.flat, grads, flat.exp_avg, flat.exp_avg_sq, dyn, self.aux_ranges, eps=ADAM_EPS,
                                     max_norm=a.max_grad_norm, norm_out=self.grad_norm)
            agent.params_updated()
        elif step_now:
            flat.step += 1
            self.aux_step += 1
            ops.clip_adam_ranges(flat.flat, grads, flat.exp_avg, flat.exp_avg_sq, flat.step, lr, self.aux_ranges,
                                 self.aux_step, lr, eps=ADAM_EPS, max_norm=a.max_grad_norm, norm_out=self.grad_norm)
            self._acc_pending = False
            agent.params_updated()

    # One CUDA graph of a whole auxiliary update (weight pack, forward, loss, backward, clip + Adam): it reads its rollout
    # columns and its (step, lr) scalars from fixed device slots filled stream-ordered before each replay, the pattern of
    # PPOEngine._capture_epoch.  Same kernels on the same operands as the eager update: bit-identical results.
    def aux_replay_ready(self):
        return (self.aux_graph and self.accum == 1 and not self._acc_pending and self.agent.uses_tc_plan()
                and self.device.type == "cuda")

    @torch.no_grad()
    def aux_minibatch_replayed(self, cols, dyn_row, stats_row):
        """``dyn_row``: device f32[4], ``adam_step_scalars`` of this update's (step, lr) for every element and for aux_critic."""
        if self._aux_g is None:
            dev, f32 = self.device, torch.float32
            self._g_cols = torch.zeros(self.R, dtype=torch.int64, device=dev)
            self._g_dyn = torch.zeros(4, dtype=f32, device=dev)
            self._g_stats = torch.zeros(4, dtype=f32, device=dev)
            self.agent.params_updated()      # the graph always starts by packing the weights it was given
            g = torch.cuda.CUDAGraph()
            if self._graph_pool is None:
                self._graph_pool = torch.cuda.graph_pool_handle()
            with torch.cuda.graph(g, pool=self._graph_pool):
                self.aux_minibatch(self._g_cols, None, self._g_stats, True, dyn=self._g_dyn)
            self.agent.pin_workspaces()
            self._aux_g = g
        self.flat.step += 1
        self.aux_step += 1
        self._g_cols.copy_(cols)
        self._g_dyn.copy_(dyn_row)
        self._aux_g.replay()
        stats_row.copy_(self._g_stats)
        self.agent.params_updated()          # no python ran inside the replay: the packed operand copies are stale

    def _aux_step_table(self, lr, n):
        """The (step, lr) scalars of the next ``n`` auxiliary updates, uploaded once (host, double, as clip_adam_ranges)."""
        hy = self.aux_hyper_h.numpy()
        for j in range(n):
            hy[j] = ops.adam_step_scalars(self.flat.step + 1 + j, lr) + ops.adam_step_scalars(self.aux_step + 1 + j, lr)
        self.aux_hyper.copy_(self.aux_hyper_h, non_blocking=True)

    @torch.no_grad()
    def aux_phase(self, lr, on_epoch=None):
        """ppg_procgen.py:420-477.  Returns the last minibatch's three losses and all of them (``per_minibatch``)."""
        self.old_policy_pass()
        # The reference zeroes gradients before every policy backward and after every auxiliary step, but not between
        # the phases: the first auxiliary backward accumulates onto the gradient the last policy update left behind,
        # which clip_grad_norm_ had scaled in place (aux_critic had none).  Kept: the drop-in follows the reference.
        a = self.ppg
        coef = torch.clamp(a.max_grad_norm / (self.grad_norm + 1e-6), max=1.0)
        torch.mul(self.flat.grad, coef, out=self.grad_acc)
        self._acc_pending = True
        aux_inds = np.arange(self.Na)
        k = 0
        if self.aux_graph and self.accum == 1 and self.agent.uses_tc_plan():
            self._aux_step_table(lr, self.aux_hyper.shape[0])
        for epoch in range(int(self.ppg.e_auxiliary)):
            if on_epoch is not None:
                on_epoch(epoch + 1)
            self._shuffle(aux_inds)          # numpy's global generator, cumulative across epochs as the reference
            self.aux_inds_h[epoch].copy_(torch.from_numpy(aux_inds))
            self.aux_inds[epoch].copy_(self.aux_inds_h[epoch], non_blocking=True)
            for i, start in enumerate(range(0, self.Na, self.R)):
                cols = self.aux_inds[epoch, start:start + self.R]
                if self.aux_replay_ready():
                    self.aux_minibatch_replayed(cols, self.aux_hyper[k], self.aux_stats[k])
                else:
                    self.aux_minibatch(cols, lr, self.aux_stats[k], (i + 1) % self.accum == 0)
                k += 1
        self.aux_stats_h[:k].copy_(self.aux_stats[:k], non_blocking=True)
        _sync()
        s = self.aux_stats_h[:k].numpy()
        out = {name: float(s[k - 1, j]) for j, name in enumerate(ops.PPG_AUX_STAT_NAMES)} if k else {}
        out["per_minibatch"] = s[:, :3].copy()
        return out
