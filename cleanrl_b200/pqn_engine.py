"""Device-resident rollout and update of cleanrl/pqn.py on libb200rl kernels.

One env step is one host-to-device copy of a pinned packet (next_obs, next_done, the previous step's reward and the
step's two CPU draws, ``torch.randint`` then ``torch.rand`` as the reference makes them), one ``pqn_act`` launch that
writes obs[step], actions[step], values[step] and the done / reward bookkeeping, and one device-to-host copy of the
actions.  ``finish_rollout`` bootstraps max Q(next_obs) and runs the Q(lambda) scan.  ``update`` shuffles with
``ops.numpy_global_shuffle`` (``np.random.shuffle``'s permutation, cumulative across epochs), uploads each epoch's
indices to a pinned slot of their own, and replays each epoch as one CUDA graph: per minibatch update, 4 library
launches (``pqn_loss_bwd``, ``pqn_wgrad``, the clip norm, RAdam), with the RAdam scalars of every update of the
iteration in a device table written once.  Nothing is read back to the host except the actions and, once per
iteration, the two logged statistics.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops

RADAM_EPS = 1e-8        # torch.optim.RAdam's default (pqn.py:152)


class PQNEngine:
    """Rollout buffers, update buffers and graphs of one ``PQNQNetwork``.  ``use_graph`` False: eager launches (the same
    kernels, the same bits)."""

    use_graph = True

    def __init__(self, q_network, args, num_envs, device):
        self.q, self.args, self.device = q_network, args, device
        self.flat = q_network.flat
        T, N = int(args.num_steps), int(num_envs)
        d, A = q_network.obs_dim, q_network.n_actions
        self.T, self.N, self.d, self.A = T, N, d, A
        self.B = T * N
        self.mbs = int(self.B // args.num_minibatches)
        if self.mbs < 1:
            raise ValueError(f"pqn: batch {self.B} is smaller than num_minibatches={args.num_minibatches}")
        self.starts = list(range(0, self.B, self.mbs))       # a batch not divisible gives a shorter last minibatch
        self.epochs = int(args.update_epochs)
        f32, i64 = torch.float32, torch.int64
        z = lambda *s, dt=f32: torch.zeros(*s, dtype=dt, device=device)     # noqa: E731
        self.obs = z(self.B, d)                    # [T * N, d]: obs[step] is rows step * N ...
        self.actions = z(self.B, dt=i64)
        self.values = z(T, N)
        self.dr = z(T + 1, 2, N)                   # per step: (next_done, the reward of the step before)
        self.rewards, self.dones, self.returns = z(T, N), z(T, N), z(T, N)
        self.next_value = z(N)
        # the packet: f32 [next_obs (N d) | next_done (N) | reward (N) | u (N)], then i64 random_actions (N)
        nf = N * d + 3 * N
        off_i = 4 * nf + (-4 * nf) % 8
        nbytes = off_i + 8 * N
        self.host_packet = torch.zeros(nbytes, dtype=torch.uint8, pin_memory=True)
        self.dev_packet = torch.zeros(nbytes, dtype=torch.uint8, device=device)

        def views(buf):
            f = buf[:4 * nf].view(f32)
            return (f[:N * d].view(N, d), f[N * d:N * d + N], f[N * d + N:N * d + 2 * N], f[N * d + 2 * N:nf],
                    buf[off_i:].view(i64), f[N * d:N * d + 2 * N])

        self.h_obs, self.h_done, self.h_rew, self.h_u, self.h_rand, _ = views(self.host_packet)
        self.d_obs, _, _, self.d_u, self.d_rand, self.d_dr = views(self.dev_packet)
        self.host_actions = torch.zeros(N, dtype=i64, pin_memory=True)
        self.step_event = torch.cuda.Event()
        # update
        self.nmb = len(self.starts)
        self.stats = z(2)
        self.ws = ops.pqn_workspace(self.mbs, device)
        self.host_inds = torch.zeros(self.epochs, self.B, dtype=i64, pin_memory=True)
        self.inds = z(self.epochs, self.B, dt=i64)
        self.host_table = torch.zeros(self.epochs * self.nmb, 4, dtype=f32, pin_memory=True)
        self.table = z(self.epochs * self.nmb, 4)
        self.update_event = torch.cuda.Event()
        self.update_event.record()
        self.radam_step = 0                        # RAdam steps taken (every parameter steps together)
        self._graphs, self._pool = {}, None

    # ---------------------------------------------------------------- rollout
    def _pack(self, next_obs, next_done, reward):
        self.h_obs.numpy()[:] = np.asarray(next_obs, dtype=np.float32).reshape(self.N, self.d)
        self.h_done.numpy()[:] = np.asarray(next_done, dtype=np.float32).reshape(self.N)
        self.h_rew.numpy()[:] = np.asarray(reward, dtype=np.float32).reshape(self.N)

    @torch.no_grad()
    def policy_step(self, step, next_obs, next_done, prev_reward, epsilon):
        """pqn.py:176-189 for rollout slot ``step``; returns the actions (numpy int64 [N])."""
        self._pack(next_obs, next_done, prev_reward)
        torch.randint(0, self.A, (self.N,), out=self.h_rand)          # the reference's two CPU draws, in its order
        torch.rand((self.N,), out=self.h_u)
        self.dev_packet.copy_(self.host_packet, non_blocking=True)
        N = self.N
        acts = self.actions[step * N:(step + 1) * N]
        ops.pqn_act(self.flat.flat, self.d_obs, self.d, self.A, self.values[step], random_actions=self.d_rand,
                    u=self.d_u, eps=epsilon, actions=acts, obs_slot=self.obs[step * N:(step + 1) * N],
                    copy=(self.d_dr, self.dr[step].view(-1)))
        self.host_actions.copy_(acts, non_blocking=True)
        self.step_event.record()
        self.step_event.synchronize()
        return self.host_actions.numpy().copy()

    @torch.no_grad()
    def finish_rollout(self, next_obs, next_done, last_reward):
        """pqn.py:205-218: next_value = max Q(next_obs), then the Q(lambda) returns."""
        self._pack(next_obs, next_done, last_reward)
        self.dev_packet.copy_(self.host_packet, non_blocking=True)
        ops.pqn_act(self.flat.flat, self.d_obs, self.d, self.A, self.next_value, copy=(self.d_dr, self.dr[self.T].view(-1)))
        self.rewards.copy_(self.dr[1:, 1])
        self.dones.copy_(self.dr[:self.T, 0])
        ops.qlambda(self.rewards, self.values, self.dones, self.next_value, self.dr[self.T, 0], self.args.gamma,
                    self.args.q_lambda, returns=self.returns)

    # ----------------------------------------------------------------- update
    def _minibatch(self, e, i):
        st = self.starts[i]
        M = min(self.mbs, self.B - st)
        rows = self.inds[e, st:st + M]
        f = self.flat
        ops.pqn_loss_bwd(f.flat, self.obs, self.d, self.A, rows, self.actions, self.returns.view(-1), self.stats, self.ws)
        ops.pqn_wgrad(self.obs, self.d, self.A, rows, self.actions, self.ws, f.grad)
        ops.clip_radam_dyn(f.flat, f.grad, f.exp_avg, f.exp_avg_sq, self.table[e * self.nmb + i], eps=RADAM_EPS,
                           max_norm=self.args.max_grad_norm)

    def _epoch(self, e):
        for i in range(self.nmb):
            self._minibatch(e, i)

    def _replay(self, e):
        g = self._graphs.get(e)
        if g is None:
            ops._workspace(self.device, "adam", ops._lib.load().b200rl_clip_adam_workspace_bytes(self.flat.flat.numel()))
            g = torch.cuda.CUDAGraph()
            if self._pool is None:
                self._pool = torch.cuda.graph_pool_handle()
            with torch.cuda.graph(g, pool=self._pool):
                self._epoch(e)
            self._graphs[e] = g
        g.replay()

    @torch.no_grad()
    def update(self, lr, use_graph=None):
        """pqn.py:220-240 at learning rate ``lr``: ``update_epochs`` shuffles of the batch indices with numpy's global
        generator and one RAdam step per minibatch.  Returns the device stats [2] (td_loss and mean q of the last
        minibatch, what the reference logs)."""
        self.update_event.synchronize()            # the pinned slots below are free once the last update has run
        for k in range(self.epochs * self.nmb):
            self.host_table[k] = torch.tensor(ops.radam_step_scalars(self.radam_step + k + 1, lr))
        self.table.copy_(self.host_table, non_blocking=True)
        b_inds = np.arange(self.B)
        graph = self.use_graph if use_graph is None else use_graph
        for e in range(self.epochs):
            ops.numpy_global_shuffle(b_inds)
            self.host_inds[e].numpy()[:] = b_inds
            self.inds[e].copy_(self.host_inds[e], non_blocking=True)
            if graph:
                self._replay(e)
            else:
                self._epoch(e)
        self.radam_step += self.epochs * self.nmb
        self.update_event.record()
        return self.stats
