"""Generative Adversarial Imitation Learning with the discriminator on the device.

Reference: tianshou/algorithm/imitation/gail.py (GailTrainingStats :24-28, constructor :34-190, rewards :193-206,
discriminator steps :214-248).

GAIL is PPO whose rewards come from a discriminator D(s, a):
  rewards  : one discriminator forward over all N rollout rows (``ts_net_gemm``), then ``ts_gail_reward_rows``
             (-logsigmoid(-D) in fp32, widened) into a scratch f64 tensor that replaces ``batch.rew`` before GAE.  The
             buffer is never written: with a full device-mirrored buffer ``batch.rew`` IS the mirror's column.
  disc     : ``N // disc_update_num``-row chunks of one ``np.random.permutation(N)`` (numpy's global stream, drawn before
             PPO's ``repeat`` permutations), each against as many expert rows from the expert buffer's own RandomState.
             Per chunk: one gather into a [policy | expert] input, one forward, ``ts_gail_disc_rows`` (loss, accuracies,
             d loss / d logit), one backward, one Adam step.  No host sync; the per-step table is read once, after PPO's.
  policy   : PPO's update, unchanged (fused epoch kernel, SIMT or layer-wise path, as PPO decides).
Single GPU, Box action spaces.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any

import numpy as np
import torch

from ... import ops
from ..._cabi import call, ptr, stream_ptr, to_device
from ...data import Batch, ReplayBuffer, SequenceSummaryStats
from ...data.batch import minibatch_bounds, numpy_global_permutation_
from ...parallel import world
from ...utils.net.common import ModuleWithVectorOutput
from ..base import _space_kind
from ..flat_params import FlatGroup, UnsupportedModelError, bind_optimizer
from ..modelfree.a2c import A2CTrainingStats
from ..modelfree.ppo import PPO
from ..modelfree.reinforce import ProbabilisticActorPolicy
from ..modelfree.sac import describe_q_critic
from ..netgraph import FusedStack
from ..optim import OptimizerFactory

# columns of the per-step discriminator table ``last_disc_table``
COL_DISC_LOSS, COL_ACC_PI, COL_ACC_EXP, COL_POLICY_ROWS = range(4)


@dataclass(kw_only=True)
class GailTrainingStats(A2CTrainingStats):
    disc_loss: SequenceSummaryStats
    acc_pi: SequenceSummaryStats
    acc_exp: SequenceSummaryStats


class GAIL(PPO):
    """Generative Adversarial Imitation Learning (arXiv:1606.03476)."""

    def __init__(
        self,
        *,
        policy: ProbabilisticActorPolicy,
        critic: torch.nn.Module,
        optim: OptimizerFactory,
        expert_buffer: ReplayBuffer,
        disc_net: torch.nn.Module,
        disc_optim: OptimizerFactory,
        disc_update_num: int = 4,
        eps_clip: float = 0.2,
        dual_clip: float | None = None,
        value_clip: bool = False,
        advantage_normalization: bool = True,
        recompute_advantage: bool = False,
        vf_coef: float = 0.5,
        ent_coef: float = 0.01,
        max_grad_norm: float | None = None,
        gae_lambda: float = 0.95,
        max_batchsize: int = 256,
        gamma: float = 0.99,
        return_scaling: bool = False,
    ) -> None:
        if not isinstance(policy.actor, ModuleWithVectorOutput):
            raise TypeError("GAIL requires the policy to use an actor with known output dimension.")
        if world()[1] > 1:
            raise UnsupportedModelError("GAIL is single-GPU")
        if _space_kind(policy.action_space) != "continuous":
            raise UnsupportedModelError("GAIL needs a Box action space: the discriminator reads concat(obs, act) rows")
        super().__init__(policy=policy, critic=critic, optim=optim, eps_clip=eps_clip, dual_clip=dual_clip, value_clip=value_clip,
                         advantage_normalization=advantage_normalization, recompute_advantage=recompute_advantage,
                         vf_coef=vf_coef, ent_coef=ent_coef, max_grad_norm=max_grad_norm, gae_lambda=gae_lambda,
                         max_batchsize=max_batchsize, gamma=gamma, return_scaling=return_scaling)
        self.disc_net = disc_net
        self.disc_optim = self._create_optimizer(self.disc_net, disc_optim)
        self.disc_update_num = disc_update_num
        self.expert_buffer = expert_buffer
        self.action_dim = self.policy.actor.get_output_dim()

        self._obs_dim, self._act_dim = self._spec.obs_dim, self._spec.act_dim
        try:
            layers, params = describe_q_critic(disc_net, self._obs_dim, self._act_dim)
        except AttributeError as e:
            raise UnsupportedModelError(f"discriminator: expected ContinuousCritic(preprocess_net=Net(concat=True)): {e}") from e
        self._g_disc = FlatGroup(params, self.device)
        bind_optimizer(self.disc_optim, self._g_disc)
        self._disc = FusedStack(layers, self._g_disc, "disc")
        self._check_expert_buffer()
        self._disc_order: torch.Tensor | None = None
        self.last_disc_table: np.ndarray | None = None

    def _check_expert_buffer(self) -> None:
        buf = self.expert_buffer
        if getattr(buf, "stack_num", 1) != 1:
            raise UnsupportedModelError("GAIL: an expert buffer with stack_num > 1 is not supported")
        keys = buf._meta.get_keys()
        if "obs" in keys and "act" in keys:
            obs_w = int(np.prod(np.asarray(buf._meta.obs).shape[1:], dtype=np.int64))
            act_w = int(np.prod(np.asarray(buf._meta.act).shape[1:], dtype=np.int64))
            if (obs_w, act_w) != (self._obs_dim, self._act_dim):
                raise UnsupportedModelError(f"GAIL: expert rows (obs width {obs_w}, act width {act_w}) do not match the networks "
                                            f"(obs {self._obs_dim}, act {self._act_dim})")

    # ------------------------------------------------------------------ rewards
    def _disc_input(self, batch: Batch, tag: str, rows: int) -> torch.Tensor:
        """concat(obs, act) of the rollout rows into the first N rows of a [rows, O + A] scratch."""
        N = batch.obs.shape[0]
        x = self._buf(tag, (rows, self._obs_dim + self._act_dim), torch.float32)
        call("ts_concat2", ptr(batch.obs), self._obs_dim, ptr(batch.act), self._act_dim, N, ptr(x), stream_ptr(self.device))
        return x

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: Any) -> Batch:
        """gail.py:193-206: rewards from the discriminator as it was before this update, then PPO's preprocessing."""
        N = batch.obs.shape[0]
        x = self._disc_input(batch, "gail_reward_x", N)
        logits = self._disc.forward(x, N, "reward")[-1]
        rew = self._buf("gail_rew", N, torch.float64)        # never the buffer's storage (the mirror's own column when full)
        call("ts_gail_reward_rows", ptr(logits), N, ptr(rew), stream_ptr(self.device))
        batch.__dict__["rew"] = rew
        return super()._preprocess_batch(batch, buffer, indices)

    # ------------------------------------------------------------------ update
    def update(self, buffer: ReplayBuffer, batch_size: int | None, repeat: int) -> GailTrainingStats:
        """The discriminator's minibatch order is drawn first (gail.py:224 runs ahead of PPO's passes), so that PPO's
        background permutation job starts from the advanced generator state."""
        if buffer is not None and self.policy.is_within_training_step:
            # Batch.split's assert fires before any draw (batch.py:1208); PPO's order job would otherwise advance the stream
            self._check_chunk_size(len(buffer))
            self._disc_order = numpy_global_permutation_(self._disc_order_rows(len(buffer)))
        try:
            return super().update(buffer=buffer, batch_size=batch_size, repeat=repeat)
        finally:
            self._disc_order = None

    def _check_chunk_size(self, n: int) -> int:
        bsz = n // self.disc_update_num
        assert bsz >= 1, f"GAIL: {n} rollout rows cannot be split into disc_update_num={self.disc_update_num} chunks"
        return bsz

    def _disc_order_rows(self, n: int) -> torch.Tensor:
        t = self._scratch.get("disc_order")
        if t is None or t.numel() != n:
            t = self._scratch["disc_order"] = torch.empty(n, dtype=torch.int32, pin_memory=True)
        return t

    def _update_with_batch(self, batch: Batch, batch_size: int | None, repeat: int) -> GailTrainingStats:
        """gail.py:214-248: the discriminator steps, then PPO's update; the two statistics tables are read at the end."""
        N = batch.obs.shape[0]
        bsz = self._check_chunk_size(N)
        order, self._disc_order = self._disc_order, None
        if order is None or order.numel() != N:
            order = numpy_global_permutation_(self._disc_order_rows(N))
        table = self._disc_steps(batch, order.numpy().astype(np.int64), bsz)
        ppo_stats = super()._update_with_batch(batch, batch_size, repeat)
        disc = table.cpu().numpy().astype(np.float64)
        self._g_disc.export_state(self.disc_optim._optim)
        self.last_disc_table = disc
        return GailTrainingStats(**ppo_stats.__dict__, disc_loss=SequenceSummaryStats.from_sequence(disc[:, COL_DISC_LOSS]),
                                 acc_pi=SequenceSummaryStats.from_sequence(disc[:, COL_ACC_PI]),
                                 acc_exp=SequenceSummaryStats.from_sequence(disc[:, COL_ACC_EXP]))

    def _disc_steps(self, batch: Batch, order: np.ndarray, bsz: int) -> torch.Tensor:
        """One Adam step per chunk of ``order``; returns the [steps][4] device table.  Rows are gathered from one source
        matrix [rollout rows | expert rows of every step] by one index vector, uploaded once."""
        dev, st = self.device, stream_ptr(self.device)
        N, W = batch.obs.shape[0], self._obs_dim + self._act_dim
        bounds = minibatch_bounds(N, bsz, merge_last=True)
        steps = len(bounds)
        # the reference samples once per step, in step order, from the expert buffer's own generator(s)
        exp_idx = np.concatenate([np.asarray(self.expert_buffer.sample_indices(bsz), dtype=np.int64) for _ in range(steps)])
        src = self._disc_input(batch, "gail_disc_src", N + steps * bsz)
        e_obs = ops.buffer_rows(self.expert_buffer, "obs", exp_idx, dev)
        e_act = ops.buffer_rows(self.expert_buffer, "act", exp_idx, dev)
        call("ts_concat2", ptr(e_obs), self._obs_dim, ptr(e_act), self._act_dim, steps * bsz, src.data_ptr() + 4 * N * W, st)
        rows = np.concatenate([np.concatenate([order[lo:hi], N + s * bsz + np.arange(bsz, dtype=np.int64)])
                               for s, (lo, hi) in enumerate(bounds)])
        table = torch.zeros((steps, 4), dtype=torch.float32, device=dev)
        self._disc_loop(src, to_device(rows, dev), bounds, bsz, table)
        return table

    def _disc_loop(self, src: torch.Tensor, rows: torch.Tensor, bounds: list[tuple[int, int]], bsz: int,
                   table: torch.Tensor) -> None:
        """Step s: rows ``rows[off:off + n]`` of ``src`` = [policy rows of chunk s | its bsz expert rows] -> forward,
        ``ts_gail_disc_rows`` into ``table[s]``, backward, Adam (no gradient clipping, gail.py:233)."""
        st = stream_ptr(self.device)
        max_rows = max(hi - lo for lo, hi in bounds) + bsz
        x_buf = self._buf("gail_disc_x", (max_rows, src.shape[1]), torch.float32)
        dlogits = self._buf("gail_dlogits", max_rows, torch.float32)
        off = 0
        for s, (lo, hi) in enumerate(bounds):
            n_pi = hi - lo
            n = n_pi + bsz
            x = ops.gather_rows(src, rows[off:off + n], out=x_buf[:n])
            off += n
            acts = self._disc.forward(x, n, "disc")
            call("ts_gail_disc_rows", ptr(acts[-1]), n_pi, bsz, ptr(dlogits), ptr(table[s]), st)
            self._disc.backward(acts, dlogits[:n].view(n, 1), n, "disc")
            self._g_disc.adam_step(self.disc_optim._optim, None)
