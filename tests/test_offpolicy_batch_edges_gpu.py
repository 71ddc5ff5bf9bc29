"""Every off-policy and offline update at the batch sizes its kernels split on, against float64 autograd, and every one of them
again after a batch of another size has used its scratch.

The row count of an update reaches the K of every weight-gradient GEMM (and with it the split-K switch), the M of
``ts_net_colsum``, the ``n`` of ``ts_mean``, the ``1 / B`` of every rows kernel, the grid of every per-row kernel (B, B x repeat
for CQL / BCQ, B x S for IQN) and the scratch caches: ``DeviceScratch.tensor`` matches on exact shape, ``FusedStack._buf`` only
grows.  Part 1 runs one update per (algorithm, batch) through each family's own float64 harness, at its own bars; part 2 runs
one batch size and then another on one instance, with every scratch tensor poisoned in between, and asks for the bits a fresh
instance in the same state computes."""
import copy

import numpy as np
import pytest
import torch

from offpolicy_testutil import (B_LARGE, B_SMALL, DEV, GEMM_BK, Box, Discrete, check_second_batch_size, gemm_splits_k, golden_cfg,
                                grid_caps, vector_buffer_from_golden)
from test_discrete_bcq_gpu import build_bcq
from test_discrete_crr_gpu import build_crr
from test_iqn_gpu import build_from_golden as build_iqn
from test_qrdqn_gpu import build_from_golden as build_qrdqn
from ts_testutil import load_golden

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------ part 1
# name -> (run(B), rows of the largest per-row launch per sampled row, rows of the largest weight-gradient GEMM per sampled row)
def _sac(B, edge):
    from test_offpolicy_gpu import sac_grad_case
    sac_grad_case(O, A, (32, 32), True, True, False, seed=14, B=B, edge=edge)


def _dsac(B, edge):
    from test_discrete_sac_gpu import grad_case
    grad_case("mlp", True, False, True, (), B=B, edge=edge)


def _cql(B, edge):
    from test_cql_gpu import grad_case
    grad_case(O, A, (32, 32), CQL_R, B=B, edge=edge)


def _td3(B, edge):
    from test_td3_gpu import grad_case
    grad_case(O, A, (32, 32), "td3", B=B, edge=edge)


def _td3bc(B, edge):
    from test_td3_gpu import grad_case
    grad_case(O, A, (32, 32), "bc", B=B, edge=edge)


def _bcq(B, edge):
    from test_bcq_gpu import grad_case
    grad_case(O, A, (32, 32), (32, 32), BCQ_L, True, B=B, edge=edge)


def _dqn(B, edge):
    from test_offpolicy_gpu import dqn_grad_case
    dqn_grad_case("mlp", "mse", True, True, 0, B=B, edge=edge)


def _qrdqn(B, edge):
    from test_qrdqn_gpu import grad_case
    grad_case("mlp", 0.0, B=B, edge=edge)


def _dcql(B, edge):
    from test_qrdqn_gpu import grad_case
    grad_case("mlp", 10.0, B=B, edge=edge)


def _iqn(B, edge):
    from test_iqn_gpu import grad_case
    grad_case("mlp", B=B, S_on=IQN_S_ON, S_t=IQN_S_T, edge=edge)


def _dbcq(B, edge):
    from test_discrete_bcq_gpu import grad_case
    grad_case("mlp_relu", "mlp", True, dict(hidden=(48, 40)), B=B, edge=edge)


def _dcrr(B, edge):
    from test_discrete_bcq_gpu import TRUNK_CASES
    from test_discrete_crr_gpu import grad_case
    grad_case(*TRUNK_CASES[0], "exp", B=B, edge=edge)


O, A, CQL_R, BCQ_N, BCQ_L, IQN_S_ON, IQN_S_T, IQN_D = 11, 3, 10, 10, 6, 6, 7, 40
# name -> (run(B, edge), rows of the largest weight-gradient GEMM per sampled row, the launches the past_grid batch takes past
# their grid caps: (launch, cap, items per sampled row))
ALGOS = {
    "sac": (_sac, 1, [("ts_squashed_gaussian", "net_ops_1d", 1), ("ts_squashed_gaussian_bwd", "net_ops_1d", A),
                      ("ts_critic_mse", "net_ops_1d", 1), ("ts_sac_target", "net_ops_1d", 1), ("ts_sac_actor_q_grad", "net_ops_1d", 1)]),
    "discrete_sac": (_dsac, 1, [("ts_discrete_sac_rows", "warp_per_row", 1), ("ts_dqn_loss", "net_ops_1d", 1)]),
    # the critic steps run on [batch; B x R current; B x R next; B x R random actions] rows; ts_cql_rows on the batch and one
    # B x R block
    "cql": (_cql, 1 + 3 * CQL_R, [("ts_cql_rows", "offpolicy_1d", 1 + CQL_R)]),
    "td3": (_td3, 1, [("ts_td3_act_rows", "offpolicy_1d", O + A), ("ts_td3_target_min", "offpolicy_1d", 1),
                      ("ts_td3_actor_head_bwd", "offpolicy_1d", A), ("ts_critic_mse", "net_ops_1d", 1)]),
    "td3_bc": (_td3bc, 1, [("ts_td3_act_rows", "offpolicy_1d", O + A), ("ts_td3_target_min", "offpolicy_1d", 1),
                           ("ts_td3_actor_head_bwd", "offpolicy_1d", A), ("ts_critic_mse", "net_ops_1d", 1)]),
    # the target decodes, perturbs and evaluates B x N sampled actions; every backward runs on B rows
    "bcq": (_bcq, 1, [("ts_bcq_decode_input", "offpolicy_1d", BCQ_N * (O + BCQ_L)), ("ts_bcq_perturb", "offpolicy_1d", BCQ_N * (O + A)),
                      ("ts_bcq_act_rows", "offpolicy_1d", BCQ_N * (O + A))]),
    "dqn": (_dqn, 1, [("ts_dqn_loss", "net_ops_1d", 1), ("ts_dqn_target", "net_ops_1d", 1)]),
    "qrdqn": (_qrdqn, 1, [("ts_qrdqn_target", "warp_per_row", 1), ("ts_qrdqn_rows", "block_per_row", 1)]),
    "discrete_cql": (_dcql, 1, [("ts_qrdqn_target", "warp_per_row", 1), ("ts_qrdqn_rows", "block_per_row", 1)]),
    # the target embeds B x S_t fractions, the online step B x S_on
    "iqn": (_iqn, IQN_S_ON, [("ts_iqn_target", "warp_per_row", 1), ("ts_iqn_rows", "block_per_row", 1), ("ts_iqn_cos", "warp_per_row", IQN_S_T),
                             ("ts_iqn_mix", "iqn_1d", IQN_S_T * IQN_D), ("ts_iqn_mix_backward", "iqn_1d", IQN_D)]),
    "discrete_bcq": (_dbcq, 1, [("ts_discrete_bcq_target", "warp_per_row", 1), ("ts_discrete_bcq_rows", "warp_per_row", 1)]),
    "discrete_crr": (_dcrr, 1, [("ts_discrete_crr_rows", "warp_per_row", 1)]),
}
BATCH_CLASSES = ["B1", "B3", "B17", "splitK_below", "splitK_above", "past_grid"]


def batch_for(name, cls):
    _, gemm_per_b, launches = ALGOS[name]
    if cls == "B1":
        return 1
    if cls == "B3":
        return 3
    if cls == "B17":
        return 17
    if cls == "splitK_below":          # the largest weight-gradient GEMM has one K chunk: unsplit
        return GEMM_BK // gemm_per_b
    if cls == "splitK_above":          # two chunks: split
        return GEMM_BK // gemm_per_b + 1
    caps = grid_caps()              # the smallest batch that takes every listed launch past its cap
    return max(caps[cap] // items + 1 for _, cap, items in launches)


@pytest.mark.parametrize("cls", BATCH_CLASSES)
@pytest.mark.parametrize("name", list(ALGOS))
def test_update_vs_fp64_autograd_at_batch_edges(name, cls):
    """One update through the family's float64 harness: every optimiser step's flat gradient (snapshotted before its Adam step),
    the losses, and where the harness checks them the n-step returns and the TD errors written back, at the harness's own
    bars, recorded under ``<family>@<class>``.  The harness asserts the update ran on the B sampled rows (B x repeat / B x S
    where the update repeats them).  ``past_grid`` is the smallest batch that takes each of the algorithm's listed launches past
    the grid cap of its kernel file."""
    run, gemm_per_b, launches = ALGOS[name]
    B = batch_for(name, cls)
    if cls.startswith("splitK"):
        assert gemm_splits_k(B * gemm_per_b) == (cls == "splitK_above")
    if cls == "past_grid":
        caps = grid_caps()
        for launch, cap, items in launches:
            assert B * items > caps[cap], f"{launch}: {B * items} items stay inside its {cap} cap of {caps[cap]}"
        assert any((B - 1) * items <= caps[cap] for _, cap, items in launches), "one batch fewer would cross every cap too"
    run(B, f"@{cls}")


# ------------------------------------------------------------------------------------------------------------ part 2
def _r_sac():
    """SAC on 96-wide hidden layers: their forward and input-gradient GEMMs have two K chunks, so they split K at every batch
    and the workspace they need grows with the rows."""
    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.sac import SAC, SACPolicy
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    from ts_testutil import synth_rollout
    O, A, H = 11, 3, (96, 96)
    torch.manual_seed(21)

    def build():
        actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H), action_shape=(A,), unbounded=True,
                                             conditioned_sigma=True).to(DEV)
        mk = lambda: ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True)).to(DEV)
        return SAC(policy=SACPolicy(actor=actor, action_space=Box(A)), policy_optim=AdamOptimizerFactory(lr=1e-3), critic=mk(),
                   critic_optim=AdamOptimizerFactory(lr=1e-3), critic2=mk(), critic2_optim=AdamOptimizerFactory(lr=1e-3), tau=0.005,
                   gamma=0.99, alpha=0.2, n_step_return_horizon=2)

    E, T = 4, 64
    buf = VectorReplayBuffer(E * T, E, device=DEV)
    for s in synth_rollout(np.random.default_rng(3), E, T, O, A, p_term=0.05, trunc_len=20):
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    return build, buf


def _r_dsac():
    from test_discrete_sac_gpu import buffer_from_golden, build_from_golden
    g = load_golden("dsac_ref_auto.npz")
    return (lambda: build_from_golden(g)), buffer_from_golden(g, False)


def _r_cql():
    from test_cql_gpu import buffer_from_golden, build_from_cfg
    g = load_golden("cql_ref_d4rl.npz")
    cfg = golden_cfg(g)
    return (lambda: build_from_cfg(cfg, g)), build_from_cfg(cfg, g).process_buffer(buffer_from_golden(g, False))   # adds the calibration returns


def _r_td3(golden):
    def make():
        from test_td3_gpu import buffer_from_golden, build_from_cfg
        g = load_golden(golden)
        return (lambda: build_from_cfg(golden_cfg(g), g)), buffer_from_golden(g, False)
    return make


def _r_bcq():
    from test_bcq_gpu import buffer_from_golden, build_from_cfg
    g = load_golden("bcq_ref_small.npz")
    return (lambda: build_from_cfg(golden_cfg(g))), buffer_from_golden(g, False)


def _r_dqn():
    from test_offpolicy_gpu import dqn_grad_setup
    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.dqn import DQN, DiscreteQLearningPolicy
    A = 6
    net, buf = dqn_grad_setup("mlp", A, seed=8, per=False)
    net0 = copy.deepcopy(net)

    def build():
        return DQN(policy=DiscreteQLearningPolicy(model=copy.deepcopy(net0), action_space=Discrete(A)), optim=AdamOptimizerFactory(lr=1e-3),
                   gamma=0.9, n_step_return_horizon=2, target_update_freq=3, is_double=True)
    return build, buf


def _r_vector(golden, build):
    """A discrete Q-learning family built from its golden, on the golden's vector buffer."""
    def make():
        g = load_golden(golden)
        return (lambda: build(g)), vector_buffer_from_golden(g, False)
    return make


REUSE = {
    "sac": _r_sac,
    "discrete_sac": _r_dsac,
    "cql": _r_cql,
    "td3": _r_td3("td3_ref_mujoco.npz"),
    "td3_bc": _r_td3("td3_ref_bc.npz"),
    "bcq": _r_bcq,
    "dqn": _r_dqn,
    "qrdqn": _r_vector("qrdqn_ref_mlp.npz", build_qrdqn),
    "discrete_cql": _r_vector("dcql_ref_mlp.npz", build_qrdqn),
    # online_sample_size 8, target_sample_size 5
    "iqn": _r_vector("iqn_ref_sizes.npz", build_iqn),
    "discrete_bcq": _r_vector("dbcq_ref_mlp.npz", build_bcq),
    "discrete_crr": _r_vector("dcrr_ref_mlp.npz", build_crr),
}


@pytest.mark.parametrize("order", ["large_then_small", "small_then_large"])
@pytest.mark.parametrize("name", list(REUSE))
def test_second_batch_size_is_bit_identical_to_a_fresh_instance(name, order):
    """``B1`` updates, every scratch tensor is filled with NaN, then a ``B2`` update: parameters, lagged parameters, Adam moments and
    steps, losses and the priorities written back must equal, bit for bit, the ``B2`` update of a fresh instance loaded from the
    same ``state_dict()`` with the same random state."""
    build, buf = REUSE[name]()
    B1, B2 = (B_LARGE, B_SMALL) if order == "large_then_small" else (B_SMALL, B_LARGE)
    check_second_batch_size(build, buf, B1, B2, name=name)
