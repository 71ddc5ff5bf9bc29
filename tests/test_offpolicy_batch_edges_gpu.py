"""Every off-policy and offline update at the batch sizes its kernels split on, against float64 autograd, and every one of them
again after a batch of another size has used its scratch.

The row count of an update reaches the K of every weight-gradient GEMM (and with it the split-K switch), the M of
``ts_net_colsum``, the ``n`` of ``ts_mean``, the ``1 / B`` of every rows kernel, the grid of every per-row kernel (B, B x repeat
for CQL / BCQ, B x S for IQN) and the scratch caches: ``DeviceScratch.tensor`` matches on exact shape, ``FusedStack._buf`` only
grows.  Part 1 runs one update per (algorithm, batch) through each family's own float64 harness, at its own bars; part 2 runs
one batch size and then another on one instance, with every scratch tensor poisoned in between, and asks for the bits a fresh
instance in the same state computes."""
import copy
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GEMM_BK = 64            # net_gemm's K chunk: a GEMM can split K only from two chunks on


def grid_caps():
    """How many items (threads, or rows for the warp- and block-per-row kernels) one launch covers before its grid is capped and
    it strides; every item past a cap is reached only by the kernel's grid-stride loop."""
    s = torch.cuda.get_device_properties(0).multi_processor_count
    return {"net_ops_1d": s * 16 * 256,      # net_ops.cu TS_LAUNCH_1D: 16 blocks of 256 threads per SM, an item per thread
            "offpolicy_1d": s * 4 * 256,     # grid_for of td3.cu / cql.cu / bcq.cu: 4 blocks of 256 threads per SM
            "warp_per_row": s * 16 * 8,      # row_grid of row_sums.cuh / discrete_sac.cu: 16 blocks of 8 warps per SM
            "block_per_row": s * 8,          # ts_qrdqn_rows / ts_iqn_rows: 8 blocks per SM, a block per row
            "iqn_1d": s * 8 * 256}           # ew_grid of iqn.cu: 8 blocks of 256 threads per SM


def gemm_splits_k(K, M=64, N=64):
    """Whether ``ts_net_gemm`` splits K for a one-tile output (every weight gradient of the small networks below)."""
    from tianshou_b200._cabi import load_library
    return int(load_library().ts_net_gemm_workspace_floats(M, N, K)) > 0


# ------------------------------------------------------------------------------------------------------------ part 1
# name -> (run(B), rows of the largest per-row launch per sampled row, rows of the largest weight-gradient GEMM per sampled row)
def _sac(B, edge):
    from test_offpolicy_gpu import _sac_grad_case
    _sac_grad_case(O, A, (32, 32), True, True, False, seed=14, B=B, edge=edge)


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
    from test_offpolicy_gpu import _dqn_grad_case
    _dqn_grad_case("mlp", "mse", True, True, 0, B=B, edge=edge)


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
    from test_offpolicy_gpu import _Box
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
        return SAC(policy=SACPolicy(actor=actor, action_space=_Box(A)), policy_optim=AdamOptimizerFactory(lr=1e-3), critic=mk(),
                   critic_optim=AdamOptimizerFactory(lr=1e-3), critic2=mk(), critic2_optim=AdamOptimizerFactory(lr=1e-3), tau=0.005,
                   gamma=0.99, alpha=0.2, n_step_return_horizon=2)

    E, T = 4, 64
    buf = VectorReplayBuffer(E * T, E, device=DEV)
    for s in synth_rollout(np.random.default_rng(3), E, T, O, A, p_term=0.05, trunc_len=20):
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    return build, buf


def _r_golden(module, golden, build, buffer):
    """``build(mod, g, cfg)`` / ``buffer(mod, g, cfg)`` with the named test module, golden file and its ``cfg_*`` entries."""
    def make():
        from ts_testutil import load_golden
        mod = __import__(module)
        g = load_golden(golden)
        cfg = mod._cfg(g) if hasattr(mod, "_cfg") else None
        return (lambda: build(mod, g, cfg)), buffer(mod, g, cfg)
    return make


def _r_simple(module, golden, builder, buffer_fn):
    return _r_golden(module, golden, lambda mod, g, cfg: getattr(mod, builder)(g), lambda mod, g, cfg: getattr(mod, buffer_fn)(g, False))


def _r_td3(golden):
    return _r_golden("test_td3_gpu", golden, lambda mod, g, cfg: mod._build(cfg, g), lambda mod, g, cfg: mod._buffer(g, False))


def _cql_buffer(mod, g, cfg):
    return mod._build(cfg, g).process_buffer(mod._buffer(g, False))       # adds the calibration returns


def _r_dqn():
    from test_offpolicy_gpu import _Discrete, _dqn_grad_setup
    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.dqn import DQN, DiscreteQLearningPolicy
    A = 6
    net, buf = _dqn_grad_setup("mlp", A, seed=8, per=False)
    net0 = copy.deepcopy(net)

    def build():
        return DQN(policy=DiscreteQLearningPolicy(model=copy.deepcopy(net0), action_space=_Discrete(A)), optim=AdamOptimizerFactory(lr=1e-3),
                   gamma=0.9, n_step_return_horizon=2, target_update_freq=3, is_double=True)
    return build, buf


REUSE = {
    "sac": _r_sac,
    "discrete_sac": _r_simple("test_discrete_sac_gpu", "dsac_ref_auto.npz", "_build_from_golden", "_buffer_from_golden"),
    "cql": _r_golden("test_cql_gpu", "cql_ref_d4rl.npz", lambda mod, g, cfg: mod._build(cfg, g), _cql_buffer),
    "td3": _r_td3("td3_ref_mujoco.npz"),
    "td3_bc": _r_td3("td3_ref_bc.npz"),
    "bcq": _r_golden("test_bcq_gpu", "bcq_ref_small.npz", lambda mod, g, cfg: mod._build(cfg), lambda mod, g, cfg: mod._buffer(g, False)),
    "dqn": _r_dqn,
    "qrdqn": _r_simple("test_qrdqn_gpu", "qrdqn_ref_mlp.npz", "build_from_golden", "buffer_from_golden"),
    "discrete_cql": _r_simple("test_qrdqn_gpu", "dcql_ref_mlp.npz", "build_from_golden", "buffer_from_golden"),
    # online_sample_size 8, target_sample_size 5
    "iqn": _r_simple("test_iqn_gpu", "iqn_ref_sizes.npz", "build_from_golden", "buffer_from_golden"),
    "discrete_bcq": _r_simple("test_discrete_bcq_gpu", "dbcq_ref_mlp.npz", "build_bcq", "buffer_from_golden"),
    "discrete_crr": _r_simple("test_discrete_crr_gpu", "dcrr_ref_mlp.npz", "build_crr", "buffer_from_golden"),
}
B_SMALL, B_LARGE = 17, 200          # one K chunk / four K chunks; CQL and BCQ repeat them to 170 / 2000 rows


def _flat_groups(algo):
    from tianshou_b200.algorithm.flat_params import FlatGroup
    out = []
    for v in vars(algo).values():
        for x in (v if isinstance(v, (list, tuple)) else (v,)):
            if isinstance(x, FlatGroup):
                out.append(x)
    return out


def _fused_stacks(algo):
    """Every FusedStack the algorithm reaches through its own (non-module) attributes: the networks' scratch owners."""
    from tianshou_b200.algorithm.netgraph import FusedStack
    found, seen = [], set()

    def walk(x, depth):
        if id(x) in seen or depth > 3 or isinstance(x, (torch.nn.Module, torch.Tensor)):
            return
        seen.add(id(x))
        if isinstance(x, FusedStack):
            found.append(x)
        elif isinstance(x, (list, tuple)):
            for y in x:
                walk(y, depth + 1)
        elif isinstance(x, dict):
            for y in x.values():
                walk(y, depth + 1)
        elif type(x).__module__.startswith("tianshou_b200.algorithm"):
            for y in vars(x).values():
                walk(y, depth + 1)

    for v in vars(algo).values():
        walk(v, 0)
    return found


def _poison(algo):
    """NaN into every floating tensor of the algorithm's DeviceScratch and every FusedStack buffer (workspace included)."""
    n = 0
    for t in list(algo._scratch.values()) + [t for s in _fused_stacks(algo) for t in s._bufs.values()]:
        if isinstance(t, torch.Tensor) and t.is_floating_point() and t.is_cuda:
            t.fill_(float("nan"))
            n += 1
    return n


def _rng_state(buf):
    return copy.deepcopy((buf.__dict__["_random_state"], buf.__dict__.get("_child_rngs")))


def _set_rng_state(buf, state):
    rs, child = copy.deepcopy(state)
    buf.__dict__["_random_state"] = rs
    if child is not None:
        buf.__dict__["_child_rngs"] = child


def _update(algo, buf, B, seed):
    """One update with every random source seeded: what it returned, and the TD errors / priorities it handed back."""
    from tianshou_b200.utils import policy_within_training_step
    cap = {}
    orig_pre, orig_post = algo._preprocess_batch, algo._postprocess_batch

    def pre(batch, buffer, indices):
        cap["indices"] = np.asarray(indices).copy()
        return orig_pre(batch, buffer, indices)

    def post(batch, buffer, indices):
        w = batch.__dict__.get("weight")
        cap["prio"] = None if w is None else torch.as_tensor(w).detach().reshape(-1).clone()
        return orig_post(batch, buffer, indices)

    algo._preprocess_batch, algo._postprocess_batch = pre, post
    np.random.seed(seed)
    torch.manual_seed(seed)
    try:
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=B)
    finally:
        algo._preprocess_batch, algo._postprocess_batch = orig_pre, orig_post
    torch.cuda.synchronize()
    scalars = {k: v for k, v in vars(stats).items() if k != "train_time" and (v is None or isinstance(v, (int, float)))}
    return cap, scalars


def _carry_outside_state_dict(a, b):
    """What the reference keeps outside ``state_dict()`` and whoever restores a run carries over by hand: the plain update
    counters, CQL's Lagrange multiplier with its Adam, AutoAlpha's Adam."""
    for attr in ("_iter", "_cnt", "_last"):
        if hasattr(a, attr):
            setattr(b, attr, copy.copy(getattr(a, attr)))
    if getattr(a, "with_lagrange", False):
        with torch.no_grad():
            b.cql_log_alpha.copy_(a.cql_log_alpha)
        b.cql_alpha_optim.load_state_dict(copy.deepcopy(a.cql_alpha_optim.state_dict()))
    alpha_optim = getattr(getattr(a, "alpha", None), "_optim", None)
    if alpha_optim is not None:
        b.alpha._optim.load_state_dict(copy.deepcopy(alpha_optim.state_dict()))


def _state(algo):
    out = []
    for g in _flat_groups(algo):
        out += [g.flat.clone(), g.exp_avg.clone(), g.exp_avg_sq.clone(), torch.tensor([g.sync_step_from_device()])]
    return out


@pytest.mark.parametrize("order", ["large_then_small", "small_then_large"])
@pytest.mark.parametrize("name", list(REUSE))
def test_second_batch_size_is_bit_identical_to_a_fresh_instance(name, order):
    """``B1`` updates, every scratch tensor is filled with NaN, then a ``B2`` update: parameters, lagged parameters, Adam moments and
    steps, losses and the priorities written back must equal, bit for bit, the ``B2`` update of a fresh instance loaded from the
    same ``state_dict()`` with the same random state."""
    build, buf = REUSE[name]()
    B1, B2 = (B_LARGE, B_SMALL) if order == "large_then_small" else (B_SMALL, B_LARGE)
    a = build()
    _update(a, buf, B1, seed=1)
    b = build()
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    _carry_outside_state_dict(a, b)
    rng = _rng_state(buf)
    assert _poison(a) > 0
    cap_a, stats_a = _update(a, buf, B2, seed=2)
    _set_rng_state(buf, rng)
    cap_b, stats_b = _update(b, buf, B2, seed=2)
    assert np.array_equal(cap_a["indices"], cap_b["indices"]) and len(cap_a["indices"]) == B2
    assert stats_a == stats_b, f"{name}: losses differ after a batch of {B1}: {stats_a} vs {stats_b}"
    assert all(v is None or math.isfinite(v) for v in stats_a.values())
    if cap_a.get("prio") is not None:
        assert cap_a["prio"].numel() == B2 and torch.equal(cap_a["prio"], cap_b["prio"])
    sa, sb = _state(a), _state(b)
    for i, (x, y) in enumerate(zip(sa, sb, strict=True)):
        assert torch.equal(x, y), f"{name}: state tensor {i} (group {i // 4}, {('flat', 'exp_avg', 'exp_avg_sq', 'step')[i % 4]}) differs"
