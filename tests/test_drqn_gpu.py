"""DRQN (DQN on ``Recurrent``) on the GPU: the LSTM cell kernels against float64, the recurrent stack's forward and backward
through time against float64 autograd of ``nn.LSTM``, ``DQN.update()`` against outputs of the imported reference
(tests/golden/drqn_ref_*.npz from oracle/gen_golden_drqn.py), one update's gradient against float64 autograd, the batch edges,
the ``state_dict()`` round trip, the cuDNN re-pointing of the LSTM weights by the torch forward, stacked flat observations for a
plain ``Net``, the refusals and the kernels' register report."""
import copy

import numpy as np
import pytest
import torch

from oracle import oracle_discrete_sac as ods
from oracle import oracle_drqn as od
from offpolicy_testutil import (B_LARGE, B_SMALL, DEV, EPS, Discrete, assert_spill_free, capture_batches, capture_grads,
                                check_final_state, check_second_batch_size, optimiser_state, ptxas_report, rng_state,
                                set_rng_state, stream)
from ts_testutil import load_golden, record_parity

gpu = pytest.mark.gpu
VARIANTS = ["drqn_ref_mlp", "drqn_ref_per", "drqn_ref_s1"]


def _cfg(g, k):
    return g[f"cfg_{k}"].item()


# ------------------------------------------------------------------------------------------------------------ cell kernels
def _cell64(pre, b_hh, c_prev):
    z = pre + b_hh
    i, f, g, o = z.chunk(4, dim=1)
    i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
    c = f * c_prev + i * g if c_prev is not None else i * g
    return torch.cat([i, f, g, o], 1), c, o * torch.tanh(c)


@gpu
@pytest.mark.parametrize("H", [1, 5, 128, 256])
@pytest.mark.parametrize("B", [1, 17, 200])
@pytest.mark.parametrize("first", [True, False])
def test_cell_kernels_vs_fp64(B, H, first):
    """Forward (gates, c, h) and backward (dgates, dc_prev) of one step against float64 autograd of the cell on the same fp32
    inputs; ``first``: t = 0 (no c_prev, and the last step: no carried dc).  Rows past B keep their sentinel and two runs are
    bit-identical.  Error model: each activation is a few roundings of a full-accuracy expf / tanhf (|err| <= 8 eps of the
    inputs' scale); the backward multiplies at most five such values."""
    from tianshou_b200._cabi import call, ptr
    g = torch.Generator().manual_seed(B * 1000 + H + first)
    f32 = lambda *s: (torch.randn(*s, generator=g) * 2).to(DEV)
    pre, b_hh = f32(B, 4 * H), f32(4 * H)
    c_prev = None if first else f32(B, H)
    pad = 3
    gates, c, h = (torch.full((B + pad, n), 7.0, device=DEV) for n in (4 * H, H, H))

    def fwd():
        call("ts_lstm_cell", ptr(pre), ptr(b_hh), None if c_prev is None else ptr(c_prev), B, H, ptr(gates), ptr(c), ptr(h), stream())
        torch.cuda.synchronize()
        return gates.clone(), c.clone(), h.clone()

    out1, out2 = fwd(), fwd()
    assert all(torch.equal(a, b) for a, b in zip(out1, out2))
    assert all(bool((t[B:] == 7.0).all()) for t in out1), "rows past B written"
    pre64 = pre.double().cpu().requires_grad_(True)
    cp64 = None if c_prev is None else c_prev.double().cpu().requires_grad_(True)
    g64, c64, h64 = _cell64(pre64, b_hh.double().cpu(), cp64)
    scale = 8 * EPS * (1 + float(pre.abs().max()) + (0 if c_prev is None else float(c_prev.abs().max())))
    for name, got, want in (("gates", gates, g64), ("c", c, c64), ("h", h, h64)):
        record_parity(f"lstm_cell/B{B}_H{H}_t{int(not first)}/{name}", got[:B].cpu().numpy(), want.detach().numpy(), rtol=0, atol=scale)
    dh = f32(B, H)
    dc = None if first else f32(B, H)
    dg = torch.full((B + pad, 4 * H), 7.0, device=DEV)
    dcp = torch.full((B + pad, H), 7.0, device=DEV)

    def bwd():
        call("ts_lstm_cell_bwd", ptr(gates), ptr(c), None if c_prev is None else ptr(c_prev), ptr(dh), None if dc is None else ptr(dc),
             B, H, ptr(dg), ptr(dcp), stream())
        torch.cuda.synchronize()
        return dg.clone(), dcp.clone()

    b1, b2 = bwd(), bwd()
    assert all(torch.equal(a, b) for a, b in zip(b1, b2)), "the backward must be bit-identical run to run"
    assert bool((dg[B:] == 7.0).all()) and bool((dcp[B:] == 7.0).all()), "rows past B written"
    # float64 autograd of the cell from the same fp32 pre-activations: dgates at the pre-activations, dc_prev
    c_prev64 = torch.zeros(B, H, dtype=torch.float64) if c_prev is None else c_prev.double().cpu()
    pre64b = pre.double().cpu().requires_grad_(True)
    c_in = c_prev64.clone().requires_grad_(True)
    _, cc, hh = _cell64(pre64b, b_hh.double().cpu(), c_in)
    loss = (hh * dh.double().cpu()).sum() + ((cc * dc.double().cpu()).sum() if dc is not None else 0.0)
    loss.backward()
    bs = 16 * EPS * float(dh.abs().max() + (0 if dc is None else dc.abs().max())) * (1 + float(pre.abs().max()))
    record_parity(f"lstm_cell_bwd/B{B}_H{H}_t{int(not first)}/dgates", dg[:B].cpu().numpy(), pre64b.grad.numpy(), rtol=0, atol=bs)
    record_parity(f"lstm_cell_bwd/B{B}_H{H}_t{int(not first)}/dc_prev", dcp[:B].cpu().numpy(), c_in.grad.numpy(), rtol=0,
                  atol=bs * (1 + float(c_prev64.abs().max())))


# ------------------------------------------------------------------------------------------------------------ the stack
def _recurrent(L, D=6, A=3, H=32, seed=0):
    from tianshou_b200.utils.net.common import Recurrent
    torch.manual_seed(seed)
    return Recurrent(layer_num=L, state_shape=D, action_shape=A, hidden_layer_size=H).to(DEV)


@gpu
@pytest.mark.parametrize("L", [1, 2, 3])
@pytest.mark.parametrize("S", [1, 4, 8])
def test_stack_forward_backward_vs_fp64_autograd(S, L):
    """Q and every parameter gradient (d sum(q * dq)) against float64 autograd of ``fc1 -> nn.LSTM -> fc2`` on the same weights,
    from zero state.  The GEMMs are fp32-faithful (bf16x3) and a gradient sums up to S * n products: 2e-4 relative plus 1e-4 of
    the tensor's largest value, as the other layered networks' gradient tests."""
    from tianshou_b200.algorithm.recurrent import RecurrentStack
    model = _recurrent(L, seed=S * 10 + L)
    ref = copy.deepcopy(model).to("cpu", torch.float64)
    stack = RecurrentStack(model, torch.device(DEV))
    n, D = 37, 6
    g = torch.Generator().manual_seed(S + 100 * L)
    obs = torch.randn(n, S, D, generator=g)
    dq = torch.randn(n, 3, generator=g)
    x = obs.transpose(0, 1).contiguous().reshape(S * n, D).to(DEV)
    acts = stack.forward(x, n, "t")
    stack.backward(acts, dq.to(DEV), n, "t")
    torch.cuda.synchronize()
    out, _ = ref.nn(ref.fc1(obs.double()))
    q64 = ref.fc2(out[:, -1])
    (q64 * dq.double()).sum().backward()
    tag = f"drqn_stack/S{S}_L{L}"
    record_parity(f"{tag}/q", acts[-1].cpu().numpy(), q64.detach().numpy(), rtol=2e-5, atol=2e-5 * float(q64.detach().abs().max()))
    grp = stack.group
    for i, (p, r) in enumerate(zip(grp.params, ref.parameters(), strict=True)):
        want = r.grad.numpy()
        got = grp.view(grp.grad, p).view(p.shape).cpu().numpy()
        record_parity(f"{tag}/grad_{i}", got, want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)


# ------------------------------------------------------------------------------------------------------------ updates
def drqn_buffer(g, mirror=False):
    """The golden's rollout in a vector buffer with its ``stack_num`` and ``obs_next`` storage, prioritised when it sets ``per``."""
    from tianshou_b200.data import Batch, PrioritizedVectorReplayBuffer, VectorReplayBuffer
    E, cap = int(_cfg(g, "E")), int(_cfg(g, "cap"))
    kw = dict(stack_num=int(_cfg(g, "stack")), ignore_obs_next=not bool(_cfg(g, "obs_next")), device=DEV, device_mirror=mirror)
    if bool(_cfg(g, "per")):
        buf = PrioritizedVectorReplayBuffer(E * cap, E, alpha=float(_cfg(g, "alpha")), beta=float(_cfg(g, "beta")), **kw)
    else:
        buf = VectorReplayBuffer(E * cap, E, **kw)
    for i in range(int(_cfg(g, "steps"))):
        s = {k: g[f"roll{i}_{k}"] for k in ("obs", "act", "rew", "terminated", "truncated", "obs_next")}
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    return buf


def build_from_golden(g):
    from tianshou_b200.algorithm import DQN, AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.dqn import DiscreteQLearningPolicy
    from tianshou_b200.utils.net.common import Recurrent
    A = int(_cfg(g, "A"))
    model = Recurrent(layer_num=int(_cfg(g, "layers")), state_shape=int(_cfg(g, "obs")), action_shape=A,
                      hidden_layer_size=int(_cfg(g, "hidden"))).to(DEV)
    ods.seeded_params(model, int(_cfg(g, "init_seed")))
    policy = DiscreteQLearningPolicy(model=model, action_space=Discrete(A))
    return DQN(policy=policy, optim=AdamOptimizerFactory(lr=float(_cfg(g, "lr"))), gamma=float(_cfg(g, "gamma")),
               n_step_return_horizon=int(_cfg(g, "n_step")), target_update_freq=int(_cfg(g, "freq")),
               is_double=bool(_cfg(g, "double")), huber_loss_delta=float(_cfg(g, "huber")) or None)


@gpu
@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("variant", VARIANTS)
def test_update_matches_reference(variant, mirror):
    """Update after update against the reference's run: the same sampled indices, n-step returns, loss and priorities written
    back, then the final parameters, Adam moments and lagged parameters, the ``state_dict()`` keys and the optimiser's
    param indices."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"{variant}.npz")
    algo, buf = build_from_golden(g), drqn_buffer(g, mirror)
    keys = [str(k) for k in g["state_dict_keys"]]
    assert list(algo.state_dict().keys()) == keys
    with capture_batches(algo) as cap:
        for u in range(int(_cfg(g, "updates"))):
            np.random.seed(700 + u)
            with policy_within_training_step(algo.policy):
                stats = algo.update(buffer=buf, sample_size=int(_cfg(g, "bs")))
            tag = f"{variant}_m{int(mirror)}_u{u}"
            assert np.array_equal(cap["indices"], g[f"u{u}_indices"]), "sampled indices differ from the reference's"
            ref_ret = g[f"u{u}_returns"].reshape(-1)
            record_parity(f"{tag}/returns", cap["returns"].cpu().numpy().reshape(-1), ref_ret, rtol=1e-4,
                          atol=1e-5 * float(np.abs(ref_ret).max()))
            record_parity(f"{tag}/losses", np.array([stats.loss]), g[f"u{u}_losses"], rtol=1e-4, atol=1e-6)
            prio = g[f"u{u}_prio"].reshape(-1)
            record_parity(f"{tag}/prio", cap["prio"].cpu().numpy().reshape(-1), prio, rtol=1e-4, atol=1e-5 * float(np.abs(prio).max()))
    check_final_state(f"{variant}_m{int(mirror)}", g, algo)
    assert list(algo.state_dict().keys()) == keys
    osd = algo.state_dict()["_optimizers"][0]
    assert list(osd["param_groups"][0]["params"]) == [int(i) for i in g["opt_param_ids"]]
    assert sorted(osd["state"].keys()) == [int(i) for i in g["opt_state_ids"]]


def _stacked(buf, idx, col, S):
    """buffer[idx].<col> stacked along the prev() chain, oldest first, on the host."""
    arr, out, cur = np.asarray(getattr(buf, col)), [], np.asarray(idx)
    for _ in range(S):
        out.insert(0, arr[cur])
        cur = buf.prev(cur)
    return np.stack(out, axis=1)


def grad_case(B, tag):
    """One update at batch ``B`` (the lagged copy is refreshed by it, so the target uses the same weights): the flat gradient
    before its Adam step against float64 autograd of the loss through the oracle's explicit LSTM on the update's own indices
    and returns.  Tolerance as in test_stack_forward_backward_vs_fp64_autograd."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("drqn_ref_mlp.npz")
    algo, buf = build_from_golden(g), drqn_buffer(g)
    model = algo.policy.model
    net = od.DrqnNet(int(_cfg(g, "layers")), int(_cfg(g, "obs")), int(_cfg(g, "A")), int(_cfg(g, "hidden")))
    od.load_from(net, list(model.parameters()))
    np.random.seed(7)
    with capture_batches(algo) as cap, capture_grads(algo._group) as grads, policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, sample_size=B)
    idx, returns = cap["indices"], cap["returns"].cpu().double().reshape(-1)
    x = torch.as_tensor(_stacked(buf, idx, "obs", int(_cfg(g, "stack"))), dtype=torch.float64)
    q = net(x)[np.arange(len(idx)), np.asarray(buf.act)[idx].astype(np.int64)]
    loss = (returns - q).pow(2).mean()
    loss.backward()
    grp = algo._group
    for i, (p, r) in enumerate(zip(grp.params, net.parameters(), strict=True)):
        want = r.grad.numpy()
        got = grp.view(grads[-1], p).view(p.shape).cpu().numpy()
        record_parity(f"drqn_grad{tag}/grad_{i}", got, want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)
    record_parity(f"drqn_grad{tag}/loss", np.array([stats.loss]), np.array([loss.item()]), rtol=2e-5, atol=2e-6)
    assert len(idx) == B


@gpu
@pytest.mark.parametrize("B", [1, 64, 65, 200])
def test_update_gradient_vs_fp64_autograd(B):
    """B = 1, the weight-gradient GEMMs at one and two K chunks of the last step (64 / 65 rows), and B_LARGE."""
    grad_case(B, f"@B{B}")


@gpu
@pytest.mark.parametrize("order", ["large_then_small", "small_then_large"])
def test_second_batch_size_is_bit_identical_to_a_fresh_instance(order):
    g = load_golden("drqn_ref_mlp.npz")
    B1, B2 = (B_LARGE, B_SMALL) if order == "large_then_small" else (B_SMALL, B_LARGE)
    check_second_batch_size(lambda: build_from_golden(g), drqn_buffer(g), B1, B2, name="drqn")


@gpu
def test_state_dict_round_trip_continues_identically():
    """A fresh algorithm loaded from another's ``state_dict()`` (and ``_iter``) continues bit for bit."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("drqn_ref_mlp.npz")
    a, buf = build_from_golden(g), drqn_buffer(g)
    for u in range(3):
        np.random.seed(u)
        with policy_within_training_step(a.policy):
            a.update(buffer=buf, sample_size=32)
    b = build_from_golden(g)
    with torch.no_grad():                      # b starts elsewhere: every value must come from the state_dict
        for p in b.policy.model.parameters():
            p.add_(1.0)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    b._iter = a._iter
    st = rng_state(buf)
    for algo in (a, b):
        set_rng_state(buf, st)
        np.random.seed(11)
        with policy_within_training_step(algo.policy):
            algo.update(buffer=buf, sample_size=32)
    for x, y in zip(optimiser_state(a), optimiser_state(b), strict=True):
        assert torch.equal(x, y)
    for x, y in zip(a.model_old.parameters(), b.model_old.parameters(), strict=True):
        assert torch.equal(x, y)


@gpu
def test_torch_forward_between_updates_keeps_device_parameters():
    """update -> the Collector's torch forward (cuDNN's flatten_parameters re-points the LSTM weights) -> update -> forward.
    Every step must see the device parameters: the torch forward reads the values the updates wrote, the second update
    continues exactly as an instance that never ran a torch forward, and neither forward touches the Adam state."""
    from tianshou_b200.data import Batch
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("drqn_ref_mlp.npz")
    a, b, buf = build_from_golden(g), build_from_golden(g), drqn_buffer(g)
    obs = torch.as_tensor(g["roll0_obs"], device=DEV)
    drawn = {}

    def step(algo, seed):         # both instances draw the same indices from the shared buffer
        if algo is a:
            drawn[seed] = rng_state(buf)
        else:
            set_rng_state(buf, drawn[seed])
        np.random.seed(seed)
        with policy_within_training_step(algo.policy):
            algo.update(buffer=buf, sample_size=32)

    def forward_and_check(algo):
        before = optimiser_state(algo)
        ref = copy.deepcopy(algo.policy.model).to("cpu", torch.float64)
        out = algo.policy(Batch(obs=obs, info=Batch()))
        torch.cuda.synchronize()
        q64, _ = ref.fc2(ref.nn(ref.fc1(obs.cpu().double().unsqueeze(1)))[0][:, -1]), None
        record_parity("drqn_flatten/q", out.logits.detach().cpu().numpy(), q64.detach().numpy(), rtol=1e-4, atol=1e-5)
        grp = algo._group
        for p in grp.params:
            assert torch.equal(p.detach(), grp.view(grp.flat, p).view(p.shape)), "the torch forward reads other weights"
        for x, y in zip(before, optimiser_state(algo), strict=True):
            assert torch.equal(x, y), "the torch forward changed the optimiser state"

    step(a, 1)
    step(b, 1)
    forward_and_check(a)
    step(a, 2)
    step(b, 2)
    for x, y in zip(optimiser_state(a), optimiser_state(b), strict=True):
        assert torch.equal(x, y), "an update after a torch forward differs from one without"
    forward_and_check(a)
    step(a, 3)
    step(b, 3)
    for x, y in zip(optimiser_state(a), optimiser_state(b), strict=True):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------------------ stacked Net
def _flat_buffer(S, D, obs_next, E=4, steps=30, seed=0):
    """Random flat episodes (ends inside the buffer, so stacks cross episode starts) in a ``stack_num=S`` buffer."""
    from tianshou_b200.data import Batch, VectorReplayBuffer
    rng = np.random.default_rng(seed)
    buf = VectorReplayBuffer(E * 40, E, stack_num=S, ignore_obs_next=not obs_next, device=DEV)
    obs = rng.standard_normal((E, D)).astype(np.float32)
    for _ in range(steps):
        nxt = rng.standard_normal((E, D)).astype(np.float32)
        term = rng.random(E) < 0.1
        buf.add(Batch(obs=obs, act=rng.integers(0, 2, E), rew=rng.standard_normal(E), terminated=term, truncated=np.zeros(E, bool),
                      obs_next=nxt), buffer_ids=np.arange(E))
        obs = np.where(term[:, None], rng.standard_normal((E, D)).astype(np.float32), nxt)
    assert buf.done.sum() > 0
    return buf


@gpu
@pytest.mark.parametrize("obs_next", [False, True])
@pytest.mark.parametrize("S", [1, 3])
def test_stacked_flat_observations_for_a_plain_net(S, obs_next):
    """A ``Net(state_shape=(S, D))`` on a ``stack_num=S`` buffer reads exactly the reference's stacked batch, flattened, for
    obs and obs_next (stored, or the stack at next(index)), and the recurrent reading is the same rows time-major."""
    from tianshou_b200.algorithm.flat_params import DeviceScratch
    from tianshou_b200.algorithm.obs_source import device_obs_source
    D = 5
    buf = _flat_buffer(S, D, obs_next)
    idx = buf.sample_indices(64)
    sc = DeviceScratch(torch.device(DEV))
    for key in ("obs", "obs_next"):
        src = device_obs_source(buf, idx, key, (S * D,), 1.0, torch.device(DEV), sc.tensor)
        if key == "obs_next" and not obs_next:
            want = _stacked(buf, buf.next(idx), "obs", S)
        else:
            want = _stacked(buf, idx, key, S)
        assert np.array_equal(src.x.cpu().numpy(), want.reshape(len(idx), S * D))
        seq = device_obs_source(buf, idx, key, (D,), 1.0, torch.device(DEV), sc.tensor, seq=True)
        assert seq.steps == S and np.array_equal(seq.x.cpu().numpy(), want.transpose(1, 0, 2).reshape(S * len(idx), D))


@gpu
def test_stacked_net_update_and_width_mismatch():
    """DQN with ``Net(state_shape=(S, D))`` on a ``stack_num=S`` buffer: the update's gradient matches float64 autograd on the
    stacked batch.  A width that is not the network's input -- ``Net(state_shape=D)`` on that buffer, or the stacked net on a
    ``stack_num=1`` buffer -- is refused before anything reads it."""
    from tianshou_b200.algorithm import DQN, AdamOptimizerFactory, UnsupportedModelError
    from tianshou_b200.algorithm.modelfree.dqn import DiscreteQLearningPolicy
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    S, D = 3, 5

    def make(shape):
        torch.manual_seed(0)
        net = Net(state_shape=shape, action_shape=2, hidden_sizes=(32,)).to(DEV)
        return DQN(policy=DiscreteQLearningPolicy(model=net, action_space=Discrete(2)), optim=AdamOptimizerFactory(lr=1e-3),
                   gamma=0.9, n_step_return_horizon=1, target_update_freq=0)

    buf = _flat_buffer(S, D, False)
    algo = make((S, D))
    ref = copy.deepcopy(algo.policy.model).to("cpu", torch.float64)
    np.random.seed(3)
    with capture_batches(algo) as cap, capture_grads(algo._group) as grads, policy_within_training_step(algo.policy):
        algo.update(buffer=buf, sample_size=48)
    idx, returns = cap["indices"], cap["returns"].cpu().double().reshape(-1)
    q = ref.model.model(torch.as_tensor(_stacked(buf, idx, "obs", S).reshape(len(idx), S * D), dtype=torch.float64))
    q = q[np.arange(len(idx)), np.asarray(buf.act)[idx].astype(np.int64)]
    (returns - q).pow(2).mean().backward()
    grp = algo._group
    for i, (p, r) in enumerate(zip(grp.params, ref.parameters(), strict=True)):
        want = r.grad.numpy()
        record_parity(f"stacked_net/grad_{i}", grp.view(grads[-1], p).view(p.shape).cpu().numpy(), want, rtol=2e-4,
                      atol=1e-4 * float(np.abs(want).max()) + 1e-12)
    for algo, b in ((make(D), buf), (make((S, D)), _flat_buffer(1, D, False))):
        with pytest.raises(UnsupportedModelError, match="the network reads"), policy_within_training_step(algo.policy):
            algo.update(buffer=b, sample_size=16)


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals():
    from torch import nn
    from tianshou_b200.algorithm import (C51, DQN, FQF, IQN, AdamOptimizerFactory, C51Policy, DiscreteBCQ, DiscreteBCQPolicy,
                                         DiscreteCQL, DiscreteCRR, DiscreteSAC, FQFPolicy, IQNPolicy, QRDQN, QRDQNPolicy,
                                         RainbowDQN, UnsupportedModelError)
    from tianshou_b200.algorithm.modelfree.discrete_sac import DiscreteSACPolicy
    from tianshou_b200.algorithm.modelfree.dqn import DiscreteQLearningPolicy
    from tianshou_b200.algorithm.modelfree.reinforce import DiscreteActorPolicy
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.discrete import (DiscreteActor, DiscreteCritic, FractionProposalNetwork, FullQuantileFunction,
                                                  ImplicitQuantileNetwork)
    A, opt = 2, lambda: AdamOptimizerFactory(lr=1e-3)

    def dqn(model):
        return DQN(policy=DiscreteQLearningPolicy(model=model, action_space=Discrete(A)), optim=opt(), target_update_freq=2)

    dqn(_recurrent(2, A=A))                     # the reference's construction builds
    for attr, kw, what in (("nn", dict(bias=False), "bias=False"), ("nn", dict(proj_size=4), "proj_size"),
                           ("nn", dict(bidirectional=True), "bidirectional"), ("nn", dict(dropout=0.5, num_layers=2), "dropout"),
                           ("nn", dict(batch_first=False), "batch_first")):
        model = _recurrent(2, A=A)
        args = dict(input_size=32, hidden_size=32, num_layers=1, batch_first=True) | kw
        setattr(model, attr, nn.LSTM(**args).to(DEV))
        with pytest.raises(UnsupportedModelError, match=what):
            dqn(model)
    # image observations: a Recurrent over flattened frames is refused at the first read of the buffer
    algo = dqn(_recurrent(1, D=16, A=A))
    buf = VectorReplayBuffer(40, 4, device=DEV)
    for _ in range(8):
        fr = np.random.default_rng(0).integers(0, 255, (4, 4, 4), dtype=np.uint8)
        buf.add(Batch(obs=fr, act=np.zeros(4, np.int64), rew=np.zeros(4), terminated=np.zeros(4, bool),
                      truncated=np.zeros(4, bool), obs_next=fr), buffer_ids=np.arange(4))
    with pytest.raises(UnsupportedModelError, match="recurrent network reads flat float"), policy_within_training_step(algo.policy):
        algo.update(buffer=buf, sample_size=8)
    # every other algorithm names DQN as the only device user of a Recurrent network
    rec = lambda: _recurrent(1, A=A)
    makers = [
        lambda: QRDQN(policy=QRDQNPolicy(model=rec(), action_space=Discrete(A)), optim=opt(), num_quantiles=4),
        lambda: DiscreteCQL(policy=QRDQNPolicy(model=rec(), action_space=Discrete(A)), optim=opt(), num_quantiles=4),
        lambda: C51(policy=C51Policy(model=rec(), action_space=Discrete(A), num_atoms=4), optim=opt()),
        lambda: RainbowDQN(policy=C51Policy(model=rec(), action_space=Discrete(A), num_atoms=4), optim=opt()),
        lambda: IQN(policy=IQNPolicy(model=ImplicitQuantileNetwork(preprocess_net=rec(), action_shape=A).to(DEV),
                                     action_space=Discrete(A)), optim=opt()),
        lambda: FQF(policy=FQFPolicy(model=FullQuantileFunction(preprocess_net=rec(), action_shape=A).to(DEV),
                                     fraction_model=FractionProposalNetwork(8, A).to(DEV), action_space=Discrete(A)),
                    optim=opt(), fraction_optim=opt(), num_fractions=8),
        lambda: DiscreteBCQ(policy=DiscreteBCQPolicy(model=DiscreteActor(preprocess_net=rec(), action_shape=A, softmax_output=False).to(DEV),
                                                     imitator=DiscreteActor(preprocess_net=rec(), action_shape=A, softmax_output=False).to(DEV),
                                                     action_space=Discrete(A)), optim=opt()),
        lambda: DiscreteCRR(policy=DiscreteActorPolicy(actor=DiscreteActor(preprocess_net=rec(), action_shape=A, softmax_output=False).to(DEV),
                                                       action_space=Discrete(A)),
                            critic=DiscreteCritic(preprocess_net=rec(), last_size=A).to(DEV), optim=opt()),
        lambda: DiscreteSAC(policy=DiscreteSACPolicy(actor=DiscreteActor(preprocess_net=rec(), action_shape=A, softmax_output=False).to(DEV),
                                                     action_space=Discrete(A)), policy_optim=opt(),
                            critic=DiscreteCritic(preprocess_net=rec(), last_size=A).to(DEV), critic_optim=opt()),
    ]
    for k, make in enumerate(makers):
        with pytest.raises(UnsupportedModelError, match="DQN only"):
            make()


# ------------------------------------------------------------------------------------------------------------ resources
def test_kernels_have_no_stack_frame_or_spills(tmp_path):
    report = ptxas_report("lstm.cu", tmp_path)
    assert len(report) == 2 and all(("lstm_cell_kernel" in e) or ("lstm_cell_bwd_kernel" in e) for e in report), report
    assert_spill_free(report)
