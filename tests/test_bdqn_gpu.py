"""BDQN on the GPU: the bdqn.cu kernels against float64 (argmax ties, end flags from truncation and unfinished episodes, B = 1,
odd B, B past the grid cap), the branch-ensemble chain of ``FusedStack`` against float64 autograd (forward, backward and the trunk
gradient that sums the value head and the branches), ``update()`` against outputs of the imported reference
(tests/golden/bdqn_ref_*.npz from oracle/gen_golden_bdqn.py) with the buffer mirror on and off, the update's gradient against
float64 autograd at bipedal_bdq.py's width, a smaller batch after a larger one, bit-identical repeats, the absence of host
synchronisation inside the update, ``state_dict()`` round trips, the refusals and the register report."""
import copy
import re

import numpy as np
import pytest
import torch

from offpolicy_testutil import DEV, MultiDiscrete, assert_spill_free, golden_cfg, load_params, ptxas_report, stream
from ts_testutil import load_golden, record_parity

gpu = pytest.mark.gpu
KEYS = ("obs", "act", "rew", "terminated", "truncated", "obs_next")
GRID_CAP_ROWS = 132 * 4 * 256 * 2       # past the grid-stride cap of bdqn.cu's row kernels on any H100 (<= 132 SMs)


def _net(O, nb, A, common, value, action, act=torch.nn.ReLU, **kw):
    from tianshou_b200.utils.net.common import BranchingNet
    return BranchingNet(state_shape=(O,), num_branches=nb, action_per_branch=A, common_hidden_sizes=list(common),
                        value_hidden_sizes=list(value), action_hidden_sizes=list(action), activation=act, **kw)


def _algo(net, lr=1e-3, **kw):
    from tianshou_b200.algorithm import BDQN, AdamOptimizerFactory, BDQNPolicy
    policy = BDQNPolicy(model=net, action_space=MultiDiscrete([net.action_per_branch] * net.num_branches))
    return BDQN(policy=policy, optim=AdamOptimizerFactory(lr=lr), **kw)


# ------------------------------------------------------------------------------------------------------------ kernels
def _q64(v, s):
    """[B, nb, A] float64 Q from v [B, 1] and s [nb, B, A]."""
    s = s.double().permute(1, 0, 2)
    return v.double().unsqueeze(1) + (s - s.mean(2, keepdim=True))


@gpu
@pytest.mark.parametrize("B,nb,A", [(1, 3, 4), (1, 1, 7), (33, 4, 25), (257, 9, 5), (GRID_CAP_ROWS + 3, 2, 3)])
def test_bdqn_kernels_vs_fp64(B, nb, A):
    from tianshou_b200._cabi import call, ptr
    g = torch.Generator().manual_seed(B * 31 + nb)
    v_on, v_tg = torch.randn(B, 1, generator=g), torch.randn(B, 1, generator=g)
    s_on, s_tg = torch.randn(nb, B, A, generator=g) * 2, torch.randn(nb, B, A, generator=g) * 2
    if A > 1:                       # exact ties of the online maximum in every third row: the first index must win
        tie = torch.arange(B) % 3 == 0
        top = s_on.max(2).values + 1.0
        s_on[:, tie, A - 1] = top[:, tie]
        s_on[:, tie, A // 2] = top[:, tie]
    n_buf = B + 11
    rew = torch.randn(n_buf, generator=g, dtype=torch.float64)
    idx = torch.randint(0, n_buf, (B,), generator=g)
    term = torch.rand(n_buf, generator=g) < 0.1
    trunc = (torch.rand(n_buf, generator=g) < 0.1) & ~term
    end = term | trunc
    end[idx[: max(1, B // 5)]] = True             # unfinished episodes' last slots: end flags set by the buffer
    act = torch.randint(0, A, (B, nb), generator=g)
    w = torch.rand(B, generator=g) + 0.1
    d = {k: t.to(DEV).contiguous() for k, t in dict(v_on=v_on, v_tg=v_tg, s_on=s_on, s_tg=s_tg, rew=rew, idx=idx,
                                                      end=end.to(torch.uint8), act=act, w=w).items()}
    gamma = 0.99
    y = torch.full((B,), float("nan"), device=DEV)
    yb = torch.full((B, nb), float("nan"), device=DEV)
    call("ts_bdqn_target", ptr(d["v_on"]), ptr(d["s_on"]), ptr(d["v_tg"]), ptr(d["s_tg"]), B, nb, A, gamma, ptr(d["rew"]),
         ptr(d["end"]), ptr(d["idx"]), ptr(y), ptr(yb), stream())
    torch.cuda.synchronize()
    q_on, q_tg = _q64(v_on, s_on), _q64(v_tg, s_tg)
    astar = q_on.argmax(-1, keepdim=True)
    if A > 1:
        assert bool((astar[tie, :, 0] == A // 2).all())
    tq = q_tg.gather(-1, astar).squeeze(-1)
    live = (~end[idx]).double()
    want_b = rew[idx].unsqueeze(1) + np.float32(gamma) * tq * live.unsqueeze(1)
    want = rew[idx] + np.float32(gamma) * tq.mean(1) * live
    tag = f"bdqn_kernels/B{B}_nb{nb}_A{A}"
    record_parity(f"{tag}/y", y.cpu().numpy(), want.numpy(), rtol=1e-5, atol=1e-5)
    record_parity(f"{tag}/y_branch", yb.cpu().numpy(), want_b.numpy(), rtol=1e-5, atol=1e-5)
    # terminated or truncated or unfinished: the target is the reward alone, exactly
    ended = end[idx].numpy()
    assert np.array_equal(y.cpu().numpy()[ended], rew[idx].numpy()[ended].astype(np.float32))

    for weighted in (False, True):
        yt = y.clone()
        td, rows, tds = (torch.full(s, float("nan"), device=DEV) for s in ((B, nb), (B,), (B,)))
        ds, dv, loss = torch.full((nb, B, A), float("nan"), device=DEV), torch.full((B, 1), float("nan"), device=DEV), \
            torch.full((1,), float("nan"), device=DEV)
        ybr = yb if B == 1 else None
        call("ts_bdqn_rows", ptr(d["v_on"]), ptr(d["s_on"]), ptr(d["act"]), ptr(yt), ptr(d["w"]) if weighted else None, ptr(ybr), B,
             nb, A, ptr(td), ptr(rows), ptr(tds), ptr(ds), ptr(dv), ptr(loss), stream())
        torch.cuda.synchronize()
        vv = v_on.double().requires_grad_(True)
        ss = s_on.double().requires_grad_(True)
        q = _q64(vv, ss)
        qa = q.gather(-1, act.unsqueeze(-1)).squeeze(-1)
        tdr = yt.cpu().double().unsqueeze(1) - qa
        wr = w.double() if weighted else torch.ones(B, dtype=torch.float64)
        lref = ((tdr.pow(2).mean(1)) * wr).mean()
        lref.backward()
        total = lref.item()
        if B == 1:
            total += float(yb.cpu().double().var(unbiased=False))
        t = f"{tag}/w{int(weighted)}"
        record_parity(f"{t}/td", td.cpu().numpy(), tdr.detach().numpy(), rtol=1e-5, atol=1e-5)
        record_parity(f"{t}/td_sum", tds.cpu().numpy(), tdr.detach().sum(1).numpy(), rtol=1e-5, atol=1e-5)
        record_parity(f"{t}/loss", loss.cpu().numpy(), np.array([total]), rtol=1e-5, atol=1e-7)
        scale = float(ss.grad.abs().max())
        record_parity(f"{t}/ds", ds.cpu().numpy(), ss.grad.numpy(), rtol=1e-5, atol=1e-6 * scale)
        record_parity(f"{t}/dv", dv.cpu().numpy(), vv.grad.numpy(), rtol=1e-5, atol=1e-6 * float(vv.grad.abs().max()))
        again = torch.empty(1, device=DEV)
        call("ts_bdqn_rows", ptr(d["v_on"]), ptr(d["s_on"]), ptr(d["act"]), ptr(yt), ptr(d["w"]) if weighted else None, ptr(ybr), B,
             nb, A, ptr(td), ptr(rows), ptr(tds), ptr(ds), ptr(dv), ptr(again), stream())
        torch.cuda.synchronize()
        assert torch.equal(again, loss)


@gpu
def test_bdqn_target_branch_mean_follows_numpy():
    """The branch mean in numpy's float32 order (np.mean over a [B, nb] row, bdqn.py:157), bit for bit, at 1 .. 128 branches.
    With A = 2, v = 0, reward 0, gamma 1 and no end the target is that mean of Q_k(a*_k) = s_k[a*] - (s_k[0] + s_k[1]) / 2."""
    from tianshou_b200._cabi import call, ptr
    B, A = 64, 2
    for nb in (1, 2, 5, 7, 8, 9, 16, 17, 31, 128):
        g = torch.Generator().manual_seed(nb)
        s = (torch.randn(nb, B, A, generator=g) * torch.exp(torch.randn(nb, B, A, generator=g) * 3)).contiguous()
        dd = [t.to(DEV).contiguous() for t in (torch.zeros(B, 1), s, torch.zeros(B, dtype=torch.float64),
                                               torch.zeros(B, dtype=torch.uint8), torch.arange(B))]
        y = torch.empty(B, device=DEV)
        call("ts_bdqn_target", ptr(dd[0]), ptr(dd[1]), ptr(dd[0]), ptr(dd[1]), B, nb, A, 1.0, ptr(dd[2]), ptr(dd[3]), ptr(dd[4]),
             ptr(y), None, stream())
        torch.cuda.synchronize()
        sn = s.permute(1, 0, 2).numpy()                     # [B, nb, A] float32
        q = sn - ((sn[..., 0] + sn[..., 1]) / np.float32(2))[..., None]
        best = np.take_along_axis(q, q.argmax(-1)[..., None], -1)[..., 0]
        assert np.array_equal(y.cpu().numpy(), np.mean(best, -1)), nb


# ------------------------------------------------------------------------------------------------------------ branch chain
@gpu
@pytest.mark.parametrize("B,nb,act,heads", [(1, 3, "relu", "mlp"), (257, 4, "relu", "mlp"), (64, 9, "tanh", "linear")])
def test_branch_stack_vs_fp64_autograd(B, nb, act, heads):
    """The trunk, the value head and the branch ensemble's forward, every parameter gradient, and the trunk gradient that sums
    the value head's and the branches' input gradients."""
    O, A = 11, 6
    hid = (24,) if heads == "mlp" else ()
    torch.manual_seed(B + nb)
    net = _net(O, nb, A, (32, 20), hid, hid, torch.nn.ReLU if act == "relu" else torch.nn.Tanh).to(DEV)
    algo = _algo(net)
    ref = copy.deepcopy(net).cpu().double()
    x = torch.randn(B, O)
    dv, ds = torch.randn(B, 1), torch.randn(nb, B, A)
    acts_c, acts_v, acts_s = algo._q_parts(x.to(DEV), B, "t")
    h = acts_c[-1]
    dh = torch.full(tuple(h.shape), float("nan"), device=DEV)
    trunk_act = (algo._common.layers[-1].act, h)
    algo._branches.backward(acts_s, ds.to(DEV), B, "t", input_grad=True, input_act=trunk_act, dx_out=dh)
    algo._value.backward(acts_v, dv.to(DEV), B, "t", input_grad=True, input_act=trunk_act, dx_out=dh, dx_accumulate=True)
    algo._common.backward(acts_c, dh, B, "t", dy_preact=True)
    torch.cuda.synchronize()
    hr = ref.common.model(x.double())
    hr.retain_grad()
    vr = ref.value.model(hr)
    sr = torch.stack([b.model(hr) for b in ref.branches], 0)
    ((vr * dv.double()).sum() + (sr * ds.double()).sum()).backward()
    tag = f"bdqn_stack/B{B}_nb{nb}_{act}_{heads}"
    record_parity(f"{tag}/v", acts_v[-1].cpu().numpy(), vr.detach().numpy(), rtol=1e-5, atol=1e-5)
    record_parity(f"{tag}/s", acts_s[-1].cpu().numpy(), sr.detach().numpy(), rtol=1e-5, atol=1e-5)
    want_dh = hr.grad.numpy()
    got_dh = dh.cpu().numpy()
    if act == "relu":                               # dh is taken after the trunk's activation derivative
        want_dh = want_dh * (hr.detach().numpy() > 0)
    else:
        want_dh = want_dh * (1 - hr.detach().numpy() ** 2)
    record_parity(f"{tag}/dtrunk", got_dh, want_dh, rtol=1e-4, atol=1e-5 * float(np.abs(want_dh).max()))
    grp = algo._group
    got = torch.cat([grp.view(grp.grad, p) for p in net.parameters()]).cpu().numpy()
    want = torch.cat([p.grad.reshape(-1) for p in ref.parameters()]).numpy()
    record_parity(f"{tag}/grad", got, want, rtol=1e-4, atol=1e-5 * float(np.abs(want).max()))


# ------------------------------------------------------------------------------------------------------------ goldens
def _build(cfg, g=None, **over):
    net = _net(int(cfg["obs"]), int(cfg["nb"]), int(cfg["A"]), [int(x) for x in cfg["common"]], [int(x) for x in cfg["value"]],
               [int(x) for x in cfg["action"]], torch.nn.Tanh if str(cfg["act_fn"]) == "tanh" else torch.nn.ReLU).to(DEV)
    if g is not None:
        load_params(net, g, "p0_net_")
    kw = dict(lr=float(cfg["lr"]), gamma=float(cfg["gamma"]), target_update_freq=int(cfg["target_update_freq"]),
              is_double=bool(cfg["is_double"]))
    kw.update(over)
    return _algo(net, **kw)


def _buffer(g, mirror):
    from tianshou_b200.data import Batch, PrioritizedReplayBuffer, ReplayBuffer, VectorReplayBuffer
    cfg = golden_cfg(g)
    size, E = int(cfg["size"]), int(cfg["envs"])
    if bool(cfg["per"]):
        buf = PrioritizedReplayBuffer(size, alpha=float(cfg["per_alpha"]), beta=float(cfg["per_beta"]), device=DEV)
    elif E > 1:
        buf = VectorReplayBuffer(size, E, device=DEV)
    else:
        buf = ReplayBuffer(size, device=DEV)
    if mirror:
        buf.enable_device_mirror()
    for i in range(0, int(cfg["adds"]), E):
        if E > 1:
            buf.add(Batch(**{k: g["add_" + k][i:i + E] for k in KEYS}, info=[{}] * E), buffer_ids=np.arange(E))
        else:
            buf.add(Batch(**{k: g["add_" + k][i] for k in KEYS}, info={}))
    for k in (*KEYS, "done"):
        assert np.array_equal(np.asarray(buf._meta[k]), g["buf_" + k]), f"rebuilt buffer differs in {k}"
    assert np.array_equal(np.sort(buf.unfinished_index()), np.sort(g["buf_unfinished"]))
    if mirror:
        buf.sync_device_mirror()
        assert buf.device_columns() is not None
    return buf


@gpu
@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("variant", ["pendulum", "bipedal", "per_trunc", "b1"])
def test_update_matches_reference(variant, mirror):
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"bdqn_ref_{variant}.npz")
    cfg = golden_cfg(g)
    algo = _build(cfg, g)
    assert sorted(algo.state_dict().keys()) == list(g["state_dict_keys"]), "state_dict() keys differ from the reference's"
    buf = _buffer(g, mirror)
    captured = {}
    orig = algo._preprocess_batch

    def hook(batch, buffer, indices):
        captured["indices"] = np.asarray(indices).copy()
        if bool(cfg["per"]):
            captured["is_weight"] = batch.weight.detach().cpu().numpy().copy()
        assert tuple(batch.act.shape) == (len(indices), int(cfg["nb"])) and batch.act.dtype == torch.int64 and batch.act.is_cuda
        return orig(batch, buffer, indices)

    algo._preprocess_batch = hook
    lr = float(cfg["lr"])
    for u in range(int(cfg["updates"])):
        np.random.seed(500 + u)
        torch.manual_seed(100 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buf, int(cfg["bs"]))
        o, tag = f"u{u}_", f"bdqn/{variant}_m{int(mirror)}_u{u}"
        assert np.array_equal(captured["indices"], g[o + "indices"]), "sampled indices differ from the reference's"
        record_parity(f"{tag}/loss", np.float64(stats.loss), g[o + "loss"], rtol=2e-5, atol=2e-6)
        if bool(cfg["per"]):
            record_parity(f"{tag}/is_weight", captured["is_weight"], g[o + "is_weight"], rtol=1e-6, atol=1e-7)
            record_parity(f"{tag}/priorities", np.asarray(buf.weight[np.arange(len(buf))]), g[o + "priorities"], rtol=1e-3,
                          atol=1e-6)
        for i, p in enumerate(algo.policy.model.parameters()):
            record_parity(f"{tag}/net_{i}", p.detach().cpu().numpy(), g[f"{o}net_{i}"], rtol=1e-3, atol=0.1 * lr)
        if algo.model_old is not None:
            for i, p in enumerate(algo.model_old.parameters()):
                record_parity(f"{tag}/old_{i}", p.detach().cpu().numpy(), g[f"{o}old_{i}"], rtol=1e-3, atol=0.1 * lr)


# ------------------------------------------------------------------------------------------------------------ gradients
def _random_buffer(O, nb, A, n, seed):
    from tianshou_b200.data import ReplayBuffer
    rng = np.random.default_rng(seed)
    term = rng.random(n) < 0.05
    term[0] = True
    trunc = (rng.random(n) < 0.03) & ~term
    return ReplayBuffer.from_data(rng.standard_normal((n, O)).astype(np.float32), rng.integers(0, A, (n, nb)), rng.standard_normal(n),
                                  term, trunc, term | trunc, rng.standard_normal((n, O)).astype(np.float32))


@gpu
@pytest.mark.parametrize("is_double", [True, False])
def test_update_gradients_vs_fp64_autograd(is_double):
    """bipedal_bdq.py's width (BipedalWalker's 24 observations, 4 branches of 25 actions, common [512, 256], value [128], action
    [128], batch 512) with a lagged network: the gradient the update's Adam step applies, against float64 autograd of the eager
    restatement on copies of the modules, with the same batch."""
    from oracle.oracle_bdqn import TARGET_GAMMA, bdqn_loss, bdqn_targets
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.utils import policy_within_training_step
    O, nb, A, B = 24, 4, 25, 512
    torch.manual_seed(3)
    net = _net(O, nb, A, (512, 256), (128,), (128,)).to(DEV)
    algo = _algo(net, lr=1e-4, target_update_freq=100, is_double=is_double)
    buf = _random_buffer(O, nb, A, 2000, seed=11)
    with torch.no_grad():                          # a lagged network that differs from the online one
        for p in algo.model_old.parameters():
            p.mul_(0.9)
    algo._iter = 1                                 # no refresh inside the recorded update
    cap = {}
    grp = algo._group
    grp.adam_step = lambda opt, mgn: (cap.update(grad=torch.cat([grp.view(grp.grad, p) for p in net.parameters()]).cpu().double()),
                                      FlatGroup.adam_step(grp, opt, mgn))
    orig = algo._preprocess_batch
    algo._preprocess_batch = lambda b, buffer, idx: (cap.update(indices=np.asarray(idx).copy()), orig(b, buffer, idx))[1]
    ref, ref_old = copy.deepcopy(net).cpu().double(), copy.deepcopy(algo.model_old.module).cpu().double()
    np.random.seed(1)
    with policy_within_training_step(algo.policy):
        stats = algo.update(buf, B)
    torch.cuda.synchronize()
    idx = cap["indices"]
    end = np.asarray(buf.done).copy()
    end[buf.unfinished_index()] = True
    returns = bdqn_targets(ref, ref_old, torch.as_tensor(buf.obs_next[idx]).double(), buf.rew[idx], end[idx], gamma=TARGET_GAMMA,
                           is_double=is_double)
    loss, _ = bdqn_loss(ref, torch.as_tensor(buf.obs[idx]).double(), torch.as_tensor(buf.act[idx]), returns)
    grads = torch.autograd.grad(loss, list(ref.parameters()))
    want = torch.cat([x.reshape(-1) for x in grads]).numpy()
    tag = f"bdqn_grad/double{int(is_double)}"
    record_parity(f"{tag}/grad", cap["grad"].numpy(), want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)
    record_parity(f"{tag}/loss", np.array([stats.loss]), np.array([loss.item()]), rtol=2e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------------------------ determinism, sync, state
def _run(algo, buf, sizes, seed0):
    from tianshou_b200.utils import policy_within_training_step
    out = []
    for u, bs in enumerate(sizes):
        np.random.seed(seed0 + u)
        with policy_within_training_step(algo.policy):
            out.append(algo.update(buf, bs).loss)
    return out


@gpu
def test_identical_updates_are_bit_identical():
    g = load_golden("bdqn_ref_bipedal.npz")
    cfg = golden_cfg(g)
    res = []
    for _ in range(2):
        algo = _build(cfg, g)
        losses = _run(algo, _buffer(g, mirror=True), [int(cfg["bs"])] * 4, 500)
        res.append((losses, algo._group.flat.clone(), algo._g_old.flat.clone()))
    assert res[0][0] == res[1][0]
    assert torch.equal(res[0][1], res[1][1]) and torch.equal(res[0][2], res[1][2])


@gpu
def test_smaller_batch_after_larger_is_bit_identical_to_a_fresh_run():
    """The scratch a larger batch sized (and left behind, here overwritten with NaN) does not leak into a smaller batch."""
    O, nb, A = 24, 4, 25
    torch.manual_seed(4)
    a = _algo(_net(O, nb, A, (64, 32), (16,), (16,)).to(DEV), target_update_freq=3)
    buf = _random_buffer(O, nb, A, 3000, seed=2)
    _run(a, buf, [2500], 7)
    b = _algo(_net(O, nb, A, (64, 32), (16,), (16,)).to(DEV), target_update_freq=3)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    b._iter = a._iter
    for store in (a._scratch, *(s._bufs for s in (a._common, a._value, a._branches))):
        for t in store.values():
            if isinstance(t, torch.Tensor) and t.is_floating_point():
                t.fill_(float("nan"))
    # each buffer draws from its own RandomState: two fresh copies give both instances the same indices
    la = _run(a, _random_buffer(O, nb, A, 3000, seed=2), [17, 3], 40)
    lb = _run(b, _random_buffer(O, nb, A, 3000, seed=2), [17, 3], 40)
    assert la == lb and np.isfinite(la).all()
    assert torch.equal(a._group.flat, b._group.flat) and torch.equal(a._g_old.flat, b._g_old.flat)


@gpu
@pytest.mark.parametrize("per", [False, True])
def test_device_update_has_no_host_sync_but_the_loss(per):
    """The update's launches run under torch.cuda.set_sync_debug_mode("error"); the loss is the one read (a prioritised
    buffer's td sums are read after it, by the priority update, as in the reference)."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("bdqn_ref_per_trunc.npz" if per else "bdqn_ref_bipedal.npz")
    cfg = golden_cfg(g)
    algo = _build(cfg, g)
    buf = _buffer(g, mirror=True)
    bs = int(cfg["bs"])
    seen = []
    orig_item = torch.Tensor.item
    with policy_within_training_step(algo.policy):
        for _ in range(2):
            batch, indices = algo._sample(buf, bs)
            batch = algo._preprocess_batch(batch, buf, indices)
            torch.cuda.synchronize()

            def item(t, *a, **k):
                torch.cuda.set_sync_debug_mode("default")
                seen.append(tuple(t.shape))
                return orig_item(t, *a, **k)

            torch.Tensor.item = item
            torch.cuda.set_sync_debug_mode("error")
            try:
                stats = algo._update_with_batch(batch)
            finally:
                torch.cuda.set_sync_debug_mode("default")
                torch.Tensor.item = orig_item
            assert np.isfinite(stats.loss)
            assert batch.weight.shape == (bs,) and batch.weight.is_cuda
            algo._postprocess_batch(batch, buf, indices)
    assert seen == [(1,), (1,)], seen


@gpu
def test_state_dict_round_trip_continues_identically():
    g = load_golden("bdqn_ref_bipedal.npz")
    cfg = golden_cfg(g)
    a = _build(cfg, g)
    _run(a, _buffer(g, mirror=False), [int(cfg["bs"])] * 3, 1)
    b = _build(cfg, g)
    with torch.no_grad():
        for p in b.parameters():
            p.add_(0.01)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    b._iter = a._iter
    la = _run(a, _buffer(g, mirror=False), [int(cfg["bs"])] * 3, 10)
    lb = _run(b, _buffer(g, mirror=False), [int(cfg["bs"])] * 3, 10)
    assert la == lb
    for ga, gb in ((a._group, b._group), (a._g_old, b._g_old)):
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals():
    from torch import nn

    from tianshou_b200.algorithm import UnsupportedModelError
    from tianshou_b200.data import Batch, PrioritizedReplayBuffer, ReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import MLP
    O, nb, A = 4, 3, 5
    make = lambda **kw: _net(O, nb, A, (8,), (8,), (8,), **kw)
    _algo(make().to(DEV))
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        _algo(make())
    with pytest.raises(UnsupportedModelError, match="outside"):
        _algo(make(norm_layer=nn.LayerNorm).to(DEV))
    with pytest.raises(UnsupportedModelError, match="ReLU / Tanh"):
        _algo(make(act=nn.GELU).to(DEV))
    odd = make()
    odd.branches[1] = MLP(input_dim=8, output_dim=A, hidden_sizes=[6])
    with pytest.raises(UnsupportedModelError, match="branch 1 differs"):
        _algo(odd.to(DEV))
    with pytest.raises(UnsupportedModelError, match="at least one branch"):
        _algo(_net(O, 0, A, (8,), (8,), (8,)).to(DEV))
    algo = _algo(make().to(DEV))
    rng = np.random.default_rng(0)

    def fill(buf, act):
        for i in range(6):
            buf.add(Batch(obs=rng.standard_normal(O).astype(np.float32), act=act, rew=1.0, terminated=False, truncated=False,
                          obs_next=rng.standard_normal(O).astype(np.float32), info={}))
        return buf

    before = algo._group.flat.clone()
    with policy_within_training_step(algo.policy):
        with pytest.raises(ValueError, match="B = 1"):
            algo.update(fill(PrioritizedReplayBuffer(10, alpha=0.6, beta=0.4, device=DEV), np.array([0, 1, 2])), 1)
        with pytest.raises(ValueError, match="rows of 3 actions"):
            algo.update(fill(ReplayBuffer(10, device=DEV), np.array([0, 1])), 4)
        with pytest.raises(ValueError, match="outputs"):
            algo.update(fill(ReplayBuffer(10, device=DEV), np.array([0, A, 1])), 4)
        with pytest.raises(ValueError, match="outputs"):
            algo.update(fill(ReplayBuffer(10, device=DEV), np.array([0, -1, 1])), 4)
        torch.cuda.synchronize()
        assert torch.equal(before, algo._group.flat)
        algo.update(fill(PrioritizedReplayBuffer(10, alpha=0.6, beta=0.4, device=DEV), np.array([0, 1, 2])), 2)     # B = 2 runs
    one = _algo(_net(O, 1, A, (8,), (8,), (8,)).to(DEV))
    with policy_within_training_step(one.policy):          # one branch at B = 1: the reference's priority update takes it
        assert np.isfinite(one.update(fill(PrioritizedReplayBuffer(10, alpha=0.6, beta=0.4, device=DEV), np.array([2])), 1).loss)


@gpu
def test_reference_construction_builds():
    """test/discrete/test_bdqn.py:84-106 against this package's imports (Pendulum's 3 observations, one branch of 40)."""
    from tianshou_b200.algorithm import BDQN
    from tianshou_b200.algorithm.modelfree.bdqn import BDQNPolicy
    from tianshou_b200.algorithm.optim import AdamOptimizerFactory
    from tianshou_b200.utils.net.common import BranchingNet
    net = BranchingNet(state_shape=(3,), num_branches=1, action_per_branch=40, common_hidden_sizes=[64, 64],
                       value_hidden_sizes=[64], action_hidden_sizes=[64]).to(DEV)
    policy = BDQNPolicy(model=net, action_space=MultiDiscrete([40]), eps_training=0.76, eps_inference=0.01)
    algorithm = BDQN(policy=policy, optim=AdamOptimizerFactory(lr=1e-3), gamma=0.9, target_update_freq=200)
    from tianshou_b200.data import Batch
    out = policy(Batch(obs=np.zeros((5, 3), np.float32), info={}))
    assert out.act.shape == (5, 1) and algorithm.use_target_network


# ------------------------------------------------------------------------------------------------------------ resources
def test_bdqn_kernels_have_no_stack_frame_or_spills(tmp_path):
    report = ptxas_report("bdqn.cu", tmp_path)
    names = sorted(re.search(r"bdqn_(target|rows|dscore|sum)_kernel", e).group(1) for e in report)
    assert names == ["dscore", "rows", "sum", "target"], report
    assert_spill_free(report)
