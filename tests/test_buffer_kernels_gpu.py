"""Edge sweep of the kernels the rollout and replay path stands on, each against the numpy / C oracle or a plain fp64
reference: the GAE scan and the running-statistics merge (`gae.cu`), the replay-buffer index and row-movement kernels
(`index.cu`), n-step returns (`nstep.cu`), the sum tree (`segtree.cu`) and the advantage-moment kernels of `mlp.cu`.

Bars:
- bit-exact for index work, row movement, n-step returns (f64; f32 = the f64 result rounded once) and the sum tree;
- GAE, which re-associates the f64 recurrence: element-wise |err| <= c * 2^-53 * S_i, where S_i is the same discounted
  sum taken over |delta| (the recurrence's condition number times |adv_i|) and c = 2 * (tiles + 48) counts the roundings
  on the longest composition chain (in-thread, warp, CTA and the look-back over every tile to the right); f32 outputs
  add one rounding;
- bit-identical between the 128-bit and the scalar GAE path, between calls that reuse one workspace, and between the
  minibatch and epoch advantage sums;
- the prioritized-replay kernels against numpy's expressions in the TD errors' dtype: the running min / max and the
  tree's parents bit-exact, every power within the documented error of CUDA's powf / pow plus the host's.
"""
import math
import warnings

import numpy as np
import pytest
import torch

from oracle import oracle_c as ocl
from oracle import oracle_np as onp
from ts_testutil import record_parity

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
EPS64 = 2.0 ** -53
TILE = 2048            # transitions per CTA of the GAE scan
TDT = {"f32": torch.float32, "f64": torch.float64}
NDT = {"f32": np.float32, "f64": np.float64}


def _cabi():
    from tianshou_b200 import _cabi as c
    return c


def ops():
    from tianshou_b200 import ops as o
    return o


def call(name, *args):
    _cabi().call(name, *args)


def ptr(t):
    return _cabi().ptr(t)


def stream():
    return _cabi().stream_ptr(torch.device(DEV))


def on_dev(a, shift=0, dtype=None):
    """Device copy of ``a`` that starts ``shift`` elements into its own allocation (torch allocations are 512-byte
    aligned, so shift 1 misaligns every vector load of the kernels)."""
    a = np.ascontiguousarray(a)
    if a.dtype == np.bool_:
        a = a.view(np.uint8)
    t = torch.from_numpy(a).reshape(-1)
    if dtype is not None:
        t = t.to(dtype)
    buf = torch.zeros(t.numel() + shift, dtype=t.dtype, device=DEV)
    view = buf[shift:]
    view.copy_(t)
    return view


def bits(t):
    return t.view(torch.int64 if t.element_size() == 8 else torch.int32)


def assert_within(key, got, ref, tol):
    got = np.asarray(got, dtype=np.float64)
    err = np.abs(got - ref)
    bad = ~(err <= tol)
    assert not bad.any(), (f"{key}: {int(bad.sum())} of {err.size} elements beyond the bound, first at "
                           f"{int(np.flatnonzero(bad)[0])}: err {err[bad][0]:.3e} > {tol[bad][0]:.3e}")
    record_parity(key, got, ref, rtol=0.0, atol=float(tol.max()) if tol.size else 0.0)


# ---------------------------------------------------------------------------------------------------------- GAE
def gae_inputs(n, seed, vdt="f64", p=0.02):
    rng = np.random.default_rng(seed)
    v_s = rng.standard_normal(n).astype(NDT[vdt])
    v_n = rng.standard_normal(n).astype(NDT[vdt])
    rew = rng.standard_normal(n)
    term, trunc, extra = (rng.random(n) < p for _ in range(3))
    return dict(v_s=v_s, v_n=v_n, rew=rew, term=term, trunc=trunc, extra=extra)


def gae_reference(x, gamma, lam, terminated_ends=True, scale=1.0):
    """(adv, un-scaled returns, bound on |adv err|) in fp64 with the C restatement of the reference's loop."""
    n = len(x["rew"])
    zeros = np.zeros(n, dtype=bool)
    term = zeros if x["term"] is None else x["term"]
    end = zeros.copy()
    for f in (x["trunc"], x["extra"], term if terminated_ends else None):
        if f is not None:
            end |= f
    vs = x["v_s"].astype(np.float64) * scale
    vn = x["v_n"].astype(np.float64) * scale * ~term
    adv = ocl.gae(vs, vn, x["rew"], end, gamma, lam)
    delta = x["rew"] + vn * gamma - vs
    cond = ocl.gae(np.zeros(n), np.zeros(n), np.abs(delta), end, gamma * lam, 1.0)
    tiles = (n + TILE - 1) // TILE
    return adv, adv + vs, 2 * (tiles + 48) * EPS64 * cond


def out_bound(ref, tol, odt):
    """The bound after the output rounding (one f32 rounding, with the f32 subnormal step as floor)."""
    if odt == "f32":
        return tol * (1 + 2.0 ** -24) + 2.0 ** -24 * np.abs(ref) + 2.0 ** -149
    return tol


GAE_PTRS = ("v_s", "v_n", "rew", "term", "trunc", "extra", "adv", "ret")


def run_gae(x, vdt, odt, gamma, lam, terminated_ends=True, shift=None, rms_state=None, batch_moments_out=None,
            workspace=None):
    """ts_gae with the argument named ``shift`` placed one element into its allocation."""
    def dev(name, dtype):
        a = x[name]
        return None if a is None else on_dev(a, 1 if shift == name else 0, dtype)
    n = len(x["rew"])
    outs = []
    for name in ("adv", "ret"):
        s = 1 if shift == name else 0
        outs.append(torch.full((n + s,), float("nan"), dtype=TDT[odt], device=DEV)[s:])
    return ops().gae(dev("v_s", TDT[vdt]), dev("v_n", TDT[vdt]), dev("rew", torch.float64), dev("term", torch.uint8),
                     dev("trunc", torch.uint8), dev("extra", torch.uint8), gamma=gamma, gae_lambda=lam,
                     rms_state=rms_state, out_dtype=TDT[odt], terminated_ends=terminated_ends, device=DEV,
                     workspace=workspace, out=tuple(outs), batch_moments_out=batch_moments_out)


def check_gae(key, x, adv, ret, odt, gamma, lam, terminated_ends=True, scale=1.0):
    ref_adv, ref_ret, tol = gae_reference(x, gamma, lam, terminated_ends, scale)
    assert_within(f"gae adv {key}", adv.cpu().numpy(), ref_adv, out_bound(ref_adv, tol, odt))
    ret_ref = ref_ret / scale
    ret_tol = tol / scale + 4 * EPS64 * np.abs(ret_ref)     # + adv + v_s and / scale, rounded on both sides
    assert_within(f"gae returns {key}", ret.cpu().numpy(), ret_ref, out_bound(ret_ref, ret_tol, odt))


GAE_SIZES = [1, 8, 9, 2047, 2048, 2049, 5 * TILE - 1, 5 * TILE + 1, 2 ** 21]
GAE_DTYPES = [("f32", "f32"), ("f32", "f64"), ("f64", "f32"), ("f64", "f64")]


@pytest.mark.parametrize("vdt,odt", GAE_DTYPES)
@pytest.mark.parametrize("n", GAE_SIZES)
def test_gae_dtypes_sizes_and_scalar_path(n, vdt, odt):
    """All four (value, output) instantiations vs fp64 under both ``terminated_ends``; then each of the eight pointers
    misaligned on its own, which sends every tile down the scalar path: bit-identical to the aligned call."""
    x = gae_inputs(n, n, vdt)
    for te in (True, False):
        adv, ret = run_gae(x, vdt, odt, 0.99, 0.95, te)
        check_gae(f"{vdt}->{odt}", x, adv, ret, odt, 0.99, 0.95, te)
    for name in GAE_PTRS:
        adv_s, ret_s = run_gae(x, vdt, odt, 0.99, 0.95, False, shift=name)
        assert torch.equal(bits(adv_s), bits(adv)), name
        assert torch.equal(bits(ret_s), bits(ret)), name


def end_pattern(name, n, rng):
    i = np.arange(n)
    if name.startswith("item"):            # one in-thread position j of the 8 items, in half of the threads
        j = int(name[4:])
        return (i % 8 == j) & (rng.random(n // 8 + 1) < 0.5)[i // 8]
    if name == "tile_edges":               # first / last transition of every warp (256) and every tile (2048)
        return (i % 256 == 0) | (i % 256 == 255)
    if name == "every_row":
        return np.ones(n, dtype=bool)
    assert name == "row0"
    return i == 0


@pytest.mark.parametrize("pattern", [f"item{j}" for j in range(8)] + ["tile_edges", "every_row", "row0"])
def test_gae_end_flag_placement(pattern):
    n = 3 * TILE + 77
    rng = np.random.default_rng(len(pattern))
    x = gae_inputs(n, 7, "f32", p=0.005)
    x["trunc"] = end_pattern(pattern, n, rng)
    for te in (True, False):
        adv, ret = run_gae(x, "f32", "f64", 0.99, 0.95, te)
        check_gae(f"end flags {pattern}", x, adv, ret, "f64", 0.99, 0.95, te)


@pytest.mark.parametrize("gamma,lam", [(0.0, 0.95), (0.99, 0.0), (1.0, 1.0), (0.5, 1.0)],
                         ids=["gamma0", "lambda0", "gl1", "gl_half"])
def test_gae_gamma_lambda_edges_without_cuts(gamma, lam):
    """2^21 rows and no end flag.  gamma lambda = 1: every advantage is a suffix sum over up to 2^21 terms, the
    bound scales with it (the condition number).  gamma lambda = 0.5: 0.5^2048 underflows to 0, so every tile's
    aggregate is exactly 0 and publishes its start value without a look-back."""
    n = 2 ** 21
    x = gae_inputs(n, 11, "f64")
    x["term"] = x["trunc"] = x["extra"] = None
    adv, ret = run_gae(x, "f64", "f64", gamma, lam)
    check_gae(f"gamma {gamma} lambda {lam} no cut", x, adv, ret, "f64", gamma, lam)


def test_gae_return_scaling_over_1024_tiles_three_calls():
    """Return scaling with the running statistics carried over three calls; returns sit 1e3 away from zero, so the
    moments must be shifted before they are squared.  rms_state vs RunningMeanStd with numpy's fp64 moments."""
    n = 1024 * TILE
    rng = np.random.default_rng(5)
    x = dict(v_s=(1e3 + rng.standard_normal(n)).astype(np.float32), v_n=(1e3 + rng.standard_normal(n)).astype(np.float32),
             rew=rng.standard_normal(n), term=rng.random(n) < 0.01, trunc=rng.random(n) < 0.01, extra=None)
    rms = onp.RunningMeanStd()
    state = torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64, device=DEV)
    for k in range(3):
        scale = float(np.sqrt(state[1].item() + 1e-8))     # the scale the kernel derives from its own state
        adv, ret = run_gae(x, "f32", "f64", 0.99, 0.95, rms_state=state)
        check_gae(f"scaled call {k}", x, adv, ret, "f64", 0.99, 0.95, scale=scale)
        rms.update(gae_reference(x, 0.99, 0.95, scale=scale)[1])
        got = state.cpu().numpy()
        assert got[2] == rms.count == (k + 1) * n
        record_parity("gae rms_state mean, var (1024 tiles, returns ~1e3)", got[:2], [rms.mean, rms.var], rtol=1e-11, atol=0)


def test_gae_batch_moments_and_workspace_reuse():
    """``batch_moments_out`` gets (count, mean, M2) of the un-scaled returns and ``rms_state`` only provides the scale;
    a second call through the same workspace is bit-identical."""
    n = 37 * TILE + 5
    x = gae_inputs(n, 3, "f32")
    x["v_s"] = x["v_s"] + np.float32(1e3)
    state = torch.tensor([3.0, 4.0, 100.0], dtype=torch.float64, device=DEV)
    before = state.clone()
    ws = torch.empty(int(_cabi().load_library().ts_gae_workspace_bytes(n)), dtype=torch.uint8, device=DEV)
    runs = []
    for _ in range(2):
        mom = torch.full((3,), float("nan"), dtype=torch.float64, device=DEV)
        adv, ret = run_gae(x, "f32", "f32", 0.99, 0.95, rms_state=state, batch_moments_out=mom, workspace=ws)
        runs.append((adv, ret, mom))
    assert torch.equal(bits(state), bits(before))
    scale = math.sqrt(4.0 + 1e-8)
    check_gae("batch moments call", x, runs[0][0], runs[0][1], "f32", 0.99, 0.95, scale=scale)
    r = gae_reference(x, 0.99, 0.95, scale=scale)[1]
    mean = math.fsum(r) / n
    m2 = math.fsum((r - mean) ** 2)
    got = runs[0][2].cpu().numpy()
    assert got[0] == n
    record_parity("gae batch_moments_out mean", got[1], mean, rtol=1e-12, atol=0)
    record_parity("gae batch_moments_out M2", got[2], m2, rtol=1e-9, atol=0)
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(bits(a), bits(b))


@pytest.mark.parametrize("parts", range(1, 9))
def test_rms_merge_parts(parts):
    """``ts_rms_merge`` of 1 .. 8 (count, mean, M2) parts, zero-count parts among them, vs RunningMeanStd.update on the
    concatenated returns."""
    rng = np.random.default_rng(parts)
    sizes = list(rng.integers(1, 5000, parts))
    if parts >= 2:
        sizes[1] = 0
    if parts >= 4:
        sizes[-1] = 0
    chunks = [7.0 + 3.0 * rng.standard_normal(k) for k in sizes]
    mom = np.array([[k, c.mean(), ((c - c.mean()) ** 2).sum()] if k else [0.0, 0.0, 0.0] for k, c in zip(sizes, chunks)],
                   dtype=np.float64)
    state = torch.tensor([0.5, 2.0, 1000.0], dtype=torch.float64, device=DEV)
    call("ts_rms_merge", ptr(state), ptr(on_dev(mom)), parts, stream())
    rms = onp.RunningMeanStd()
    rms.mean, rms.var, rms.count = 0.5, 2.0, 1000
    rms.update(np.concatenate(chunks))
    got = state.cpu().numpy()
    assert got[2] == rms.count
    record_parity("ts_rms_merge mean, var", got[:2], [rms.mean, rms.var], rtol=1e-12, atol=0)


def test_rms_merge_all_parts_empty_leaves_state():
    state = torch.tensor([0.5, 2.0, 1000.0], dtype=torch.float64, device=DEV)
    before = state.clone()
    call("ts_rms_merge", ptr(state), ptr(on_dev(np.zeros((3, 3)))), 3, stream())
    assert torch.equal(bits(state), bits(before))


# -------------------------------------------------------------------------------------------------- index kernels
def make_buffer(E, seed):
    """E sub-buffers of unequal capacity, each empty, with one row, two rows, full or partly filled; the state an
    ``add()``-filled buffer has (insertion index = last_index + 1), plus an independent insertion index as
    ``from_data`` / ``dropnull`` leave it."""
    rng = np.random.default_rng(seed)
    caps = rng.integers(1, 9, E)
    caps[:5] = [8, 5, 1, 3, 2][:E]
    offset = np.concatenate([[0], np.cumsum(caps)]).astype(np.int64)
    start = offset[:-1]
    kind = rng.integers(0, 5, E)
    kind[:5] = [4, 3, 0, 1, 2][:E]
    partial = np.where(caps > 1, rng.integers(1, np.maximum(caps, 2)), 1)
    lengths = np.choose(kind, [np.zeros(E, np.int64), np.ones(E, np.int64), np.full(E, 2), caps, partial])
    lengths = np.minimum(lengths, caps).astype(np.int64)
    full = lengths == caps
    last = np.where(full, start + rng.integers(0, 1 << 30, E) % caps, start + np.maximum(lengths - 1, 0))
    ins = np.where(lengths > 0, rng.integers(0, 1 << 30, E) % (lengths + 1), 0).astype(np.int64)
    done = rng.random(offset[-1]) < 0.25
    return offset, done, last.astype(np.int64), lengths, ins


def sample_all(meta, capacity):
    """ts_sample_all_indices into a sentinel-filled output of ``capacity`` + 16 slots: (out, seg_start, total)."""
    out = torch.full((capacity + 16,), -7, dtype=torch.int64, device=DEV)
    seg = torch.full((meta.E + 1,), -7, dtype=torch.int64, device=DEV)
    tot = torch.full((1,), -7, dtype=torch.int64, device=DEV)
    call("ts_sample_all_indices", ptr(meta.offset), meta.E, ptr(meta.last_index), ptr(meta.lengths), ptr(meta.ins),
         ptr(seg), ptr(out), capacity, ptr(tot), stream())
    return out.cpu().numpy(), seg.cpu().numpy(), int(tot.item())


@pytest.mark.parametrize("ins_given", [False, True], ids=["derived_ins", "given_ins"])
@pytest.mark.parametrize("E", [1, 2, 1023, 1024, 1025, 5000])
def test_index_kernels_unequal_subbuffers(E, ins_given):
    offset, done, last, lengths, ins = make_buffer(E, E)
    ins = ins if ins_given else None
    meta = ops().DeviceBufferMeta.from_host(offset, done, last, lengths, DEV, ins=ins)
    total = int(offset[-1])
    rng = np.random.default_rng(E + 1)
    q = np.concatenate([offset[:-1], offset[1:] - 1, offset[:-1] - 1, last, np.flatnonzero(done),
                        [-1, -2, -total, -total - 1, -3 * total + 5, total, total + 1, 2 * total + 7],
                        rng.integers(-2 * total, 3 * total, 1000)]).astype(np.int64)
    assert np.array_equal(ops().next_index(meta, q).cpu().numpy(), onp.next_index(q, offset, done, last, lengths))
    assert np.array_equal(ops().prev_index(meta, q).cpu().numpy(), onp.prev_index(q, offset, done, last, lengths))
    ref_unf = onp.unfinished_index(offset, done, last, lengths, ins)
    assert np.array_equal(ops().unfinished_index(meta).cpu().numpy(), ref_unf)
    ref_all = onp.sample_all_indices(offset, last, lengths, ins)
    assert len(ref_all) == lengths.sum()
    for cap in sorted({len(ref_all), len(ref_all) // 2 + 1, 1, 0}):
        out, seg, tot = sample_all(meta, cap)
        assert tot == len(ref_all)
        assert np.array_equal(seg, np.concatenate([[0], np.cumsum(lengths)]))
        k = min(cap, len(ref_all))
        assert np.array_equal(out[:k], ref_all[:k]), cap
        assert np.all(out[k:] == -7), cap
    if not ins_given:   # next / prev / stacks do not read the insertion index
        sq = rng.choice(q, min(len(q), 3000), replace=False)
        for n_step in (1, 17):
            got = ops().stack_next_indices(meta, sq, n_step).cpu().numpy()
            rows = [sq]
            for _ in range(n_step - 1):
                rows.append(onp.next_index(rows[-1], offset, done, last, lengths))
            assert np.array_equal(got, np.stack(rows)), n_step


@pytest.mark.parametrize("B", [1, 15, 16, 17, 1000, 4096 + 9])
@pytest.mark.parametrize("done_shift,out_shift", [(0, 0), (1, 0), (0, 1)])
def test_buffer_end_flags_tail_and_misaligned(B, done_shift, out_shift):
    """The byte tail (B % 16 != 0) and a ``done`` / output one byte into its allocation; bytes past B stay as they were."""
    rng = np.random.default_rng(B)
    caps = np.array([B]) if B < 3 else np.array([B // 3, B // 3, B - 2 * (B // 3)])
    offset = np.concatenate([[0], np.cumsum(caps)]).astype(np.int64)
    lengths = np.minimum(caps, rng.integers(0, B + 1, len(caps))).astype(np.int64)
    last = (offset[:-1] + np.maximum(lengths - 1, 0)).astype(np.int64)
    done = rng.random(B) < 0.3
    meta = ops().DeviceBufferMeta.from_host(offset, done, last, lengths, DEV)
    dbuf = torch.zeros(B + 32, dtype=torch.uint8, device=DEV)
    dbuf[done_shift:done_shift + B] = meta.done
    obuf = torch.full((B + 32,), 0xAB, dtype=torch.uint8, device=DEV)
    call("ts_buffer_end_flags", ptr(dbuf[done_shift:done_shift + B]), ptr(meta.offset), ptr(meta.last_index),
         ptr(meta.lengths), meta.E, ptr(obuf[out_shift:out_shift + B]), stream())
    got = obuf.cpu().numpy()
    assert np.array_equal(got[out_shift:out_shift + B].astype(bool), onp.buffer_end_flags(done, last, lengths))
    assert np.all(got[:out_shift] == 0xAB) and np.all(got[out_shift + B:] == 0xAB)


@pytest.mark.parametrize("count", [None, 0, 5, 37], ids=["all", "count0", "count5", "count37"])
def test_mark_members_edges(count):
    """Members that are -1 or >= table_size are skipped, duplicates are harmless, a device count below the capacity
    limits the list, and the table is all zero again on return (it is reused across calls)."""
    rng = np.random.default_rng(0 if count is None else count + 1)
    table_size = 1000
    members = np.concatenate([[-1, 3, table_size, 3, table_size - 1, 0, 5000, -7, 3, 512],
                              rng.integers(0, table_size, 30)]).astype(np.int64)
    idx = np.concatenate([rng.integers(0, table_size, 3000), members[(members >= 0) & (members < table_size)]])
    table = torch.zeros(table_size, dtype=torch.uint8, device=DEV)
    cnt = None if count is None else torch.tensor([count], dtype=torch.int64, device=DEV)
    valid = members if count is None else members[:count]
    for _ in range(2):
        mark = ops().mark_members(on_dev(idx), on_dev(members), table_size, table=table, count=cnt)
        assert np.array_equal(mark.cpu().numpy().astype(bool), np.isin(idx, valid))
        assert int(table.sum().item()) == 0


def test_value_mask_rows_special_values():
    """``tq *= mask`` on terminated rows: -0, +-inf and NaN keep numpy's float32 product (sign of zero included).
    NaN payloads are not compared: the GPU returns its canonical NaN for inf * 0 and NaN * 0."""
    rng = np.random.default_rng(2)
    B, I, A = 500, 300, 7
    term = rng.random(B) < 0.5
    idx = rng.integers(0, B, I)
    tq = rng.standard_normal((I, A)).astype(np.float32)
    special = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, -1e-45, 3e38], dtype=np.float32)
    for r in range(0, I, 3):
        tq[r] = np.roll(special, r)
    d_tq = on_dev(tq)
    ops().value_mask_rows(d_tq, on_dev(term), on_dev(idx))
    got = d_tq.cpu().numpy().reshape(I, A)
    with np.errstate(invalid="ignore"):
        ref = tq * (~term[idx]).astype(np.float32)[:, None]
    assert ref.dtype == np.float32
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    assert np.array_equal(got[ok].view(np.uint32), ref[ok].view(np.uint32))


# ------------------------------------------------------------------------------------------------------- n-step
@pytest.mark.parametrize("gamma", [0.0, 1.0, 0.99])
@pytest.mark.parametrize("n_step", [1, 2, 7, 8, 9, 16, 17])
def test_nstep_end_flag_at_every_window_position(n_step, gamma):
    """Sample i has one end flag at window row i % (n + 2) (none when that is n, random flags when it is n + 1), so
    every row of the window cuts some samples; n > 8 runs the gather-then-fold chunk loop more than once."""
    rng = np.random.default_rng(n_step)
    I = 300
    B = I * n_step + 11
    idx = rng.permutation(B)[: I * n_step].reshape(n_step, I).astype(np.int64)
    end = np.zeros(B, dtype=bool)
    pos = np.arange(I) % (n_step + 2)
    for i in range(I):
        if pos[i] < n_step:
            end[idx[pos[i], i]] = True
        elif pos[i] == n_step + 1:
            end[idx[:, i]] = rng.random(n_step) < 0.3
    rew = rng.standard_normal(B)
    d_rew, d_end, d_idx = on_dev(rew), on_dev(end), on_dev(idx).reshape(n_step, I)
    for A in (1, 6, 18):
        tq = rng.standard_normal((I, A)).astype(np.float32)
        ref = onp.nstep_return(rew, end, tq, idx, gamma, n_step)
        d_tq = on_dev(tq).reshape(I, A)
        out64 = ops().nstep_return(d_rew, d_end, d_tq, d_idx, gamma, n_step, torch.float64).cpu().numpy()
        assert np.array_equal(out64, ref), A
        out32 = ops().nstep_return(d_rew, d_end, d_tq, d_idx, gamma, n_step, torch.float32).cpu().numpy()
        assert np.array_equal(out32, ref.astype(np.float32)), A


# ----------------------------------------------------------------------------------------------------- sum tree
TREE_SIZES = [1, 2, 3, 5, 1000, 2 ** 20, 2 ** 20 + 1]


def make_tree(size):
    from tianshou_b200.data import SegmentTree
    tree = SegmentTree(size, device=DEV)
    return tree, np.zeros(2 * tree.bound)


@pytest.mark.parametrize("vdt", ["f32", "f64"])
@pytest.mark.parametrize("size", TREE_SIZES)
def test_segtree_setitem_batches_with_duplicates(size, vdt):
    """Batches of 1 .. 32768 items drawn from a small pool: duplicates everywhere, last write wins, including items
    31744 .. 32767 (bit 31 of each thread's win mask).  The whole tree is bit-identical to the oracle after every batch."""
    rng = np.random.default_rng(size)
    tree, ref = make_tree(size)
    pool = rng.choice(size, min(size, 3000), replace=False)
    for b in (1, 1023, 1024, 1025, 32768):
        idx = pool[rng.integers(0, len(pool), b)].astype(np.int64)
        val = rng.random(b).astype(NDT[vdt])
        val[rng.random(b) < 0.1] = 0
        ops().segtree_setitem(tree.tree, tree.bound, on_dev(idx), on_dev(val))
        onp.segtree_setitem(ref, tree.bound, idx, val)
        assert np.array_equal(tree.tree.cpu().numpy(), ref), b


def test_segtree_setitem_device_duplicates_across_chunks():
    rng = np.random.default_rng(1)
    tree, ref = make_tree(5000)
    idx = rng.integers(0, 700, 3 * 32768 + 1234).astype(np.int64)
    val = rng.random(len(idx))
    tree.setitem_device(on_dev(idx), on_dev(val))
    onp.segtree_setitem(ref, tree.bound, idx, val)
    assert np.array_equal(tree.tree.cpu().numpy(), ref)


def fill_tree(size, weights):
    tree, ref = make_tree(size)
    idx = np.arange(size, dtype=np.int64)
    tree.setitem_device(on_dev(idx), on_dev(weights))
    onp.segtree_setitem(ref, tree.bound, idx, weights)
    assert np.array_equal(tree.tree.cpu().numpy(), ref)
    return tree, ref


@pytest.mark.parametrize("size", [1, 2, 3, 5, 1000, 2 ** 20 + 1])
def test_segtree_reduce_ranges(size):
    rng = np.random.default_rng(size)
    w = rng.random(size)
    w[rng.random(size) < 0.2] = 0
    tree, ref = fill_tree(size, w)
    if size <= 5:
        ranges = [(s, e) for s in range(size + 1) for e in range(s, size + 1)]
    else:
        lo = rng.integers(0, size, 100)
        ranges = [(int(s), int(rng.integers(s, size + 1))) for s in lo] + [(0, size), (7, 7), (size - 1, size)]
    for s, e in ranges:
        got = ops().segtree_reduce(tree.tree, tree.bound, s, e).item()
        assert got == onp.segtree_reduce(ref, tree.bound, s, e), (s, e)


@pytest.mark.parametrize("size", [1, 2, 3, 5, 1000, 2 ** 20 + 1])
def test_segtree_prefix_queries_ties_and_edges(size):
    """Dyadic weights keep every cumulative sum exact, so a query equal to one ties at some node of the descent (the
    reference sends ties left); runs of zero-weight leaves, 0 and nextafter(total, 0).  ``sample_device(u)`` must
    equal the prefix query of ``u * total``."""
    rng = np.random.default_rng(size)
    w = rng.integers(0, 8, size) * 0.25
    for s in rng.integers(0, size, max(1, size // 50)):
        w[s:s + int(rng.integers(1, 40))] = 0.0
    w[-1] = 1.0
    tree, ref = fill_tree(size, w)
    total = ref[1]
    cs = np.cumsum(w)
    assert cs[-1] == total
    q = np.concatenate([[0.0], cs[:-1], [np.nextafter(total, 0.0)], rng.random(1000) * total])
    got = ops().segtree_prefix_sum_idx(tree.tree, tree.bound, on_dev(q)).cpu().numpy()
    assert np.array_equal(got, onp.segtree_prefix_sum_idx(ref, tree.bound, q))
    u = np.concatenate([[0.0, np.nextafter(1.0, 0.0)], rng.random(4096)])
    got = tree.sample_device(on_dev(u)).cpu().numpy()
    assert np.array_equal(got, onp.segtree_prefix_sum_idx(ref, tree.bound, u * total))


# ------------------------------------------------------------------------------------------ prioritized replay
# The CUDA C++ Programming Guide (appendix "Mathematical Functions") documents a maximum error of 4 ulp for powf and of
# 2 ulp for pow over their full range; numpy's float32 / float64 power calls the host libm, which is within 1 ulp.  So a
# device power lies within 5 (float32) or 3 (float64) ulp of numpy's, and one ulp of x is at most eps(type) * |x|.
POW_ULP = {"f32": 4 + 1, "f64": 2 + 1}
EPS = {"f32": 2.0 ** -23, "f64": 2.0 ** -52}
PRIO_EPS = np.finfo(np.float32).eps.item()          # prio.py: self._eps, a Python float


def prio_update(tree, minmax, idx, td, alpha, eps=PRIO_EPS):
    c = _cabi()
    dt = c.TS_F32 if td.dtype == np.float32 else c.TS_F64
    d_idx, d_td = on_dev(idx), on_dev(td)       # held: a freed temporary's block would be handed to the next one
    call("ts_prio_update_weight", ptr(tree.tree), tree.bound, ptr(d_idx), ptr(d_td), dt, len(idx), alpha, eps,
         ptr(minmax), stream())


def prio_update_reference(td, alpha, eps=PRIO_EPS):
    """The reference's own expressions (prio.py update_weight): numpy keeps a float32 array combined with a Python float in
    float32, so w and w ** alpha are float32 for float32 TD errors."""
    w = np.abs(td) + eps
    leaf = w ** alpha
    assert w.dtype == leaf.dtype == td.dtype
    return w, leaf


@pytest.mark.parametrize("tdt", ["f32", "f64"])
@pytest.mark.parametrize("n", [1, 1000, 1025, 32768])
def test_prio_update_weight_matches_numpy_expressions(n, tdt):
    """``ts_prio_update_weight`` against numpy's ``|td| + eps`` and ``w ** alpha`` in the TD errors' own dtype, twice on one
    tree.  Each batch draws its indices from a small pool (duplicates everywhere) and starts with two items that lose to a
    later duplicate of their index: one carries the batch's largest w, the other the smallest (td = 0).  ``prio_minmax`` is
    bit-exact (the losers count, as ``weight.max()`` / ``min()`` see every item); each leaf holds the last duplicate's value
    within POW_ULP; float32 leaves are float32 numbers; untouched leaves keep their bits; every parent is exactly
    ``left + right`` of the device's own children."""
    rng = np.random.default_rng(n + (0 if tdt == "f32" else 7))
    size = 5000
    tree, _ = make_tree(size)
    bound = tree.bound
    init = rng.random(size)
    ops().segtree_setitem(tree.tree, bound, on_dev(np.arange(size, dtype=np.int64)), on_dev(init))
    minmax = torch.tensor([1.0, 1.0], dtype=torch.float64, device=DEV)
    ref_max, ref_min = 1.0, 1.0
    alpha = 0.6
    pool = rng.choice(size, max(1, min(size, n // 3)), replace=False)
    for call_no in range(2):
        idx = pool[rng.integers(0, len(pool), n)].astype(np.int64)
        td = (rng.standard_normal(n) * (3.0 if call_no else 0.2)).astype(NDT[tdt])
        td[rng.random(n) < 0.05] = 0
        if n >= 3:
            idx[0] = idx[1] = idx[-1]
            td[0] = NDT[tdt](50.0 + call_no)
            td[1] = 0
        before = tree.tree.cpu().numpy()
        prio_update(tree, minmax, idx, td, alpha)
        got = tree.tree.cpu().numpy()
        w, leaf = prio_update_reference(td, alpha)
        ref_max, ref_min = max(ref_max, w.max()), min(ref_min, w.min())           # prio.py: max(self._max_prio, weight.max())
        mm = minmax.cpu().numpy()
        assert mm[0] == float(ref_max) and mm[1] == float(ref_min), (call_no, mm, ref_max, ref_min)
        last = {}
        for k, i in enumerate(idx):
            last[int(i)] = k                      # last write wins
        slots = np.array(sorted(last), dtype=np.int64)
        winners = np.array([last[int(i)] for i in slots])
        g_leaf = got[bound + slots]
        r_leaf = leaf[winners].astype(np.float64)
        tol = POW_ULP[tdt] * EPS[tdt] * np.abs(r_leaf)
        assert_within(f"ts_prio_update_weight {tdt} leaves vs numpy w ** alpha", g_leaf, r_leaf, tol)
        if tdt == "f32":
            assert np.array_equal(g_leaf, g_leaf.astype(np.float32).astype(np.float64)), "f32 leaves must be float32 numbers"
        if n >= 3:                                # the losers' values are 50 ** 0.6 and eps ** 0.6, far from the winner's
            assert abs(got[bound + idx[-1]] - leaf[-1]) <= POW_ULP[tdt] * EPS[tdt] * abs(float(leaf[-1]))
        untouched = np.ones(bound, dtype=bool)
        untouched[slots] = False
        assert np.array_equal(got[bound:][untouched], before[bound:][untouched])
        parents = np.arange(1, bound)
        assert np.array_equal(got[parents], got[2 * parents] + got[2 * parents + 1])


def test_prio_update_weight_batch_limit():
    """One CTA resolves duplicates with a 32-bit win mask per thread: 32 x 1024 items per call, more are refused."""
    tree, _ = make_tree(100)
    minmax = torch.tensor([1.0, 1.0], dtype=torch.float64, device=DEV)
    idx = np.zeros(32 * 1024 + 1, dtype=np.int64)
    with pytest.raises(RuntimeError, match="at most 32768 items"):
        prio_update(tree, minmax, idx, np.ones(len(idx), dtype=np.float32), 0.6)


@pytest.mark.parametrize("weight_norm", [0, 1], ids=["raw", "weight_norm"])
@pytest.mark.parametrize("n", [1, 1000, 1025, 5000])
def test_prio_get_weight_matches_numpy_expressions(n, weight_norm):
    """``ts_prio_get_weight`` against ``(weight[index] / min_prio) ** (-beta)`` and ``weight / weight.max()`` in float64.  The
    quotient is one correctly rounded division on both sides, so the power's error is all there is: POW_ULP of the result;
    dividing by the batch maximum (itself a power) doubles that and adds one rounding on each side.  With weight_norm the batch's largest entry is exactly 1.
    n > 1024 makes the kernel's single block loop."""
    rng = np.random.default_rng(n + 10 * weight_norm)
    size = 3000
    tree, _ = make_tree(size)
    leaves = rng.uniform(1e-4, 3.0, size) ** 0.6
    ops().segtree_setitem(tree.tree, tree.bound, on_dev(np.arange(size, dtype=np.int64)), on_dev(leaves))
    min_prio = float(np.float32(1.2e-4))
    minmax = torch.tensor([3.0, min_prio], dtype=torch.float64, device=DEV)
    for beta in (0.4, 1.0, 0.0):
        idx = rng.integers(0, size, n).astype(np.int64)
        out = torch.full((n,), float("nan"), dtype=torch.float64, device=DEV)
        d_idx = on_dev(idx)
        call("ts_prio_get_weight", ptr(tree.tree), tree.bound, ptr(d_idx), n, ptr(minmax), beta, weight_norm, ptr(out),
             stream())
        got = out.cpu().numpy()
        ref = (leaves[idx] / min_prio) ** (-beta)
        if weight_norm:
            ref = ref / np.max(ref)
            assert got.max() == 1.0
        tol = (2 * POW_ULP["f64"] + 1 if weight_norm else POW_ULP["f64"]) * EPS["f64"] * np.abs(ref)
        assert_within(f"ts_prio_get_weight beta {beta} weight_norm {weight_norm}", got, ref, tol)
        if beta == 0.0:
            assert np.all(got == 1.0)


# ------------------------------------------------------------------------------------------------- row movement
ROW_BYTES = [1, 2, 3, 4, 6, 8, 12, 16, 48, 68]
# (src, dst) byte offsets into their allocations: 16-aligned, 4- but not 16-aligned, 1- and 2-byte misaligned
OFFSETS = [(0, 0), (4, 8), (8, 4), (1, 0), (0, 2), (3, 1)]


def byte_rows(rng, n, rb, off):
    """(whole allocation, [n, rb] uint8 view starting ``off`` bytes into it), random contents."""
    buf = torch.from_numpy(rng.integers(0, 256, n * rb + off + 16, dtype=np.uint8)).to(DEV)
    return buf, buf[off:off + n * rb].view(n, rb)


def check_gather_scatter(rng, rb, off, n_src, n):
    so, do = off
    _, src = byte_rows(rng, n_src, rb, so)
    src_np = src.cpu().numpy()
    idx = rng.integers(0, n_src, n)
    dbuf, dst = byte_rows(rng, n, rb, do)
    before = dbuf.cpu().numpy()
    ops().gather_rows(src, on_dev(idx), out=dst)
    ref = before.copy()
    ref[do:do + n * rb] = src_np[idx].reshape(-1)
    assert np.array_equal(dbuf.cpu().numpy(), ref), ("gather", rb, off)
    # scatter: distinct slots, every other row of the destination untouched
    sbuf, dst2 = byte_rows(rng, n_src, rb, do)
    _, rows = byte_rows(rng, n, rb, so)
    slots = rng.permutation(n_src)[:n]
    before = sbuf.cpu().numpy()
    call("ts_scatter_rows", ptr(rows), rb, ptr(on_dev(slots)), n, ptr(dst2), stream())
    ref = before.copy()
    view = ref[do:do + n_src * rb].reshape(n_src, rb)
    view[slots] = rows.cpu().numpy()
    assert np.array_equal(sbuf.cpu().numpy(), ref), ("scatter", rb, off)


@pytest.mark.parametrize("off", OFFSETS, ids=[f"src{s}_dst{d}" for s, d in OFFSETS])
@pytest.mark.parametrize("rb", ROW_BYTES)
def test_gather_scatter_rows_alignment(rb, off):
    check_gather_scatter(np.random.default_rng(rb), rb, off, 1000, 777)


@pytest.mark.parametrize("rb,off", [(16, (0, 0)), (4, (4, 8)), (1, (0, 0)), (3, (1, 2))],
                         ids=["16B", "4B", "single_byte", "bytewise"])
def test_gather_scatter_rows_past_the_grid(rb, off):
    """n x row words beyond the num_sms x 32 x 256 threads of the capped grid, so the grid-stride loop runs."""
    cap = torch.cuda.get_device_properties(0).multi_processor_count * 32 * 256
    word = 16 if rb == 16 else (4 if rb == 4 and off[0] % 4 == 0 and off[1] % 4 == 0 else 1)
    n = (cap + 4099) * word // rb
    check_gather_scatter(np.random.default_rng(rb), rb, off, n + 5, n)


def test_narrow_i64_i32_near_int32_limits():
    rng = np.random.default_rng(0)
    edge = np.array([-2 ** 31, -2 ** 31 + 1, -1, 0, 1, 2 ** 31 - 2, 2 ** 31 - 1], dtype=np.int64)
    v = np.concatenate([edge, rng.integers(-2 ** 31, 2 ** 31, 1000), 2 ** 31 - 1 - rng.integers(0, 300, 300)])
    got = ops().narrow_i64_i32(on_dev(v)).cpu().numpy()
    assert got.dtype == np.int32 and np.array_equal(got, v.astype(np.int32))


# --------------------------------------------------------------------------------------------- advantage moments
def adv_moments_fp64(x):
    n = len(x)
    mean = math.fsum(x) / n
    std = math.sqrt(math.fsum((x - mean) ** 2) / (n - 1)) if n > 1 else 0.0
    return mean, std


@pytest.mark.parametrize("with_perm", [False, True], ids=["no_perm", "perm"])
@pytest.mark.parametrize("S", [2, 255, 256, 257, 16384])
def test_adv_moments_minibatch_and_epoch_paths(S, with_perm):
    """Three minibatches from lo0 = 5, the last one ragged (S + S // 2 + 1 rows), advantages with mean / std = 1e3, over
    world = 1 .. 4 rank shards whose sums are added as the all-reduce would.  Both entry points vs fp64 mean and
    unbiased std; the minibatch sums equal the epoch sums bit for bit, and a repeated call is bit-identical."""
    rng = np.random.default_rng(S)
    lo0, n_mb = 5, 3
    end = lo0 + 2 * S + S + S // 2 + 1
    N = end + 3
    bounds = [(lo0 + m * S, lo0 + (m + 1) * S if m < n_mb - 1 else end) for m in range(n_mb)]
    shards = []
    for _ in range(4):
        adv = (1e3 + rng.standard_normal(N)).astype(np.float32)
        perm = rng.permutation(N).astype(np.int32) if with_perm else None
        shards.append((adv, perm, on_dev(adv), None if perm is None else on_dev(perm)))
    epoch_sums = []
    for _, _, d_adv, d_perm in shards:
        sums = torch.full((2 * n_mb,), float("nan"), dtype=torch.float64, device=DEV)
        call("ts_epoch_adv_sums", ptr(d_adv), ptr(d_perm), lo0, S, end, n_mb, ptr(sums), stream())
        epoch_sums.append(sums)
    for world in range(1, 5):
        total = epoch_sums[0].clone()
        for s in epoch_sums[1:world]:
            total += s
        mom = torch.empty(2 * n_mb, dtype=torch.float32, device=DEV)
        call("ts_epoch_adv_finalize", ptr(total), lo0, S, end, n_mb, world, ptr(mom), stream())
        mom = mom.cpu().numpy()
        for m, (lo, hi) in enumerate(bounds):
            rows = np.concatenate([(a[p[lo:hi]] if p is not None else a[lo:hi]).astype(np.float64)
                                   for a, p, _, _ in shards[:world]])
            ref = adv_moments_fp64(rows)
            record_parity("epoch adv moments (mean, std) vs fp64", mom[2 * m:2 * m + 2], ref, rtol=2.0 ** -23, atol=0)
            # the minibatch entry point on the same rows
            part = []
            for r, (_, _, d_adv, d_perm) in enumerate(shards[:world]):
                sums = torch.full((2,), float("nan"), dtype=torch.float64, device=DEV)
                call("ts_minibatch_adv_sums", ptr(d_adv), ptr(d_perm), lo, hi, ptr(sums), stream())
                again = torch.full((2,), float("nan"), dtype=torch.float64, device=DEV)
                call("ts_minibatch_adv_sums", ptr(d_adv), ptr(d_perm), lo, hi, ptr(again), stream())
                assert torch.equal(bits(sums), bits(again))
                assert torch.equal(bits(sums), bits(epoch_sums[r][2 * m:2 * m + 2]))
                part.append(sums)
            tot = part[0].clone()
            for s in part[1:]:
                tot += s
            mb = torch.empty(2, dtype=torch.float32, device=DEV)
            call("ts_adv_moments_finalize", ptr(tot), (hi - lo) * world, ptr(mb), stream())
            mb = mb.cpu().numpy()
            record_parity("minibatch adv moments (mean, std) vs fp64", mb, ref, rtol=2.0 ** -23, atol=0)
            assert np.array_equal(mb.view(np.uint32), mom[2 * m:2 * m + 2].view(np.uint32))


def test_adv_moments_single_row_std_is_zero_where_torch_gives_nan():
    """A one-row minibatch: the kernels return std 0, the reference's ``minibatch.adv.std()`` is NaN (DESIGN.md 4)."""
    adv = on_dev(np.array([0.0, 3.5, 1.0], dtype=np.float32))
    sums = torch.full((2,), float("nan"), dtype=torch.float64, device=DEV)
    call("ts_minibatch_adv_sums", ptr(adv), None, 1, 2, ptr(sums), stream())
    mb = torch.empty(2, dtype=torch.float32, device=DEV)
    call("ts_adv_moments_finalize", ptr(sums), 1, ptr(mb), stream())
    ep_sums = torch.full((2,), float("nan"), dtype=torch.float64, device=DEV)
    call("ts_epoch_adv_sums", ptr(adv), None, 1, 1, 2, 1, ptr(ep_sums), stream())
    ep = torch.empty(2, dtype=torch.float32, device=DEV)
    call("ts_epoch_adv_finalize", ptr(ep_sums), 1, 1, 2, 1, 1, ptr(ep), stream())
    assert mb.cpu().tolist() == [3.5, 0.0] and ep.cpu().tolist() == [3.5, 0.0]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")          # torch warns about the zero degrees of freedom
        assert torch.isnan(torch.tensor([3.5]).std())
