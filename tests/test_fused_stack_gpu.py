"""``FusedStack`` (algorithm/netgraph.py) in every mode its callers use, on its own and against float64 references of the same
modules: the forward with the live and with another parameter buffer, the parameter and input gradients of ``backward``
(``input_cols``, ``input_act``, ``dx_out``, ``dx_accumulate``, ``dy_preact``, ``param_grads=False``), the tangent pass
``jvp``, repeatability and the separation of the scratch buffers by tag and row count.  Then ``compile_sequential``'s
accepted and refused chains (no GPU needed).

The GEMM underneath is swept on its own in ``test_net_gpu.py``; what is under test here is the glue: the weight, bias and
mask pointers, the leading dimensions, which activation masks which gradient, and the accumulate flags.  The chains sit on
the GEMM's tile edges (widths 1, 3, 5, 17, 23, 64, 127, 129, 256, 257, 393; depths 1 .. 4; ReLU, Tanh and no activation
mixed; a width-1 hidden layer; the Humanoid critic 393 -> 256 -> 256 -> 1; a conv -> flatten -> Linear chain), at 1, 37,
129, 4099 and 8209 rows (8209: every forward GEMM of the sweep runs unsplit, asserted).  The fp64 references take the
stack's own ReLU decisions, as ``test_conv_kernels_gpu.py`` explains."""
import copy

import numpy as np
import pytest
import torch
from torch import nn
from torch.func import functional_call, jvp

from test_conv_kernels_gpu import U, _bounded, _check_layers, _exact, _flat_modules
from ts_testutil import record_parity

DEV = "cuda:0"
gpu = pytest.mark.gpu
ACT_NONE, ACT_RELU, ACT_TANH = 0, 1, 2        # TS_ACT_* of include/ts_b200.h


def _conv_chain():
    # 3 x 9 x 11 -> (k 3, s 2) 4 x 4 x 5 -> flatten 80 -> 17 Tanh -> 3; the Linear after the flatten masks its input
    # gradient with the convolution's ReLU, looking through the flatten
    return nn.Sequential(nn.Conv2d(3, 4, 3, 2), nn.ReLU(), nn.Flatten(), nn.Linear(80, 17), nn.Tanh(), nn.Linear(17, 3)), (3, 9, 11)


CHAINS = {
    "lin17-5": lambda: (nn.Sequential(nn.Linear(17, 5)), (17,)),
    "relu23-64-3": lambda: (nn.Sequential(nn.Linear(23, 64), nn.ReLU(), nn.Linear(64, 3)), (23,)),
    "tanh5-17-1-23": lambda: (nn.Sequential(nn.Linear(5, 17), nn.Tanh(), nn.Linear(17, 1), nn.Tanh(), nn.Linear(1, 23)), (5,)),
    "in1-256-129-1": lambda: (nn.Sequential(nn.Linear(1, 256), nn.Tanh(), nn.Linear(256, 129), nn.ReLU(), nn.Linear(129, 1)), (1,)),
    "mix129-127-257-256-5": lambda: (nn.Sequential(nn.Linear(129, 127), nn.ReLU(), nn.Linear(127, 257), nn.Linear(257, 256), nn.Tanh(),
                                                   nn.Linear(256, 5)), (129,)),
    "humanoid393-256-256-1": lambda: (nn.Sequential(nn.Linear(393, 256), nn.ReLU(), nn.Linear(256, 256), nn.ReLU(),
                                                    nn.Linear(256, 1)), (393,)),
    "conv3x9x11": _conv_chain,
}
MLP_CHAINS = [n for n in CHAINS if not n.startswith("conv")]
WIDE_CHAINS = ["relu23-64-3", "mix129-127-257-256-5", "humanoid393-256-256-1"]     # in_dim >= 23: room for input_cols
ROWS = [1, 37, 129, 4099, 8209]
BIG = ROWS[-1]


class _Case:
    def __init__(self, name: str, seed: int) -> None:
        from tianshou_b200.algorithm.flat_params import FlatGroup
        from tianshou_b200.algorithm.netgraph import FusedStack, compile_sequential
        torch.manual_seed(seed)
        net, self.shape = CHAINS[name]()
        self.net = net.to(DEV)
        self.net64 = copy.deepcopy(self.net).to("cpu", torch.float64)
        self.layers = compile_sequential(list(self.net), self.shape)
        self.params = [p for L in self.layers if L.weight is not None for p in (L.weight, L.bias)]
        self.group = FlatGroup(self.params, torch.device(DEV))
        self.stack = FusedStack(self.layers, self.group)
        self.out_dim = self.layers[-1].out_dim

    def input(self, rng, rows):
        """(device input rows, the same values in fp64 in torch's layout): NHWC rows for a convolution, NCHW for torch."""
        if len(self.shape) == 1:
            x = rng.standard_normal((rows, self.shape[0])).astype(np.float32)
            return torch.from_numpy(x).to(DEV), torch.from_numpy(x).double()
        C, H, W = self.shape
        x = rng.standard_normal((rows, H, W, C)).astype(np.float32)
        return torch.from_numpy(x).to(DEV), torch.from_numpy(x).double().permute(0, 3, 1, 2).contiguous()

    def ref(self, acts, rows):
        return _Layers64(self, acts, rows)


class _Keep(nn.Module):
    """ReLU with the decisions of the stack's own forward."""

    def __init__(self, keep: torch.Tensor) -> None:
        super().__init__()
        self.keep = keep

    def forward(self, x):
        return x * self.keep


class _Layers64(nn.Module):
    """The fp64 copy of the case's modules, one block per compiled layer, returning every layer's output; ReLU takes the
    decisions of the stack's forward ``acts``.  Its parameters come in the flat group's order."""

    def __init__(self, case: _Case, acts, rows: int) -> None:
        super().__init__()
        mods = [m for m in _flat_modules(list(case.net64)) if isinstance(m, (nn.Conv2d, nn.Linear, nn.Flatten))]
        blocks = []
        for i, (L, m) in enumerate(zip(case.layers, mods, strict=True)):
            parts = [m]
            if L.act == ACT_RELU:
                keep = (acts[i + 1] > 0).cpu().double()
                parts.append(_Keep(keep.view(rows, L.Ho, L.Wo, L.out_dim).permute(0, 3, 1, 2) if L.kind == "conv"
                                   else keep.view(rows, L.out_dim)))
            elif L.act == ACT_TANH:
                parts.append(nn.Tanh())
            blocks.append(nn.Sequential(*parts))
        self.blocks = nn.ModuleList(blocks)

    def forward(self, x):
        outs = []
        for b in self.blocks:
            x = b(x)
            outs.append(x)
        return tuple(outs)


def _h(t):
    return t.detach().cpu().numpy()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _grad_bar(key, got, ref):
    """The conv stack test's gradient bar: 1e-4 relative + 2e-5 x max |ref|."""
    ref = np.asarray(ref)
    return record_parity(key, got, ref, rtol=1e-4, atol=2e-5 * float(np.abs(ref).max()))


def _seed(name, rows):
    return list(CHAINS).index(name) * 10007 + rows


# ------------------------------------------------------------------------------------- forward + parameter gradients
@gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("name", list(CHAINS))
def test_forward_and_gradients_vs_fp64(name, rows):
    """Each layer's output on its own fp32 input within gamma(K) (|W| |a| + |b|) (+ 4 ulp of tanhf); every weight and bias
    gradient of sum(coef * y_L), and d loss / d input over all columns, against fp64 autograd.  ``param_grads=False`` leaves
    the gradient buffer bit-unchanged.  A convolution in front refuses the input gradient."""
    from tianshou_b200.algorithm.flat_params import UnsupportedModelError
    case = _Case(name, _seed(name, rows))
    rng = np.random.default_rng(_seed(name, rows))
    x, x64 = case.input(rng, rows)
    coef = rng.standard_normal((rows, case.out_dim)).astype(np.float32)
    acts = case.stack.forward(x, rows, "t")
    case.stack.backward(acts, _dev(coef), rows, "t")
    torch.cuda.synchronize()
    grad = case.group.grad.clone()
    tag = f"fused_stack/fwd_bwd/{name}/r{rows}"
    with torch.no_grad():
        _check_layers(tag, case.layers, list(case.net64), acts, x64, rows)
    ref = case.ref(acts, rows)
    xg = x64.clone().requires_grad_(True)
    (ref(xg)[-1] * torch.from_numpy(coef).double()).sum().backward()
    for i, (p, rp) in enumerate(zip(case.params, ref.parameters(), strict=True)):
        _grad_bar(f"{tag}/grad{i}", _h(case.group.view(grad, p)).reshape(p.shape), rp.grad.numpy())
    case.group.grad.fill_(-7.25)
    if case.layers[0].kind == "conv":
        with pytest.raises(UnsupportedModelError):
            case.stack.backward(acts, _dev(coef), rows, "t", param_grads=False, input_grad=True)
        return
    dx = case.stack.backward(acts, _dev(coef), rows, "t", param_grads=False, input_grad=True)
    torch.cuda.synchronize()
    assert torch.equal(case.group.grad, torch.full_like(case.group.grad, -7.25)), "param_grads=False must not touch the gradients"
    _grad_bar(f"{tag}/dx", _h(dx), xg.grad.numpy())


# -------------------------------------------------------------------------------------------------- input gradients
def _producer_output(rng, rows, width, kind):
    """Rows of the stack's input as the activation ``kind`` left them: ReLU outputs with +0.0 and -0.0 among the positives
    (only > 0 passes the mask), tanh outputs spread over (-1, 1); unconstrained rows without a producing activation."""
    z = rng.standard_normal((rows, width))
    if kind == "relu":
        y = np.maximum(z, 0.0)
        y[(z < 0) & (rng.random(z.shape) < 0.5)] = -0.0
        return y.astype(np.float32)
    if kind == "tanh":
        return np.tanh(1.5 * z).astype(np.float32)
    return z.astype(np.float32)


@gpu
@pytest.mark.parametrize("input_act", ["none", "relu", "tanh"])
@pytest.mark.parametrize("rows", [1, 37, 4099])
@pytest.mark.parametrize("name", WIDE_CHAINS)
def test_input_gradient_modes_vs_fp64(name, rows, input_act):
    """d loss / d input against fp64 autograd, times the derivative of the activation that produced the input when
    ``input_act`` names one, for all columns and for ``input_cols`` (17, 18) and (17, 23) (a start that is not a multiple
    of 4, widths 1 and 6): returned from the stack's scratch, written into a NaN-filled ``dx_out`` (bit-identical to the
    former), and added onto a non-zero ``dx_out`` with ``dx_accumulate`` (the stored result plus the prior in one fp32
    rounding).  The parameter gradients stay untouched throughout (``param_grads=False``)."""
    case = _Case(name, _seed(name, rows) + 1)
    rng = np.random.default_rng(_seed(name, rows) + 2)
    K = case.layers[0].in_dim
    xn = _producer_output(rng, rows, K, input_act)
    x, x64 = _dev(xn), torch.from_numpy(xn).double()
    coef = rng.standard_normal((rows, case.out_dim)).astype(np.float32)
    acts = case.stack.forward(x, rows, "t")
    ref = case.ref(acts, rows)
    xg = x64.clone().requires_grad_(True)
    (ref(xg)[-1] * torch.from_numpy(coef).double()).sum().backward()
    deriv = {"none": torch.ones_like(x64), "relu": (x64 > 0).double(), "tanh": 1.0 - x64 * x64}[input_act]
    want = (xg.grad * deriv).numpy()
    ia = None if input_act == "none" else ({"relu": ACT_RELU, "tanh": ACT_TANH}[input_act], x)
    case.group.grad.fill_(3.5)
    for cols in (None, (17, 18), (17, 23)):
        lo, hi = cols if cols is not None else (0, K)
        tag = f"fused_stack/dx/{name}/r{rows}/{input_act}/cols{lo}-{hi}"
        kw = dict(param_grads=False, input_grad=True, input_cols=cols, input_act=ia)
        stored = case.stack.backward(acts, _dev(coef), rows, "t", **kw).clone()
        _grad_bar(tag, _h(stored), want[:, lo:hi])
        out = torch.full((rows, hi - lo), float("nan"), device=DEV)
        ret = case.stack.backward(acts, _dev(coef), rows, "t", dx_out=out, **kw)
        assert ret is out
        _exact(tag + "/dx_out", _h(out), _h(stored))
        prior = rng.standard_normal((rows, hi - lo)).astype(np.float32)
        out = _dev(prior)
        case.stack.backward(acts, _dev(coef), rows, "t", dx_out=out, dx_accumulate=True, **kw)
        s = _h(stored)
        if input_act == "tanh":
            # x * (1 - y^2) + prior may be contracted into one FMA: one rounding of the exact product plus the prior
            _bounded(tag + "/accumulate", _h(out), s.astype(np.float64) + prior, 4 * U * (np.abs(s) + np.abs(prior)))
        else:
            _exact(tag + "/accumulate", _h(out), s + prior)
    torch.cuda.synchronize()
    assert torch.equal(case.group.grad, torch.full_like(case.group.grad, 3.5)), "param_grads=False must not touch the gradients"


# ---------------------------------------------------------------------------------------------------------- dy_preact
@gpu
@pytest.mark.parametrize("rows", [1, 37, 4099])
def test_dy_preact_gradients_vs_fp64(rows):
    """A trunk ending in Tanh under a head: ``dy`` is the gradient w.r.t. the last pre-activation, and every parameter
    gradient of sum(coef * z_L) matches fp64 autograd.  Without ``dy_preact`` the stack refuses."""
    from tianshou_b200.algorithm.flat_params import FlatGroup, UnsupportedModelError
    from tianshou_b200.algorithm.netgraph import FusedStack, compile_sequential
    torch.manual_seed(rows)
    net = nn.Sequential(nn.Linear(23, 17), nn.ReLU(), nn.Linear(17, 5), nn.Tanh()).to(DEV)
    net64 = copy.deepcopy(net).to("cpu", torch.float64)
    layers = compile_sequential(list(net), (23,))
    params = [p for L in layers for p in (L.weight, L.bias)]
    group = FlatGroup(params, torch.device(DEV))
    stack = FusedStack(layers, group)
    rng = np.random.default_rng(rows + 5)
    xn = rng.standard_normal((rows, 23)).astype(np.float32)
    coef = rng.standard_normal((rows, 5)).astype(np.float32)
    acts = stack.forward(_dev(xn), rows, "t")
    with pytest.raises(UnsupportedModelError):
        stack.backward(acts, _dev(coef), rows, "t")
    stack.backward(acts, _dev(coef), rows, "t", dy_preact=True)
    torch.cuda.synchronize()
    keep = (acts[1] > 0).cpu().double()
    l0, l1 = net64[0], net64[2]
    z = l1(l0(torch.from_numpy(xn).double()) * keep)
    (z * torch.from_numpy(coef).double()).sum().backward()
    for i, (p, rp) in enumerate(zip(params, [l0.weight, l0.bias, l1.weight, l1.bias], strict=True)):
        _grad_bar(f"fused_stack/dy_preact/r{rows}/grad{i}", _h(group.view(group.grad, p)).reshape(p.shape), rp.grad.numpy())


# --------------------------------------------------------------------------------------------------------------- jvp
@gpu
@pytest.mark.parametrize("rows", [1, 37, 4099, BIG])
@pytest.mark.parametrize("name", MLP_CHAINS)
def test_jvp_vs_torch_func_jvp(name, rows):
    """Every layer's tangent along a flat parameter direction (the group's layout), with the input as data (``x_dot``
    None) and with an input tangent, against ``torch.func.jvp`` of the fp64 modules through ``functional_call``; the FVP
    test's bar, 2e-4 relative + 1e-4 x max per layer."""
    case = _Case(name, _seed(name, rows) + 3)
    rng = np.random.default_rng(_seed(name, rows) + 4)
    x, x64 = case.input(rng, rows)
    acts = case.stack.forward(x, rows, "t")
    v = rng.standard_normal(case.group.n).astype(np.float32)
    vt = torch.from_numpy(v)
    ref = case.ref(acts, rows)
    names = [n for n, _ in ref.named_parameters()]
    primals = tuple(p.detach() for _, p in ref.named_parameters())
    tangents = tuple(case.group.view(vt, p).view(p.shape).double() for p in case.params)

    def f(xx, *ps):
        return functional_call(ref, dict(zip(names, ps, strict=True)), (xx,))

    for with_xdot in (False, True):
        xd = rng.standard_normal(x64.shape).astype(np.float32) if with_xdot else None
        _, want = jvp(f, (x64, *primals), (torch.from_numpy(xd).double() if with_xdot else torch.zeros_like(x64), *tangents))
        got = case.stack.jvp(acts, _dev(v), rows, "t", x_dot=_dev(xd) if with_xdot else None)
        assert len(got) == len(want)
        for i, (g, w) in enumerate(zip(got, want)):
            w = w.numpy()
            record_parity(f"fused_stack/jvp/{name}/r{rows}/{'xdot' if with_xdot else 'data'}/layer{i}", _h(g), w, rtol=2e-4,
                          atol=1e-4 * float(np.abs(w).max()))


@gpu
def test_refusals_of_the_conv_chain():
    """Tangent passes exist for Linear layers only, and the input gradient stops at a first convolution: both raise
    ``UnsupportedModelError``."""
    from tianshou_b200.algorithm.flat_params import UnsupportedModelError
    case = _Case("conv3x9x11", 0)
    rng = np.random.default_rng(0)
    x, _ = case.input(rng, 5)
    acts = case.stack.forward(x, 5, "t")
    with pytest.raises(UnsupportedModelError, match="Linear layers only"):
        case.stack.jvp(acts, torch.zeros(case.group.n, device=DEV), 5, "t")
    with pytest.raises(UnsupportedModelError, match="first convolution"):
        case.stack.backward(acts, torch.zeros(5, 3, device=DEV), 5, "t", input_grad=True)


# ---------------------------------------------------------------------------------------------------- forward(params=)
@gpu
@pytest.mark.parametrize("rows", [37, 4099])
@pytest.mark.parametrize("name", list(CHAINS))
def test_forward_with_other_params_reads_only_them(name, rows):
    """``forward(params=other)`` is bit-identical to the forward of a stack built on a group holding ``other``, and reads
    nothing of the live buffer: it is NaN for the call."""
    case = _Case(name, _seed(name, rows) + 6)
    twin = _Case(name, _seed(name, rows) + 7)
    rng = np.random.default_rng(_seed(name, rows) + 8)
    other = (case.group.flat + 0.25 * torch.from_numpy(rng.standard_normal(case.group.n).astype(np.float32)).to(DEV)).contiguous()
    twin.group.flat.copy_(other)
    x, _ = case.input(rng, rows)
    want = [a.clone() for a in twin.stack.forward(x, rows, "t")[1:]]
    live = case.group.flat.clone()
    case.group.flat.fill_(float("nan"))
    try:
        got = case.stack.forward(x, rows, "t", params=other)[1:]
        torch.cuda.synchronize()
        got = [g.clone() for g in got]
    finally:
        case.group.flat.copy_(live)
    for i, (g, w) in enumerate(zip(got, want, strict=True)):
        _exact(f"fused_stack/params/{name}/r{rows}/layer{i}", _h(g), _h(w))


# -------------------------------------------------------------------------------------- determinism and scratch reuse
def _sequence(case, data, rows, tag, stack=None):
    """forward + backward (parameter gradients) + input gradient + jvp; every output cloned."""
    stack = stack or case.stack
    x, dy, v, xd = data[rows]
    acts = stack.forward(x, rows, tag)
    stack.backward(acts, dy, rows, tag)
    out = [a.clone() for a in acts[1:]] + [case.group.grad.clone()]
    if case.layers[0].kind == "linear":
        out.append(stack.backward(acts, dy, rows, tag, param_grads=False, input_grad=True).clone())
        out += [t.clone() for t in stack.jvp(acts, v, rows, tag, x_dot=xd)]
    torch.cuda.synchronize()
    return out


def _same(key, got, want):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        _exact(f"{key}/{i}", _h(g), _h(w))


@gpu
@pytest.mark.parametrize("name", list(CHAINS))
def test_repeatable_and_scratch_separated_by_tag_and_rows(name):
    """Two identical forward + backward + jvp sequences are bit-identical.  A forward on tag "a", a forward on tag "b"
    with other rows, then a backward on "a" gives "a"'s gradients.  On one tag, 4099 rows after 37 (the scratch grows) and 37
    after 4099 give what a fresh stack gives."""
    from tianshou_b200.algorithm.netgraph import FusedStack
    case = _Case(name, _seed(name, 0) + 9)
    rng = np.random.default_rng(_seed(name, 0) + 10)
    data = {}
    for rows in (37, 129, 4099):
        x, _ = case.input(rng, rows)
        data[rows] = (x, _dev(rng.standard_normal((rows, case.out_dim)).astype(np.float32)),
                      _dev(rng.standard_normal(case.group.n).astype(np.float32)),
                      _dev(rng.standard_normal(tuple(x.shape)).astype(np.float32)))
    tag = f"fused_stack/repeat/{name}"
    first = _sequence(case, data, 129, "a")
    _same(tag + "/twice", _sequence(case, data, 129, "a"), first)
    acts_a = case.stack.forward(data[129][0], 129, "a")
    case.stack.forward(data[4099][0], 4099, "b")
    case.stack.backward(acts_a, data[129][1], 129, "a")
    torch.cuda.synchronize()
    n_acts = len(case.layers)
    _same(tag + "/tags", [a.clone() for a in acts_a[1:]] + [case.group.grad.clone()], first[:n_acts + 1])
    fresh = {rows: _sequence(case, data, rows, "t", FusedStack(case.layers, case.group)) for rows in (37, 4099)}
    for rows in (37, 4099, 37):
        _same(f"{tag}/rows{rows}", _sequence(case, data, rows, "t"), fresh[rows])


@gpu
def test_sweep_runs_split_and_unsplit_gemms():
    """The row counts put forward GEMMs on both paths of ``ts_net_gemm``: split-K at some counts, and every forward GEMM
    of every chain unsplit at the largest."""
    from tianshou_b200._cabi import load_library
    from tianshou_b200.algorithm.netgraph import compile_sequential
    lib = load_library()
    split = {}
    for name, make in CHAINS.items():
        net, shape = make()
        for L in compile_sequential(list(net), shape):
            if L.kind == "flatten":
                continue
            for rows in ROWS:
                M = rows * L.Ho * L.Wo if L.kind == "conv" else rows
                split[(name, rows, L.in_dim, L.out_dim)] = int(lib.ts_net_gemm_workspace_floats(M, L.out_dim, L.in_dim)) > 0
    assert any(split.values())
    assert not any(s for (_, rows, _, _), s in split.items() if rows == BIG)
    assert any(s for (_, rows, K, _), s in split.items() if rows == 4099 and K > 64)


# ------------------------------------------------------------------------------------ compile_sequential (no GPU needed)
def _sig(layers):
    return [(L.kind, L.act, L.in_dim, L.out_dim, L.C, L.H, L.W, L.k, L.s, L.Ho, L.Wo) for L in layers]


ACCEPTED = {
    "linear": (lambda: [nn.Linear(5, 3)], (5,), [("linear", ACT_NONE, 5, 3)]),
    "relu_tanh_mlp": (lambda: [nn.Linear(5, 7), nn.ReLU(), nn.Linear(7, 4), nn.Tanh(), nn.Linear(4, 2)], (5,),
                      [("linear", ACT_RELU, 5, 7), ("linear", ACT_TANH, 7, 4), ("linear", ACT_NONE, 4, 2)]),
    "flatten_of_a_vector_is_nothing": (lambda: [nn.Flatten(), nn.Linear(5, 2)], (5,), [("linear", ACT_NONE, 5, 2)]),
    "conv_relu_flatten_linear": (lambda: [nn.Conv2d(2, 3, 3, 2), nn.ReLU(), nn.Flatten(), nn.Linear(18, 4)], (2, 5, 7),
                                 [("conv", ACT_RELU, 18, 3), ("flatten", ACT_NONE, 18, 18), ("linear", ACT_NONE, 18, 4)]),
    "conv_flatten_without_activation": (lambda: [nn.Conv2d(2, 3, 3, 2), nn.Flatten(), nn.Linear(18, 4)], (2, 5, 7),
                                        [("conv", ACT_NONE, 18, 3), ("flatten", ACT_NONE, 18, 18), ("linear", ACT_NONE, 18, 4)]),
}

REFUSED = {
    "linear_without_bias": (lambda: [nn.Linear(5, 3, bias=False)], (5,)),
    "sigmoid": (lambda: [nn.Linear(5, 3), nn.Sigmoid(), nn.Linear(3, 2)], (5,)),
    "gelu": (lambda: [nn.Linear(5, 3), nn.GELU(), nn.Linear(3, 2)], (5,)),
    "activation_first": (lambda: [nn.ReLU(), nn.Linear(5, 2)], (5,)),
    "activation_after_flatten": (lambda: [nn.Conv2d(2, 3, 3, 2), nn.Flatten(), nn.ReLU(), nn.Linear(18, 4)], (2, 5, 7)),
    "two_activations": (lambda: [nn.Linear(5, 3), nn.ReLU(), nn.Tanh(), nn.Linear(3, 2)], (5,)),
    "tanh_before_conv": (lambda: [nn.Conv2d(2, 3, 1, 1), nn.Tanh(), nn.Conv2d(3, 3, 3, 2), nn.Flatten(), nn.Linear(18, 4)], (2, 5, 7)),
    "tanh_before_flatten": (lambda: [nn.Conv2d(2, 3, 3, 2), nn.Tanh(), nn.Flatten(), nn.Linear(18, 4)], (2, 5, 7)),
    "leading_flatten_of_3d_input": (lambda: [nn.Flatten(), nn.Linear(24, 5), nn.ReLU(), nn.Linear(5, 2)], (2, 3, 4)),
    "nested_leading_flatten": (lambda: [nn.Sequential(nn.Flatten(), nn.Linear(24, 5)), nn.Linear(5, 2)], (2, 3, 4)),
    "linear_width_mismatch": (lambda: [nn.Linear(5, 3), nn.Linear(4, 2)], (5,)),
    "linear_on_3d_input": (lambda: [nn.Linear(24, 5)], (2, 3, 4)),
}


@pytest.mark.parametrize("case", list(ACCEPTED))
def test_compile_sequential_accepts(case):
    from tianshou_b200.algorithm.netgraph import compile_sequential
    make, shape, want = ACCEPTED[case]
    assert [s[:4] for s in _sig(compile_sequential(make(), shape))] == want


@pytest.mark.parametrize("case", list(REFUSED))
def test_compile_sequential_refuses(case):
    """Layers and orders the fused stack has no kernels for raise ``UnsupportedModelError`` when the chain is compiled,
    not at the first forward or backward.  A Flatten of a (C, H, W) network input is one: the stack's flatten permutes a
    convolution's NHWC rows into NCHW order, and a network input has no such rows (with the frame source, none at all)."""
    from tianshou_b200.algorithm.flat_params import UnsupportedModelError
    from tianshou_b200.algorithm.netgraph import compile_sequential
    make, shape = REFUSED[case]
    with pytest.raises(UnsupportedModelError):
        compile_sequential(make(), shape)


def test_nested_sequential_and_identity_compile_like_the_flat_chain():
    """Nested ``nn.Sequential`` containers (one starting with the Flatten of the outer chain's convolution, one starting
    with the activation of the outer chain's Linear) and ``nn.Identity`` anywhere compile to the same layers, on the same
    parameters, as the flat chain."""
    from tianshou_b200.algorithm.netgraph import compile_sequential
    c1, c2, l1, l2 = nn.Conv2d(2, 3, 3, 2), nn.Conv2d(3, 4, 1, 1), nn.Linear(24, 6), nn.Linear(6, 2)
    flat = [c1, nn.ReLU(), c2, nn.Flatten(), l1, nn.Tanh(), l2]
    nested = [nn.Identity(), nn.Sequential(nn.Sequential(c1, nn.ReLU()), nn.Identity(), c2), nn.Sequential(nn.Flatten(), l1),
              nn.Sequential(nn.Tanh(), nn.Identity(), nn.Sequential(l2)), nn.Identity()]
    want = compile_sequential(flat, (2, 5, 7))
    got = compile_sequential(nested, (2, 5, 7))
    assert _sig(got) == _sig(want)
    assert [(id(L.weight), id(L.bias)) for L in got] == [(id(L.weight), id(L.bias)) for L in want]
    assert [id(L.weight) for L in want if L.weight is not None] == [id(m.weight) for m in (c1, c2, l1, l2)]
    assert want[0].Ho == 2 and want[0].Wo == 3 and want[2].out_dim == 24
