"""``Batch`` -- the dict-like container of numpy arrays / torch tensors / nested Batches that
travels between Collector, ReplayBuffer and Algorithm.

API contract mirrored from the reference (tianshou/data/batch.py:625-1372): attribute and key
access, row indexing of every leaf (``__getitem__`` :714-738), row assignment from a compatible
Batch (``__setitem__`` :769-793), ``cat``/``stack`` with zero padding of partially-present keys
(:907-1123), ``split`` with the *global* ``np.random.permutation`` and ``merge_last`` rule
(:1199-1215), ``len`` = min over leaves (:1162-1182), ``to_torch_``/``to_numpy_`` (:860-905).

This is an independent implementation written against that contract; leaves are normalised once
on insertion (``_coerce``) so every other method can rely on {Batch, ndarray, Tensor, None}.
"""
from __future__ import annotations

import pprint
from collections.abc import Callable, Collection, Iterable, Iterator, KeysView, Sequence
from copy import deepcopy
from numbers import Number
from typing import Any, Union

import numpy as np
import torch
from torch.distributions import Categorical, Distribution, Independent, Normal

IndexType = Union[slice, int, np.ndarray, list]
TArr = Union[torch.Tensor, np.ndarray]

_NUMERIC = (np.bool_, np.number)


def _numeric_array(a: Any) -> bool:
    return isinstance(a, np.ndarray) and issubclass(a.dtype.type, _NUMERIC)


def _is_record_list(obj: Any) -> bool:
    """A "batch set": non-empty list/tuple (or 1-d+ object array) of dict/Batch records."""
    if isinstance(obj, np.ndarray):
        return (
            obj.shape != ()
            and obj.dtype == object
            and all(isinstance(e, (dict, Batch)) for e in obj)
        )
    return (
        isinstance(obj, (list, tuple))
        and len(obj) > 0
        and all(isinstance(e, (dict, Batch)) for e in obj)
    )


def _is_scalar(v: Any) -> bool:
    if isinstance(v, torch.Tensor):
        return v.dim() == 0
    return np.isscalar(v)


def _as_typed_array(obj: Any) -> np.ndarray:
    """ndarray with bool/number dtype, otherwise object dtype (strings, None, ragged)."""
    if _numeric_array(obj):
        return obj
    try:
        arr = np.asanyarray(obj)
    except ValueError:
        arr = np.asanyarray(obj, dtype=object)
    if not issubclass(arr.dtype.type, _NUMERIC):
        arr = arr.astype(object)
    if arr.dtype == object:
        if arr.shape == ():
            return arr.item(0)
        flat = arr.reshape(-1)
        if all(isinstance(e, np.ndarray) for e in flat):
            return arr
        if any(isinstance(e, torch.Tensor) for e in flat):
            raise ValueError("Numpy arrays of tensors are not supported yet.")
    return arr


def _coerce(obj: Any) -> Any:
    """Normalise a value stored in a Batch to Batch | ndarray | Tensor | None | Distribution."""
    if isinstance(obj, Batch) or obj is None or isinstance(obj, torch.Tensor) or _numeric_array(obj):
        return obj
    if isinstance(obj, (Number, np.number, np.bool_)):
        return np.asanyarray(obj)
    if isinstance(obj, dict):
        return Batch(obj)
    if type(obj).__name__ == "Batch" and hasattr(obj, "get_keys") and hasattr(obj, "__getitem__"):
        # a Batch of another implementation with the same protocol (the reference Collector builds its own when it drives
        # this package's buffers / policies, INTEGRATION.md): adopt its entries
        return Batch({k: obj[k] for k in obj.get_keys()})
    if isinstance(obj, Distribution):
        return obj
    if (
        not isinstance(obj, np.ndarray)
        and isinstance(obj, Collection)
        and len(obj) > 0
        and all(isinstance(e, torch.Tensor) for e in obj)
    ):
        try:
            return torch.stack(list(obj))
        except RuntimeError as e:
            raise TypeError(
                "Batch does not support non-stackable iterable of torch.Tensor as unique value yet."
            ) from e
    if _is_record_list(obj):
        return Batch(obj)
    try:
        return _as_typed_array(obj)
    except ValueError as e:
        raise TypeError(
            "Batch does not support heterogeneous list/tuple of tensors as unique value yet."
        ) from e


def create_value(inst: Any, size: int, stack: bool = True) -> Union["Batch", np.ndarray, torch.Tensor]:
    """Zero/None-filled storage for ``size`` rows shaped like ``inst`` (reference batch.py:147-182).

    ``stack=True``: ``inst`` is one row; ``stack=False``: ``inst`` already has a leading row axis.
    """
    scalar = _is_scalar(inst)
    if not stack and scalar:
        raise TypeError(f"cannot concatenate with {inst} which is scalar")
    if isinstance(inst, (np.ndarray, torch.Tensor)):
        shape = (size, *inst.shape) if stack else (size, *inst.shape[1:])
        if isinstance(inst, torch.Tensor):
            return torch.zeros(shape, dtype=inst.dtype, device=inst.device)
        if issubclass(inst.dtype.type, _NUMERIC):
            return np.zeros(shape, dtype=inst.dtype)
        return np.full(shape, None, dtype=object)
    if isinstance(inst, (dict, Batch)):
        out = Batch()
        for k, v in inst.items():
            out.__dict__[k] = create_value(v, size, stack=stack)
        return out
    if scalar:
        return create_value(np.asarray(inst), size, stack=stack)
    return np.full((size,), None, dtype=object)


def alloc_by_keys_diff(meta: "Batch", batch: "Batch", size: int, stack: bool = True) -> None:
    """Add storage to ``meta`` for keys of ``batch`` it lacks (reference batch.py:230-247)."""
    for key in batch.get_keys():
        if key in meta.get_keys():
            mv, bv = meta[key], batch[key]
            if isinstance(mv, Batch) and isinstance(bv, Batch):
                alloc_by_keys_diff(mv, bv, size, stack)
            elif isinstance(mv, Batch) and len(mv.get_keys()) == 0:
                meta[key] = create_value(bv, size, stack)
        else:
            meta[key] = create_value(batch[key], size, stack)


def get_sliced_dist(dist: Distribution, index: IndexType) -> Distribution:
    """Row-slice a torch distribution (reference batch.py:265-277)."""
    if isinstance(dist, Categorical):
        return Categorical(probs=dist.probs[index])
    if isinstance(dist, Normal):
        return Normal(loc=dist.loc[index], scale=dist.scale[index])
    if isinstance(dist, Independent):
        return Independent(get_sliced_dist(dist.base_dist, index), dist.reinterpreted_batch_ndims)
    raise NotImplementedError(f"Unsupported distribution for slicing: {dist}")


def get_len_of_dist(dist: Distribution) -> int:
    if len(dist.batch_shape) == 0:
        raise TypeError(f"scalar Distribution has no length: {dist=}")
    return dist.batch_shape[0]


def _empty(b: Any) -> bool:
    return isinstance(b, Batch) and len(b.__dict__) == 0


class Batch:
    """Dict-like container; see module docstring."""

    def __init__(
        self,
        batch_dict: dict | "Batch" | Sequence[dict | "Batch"] | np.ndarray | None = None,
        copy: bool = False,
        **kwargs: Any,
    ) -> None:
        if copy:
            batch_dict = deepcopy(batch_dict)
        if batch_dict is not None:
            if isinstance(batch_dict, (dict, Batch)):
                keys = list(batch_dict.keys())
                assert all(isinstance(k, str) for k in keys), f"keys should all be string, but got {keys}"
                for k, v in batch_dict.items():
                    self.__dict__[k] = _coerce(v)
            elif _is_record_list(batch_dict):
                self.stack_(batch_dict)  # type: ignore[arg-type]
        if kwargs:
            Batch.__init__(self, kwargs, copy=copy)

    # ---------------------------------------------------------------- mapping surface
    def get_keys(self) -> KeysView:
        return self.__dict__.keys()

    def keys(self) -> KeysView:
        return self.__dict__.keys()

    def values(self):
        return self.__dict__.values()

    def items(self):
        return self.__dict__.items()

    def get(self, key: str, default: Any | None = None) -> Any:
        return self.__dict__.get(key, default)

    def pop(self, key: str, default: Any | None = None) -> Any:
        return self.__dict__.pop(key, default)

    def to_dict(self, recursive: bool = True) -> dict[str, Any]:
        return {
            k: (v.to_dict(recursive=True) if recursive and isinstance(v, Batch) else v)
            for k, v in self.__dict__.items()
        }

    def to_list_of_dicts(self) -> list[dict[str, Any]]:
        return [row.to_dict() for row in self]

    def __setattr__(self, key: str, value: Any) -> None:
        self.__dict__[key] = _coerce(value)

    def __getattr__(self, key: str) -> Any:
        # only reached when normal lookup fails -> mimic dict attribute fall-through
        return getattr(self.__dict__, key)

    def __contains__(self, key: str) -> bool:
        return key in self.__dict__

    def __getstate__(self) -> dict[str, Any]:
        return {k: (v.__getstate__() if isinstance(v, Batch) else v) for k, v in self.items()}

    def __setstate__(self, state: dict[str, Any]) -> None:
        Batch.__init__(self, **state)

    # ---------------------------------------------------------------- indexing
    def __getitem__(self, index: str | IndexType) -> Any:
        if isinstance(index, str):
            return self.__dict__[index]
        if not self.__dict__:
            raise IndexError("Cannot access item from empty Batch object.")
        out = Batch()
        for k, v in self.__dict__.items():
            if v is None:
                out.__dict__[k] = None
            elif _empty(v):
                out.__dict__[k] = Batch()
            elif isinstance(v, Distribution):
                out.__dict__[k] = get_sliced_dist(v, index)
            else:
                out.__dict__[k] = v[index]
        return out

    def __setitem__(self, index: str | IndexType, value: Any) -> None:
        value = _coerce(value)
        if isinstance(index, str):
            self.__dict__[index] = value
            return
        if not isinstance(value, Batch):
            raise ValueError(
                "Batch does not supported tensor assignment. Use a compatible Batch or dict instead."
            )
        if not set(value.keys()).issubset(self.__dict__.keys()):
            raise ValueError("Creating keys is not supported by item assignment.")
        for k, cur in self.__dict__.items():
            if cur is None:
                continue
            if k in value.__dict__:
                cur[index] = value.__dict__[k]
            elif isinstance(cur, Batch):
                cur[index] = Batch()
            elif isinstance(cur, torch.Tensor) or _numeric_array(cur):
                cur[index] = 0
            else:
                cur[index] = None

    def __iter__(self) -> Iterator["Batch"]:
        if not self.__dict__:
            return
        for i in range(len(self)):
            yield self[i]

    def __len__(self) -> int:
        lens = []
        for k, v in self.__dict__.items():
            if v is None or (isinstance(v, Batch) and len(v) == 0):
                continue
            if isinstance(v, Distribution):
                lens.append(get_len_of_dist(v))
            elif isinstance(v, Batch) or (hasattr(v, "__len__") and v.ndim > 0):
                lens.append(len(v))
            else:
                raise TypeError(f"Entry for {k} in {self} is {v} has no len()")
        return min(lens) if lens else 0

    @property
    def shape(self) -> list[int]:
        if not self.__dict__:
            return []
        shapes = []
        for v in self.__dict__.values():
            try:
                shapes.append(list(v.shape))
            except AttributeError:
                shapes.append([])
        return list(map(min, zip(*shapes, strict=False))) if len(shapes) > 1 else shapes[0]

    # ---------------------------------------------------------------- arithmetic
    def _inplace_op(self, other: Any, fn: Callable[[Any, Any], Any], name: str) -> "Batch":
        if isinstance(other, Batch):
            for (k, v), ov in zip(self.__dict__.items(), other.__dict__.values(), strict=True):
                if _empty(v):
                    continue
                self.__dict__[k] = fn(v, ov)
            return self
        if isinstance(other, (Number, np.number, np.bool_)):
            for k, v in self.__dict__.items():
                if _empty(v):
                    continue
                self.__dict__[k] = fn(v, other)
            return self
        raise TypeError(f"Only {name} of Batch or number is supported.")

    def __iadd__(self, other: Any) -> "Batch":
        def add(a: Any, b: Any) -> Any:
            a += b
            return a

        return self._inplace_op(other, add, "addition")

    def __add__(self, other: Any) -> "Batch":
        return deepcopy(self).__iadd__(other)

    def __imul__(self, value: Any) -> "Batch":
        assert isinstance(value, (Number, np.number, np.bool_)), "Only multiplication by a number is supported."

        def mul(a: Any, b: Any) -> Any:
            a *= b
            return a

        return self._inplace_op(value, mul, "multiplication")

    def __mul__(self, value: Any) -> "Batch":
        return deepcopy(self).__imul__(value)

    def __itruediv__(self, value: Any) -> "Batch":
        assert isinstance(value, (Number, np.number, np.bool_)), "Only division by a number is supported."

        def div(a: Any, b: Any) -> Any:
            a /= b
            return a

        return self._inplace_op(value, div, "division")

    def __truediv__(self, value: Any) -> "Batch":
        return deepcopy(self).__itruediv__(value)

    def __repr__(self) -> str:
        s = self.__class__.__name__ + "(\n"
        any_key = False
        for k, v in self.__dict__.items():
            pad = " " * (6 + len(k))
            s += f"    {k}: " + pprint.pformat(v).replace("\n", "\n" + pad) + ",\n"
            any_key = True
        return s + ")" if any_key else self.__class__.__name__ + "()"

    def __eq__(self, other: Any) -> bool:
        if not isinstance(other, self.__class__):
            return False

        def same(a: Any, b: Any) -> bool:
            if isinstance(a, Batch) or isinstance(b, Batch):
                if not (isinstance(a, Batch) and isinstance(b, Batch)):
                    return False
                if set(a.keys()) != set(b.keys()):
                    return False
                return all(same(a[k], b[k]) for k in a.keys())
            if a is None or b is None:
                return a is None and b is None
            if isinstance(a, torch.Tensor):
                a = a.detach().cpu().numpy()
            if isinstance(b, torch.Tensor):
                b = b.detach().cpu().numpy()
            if isinstance(a, Distribution) or isinstance(b, Distribution):
                return a is b
            a, b = np.atleast_1d(a), np.atleast_1d(b)
            if a.shape != b.shape:
                return False
            if a.dtype == object or b.dtype == object:
                return all(x == y for x, y in zip(a.reshape(-1), b.reshape(-1), strict=True))
            return bool(np.array_equal(a, b, equal_nan=True))

        return same(self, other)

    __hash__ = None  # type: ignore[assignment]

    # ---------------------------------------------------------------- conversions
    def apply_values_transform(self, values_transform: Callable, inplace: bool = False) -> "Batch | None":
        def rec(b: Batch) -> Batch:
            out = b if inplace else Batch()
            for k, v in list(b.__dict__.items()):
                out.__dict__[k] = rec(v) if isinstance(v, Batch) else values_transform(v)
            return out

        result = rec(self)
        return None if inplace else result

    def to_numpy_(self) -> None:
        self.apply_values_transform(
            lambda a: a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a, inplace=True
        )

    def to_numpy(self) -> "Batch":
        out = deepcopy(self)
        out.to_numpy_()
        return out

    def to_torch_(self, dtype: torch.dtype | None = None, device: str | int | torch.device = "cpu") -> None:
        if not isinstance(device, torch.device):
            device = torch.device(device)

        def conv(a: Any) -> Any:
            if isinstance(a, np.ndarray):
                return torch.from_numpy(a).to(device)
            if isinstance(a, torch.Tensor):
                if dtype is not None and a.dtype != dtype:
                    a = a.type(dtype)
                if a.device.type != device.type or device.index != a.device.index:
                    a = a.to(device)
            return a

        self.apply_values_transform(conv, inplace=True)

    def to_torch(self, dtype: torch.dtype | None = None, device: str | int | torch.device = "cpu") -> "Batch":
        out = deepcopy(self)
        out.to_torch_(dtype=dtype, device=device)
        return out

    def to_at_least_2d(self) -> "Batch":
        def f(a: Any) -> Any:
            if isinstance(a, torch.Tensor):
                return torch.atleast_2d(a)
            if isinstance(a, np.ndarray):
                return np.atleast_2d(a)
            return a

        return self.apply_values_transform(f)  # type: ignore[return-value]

    # ---------------------------------------------------------------- cat / stack
    @staticmethod
    def _normalise_inputs(batches: Any, op: str) -> list["Batch"]:
        if isinstance(batches, (Batch, dict)):
            batches = [batches]
        out = []
        for b in batches:
            if isinstance(b, dict):
                b = Batch(b)
            if not isinstance(b, Batch):
                raise ValueError(f"Cannot {op} {type(b)} in Batch.{op}_")
            if len(b.__dict__) == 0:
                continue
            out.append(b)
        return out

    def _cat_into(self, batches: Sequence["Batch"], lens: list[int]) -> None:
        """Concatenate along rows; keys present in only some inputs are zero-padded."""
        starts = np.concatenate([[0], np.cumsum(lens)]).astype(int)
        total = int(starts[-1])
        live = [{k for k, v in b.items() if not _empty(v)} for b in batches]
        shared = set.intersection(*live)
        every = set.union(*[set(b.keys()) for b in batches])
        for k in [k for k in batches[0].keys() if k in shared] + sorted(
            shared - set(batches[0].keys())
        ):
            vals = [b[k] for b in batches]
            if all(isinstance(v, (dict, Batch)) for v in vals):
                holder = Batch()
                holder._cat_into(vals, lens)
                self.__dict__[k] = holder
            elif all(isinstance(v, torch.Tensor) for v in vals):
                self.__dict__[k] = torch.cat(vals)
            else:
                self.__dict__[k] = _as_typed_array(np.concatenate(vals))
        reserved = every - set.union(*live)
        for k in every - shared:
            if k in reserved:
                self.__dict__[k] = Batch()
                continue
            for i, b in enumerate(batches):
                v = b.__dict__.get(k)
                if v is None or _empty(v):
                    continue
                if k not in self.__dict__:
                    self.__dict__[k] = create_value(v, total, stack=False)
                self.__dict__[k][starts[i] : starts[i + 1]] = v

    def cat_(self, batches: "Batch | Sequence[dict | Batch]") -> None:
        """In-place row concatenation of ``self`` followed by ``batches`` (ref. batch.py:976-1034)."""
        blist = self._normalise_inputs(batches, "concatenate")
        if not blist:
            return
        try:
            lens = [0 if len(b.get_keys()) == 0 else len(b) for b in blist]
        except TypeError as e:
            raise ValueError(
                f"Batch.cat_ meets an exception. Maybe because there is any scalar in {blist} "
                "but Batch.cat_ does not support the concatenation of scalar."
            ) from e
        if self.__dict__:
            blist = [self, *blist]
            # ``self`` may hold only reserved (empty) keys
            lens = [0 if all(_empty(v) for v in self.values()) else len(self), *lens]
        merged = Batch()
        merged._cat_into(blist, lens)
        self.__dict__.clear()
        self.__dict__.update(merged.__dict__)

    @staticmethod
    def cat(batches: Sequence[dict | "Batch"]) -> "Batch":
        out = Batch()
        out.cat_(batches)
        return out

    def stack_(self, batches: Sequence[dict | "Batch"], axis: int = 0) -> None:
        """In-place stacking of records along a new axis (ref. batch.py:1041-1117)."""
        blist = self._normalise_inputs(batches, "stack")
        if not blist:
            return
        if self.__dict__:
            blist = [self, *blist]
        live = [{k for k, v in b.items() if not _empty(v)} for b in blist]
        shared = set.intersection(*live)
        ordered_shared = [k for k in blist[0].keys() if k in shared]
        result: dict[str, Any] = {}
        for k in ordered_shared:
            vals = [b[k] for b in blist]
            if all(isinstance(v, torch.Tensor) for v in vals):
                result[k] = torch.stack(vals, axis)
            elif all(isinstance(v, (Batch, dict)) for v in vals):
                result[k] = Batch.stack(vals, axis)
            else:
                try:
                    result[k] = _as_typed_array(np.stack(vals, axis))
                except ValueError:
                    arr = np.empty(len(vals), dtype=object)
                    arr[:] = vals
                    result[k] = arr
        every = set.union(*[set(b.keys()) for b in blist])
        reserved = every - set.union(*live)
        partial = every - shared - reserved
        if partial and axis != 0:
            raise ValueError(
                f"Stack of Batch with non-shared keys {partial} is only supported with axis=0, "
                f"but got axis={axis}!"
            )
        for k in reserved:
            result[k] = Batch()
        for k in partial:
            for i, b in enumerate(blist):
                v = b.__dict__.get(k)
                if v is None or _empty(v):
                    continue
                if k not in result:
                    result[k] = create_value(v, len(blist))
                result[k][i] = v
        self.__dict__.clear()
        self.__dict__.update(result)

    @staticmethod
    def stack(batches: Sequence[dict | "Batch"], axis: int = 0) -> "Batch":
        out = Batch()
        out.stack_(batches, axis)
        return out

    def empty_(self, index: IndexType | None = None) -> "Batch":
        """Reset rows (all, or ``index``) to 0 / None (ref. batch.py:1125-1148)."""
        for k, v in self.__dict__.items():
            if isinstance(v, torch.Tensor):
                if index is None:
                    v.zero_()
                else:
                    v[index] = 0
            elif v is None:
                continue
            elif isinstance(v, np.ndarray):
                fill = None if v.dtype == object else 0
                if index is None:
                    v.fill(fill)  # type: ignore[arg-type]
                else:
                    v[index] = fill
            elif isinstance(v, Batch):
                v.empty_(index=index)
            else:
                self.__dict__[k] = None
        return self

    @staticmethod
    def empty(batch: "Batch", index: IndexType | None = None) -> "Batch":
        return deepcopy(batch).empty_(index)

    def update(self, batch: "dict | Batch | None" = None, **kwargs: Any) -> None:
        if batch is not None:
            for k, v in batch.items():
                self.__dict__[k] = _coerce(v)
        if kwargs:
            self.update(kwargs)

    # ---------------------------------------------------------------- minibatching
    def split(self, size: int, shuffle: bool = True, merge_last: bool = False) -> Iterator["Batch"]:
        """Yield row minibatches.  The shuffle order is ONE draw of the *global* numpy RNG
        (``np.random.permutation``), exactly as the reference (batch.py:1209) so that index
        streams stay identical; a short tail is folded into the previous chunk when
        ``merge_last`` (:1210-1215).
        """
        n = len(self)
        if size == -1:
            size = n
        assert size >= 1
        order = np.random.permutation(n) if shuffle else np.arange(n)
        for lo, hi in minibatch_bounds(n, size, merge_last):
            yield self[order[lo:hi]]

    # ---------------------------------------------------------------- null handling
    def set_array_at_key(
        self,
        arr: np.ndarray,
        key: str,
        index: IndexType | None = None,
        default_value: float | None = None,
    ) -> None:
        if index is None:
            if len(arr) != len(self):
                raise ValueError(
                    f"Sequence length {len(arr)} does not match batch length {len(self)}. For setting a "
                    "subsequence with missing entries filled up by default values, consider passing an index."
                )
            self[key] = arr
            return
        if key not in self.get_keys():
            try:
                self[key] = np.array([default_value] * len(self), dtype=arr.dtype)
            except TypeError as e:
                raise TypeError(
                    f"Cannot create a sequence of dtype {arr.dtype} with default value {default_value}."
                ) from e
        elif isinstance(self[key], Batch):
            raise ValueError(
                f"Cannot set sequence at key {key} because it is a nested batch, "
                "can only set a subsequence of an array."
            )
        self[key][index] = arr

    def isnull(self) -> "Batch":
        def f(a: Any) -> Any:
            if isinstance(a, torch.Tensor):
                return torch.isnan(a).cpu().numpy() if a.is_floating_point() else np.zeros(a.shape, bool)
            if a is None:
                return np.array(True)
            a = np.asarray(a)
            if a.dtype == object:
                flat = np.array([e is None or (isinstance(e, float) and e != e) for e in a.reshape(-1)])
                return flat.reshape(a.shape)
            if issubclass(a.dtype.type, np.floating):
                return np.isnan(a)
            return np.zeros(a.shape, bool)

        return self.apply_values_transform(f)  # type: ignore[return-value]

    def hasnull(self) -> bool:
        def any_true(b: Batch) -> bool:
            for v in b.values():
                if isinstance(v, Batch):
                    if any_true(v):
                        return True
                elif bool(np.any(v)):
                    return True
            return False

        return any_true(self.isnull())

    def dropnull(self) -> "Batch":
        keep = []
        for row in self:
            if row.hasnull():
                continue
            keep.append(row.apply_values_transform(np.atleast_1d))
        return Batch.cat(keep)

    def replace_empty_batches_by_none(self) -> None:
        for k, v in self.items():
            if isinstance(v, Batch):
                if len(v.get_keys()) == 0:
                    self.__dict__[k] = None
                else:
                    v.replace_empty_batches_by_none()


def minibatch_bounds(n: int, size: int, merge_last: bool) -> list[tuple[int, int]]:
    """[lo, hi) positions of each minibatch for ``Batch.split`` (ref. batch.py:1210-1215).

    Shared by the host iterator above and by the fused device update so both cut the permuted
    index array identically.
    """
    merge = merge_last and n % size > 0
    out = []
    for lo in range(0, n, size):
        if merge and lo + size + size >= n:
            out.append((lo, n))
            break
        out.append((lo, min(lo + size, n)))
    return out


def numpy_global_permutation_(out: "torch.Tensor") -> "torch.Tensor":
    """``out[:] = np.random.permutation(len(out))`` (int32, host tensor -- typically pinned) drawn from numpy's
    GLOBAL legacy RandomState exactly as ``Batch.split(shuffle=True)`` does (batch.py:1209): same values, same
    state afterwards.  Runs the reference's algorithm (MT19937 + masked rejection + backward Fisher-Yates) as a
    tight int32 loop in the C library (``ts_host_mt19937_permutation``), ~3x faster than numpy + astype + copy."""
    import ctypes as C

    from .._cabi import call
    n = out.numel()
    st = np.random.get_state()
    if st[0] != "MT19937" or out.dtype != torch.int32 or out.is_cuda or not out.is_contiguous():
        out.copy_(torch.from_numpy(np.random.permutation(n).astype(np.int32)))
        return out
    key = np.ascontiguousarray(st[1], dtype=np.uint32).copy()
    pos = C.c_int32(int(st[2]))
    call("ts_host_mt19937_permutation", key.ctypes.data_as(C.c_void_p), C.byref(pos), n, C.c_void_p(out.data_ptr()))
    np.random.set_state((st[0], key, pos.value, st[3], st[4]))
    return out


class NumpyGlobalPermutationJob:
    """All ``repeat`` draws ``np.random.permutation(n)`` of one ``update()`` from numpy's GLOBAL legacy stream,
    produced ahead of the passes that use them by background threads of the C library
    (``ts_host_perm_job_*``, csrc/hostperm.cu): bit-identical rows and final generator state, but row r is
    ready ~4 + 2 r ms after the start instead of after (r + 1) x 14 ms of ``np.random.permutation + astype``.
    ``rows``: int32 host tensor [>= repeat, n] (pinned).  Use as a context manager; ``wait(r)`` blocks until row r is
    complete; leaving the context joins the threads and writes the advanced state back into numpy.  ``handle``: the C
    job (what ``ts_host_perm_feed_start`` takes), None when the rows were drawn up front."""

    def __init__(self, rows: "torch.Tensor", repeat: int, n_workers: int | None = None) -> None:
        import ctypes as C
        import os

        from .._cabi import call
        assert rows.dtype == torch.int32 and not rows.is_cuda and rows.is_contiguous() and rows.shape[0] >= repeat
        self.rows, self._repeat, self._n = rows, repeat, rows.shape[1]
        self.shape = (repeat, self._n)
        self._st = np.random.get_state()
        self.handle = None
        if self._st[0] != "MT19937":          # not the legacy MT19937 state: plain numpy draws, in order, up front
            self._draw_serially()
            return
        self._key = np.ascontiguousarray(self._st[1], dtype=np.uint32).copy()
        # generator + walker + nw appliers per process; under torchrun every local rank runs its own job on the same host cores
        local_world = max(1, int(os.environ.get("LOCAL_WORLD_SIZE", "1") or 1))
        cores = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 2)
        # a row beyond ~1 M entries no longer fits a core's L2: its swaps cost ~4x as much each, so give the appliers twice the width
        nw = (n_workers or int(os.environ.get("TS_B200_PERM_WORKERS", "0") or 0)
              or max(1, min(repeat, 8 if self._n >= (1 << 20) else (2 if local_world >= 4 else 4), cores // local_world - 2)))
        # (>= 4 local ranks: two appliers per rank still finish every row ahead of the GPU and leave the host threads that feed the
        # GPUs more room)
        h = C.c_void_p()
        try:
            call("ts_host_perm_job_start", self._key.ctypes.data_as(C.c_void_p), int(self._st[2]), self._n, repeat,
                 C.c_void_p(rows.data_ptr()), nw, C.byref(h))
            self.handle = h
        except RuntimeError:      # no threads / memory for the job: same stream, drawn serially (in order) right now
            self.handle = None
            self._draw_serially()

    def _draw_serially(self) -> None:
        for r in range(self._repeat):
            numpy_global_permutation_(self.rows[r])

    def wait(self, r: int) -> "torch.Tensor":
        from .._cabi import call
        if self.handle is not None:
            call("ts_host_perm_job_wait", self.handle, r)
        return self.rows[r]

    def __enter__(self) -> "NumpyGlobalPermutationJob":
        return self

    def __exit__(self, *exc: Any) -> None:
        import ctypes as C

        from .._cabi import call
        if self.handle is not None:
            pos = C.c_int32(0)
            call("ts_host_perm_job_finish", self.handle, self._key.ctypes.data_as(C.c_void_p), C.byref(pos))
            self.handle = None
            cur = np.random.get_state()
            if cur[2] != self._st[2] or not np.array_equal(cur[1], self._st[1]):
                # somebody drew from numpy's GLOBAL stream while the update was running (an lr-scheduler lambda, user
                # callbacks, another thread): the `repeat` permutations were taken from the state at the START of update(), as
                # the reference would have taken them had that draw come later.  Writing the advanced state back would replay /
                # drop that draw, so the foreign stream position wins and the divergence is reported.
                import warnings
                warnings.warn("numpy's global RNG was used while Algorithm.update() was drawing its minibatch permutations; "
                              "the global stream is left as that draw put it (it no longer matches the reference's)", RuntimeWarning,
                              stacklevel=2)
                return
            np.random.set_state((self._st[0], self._key, pos.value, self._st[3], self._st[4]))
