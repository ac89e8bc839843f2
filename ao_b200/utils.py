"""Tensor-subclass base for quantized weights + small helpers.

``TorchAOBaseTensor`` plays the role of torchao/utils.py:720-1067: a wrapper subclass whose
payload lives in named attributes (``tensor_data_names`` + ``tensor_attribute_names`` +
optional variants, in ``__init__`` order), with per-class dispatch tables filled by
``@cls.implements(aten_op)`` / ``@cls.implements_torch_function(fn)``.  ``F.linear`` on a module
whose weight is such a subclass lands in the handler that calls ``torch.ops.ao_b200.*``.
Unhandled ops raise NotImplementedError (reference: utils.py:678-697).
"""
from __future__ import annotations

import functools
from typing import Any, Callable, Dict, List

import torch
from torch.utils._python_dispatch import return_and_correct_aliasing

aten = torch.ops.aten

__all__ = [
    "TorchAOBaseTensor", "find_multiple", "rows_for_kernel", "fill_defaults", "is_sm_at_least_100", "is_sm_at_least_90",
    "is_sm_at_least_89", "torch_version_at_least", "get_model_size_in_bytes",
]


def rows_for_kernel(x2: torch.Tensor) -> torch.Tensor:
    """2-D activations as this engine's kernels take them: unit inner stride, row pitch a multiple of 8 elements,
    16-byte aligned start.  A column slice of a wider buffer (the q part of a fused q|k|v output) qualifies and is
    passed through WITHOUT a copy -- the kernels get the pitch; anything else is made contiguous, which is what the
    reference's handlers always do.  (Alignment is judged from the storage offset, not data_ptr(): handlers must
    stay traceable with fake tensors.)"""
    if x2.dim() == 2 and x2.stride(-1) == 1 and x2.stride(0) >= x2.shape[-1] and x2.stride(0) % 8 == 0 and x2.storage_offset() % 8 == 0:
        return x2
    return x2.contiguous()


def find_multiple(n: int, k: int) -> int:
    return n if n % k == 0 else n + k - (n % k)


def fill_defaults(args, n, defaults_tail):
    """Right-fill ``args`` to length n from ``defaults_tail`` (reference: utils.py fill_defaults)."""
    if len(args) + len(defaults_tail) < n:
        raise RuntimeError("not enough defaults to fill arguments")
    r = list(args)
    for i in range(len(args), n):
        r.append(defaults_tail[i - n + len(defaults_tail)])
    return r


def _cap():
    return torch.cuda.get_device_capability() if torch.cuda.is_available() else (0, 0)


def is_sm_at_least_89():
    return _cap() >= (8, 9)


def is_sm_at_least_90():
    return _cap() >= (9, 0)


def is_sm_at_least_100():
    return _cap() >= (10, 0)


def torch_version_at_least(v: str) -> bool:
    from packaging.version import parse

    return parse(torch.__version__.split("+")[0]) >= parse(v)


def get_model_size_in_bytes(model, ignore_embeddings=False):
    def flat_size(t):
        if hasattr(t, "__tensor_flatten__"):
            names, _ = t.__tensor_flatten__()
            return sum(flat_size(getattr(t, n)) for n in names)
        return t.numel() * t.element_size()

    total = 0
    for _, m in model.named_modules():
        if ignore_embeddings and isinstance(m, torch.nn.Embedding):
            continue
        for p in list(m.parameters(recurse=False)) + list(m.buffers(recurse=False)):
            total += flat_size(p)
    return total


class TorchAOBaseTensor(torch.Tensor):
    """Wrapper-subclass base; see module docstring."""

    # per-class tables: {cls: {op: handler}}
    _ATEN_OP_TABLE: Dict[type, Dict[Any, Callable]] = {}
    _TORCH_FN_TABLE: Dict[type, Dict[Any, Callable]] = {}

    def __init_subclass__(cls, **kwargs):
        super().__init_subclass__(**kwargs)
        TorchAOBaseTensor._ATEN_OP_TABLE.setdefault(cls, {})
        TorchAOBaseTensor._TORCH_FN_TABLE.setdefault(cls, {})
        for parent in cls.__bases__:
            TorchAOBaseTensor._ATEN_OP_TABLE[cls].update(TorchAOBaseTensor._ATEN_OP_TABLE.get(parent, {}))
            TorchAOBaseTensor._TORCH_FN_TABLE[cls].update(TorchAOBaseTensor._TORCH_FN_TABLE.get(parent, {}))
        if "tensor_data_names" in cls.__dict__ and "tensor_attribute_names" in cls.__dict__:
            _register_common_ops(cls)

    # ---- registration decorators -------------------------------------------------------
    @classmethod
    def implements(cls, ops):
        if not isinstance(ops, (list, tuple)):
            ops = [ops]

        def deco(fn):
            for op in ops:
                TorchAOBaseTensor._ATEN_OP_TABLE.setdefault(cls, {})[op] = fn
            return fn

        return deco

    @classmethod
    def implements_torch_function(cls, fns):
        if not isinstance(fns, (list, tuple)):
            fns = [fns]

        def deco(fn):
            for f in fns:
                TorchAOBaseTensor._TORCH_FN_TABLE.setdefault(cls, {})[f] = fn
            return fn

        return deco

    # ---- dispatch ----------------------------------------------------------------------
    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        table = TorchAOBaseTensor._TORCH_FN_TABLE.get(cls, {})
        if func in table:
            return table[func](func, types, args, kwargs)
        with torch._C.DisableTorchFunctionSubclass():
            return func(*args, **kwargs)

    @classmethod
    def __torch_dispatch__(cls, func, types, args, kwargs):
        kwargs = kwargs or {}
        table = TorchAOBaseTensor._ATEN_OP_TABLE.get(cls, {})
        if func in table:
            return table[func](func, types, args, kwargs)
        raise NotImplementedError(
            f"{cls.__name__} dispatch: attempting to run unimplemented operator/function: {func=}, {types=}, "
            f"arg_types={tuple(type(a) for a in args)}, kwarg_types={ {k: type(v) for k, v in kwargs.items()} }"
        )

    # ---- flatten / unflatten (torch.compile, state_dict, safetensors) -------------------
    def _all_names(self):
        return (list(self.tensor_data_names), list(self.tensor_attribute_names),
                list(getattr(self, "optional_tensor_data_names", [])),
                list(getattr(self, "optional_tensor_attribute_names", [])))

    def __tensor_flatten__(self):
        td, ta, otd, ota = self._all_names()
        names = td + [n for n in otd if getattr(self, n) is not None]
        attrs = {n: getattr(self, n) for n in ta + ota}
        return names, attrs

    @classmethod
    def __tensor_unflatten__(cls, tensor_data_dict, tensor_attributes, outer_size, outer_stride):
        req_t = [tensor_data_dict[n] for n in cls.tensor_data_names]
        req_a = [tensor_attributes[n] for n in cls.tensor_attribute_names]
        opt_t = {n: tensor_data_dict.get(n, None) for n in getattr(cls, "optional_tensor_data_names", [])}
        opt_a = {n: tensor_attributes[n] for n in getattr(cls, "optional_tensor_attribute_names", [])}
        return cls(*req_t, *req_a, **opt_t, **opt_a)

    def _apply_fn_to_data(self, fn):
        td, ta, otd, ota = self._all_names()
        req_t = [fn(getattr(self, n)) for n in td]
        req_a = [getattr(self, n) for n in ta]
        opt_t = {n: (fn(getattr(self, n)) if getattr(self, n) is not None else None) for n in otd}
        opt_a = {n: getattr(self, n) for n in ota}
        return self.__class__(*req_t, *req_a, **opt_t, **opt_a)

    def __setstate__(self, state):
        # checkpoints written before an optional attribute existed: fill with None (BC,
        # reference utils.py:639-656).  Names the class itself provides (Float8Tensor's `dtype` is the wrapper's own,
        # read-only) are not instance state
        torch._utils._set_obj_state(self, state)
        for n in list(getattr(self, "optional_tensor_data_names", [])) + list(
                getattr(self, "optional_tensor_attribute_names", [])):
            if n not in self.__dict__ and not hasattr(type(self), n):
                setattr(self, n, None)

    def __repr__(self):
        td, ta, otd, ota = self._all_names()
        parts = [f"{n}={getattr(self, n)}" for n in td + ta + otd + ota]
        return f"{self.__class__.__name__}({', '.join(parts)})"

    def _get_to_kwargs(self, *args, **kwargs):
        device, dtype, _, memory_format = torch._C._nn._parse_to(*args, **kwargs)
        device = self.device if device is None else device
        dtype = self.dtype if dtype is None else dtype
        memory_format = memory_format if memory_format is not None else torch.preserve_format
        return {"device": device, "dtype": dtype, "memory_format": memory_format}

    def to(self, *args, **kwargs):
        kw = self._get_to_kwargs(*args, **kwargs)
        dev = kw["device"]
        out = self._apply_fn_to_data(lambda t: t.to(device=dev))
        if kw["dtype"] != self.dtype and hasattr(out, "dtype_attr_name"):
            setattr(out, out.dtype_attr_name, kw["dtype"])
        return out


def _same_metadata(a: TorchAOBaseTensor, b: TorchAOBaseTensor) -> bool:
    if type(a) is not type(b) or a.shape != b.shape:
        return False
    td, ta, otd, ota = a._all_names()
    for n in td:
        if getattr(a, n).shape != getattr(b, n).shape:
            return False
    for n in otd:
        x, y = getattr(a, n), getattr(b, n)
        if (x is None) != (y is None) or (x is not None and x.shape != y.shape):
            return False
    for n in ta + ota:
        if getattr(a, n) != getattr(b, n):
            return False
    return True


def _register_common_ops(cls):
    """detach / clone / alias / contiguous / _to_copy / copy_ for every payload-carrying subclass
    (reference: utils.py:480-636)."""

    @cls.implements([aten.detach.default, aten.alias.default])
    def _(func, types, args, kwargs):
        return return_and_correct_aliasing(func, args, kwargs, args[0]._apply_fn_to_data(lambda t: t.detach()))

    @cls.implements(aten.clone.default)
    def _(func, types, args, kwargs):
        return return_and_correct_aliasing(func, args, kwargs, args[0]._apply_fn_to_data(torch.clone))

    @cls.implements(aten.contiguous.default)
    def _(func, types, args, kwargs):
        return args[0]._apply_fn_to_data(lambda t: t.contiguous())

    @cls.implements(aten._to_copy.default)
    def _(func, types, args, kwargs):
        dev = kwargs.get("device", None)
        self = args[0]
        out = self._apply_fn_to_data(lambda t: t.to(device=dev) if dev is not None else t.clone())
        return return_and_correct_aliasing(func, args, kwargs, out)

    @cls.implements(aten.copy_.default)
    def _(func, types, args, kwargs):
        dst, src = args[0], args[1]
        if not isinstance(src, TorchAOBaseTensor) or not _same_metadata(dst, src):
            raise ValueError(
                f"Not supported args for copy_ due to metadata mismatch: {type(dst).__name__}{tuple(dst.shape)} "
                f"<- {type(src).__name__}{tuple(src.shape)}")
        td, _, otd, _ = dst._all_names()
        for n in td + otd:
            d = getattr(dst, n)
            if d is not None:
                d.copy_(getattr(src, n))
        return dst

    @cls.implements_torch_function(torch.Tensor.contiguous)
    def _(func, types, args, kwargs):
        return args[0]._apply_fn_to_data(lambda t: t.contiguous())
