"""JSON side of the safetensors wire format of quantized tensors (SURVEY §8f rank 3).

Mirrors the on-disk convention of the reference (`torchao/prototype/safetensors/safetensors_utils.py:30-256`), which
HF transformers reads and writes (`transformers/integrations/torchao.py`): every quantized tensor becomes one JSON
string ``{"_type": <class name>, "_data": {non-tensor attributes}, "_tensor_data_names": [...]}``; nested values
(kwargs dataclasses, NamedTuples, enums, dtypes, granularities) are tagged ``{"_type", "_data"}`` objects; decoding
only instantiates names from an allow-list.
"""
from __future__ import annotations

import dataclasses
import enum
import json
from typing import Any, Dict

import torch

from ao_b200.float8.inference import Float8MMConfig
from ao_b200.prototype.mx_formats.mx_tensor import MXTensor, QuantizeTensorToMXKwargs, ScaleCalculationMode
from ao_b200.prototype.mx_formats.nvfp4_tensor import NVFP4Tensor, QuantizeTensorToNVFP4Kwargs
from ao_b200.quantization.granularity import PerBlock, PerRow, PerTensor
from ao_b200.quantization.quant_primitives import MappingType
from ao_b200.quantization.quantize_.common.kernel_preference import KernelPreference
from ao_b200.quantization.quantize_.workflows.float8.float8_tensor import Float8Tensor, QuantizeTensorToFloat8Kwargs
from ao_b200.quantization.quantize_.workflows.int4.int4_tile_packed_to_4d_tensor import Int4TilePackedTo4dTensor
from ao_b200.quantization.quantize_.workflows.int8.int8_tensor import Int8Tensor, QuantizeTensorToInt8Kwargs

__all__ = ["ALLOWED_CLASSES", "ALLOWED_TENSORS_SUBCLASSES", "TensorSubclassAttributeJSONEncoder", "object_from_dict",
           "is_metadata_torchao"]

# tensor subclasses of the hot path (the reference's list also names formats outside SURVEY §8: Int4Tensor,
# Int4PlainInt32Tensor, IntxUnpackedToInt8Tensor; metadata naming them is recognised but cannot be rebuilt here)
_TENSOR_CLASSES = {c.__name__: c for c in (Float8Tensor, Int4TilePackedTo4dTensor, Int8Tensor, MXTensor, NVFP4Tensor)}
_REFERENCE_ONLY_TENSORS = ("Int4Tensor", "IntxUnpackedToInt8Tensor", "Int4PlainInt32Tensor")
ALLOWED_TENSORS_SUBCLASSES = list(_TENSOR_CLASSES) + list(_REFERENCE_ONLY_TENSORS)
ALLOWED_CLASSES: Dict[str, type] = dict(_TENSOR_CLASSES)
ALLOWED_CLASSES.update({c.__name__: c for c in (Float8MMConfig, QuantizeTensorToFloat8Kwargs, QuantizeTensorToInt8Kwargs,
                                                 QuantizeTensorToMXKwargs, QuantizeTensorToNVFP4Kwargs, PerBlock, PerRow, PerTensor,
                                                 KernelPreference, MappingType, ScaleCalculationMode)})


def _names(obj, attr):
    return list(getattr(obj, attr, None) or [])


class TensorSubclassAttributeJSONEncoder(json.JSONEncoder):
    """``json.dumps(tensor, cls=TensorSubclassAttributeJSONEncoder)`` -> the tensor's metadata string."""

    def default(self, o):
        if type(o).__name__ in ALLOWED_TENSORS_SUBCLASSES:
            attrs = {name: self.encode_value(getattr(o, name))
                     for name in _names(o, "optional_tensor_attribute_names") + _names(o, "tensor_attribute_names")}
            present = [name for name in _names(o, "optional_tensor_data_names") + _names(o, "tensor_data_names")
                       if getattr(o, name) is not None]
            return {"_type": type(o).__name__, "_data": attrs, "_tensor_data_names": present}
        if isinstance(o, tuple) and hasattr(o, "_fields"):  # NamedTuple (Float8MMConfig)
            return {"_type": type(o).__name__, "_data": {k: self.encode_value(v) for k, v in o._asdict().items()}}
        if dataclasses.is_dataclass(o) and not isinstance(o, type):
            return {"_type": type(o).__name__,
                    "_data": {f.name: self.encode_value(getattr(o, f.name)) for f in dataclasses.fields(o)}}
        if isinstance(o, torch.dtype):
            return {"_type": "torch.dtype", "_data": str(o).rsplit(".", 1)[-1]}
        if isinstance(o, enum.Enum):
            return {"_type": type(o).__name__, "_data": o.name}
        if isinstance(o, list):
            return [self.encode_value(v) for v in o]
        if isinstance(o, dict):
            return {k: self.encode_value(v) for k, v in o.items()}
        return super().default(o)

    def encode_value(self, value):
        """Tagged encoding where one applies, the value itself (left to the stock encoder) otherwise."""
        try:
            return self.default(value)
        except TypeError:
            return value


def _is_tagged(v) -> bool:
    return isinstance(v, dict) and "_type" in v and "_data" in v


def object_from_dict(data: Dict[str, Any]):
    """Inverse of the encoder for one tagged object (tensor subclasses included once their tensors are in ``_data``)."""
    if not isinstance(data, dict):
        raise TypeError(f"Expected dictionary, got {type(data)}")
    if "_type" not in data or "_data" not in data:
        raise ValueError("Input dictionary missing required '_type' or '_data' fields")
    type_name, payload = data["_type"], data["_data"]
    if type_name == "torch.dtype":
        return getattr(torch, payload)
    cls = ALLOWED_CLASSES.get(type_name)
    if cls is None:
        raise ValueError(f"Failed to find class {type_name} in any of the allowed modules: {', '.join(ALLOWED_CLASSES)}")
    if not isinstance(payload, dict):
        if issubclass(cls, enum.Enum):
            return getattr(cls, payload)
        try:
            return cls(payload)
        except Exception:
            return payload
    kwargs = {}
    for key, value in payload.items():
        if _is_tagged(value):
            kwargs[key] = object_from_dict(value)
        elif isinstance(value, list):
            kwargs[key] = [object_from_dict(v) if _is_tagged(v) else v for v in value]
        elif isinstance(value, tuple):
            raise NotImplementedError(f"Tuples are serialized as lists in JSON; use lists to avoid surprises. got: {value}")
        elif isinstance(value, dict):
            kwargs[key] = {k: object_from_dict(v) if _is_tagged(v) else v for k, v in value.items()}
        else:
            kwargs[key] = value
    try:
        return cls(**kwargs)
    except Exception as e:
        raise ValueError(f"Failed to create instance of {cls.__name__}: {e}")


def is_metadata_torchao(metadata: Dict[str, Any]) -> bool:
    """True when a safetensors header's metadata dict was written by flatten_tensor_state_dict."""
    if not metadata or "tensor_names" not in metadata:
        return False
    try:
        names = json.loads(metadata["tensor_names"])
    except (TypeError, json.JSONDecodeError, UnicodeDecodeError):
        return False
    if not names or not isinstance(names, list):
        return False
    for name in names:
        entry = metadata.get(name)
        if not isinstance(entry, str):
            return False
        try:
            kind = json.loads(entry).get("_type")
        except (TypeError, json.JSONDecodeError, UnicodeDecodeError, AttributeError):
            return False
        if kind not in ALLOWED_TENSORS_SUBCLASSES and kind != "Tensor":
            return False
    return True
