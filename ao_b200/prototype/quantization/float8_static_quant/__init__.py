from .prototype_float8_tensor import PrototypeFloat8Tensor  # noqa: F401
