from .nf4_tensor import NF4Tensor, linear_nf4, to_nf4  # noqa: F401
