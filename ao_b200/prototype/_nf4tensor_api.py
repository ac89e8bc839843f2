"""``NF4WeightOnlyConfig``: QLoRA NF4 weights (reference torchao/prototype/_nf4tensor_api.py), served by the sm_90a
NF4 kernel (``ao_b200.quantization.NF4Tensor``)."""
import logging

import torch

from ao_b200.core.config import AOBaseConfig
from ao_b200.quantization import NF4Tensor
from ao_b200.quantization.transform_module import register_quantize_module_handler

logger = logging.getLogger(__name__)


class NF4WeightOnlyConfig(AOBaseConfig):
    """NF4 weight-only quantization with ``block_size`` elements per scaler and ``scaler_block_size`` scalers per
    quantization factor (class attributes, as in the reference)."""

    block_size: int = 64
    scaler_block_size: int = 256


# for bc
nf4_weight_only = NF4WeightOnlyConfig


def _nf4_kernel_skip_reason(weight: torch.Tensor, block_size: int) -> str:
    """Why the sm_90a kernel cannot serve this weight ('' when it can)."""
    K = weight.shape[-1]
    if weight.dtype != torch.bfloat16:
        return f"weight dtype {weight.dtype} needs to be torch.bfloat16"
    if weight.dim() != 2:
        return f"a {weight.dim()}-D weight needs to be 2-D"
    if block_size % 16 != 0:
        return f"block_size={block_size} needs to be a multiple of 16 (a k16 step within one block)"
    if K % block_size != 0:
        return f"in_features={K} needs to be a multiple of block_size={block_size} (no block across two rows)"
    if K % 32 != 0:
        return f"in_features={K} needs to be a multiple of 32 (the row pitch of the codes)"
    return ""


@register_quantize_module_handler(NF4WeightOnlyConfig)
def _nf4_weight_only_transform(module: torch.nn.Module, config: NF4WeightOnlyConfig, *,
                               parameter_name: str = "weight") -> torch.nn.Module:
    weight = getattr(module, parameter_name)
    n_blocks = weight.numel() // config.block_size
    # the reference's own checks first: these layers fail there too, with the same exception
    assert weight.numel() % config.block_size == 0, (
        f"Input tensor must be divisible by block size, got {weight.numel()} and {config.block_size}")
    assert n_blocks % config.scaler_block_size == 0, (
        f"Number of scalers must be divisible by scaler block size, got {n_blocks} scaler_block_size "
        f"{config.scaler_block_size} ")
    reason = _nf4_kernel_skip_reason(weight, config.block_size)
    if reason:
        # no fallback: the layer stays unquantized, as the weight-only float8 flow does
        logger.info(f"Skipping nf4 weight only quantization of weight shape {tuple(weight.shape)}: {reason} for the "
                    f"sm_90a kernel")
        return module
    new_weight = NF4Tensor.from_tensor(weight.detach(), config.block_size, config.scaler_block_size)
    setattr(module, parameter_name, torch.nn.Parameter(new_weight, requires_grad=False))
    return module


torch.serialization.add_safe_globals([NF4WeightOnlyConfig])
