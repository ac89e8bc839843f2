"""``ao_b200.quantization`` — same import surface as ``torchao.quantization`` for the hot path."""
from .granularity import Granularity, PerAxis, PerBlock, PerGroup, PerRow, PerTensor, PerToken  # noqa: F401
from .quant_primitives import MappingType  # noqa: F401
from .quantize_.common import KernelPreference  # noqa: F401
from .quantize_.workflows import (  # noqa: F401
    Float8PackingFormat, Float8Sparse2x4_2DData2DMetadataTensor, Float8Tensor, Int4ChooseQParamsAlgorithm,
    Int4PackingFormat, Int4TilePackedTo4dTensor, Int8Tensor, NF4Tensor, QuantizeTensorToFloat8Kwargs,
    QuantizeTensorToInt8Kwargs, to_nf4)
from .quant_api import (  # noqa: F401
    Float8DynamicActivationFloat8WeightConfig, Float8WeightOnlyConfig, FqnToConfig, Int4WeightOnlyConfig,
    Int8DynamicActivationInt8WeightConfig, Int8StaticActivationInt8WeightConfig, Int8WeightOnlyConfig, ModuleFqnToConfig,
    fqn_matches_fqn_config, quantize_)
from .transform_module import register_quantize_module_handler  # noqa: F401
from .utils import compute_error  # noqa: F401
from ao_b200.float8.inference import Float8MMConfig  # noqa: F401
from ao_b200.prototype.quantization.quant_api import Float8StaticActivationFloat8WeightConfig  # noqa: F401,E402

import torch as _torch

_torch.serialization.add_safe_globals([Granularity, PerAxis, PerBlock, PerGroup, PerRow, PerTensor, PerToken,
                                       KernelPreference, MappingType, Int4PackingFormat, Int4ChooseQParamsAlgorithm,
                                       Float8PackingFormat, Float8MMConfig])
