from .int4.int4_packing_format import Int4PackingFormat  # noqa: F401
from .int4.int4_choose_qparams_algorithm import Int4ChooseQParamsAlgorithm  # noqa: F401
from .int4.int4_tile_packed_to_4d_tensor import Int4TilePackedTo4dTensor  # noqa: F401
from .int8.int8_tensor import Int8Tensor, QuantizeTensorToInt8Kwargs  # noqa: F401
from .float8.float8_tensor import Float8Tensor, QuantizeTensorToFloat8Kwargs  # noqa: F401
from .float8.float8_packing_format import Float8PackingFormat  # noqa: F401
from .float8.float8_sparse_2x4_2d_data_2d_metadata_tensor import Float8Sparse2x4_2DData2DMetadataTensor  # noqa: F401
from .nf4.nf4_tensor import NF4Tensor, to_nf4  # noqa: F401

Sparse2x4CUTLASSFloat8Tensor = Float8Sparse2x4_2DData2DMetadataTensor
