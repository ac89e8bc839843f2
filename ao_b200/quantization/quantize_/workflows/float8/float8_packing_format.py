from enum import Enum


class Float8PackingFormat(str, Enum):
    """reference: workflows/float8/float8_packing_format.py.  PLAIN and SPARSE_2D_DATA_2D_METADATA (2:4-sparse e4m3 in
    CUTLASS's Sm90 layout) have kernels here; SPARSE_1D_DATA_1D_METADATA is the reference's hipSPARSELt (ROCm) format
    and is accepted by the enum only."""

    PLAIN = "plain"
    SPARSE_2D_DATA_2D_METADATA = "sparse_2d_data_2d_metadata"
    SPARSE_1D_DATA_1D_METADATA = "sparse_1d_data_1d_metadata"
    OPAQUE = "opaque"


# the reference's earlier name, kept as an alias (not a member) as the reference keeps it
Float8PackingFormat.SPARSE_CUTLASS = Float8PackingFormat.SPARSE_2D_DATA_2D_METADATA
