"""Golden fixture for 2:4-sparse fp8 (Float8DynamicActivationFloat8WeightConfig with granularity PerRow() and
packing_format SPARSE_2D_DATA_2D_METADATA) from the REFERENCE on the CPU: config_to_dict of the config
(``config_json``), the Float8PackingFormat members and values (``packing_formats``) and what its SPARSE_CUTLASS alias
names (``sparse_cutlass``).  The reference's compressor and GEMM are CUDA-only CUTLASS kernels; the GPU tests compare
against them directly (oracle/ref_sparse.py).

    AO_REFERENCE=<reference checkout> python tests/golden/make_golden_fp8_sparse.py
-> fp8_sparse.npz (JSON strings as 0-d arrays)."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.environ["AO_REFERENCE"])
HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    from torchao.core.config import config_to_dict
    from torchao.quantization import Float8DynamicActivationFloat8WeightConfig, PerRow
    from torchao.quantization.quantize_.workflows.float8.float8_packing_format import Float8PackingFormat

    c = Float8DynamicActivationFloat8WeightConfig(granularity=PerRow(),
                                                  packing_format=Float8PackingFormat.SPARSE_2D_DATA_2D_METADATA)
    out = {
        "config_json": np.array(json.dumps(config_to_dict(c), sort_keys=True)),
        "packing_formats": np.array(json.dumps({m.name: m.value for m in Float8PackingFormat})),
        "sparse_cutlass": np.array(json.dumps([Float8PackingFormat.SPARSE_CUTLASS.name,
                                               Float8PackingFormat.SPARSE_CUTLASS.value])),
    }
    np.savez_compressed(os.path.join(HERE, "fp8_sparse.npz"), **out)
    for k, v in out.items():
        print(k, v)


if __name__ == "__main__":
    main()
