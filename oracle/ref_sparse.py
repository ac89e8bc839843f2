"""The reference's own 2:4-sparse fp8 kernels as a test oracle: its CUTLASS compressor
(``torchao::to_sparse_semi_structured_cutlass_sm9x_f8``) and GEMM (``torchao::rowwise_scaled_linear_sparse_cutlass_f8f8``),
compiled in place from a torchao source tree by ``ref_sparse.mk`` into ``oracle/_ref/libref_sparse_f8.so``.

TEST INFRASTRUCTURE ONLY: used by tests/test_fp8_sparse_gpu.py and scripts/measure_fp8_sparse.py, never by ao_b200/.
The tree is the first of ``$AO_B200_REFERENCE_TREE``, ``reference`` beside this repository and ``/root/reference`` that
holds the reference's CUDA sources.  Where no tree is present, an already-built library is kept (it travels with the
working tree) and ``build()`` does not fail; it says so when there is neither a tree nor a library.
"""
from __future__ import annotations

import os
import subprocess
import sys
import sysconfig
from pathlib import Path
from typing import Optional

_DIR = Path(__file__).resolve().parent
LIB = _DIR / "_ref" / "libref_sparse_f8.so"
_CSRC = Path("torchao") / "csrc" / "cuda"
_GEMM = _CSRC / "rowwise_scaled_linear_sparse_cutlass"
SOURCES = [_CSRC / "to_sparse_semi_structured_cutlass_sm9x" / "to_sparse_semi_structured_cutlass_sm9x_f8.cu",
           _CSRC / "to_sparse_semi_structured_cutlass_sm9x" / "to_sparse_semi_structured_cutlass_sm9x.cuh",
           _GEMM / "rowwise_scaled_linear_sparse_cutlass.cuh",
           _GEMM / "rowwise_scaled_linear_sparse_cutlass_f8f8.cu"] + [
    _GEMM / f"rowwise_scaled_linear_sparse_cutlass_{a}{b}.{ext}" for a in ("e4m3", "e5m2") for b in ("e4m3", "e5m2")
    for ext in ("cu", "h")]
# the schemas the reference defines in torchao/ops.py (its C++ registers implementations only)
SCHEMAS = [
    "rowwise_scaled_linear_sparse_cutlass_f8f8(Tensor input, Tensor input_scale, Tensor weight, Tensor weight_meta, "
    "Tensor weight_scale, Tensor? bias=None, ScalarType? out_dtype=None) -> Tensor",
    "to_sparse_semi_structured_cutlass_sm9x_f8(Tensor weight) -> (Tensor, Tensor)",
]


def reference_tree() -> Optional[Path]:
    env = os.environ.get("AO_B200_REFERENCE_TREE")
    for tree in ([Path(env)] if env else []) + [_DIR.parent.parent / "reference", Path("/root/reference")]:
        if (tree / _CSRC).is_dir():
            return tree
    return None


def build(jobs: int = 8) -> Optional[Path]:
    """(Re)build the library when a reference tree is present and the library is missing or older than its sources
    or recipe; returns the library path, or None when there is neither a tree nor a library."""
    tree = reference_tree()
    if tree is None:
        if LIB.exists():
            return LIB
        print(f"oracle/ref_sparse: no torchao source tree found ($AO_B200_REFERENCE_TREE, ../reference, "
              f"/root/reference) and no {LIB.relative_to(_DIR.parent)}: the GPU tests against the reference's sparse "
              f"fp8 kernels will skip", file=sys.stderr)
        return None
    deps = [tree / s for s in SOURCES] + [_DIR / "ref_sparse.mk"]
    if LIB.exists() and all(d.stat().st_mtime <= LIB.stat().st_mtime for d in deps if d.exists()):
        return LIB
    import torch
    from torch.utils import cpp_extension

    inc = cpp_extension.include_paths() + [sysconfig.get_paths()["include"]]
    torch_lib = Path(torch.__file__).resolve().parent / "lib"
    cmd = ["make", "-C", str(_DIR), "-f", "ref_sparse.mk", f"-j{jobs}", f"REF={tree}", f"PY_INC={' '.join(inc)}",
           f"TORCH_LIB={torch_lib}"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("reference sparse fp8 oracle build failed:\n" + r.stdout[-8000:])
    return LIB


_LOADED = False


def load():
    """Define the two torchao:: schemas and load the library; returns torch.ops.torchao.  Raises FileNotFoundError
    naming the library when it has not been built."""
    global _LOADED
    import torch

    if not _LOADED:
        if not LIB.exists():
            raise FileNotFoundError(f"{LIB} (built by oracle/ref_sparse.py from a torchao source tree)")
        lib = torch.library.Library("torchao", "FRAGMENT")
        for s in SCHEMAS:
            lib.define(s)
        load.lib = lib   # keep the definitions alive
        torch.ops.load_library(str(LIB))
        _LOADED = True
    return torch.ops.torchao


if __name__ == "__main__":
    print(build() or "no reference tree and no library", file=sys.stderr)
