"""Build the native pieces in-tree (no JIT cache): the C-ABI CUDA library
``ao_b200/lib/libao_b200.so`` (nvcc, sm_90a only) and the torch.library binding
``ao_b200/lib/ao_b200_torch.so`` (g++ against the installed torch headers).

Run ``python -m ao_b200._build`` or call :func:`build_all`.  Nothing here needs a GPU.
"""
from __future__ import annotations

import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
LIB = ROOT / "lib"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-diag-suppress", "177",
]


def _newer(target: Path, sources) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(s).stat().st_mtime > t for s in sources)


def nvcc_path() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def build_cuda_lib(force: bool = False, verbose: bool = False) -> Path:
    LIB.mkdir(exist_ok=True)
    out = LIB / "libao_b200.so"
    cu = sorted(CSRC.glob("*.cu"))
    deps = cu + sorted(CSRC.glob("*.h")) + sorted(CSRC.glob("*.cuh")) + [ROOT.parent / "include" / "ao_b200.h"]
    if not force and not _newer(out, deps):
        return out
    objs = []
    procs = []
    objdir = LIB / "obj"
    objdir.mkdir(exist_ok=True)
    for src in cu:
        obj = objdir / (src.stem + ".o")
        objs.append(obj)
        if not force and not _newer(obj, [src] + [d for d in deps if d.suffix in (".h", ".cuh")]):
            continue
        cmd = [nvcc_path(), *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        log, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{log}")
        if verbose:
            print(log)
    cmd = [nvcc_path(), "-shared", "-o", str(out), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc link failed:\n{r.stdout}")
    return out


def build_torch_binding(force: bool = False) -> Path:
    """Compile csrc/torch_binding.cpp (TORCH_LIBRARY(ao_b200, ...)) against libao_b200.so."""
    import torch
    from torch.utils import cpp_extension as ce

    LIB.mkdir(exist_ok=True)
    out = LIB / "ao_b200_torch.so"
    src = CSRC / "torch_binding.cpp"
    if not src.exists():
        raise FileNotFoundError(src)
    if not force and not _newer(out, [src, CSRC / "torch_binding_lowp.inc", ROOT.parent / "include" / "ao_b200.h", LIB / "libao_b200.so"]):
        return out
    inc = []
    for p in ce.include_paths():
        inc += ["-isystem", p]
    inc += ["-I", "/usr/local/cuda/include", "-I", str(ROOT.parent / "include")]
    torch_lib = os.path.join(os.path.dirname(torch.__file__), "lib")
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    cmd = [
        "g++", "-O2", "-std=c++17", "-fPIC", "-shared", f"-D_GLIBCXX_USE_CXX11_ABI={abi}",
        "-DTORCH_EXTENSION_NAME=ao_b200_torch",
        *inc, str(src), "-o", str(out),
        f"-L{LIB}", "-lao_b200", f"-L{torch_lib}", "-ltorch", "-ltorch_cpu", "-lc10", "-ltorch_cuda", "-lc10_cuda",
        "-Wl,-rpath,$ORIGIN", f"-Wl,-rpath,{torch_lib}",
    ]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"g++ failed for torch binding:\n{r.stdout[-6000:]}")
    return out


def build_all(force: bool = False, verbose: bool = False):
    a = build_cuda_lib(force=force, verbose=verbose)
    b = build_torch_binding(force=force)
    return a, b


if __name__ == "__main__":
    force = "--force" in sys.argv
    verbose = "-v" in sys.argv
    if "--dry-run" in sys.argv:   # what would be compiled, without compiling (also: the clean-checkout test)
        print("nvcc:", nvcc_path(), " ".join(NVCC_FLAGS))
        for src in sorted(CSRC.glob("*.cu")):
            print("  ", src.relative_to(ROOT.parent))
        print("  ", (CSRC / "torch_binding.cpp").relative_to(ROOT.parent))
        sys.exit(0)
    for p in build_all(force=force, verbose=verbose):
        print("built", p)
