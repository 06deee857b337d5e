"""In-tree builder / loader for the two native extensions.

* ``_psb200_host``  — g++ only (pybind11): shm transport, tensor packing, byte shuffle.
* ``_psb200_cuda``  — nvcc ``-gencode arch=compute_90a,code=sm_90a -lineinfo`` kernels (pure
  CUDA translation units, no torch headers → seconds per file) + the C++ VMM symmetric-memory
  runtime + one torch-aware ``bindings.cpp``.

Both ``.so`` files are written next to this package (git-ignored) and are imported straight from that path — there is no JIT cache and no
silent fallback: on a GPU box a missing CUDA extension raises.
"""
from __future__ import annotations

import importlib.machinery
import importlib.util
import os
import subprocess
import sys
import sysconfig
import threading
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from typing import List, Optional

PKG = Path(__file__).resolve().parent.parent
CSRC = PKG / "csrc"
OBJ = PKG / "_build"
SUFFIX = sysconfig.get_config_var("EXT_SUFFIX")
HOST_SO = PKG / f"_psb200_host{SUFFIX}"
CUDA_SO = PKG / f"_psb200_cuda{SUFFIX}"

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
              "--expt-relaxed-constexpr", "-Xptxas", "-v"]

_lock = threading.Lock()
_host_mod = None
_cuda_mod = None


def _run(cmd: List[str], log: Optional[Path] = None) -> str:
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if log is not None:
        log.write_text(" ".join(cmd) + "\n" + p.stdout)
    if p.returncode != 0:
        raise RuntimeError(f"build step failed ({p.returncode}): {' '.join(cmd)}\n{p.stdout[-6000:]}")
    return p.stdout


def _newer(target: Path, deps: List[Path]) -> bool:
    if not target.exists():
        return False
    t = target.stat().st_mtime
    return all(d.stat().st_mtime <= t for d in deps if d.exists())


def _py_includes() -> List[str]:
    import pybind11
    return ["-I" + sysconfig.get_paths()["include"], "-I" + pybind11.get_include()]


def nvcc_path() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    return "nvcc"


def cuda_home() -> str:
    return os.environ.get("CUDA_HOME", "/usr/local/cuda")


# ---------------------------------------------------------------------------------------
def build_host(force: bool = False, verbose: bool = False) -> Path:
    src = CSRC / "runtime" / "host_ext.cpp"
    if not force and _newer(HOST_SO, [src]):
        return HOST_SO
    OBJ.mkdir(exist_ok=True)
    cmd = ["g++", "-O3", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-pthread",
           *_py_includes(), str(src), "-o", str(HOST_SO), "-lrt"]
    out = _run(cmd, OBJ / "host_ext.log")
    if verbose:
        print(out)
    return HOST_SO


def cuda_sources() -> List[Path]:
    return sorted((CSRC / "kernels").glob("*.cu"))


def build_cuda(force: bool = False, verbose: bool = False) -> Path:
    """Compile every ``csrc/kernels/*.cu`` for sm_90a, the runtime and the bindings; link."""
    import torch
    from torch.utils import cpp_extension as ce

    OBJ.mkdir(exist_ok=True)
    cus = cuda_sources()
    headers = list((CSRC / "kernels").glob("*.cuh")) + list((CSRC / "kernels").glob("*.h")) + \
        list((CSRC / "runtime").glob("*.h"))
    cpps = [CSRC / "runtime" / "symm_mem.cpp", CSRC / "bindings.cpp", CSRC / "gemm_bindings.cpp"]
    all_src = cus + cpps + headers
    if not force and _newer(CUDA_SO, all_src):
        return CUDA_SO
    inc = ["-I" + str(CSRC / "kernels"), "-I" + str(CSRC / "runtime"), "-I" + cuda_home() + "/include"]
    jobs = []
    objs = []
    for cu in cus:
        o = OBJ / (cu.stem + ".o")
        objs.append(o)
        if force or not _newer(o, [cu] + headers):
            jobs.append(([nvcc_path(), *ARCH_FLAGS, *NVCC_FLAGS, *inc, "-c", str(cu), "-o", str(o)],
                         OBJ / (cu.stem + ".nvcc.log")))
    torch_inc = ["-I" + p for p in ce.include_paths()]
    abi = getattr(torch._C, "_GLIBCXX_USE_CXX11_ABI", True)
    cxx = ["g++", "-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-pthread",
           f"-D_GLIBCXX_USE_CXX11_ABI={int(abi)}", "-DTORCH_EXTENSION_NAME=_psb200_cuda",
           "-DTORCH_API_INCLUDE_EXTENSION_H", *inc, *_py_includes(), *torch_inc]
    for cp in cpps:
        o = OBJ / (cp.stem + ".o")
        objs.append(o)
        if force or not _newer(o, [cp] + headers):
            jobs.append(([*cxx, "-c", str(cp), "-o", str(o)], OBJ / (cp.stem + ".cxx.log")))
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        outs = list(ex.map(lambda j: _run(*j), jobs))
    if verbose:
        for o in outs:
            print(o)
    libdirs = ce.library_paths() + [cuda_home() + "/lib64"]
    link = ["g++", "-shared", "-o", str(CUDA_SO), *map(str, objs),
            *["-L" + d for d in libdirs], *["-Wl,-rpath," + d for d in libdirs],
            "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
            "-lcudart", "-ldl", "-lrt", "-pthread"]
    _run(link, OBJ / "link.log")
    return CUDA_SO


def build_all(force: bool = False, verbose: bool = False) -> None:
    build_host(force, verbose)
    build_cuda(force, verbose)


# ---------------------------------------------------------------------------------------
def _load(name: str, path: Path):
    loader = importlib.machinery.ExtensionFileLoader(name, str(path))
    spec = importlib.util.spec_from_file_location(name, str(path), loader=loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    sys.modules[name] = mod
    return mod


def host_available() -> bool:
    return _host_mod is not None or HOST_SO.exists()


def host():
    """The host extension (built on first use if the compiler is around)."""
    global _host_mod
    with _lock:
        if _host_mod is None:
            if not HOST_SO.exists():
                build_host()
            _host_mod = _load("_psb200_host", HOST_SO)
        return _host_mod


def cuda_available() -> bool:
    return _cuda_mod is not None or CUDA_SO.exists()


def cuda():
    """The CUDA extension.  Never falls back: a GPU path without its kernels is an error."""
    global _cuda_mod
    with _lock:
        if _cuda_mod is None:
            if not CUDA_SO.exists():
                if os.environ.get("PSB200_NO_AUTOBUILD"):
                    raise RuntimeError(f"{CUDA_SO.name} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
                build_cuda()
            import torch  # noqa: F401  (libtorch must be loaded before the extension)
            _cuda_mod = _load("_psb200_cuda", CUDA_SO)
        return _cuda_mod


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built:", HOST_SO.name, CUDA_SO.name)
