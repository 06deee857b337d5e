"""The native extensions exist, import on a CPU-only box, and the CUDA objects really are sm_90a code
using the Hopper paths (wgmma, TMA loads / multicast / stores in the SASS)."""
import shutil
import subprocess

import pytest

from pytorch_ps_mpi_b200.ops import ext


def test_host_extension_imports_and_works():
    h = ext.host()
    assert h.ANY_SOURCE == -1
    raw = bytes(range(64))
    assert bytes(h.byteunshuffle(h.byteshuffle(raw, 4), 4)) == raw


def test_cuda_extension_imports_without_a_gpu():
    if not ext.CUDA_SO.exists():
        pytest.skip("CUDA extension not built yet (run __graft_entry__.build())")
    m = ext.cuda()
    for name in ("SymmBlock", "UpdatePlan", "encode", "signal", "wait_flags", "select_ready", "bcast_gemm",
                 "bn_forward", "bn_backward", "maxpool_forward", "im2col_stem", "normalize_nhwc3", "launch_count"):
        assert hasattr(m, name), name
    assert m.TILE == 2048 and m.MAX_RANKS >= 8


def _sass(obj):
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    return subprocess.run([exe, "-sass", str(obj)], stdout=subprocess.PIPE, text=True, check=True).stdout


def test_sass_shows_hopper_paths():
    gemm, psk = ext.OBJ / "bcast_gemm.o", ext.OBJ / "ps_kernels.o"
    if not gemm.exists() or not psk.exists():
        pytest.skip("object files not present (built elsewhere)")
    s = _sass(gemm)
    assert "sm_90a" in s or "EF_CUDA_SM90" in s
    for mnemonic in ("HGMMA.64x128x16.F32.BF16", "HGMMA.64x64x16.F32.BF16", "UTMALDG.2D", "UTMALDG.2D.MULTICAST", "UTMASTG.2D"):
        assert mnemonic in s, f"{mnemonic} missing from bcast_gemm SASS"
    p = _sass(psk)
    assert "STRONG.SYS" in p            # system-scope peer loads/stores of the gather / broadcast
    assert "HMMA" not in s.replace("HGMMA", "")        # no legacy mma.sync tensor path in the GEMM


def test_sass_of_the_fused_stem_and_gemm_epilogues():
    """The fused stem and the GEMM (TMA-store epilogue) are real wgmma / TMA code, and spill nothing."""
    stem, gemm = ext.OBJ / "stem_kernels.o", ext.OBJ / "bcast_gemm.o"
    if not stem.exists() or not gemm.exists():
        pytest.skip("object files not present (built elsewhere)")
    s = _sass(stem)
    for mnemonic in ("HGMMA.64x64x16.F32.BF16", "UTMALDG.2D", "UTMASTG.2D", "LDGSTS"):
        assert mnemonic in s, f"{mnemonic} missing from stem_kernels SASS"
    g = _sass(gemm)
    for mnemonic in ("HGMMA.64x128x16.F32.BF16", "UTMALDG.2D.MULTICAST", "UTMASTG.2D"):
        assert mnemonic in g, f"{mnemonic} missing from bcast_gemm SASS"
    for log in ("stem_kernels.nvcc.log", "bcast_gemm.nvcc.log", "bn_kernels.nvcc.log", "pool_kernels.nvcc.log"):
        p = ext.OBJ / log
        if p.exists():
            for line in p.read_text().splitlines():
                if "spill" in line:
                    assert "0 bytes spill stores, 0 bytes spill loads" in line, f"{log}: {line.strip()}"


def test_ps_kernels_spill_budget():
    """``ps_kernels.cu`` at ``__launch_bounds__(256, 3)`` (85 registers, so that the whole grid is co-resident): nothing spills
    except the dense-coding update kernels with a 32- or 16-bit wire (fp32 / bf16 / fp16 gathers per rank in flight), and those
    no more than sm_90a's ptxas spills today: 80 bytes with an fp32 wire, 16 bytes with a bf16 / fp16 wire."""
    p = ext.OBJ / "ps_kernels.nvcc.log"
    if not p.exists():
        pytest.skip("build log not present (built elsewhere)")
    budget = {"psb_update_kernelILi0ELi0E": 80, "psb_update_kernelILi0ELi1E": 16, "psb_update_kernelILi0ELi2E": 16}
    entry = None
    for line in p.read_text().splitlines():
        if "Compiling entry function" in line:
            entry = line.split("'")[1]
        if "spill" in line and "0 bytes spill stores, 0 bytes spill loads" not in line:
            limit = next((v for k, v in budget.items() if k in entry), None)
            assert limit is not None, f"{entry}: {line.strip()}"
            assert int(line.split("bytes stack frame,")[1].split("bytes spill stores")[0]) <= limit, f"{entry}: {line.strip()}"


def test_built_extensions_are_not_older_than_their_sources():
    """The in-tree ``.so`` files travel to the GPU box as they are: a kernel edited after the last build would be tested (and
    benchmarked) in its OLD form there.  ``make build`` / ``__graft_entry__.build()`` refreshes them."""
    if not ext.CUDA_SO.exists() or not ext.HOST_SO.exists():
        pytest.skip("extensions not built yet (run __graft_entry__.build())")
    native = ext.cuda_sources() + list((ext.CSRC / "kernels").glob("*.cuh")) + list((ext.CSRC / "kernels").glob("*.h")) + \
        list((ext.CSRC / "runtime").glob("*.h")) + [ext.CSRC / "runtime" / "symm_mem.cpp", ext.CSRC / "bindings.cpp",
                                                     ext.CSRC / "gemm_bindings.cpp"]
    def stale():
        return [p.name for p in native if p.stat().st_mtime > ext.CUDA_SO.stat().st_mtime]

    if stale() and shutil.which("g++") and shutil.which(ext.nvcc_path()):
        ext.build_cuda()                  # what `make test` does first (a checkout may also have touched the sources)
    assert not stale(), f"{ext.CUDA_SO.name} is older than {stale()}: rebuild"
    if (ext.CSRC / "runtime" / "host_ext.cpp").stat().st_mtime > ext.HOST_SO.stat().st_mtime and shutil.which("g++"):
        ext.build_host()
    assert (ext.CSRC / "runtime" / "host_ext.cpp").stat().st_mtime <= ext.HOST_SO.stat().st_mtime, "host extension is stale"
