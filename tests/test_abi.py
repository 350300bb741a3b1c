"""CPU: the C-ABI library builds, loads, exports every symbol include/wax_vs_cuda.h declares, and fails
loudly (never falls back) when no CUDA device is present."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
HEADER = ROOT / "include" / "wax_vs_cuda.h"


def _declared_symbols():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    return sorted(set(re.findall(r"\b(wax_vs_[a-z_0-9]+)\s*\(", text)))


def test_header_declares_what_the_binding_binds():
    from wax_b200 import _lib
    assert _declared_symbols() == sorted(_lib.SIGNATURES)


def test_library_exports_every_declared_symbol():
    from wax_b200 import _lib, build
    lib_path = build.build()
    assert lib_path.exists()
    out = subprocess.run(["nm", "-D", "--defined-only", str(lib_path)], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (wax_vs_[a-z_0-9]+)", out))
    assert exported == set(_declared_symbols())
    handle = _lib.lib()
    for name in _lib.SIGNATURES:
        assert getattr(handle, name) is not None
    assert b"sm_90a" in handle.wax_vs_version()


def test_library_contains_sm90a_tma_code():
    from wax_b200 import build
    out = subprocess.run(["cuobjdump", "-lelf", str(build.build())], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_candidate_struct_layout():
    from wax_b200 import _lib
    from wax_b200.sharded import CAND_DTYPE
    assert C.sizeof(_lib.Candidate) == 24 == CAND_DTYPE.itemsize
    assert [(_lib.Candidate.distance.offset), _lib.Candidate.valid.offset, _lib.Candidate.row.offset,
            _lib.Candidate.frame_id.offset] == [0, 4, 8, 16]
    assert [CAND_DTYPE.fields[n][1] for n in ("distance", "valid", "row", "frame_id")] == [0, 4, 8, 16]


def test_argument_validation_without_a_device():
    """These checks run before any CUDA call, so they hold on a CPU-only box too."""
    from wax_b200 import _lib
    L = _lib.lib()
    h = C.c_void_p()
    assert L.wax_vs_create(0, 0, None, 0, C.byref(h)) == _lib.ERR_ARGUMENT       # dimensions must be > 0
    assert "dimensions must be > 0" in _lib.last_error()
    assert L.wax_vs_create(1_000_001, 0, None, 0, C.byref(h)) == _lib.ERR_CAPACITY
    assert L.wax_vs_create(4, 3, None, 0, C.byref(h)) == _lib.ERR_ARGUMENT
    assert L.wax_vs_create(4, 0, None, 0, None) == _lib.ERR_NULL
    assert L.wax_vs_device_count(None) == _lib.ERR_NULL
    assert L.wax_vs_count(None, None) == _lib.ERR_NULL
    assert L.wax_vs_debug_shadow_nominations(None, None, 10, None, None, None, None, None) == _lib.ERR_NULL
    assert L.wax_vs_debug_read_shadow(None, 0, 1, None) == _lib.ERR_NULL
    out = (C.c_uint32 * 10)()
    assert L.wax_vs_debug_last_scan(None, out) == _lib.ERR_NULL
    assert L.wax_vs_debug_last_scan(None, None) == _lib.ERR_NULL
    L.wax_vs_destroy(None)  # no-op


def test_no_silent_cpu_fallback():
    """Without a GPU the product path must raise, not compute on the CPU."""
    import wax_b200
    if wax_b200.CUDAVectorEngine.is_available():
        pytest.skip("CUDA device present")
    with pytest.raises(wax_b200.InvalidToc, match="CUDA device not available"):
        wax_b200.CUDAVectorEngine(wax_b200.VectorMetric.cosine, 4)


def test_product_package_never_touches_the_oracle():
    """No import / include / link of anything under oracle/ from the product package (comments may cite it)."""
    from wax_b200 import build
    for path in (ROOT / "wax_b200").rglob("*"):
        if path.suffix == ".py":
            for line in path.read_text().splitlines():
                code = line.split("#", 1)[0]
                assert not re.search(r"^\s*(from|import)\s+oracle\b", code), (path, line)
                assert "libwax_oracle" not in code and "oracle/" not in code.replace("oracle/wax_oracle", ""), (path, line)
        elif path.suffix in {".cu", ".cuh", ".cpp", ".h", ".hpp"}:
            for line in path.read_text().splitlines():
                if line.lstrip().startswith("#include"):
                    assert "oracle" not in line, (path, line)
    # helper scripts are not test infrastructure either: only tests/, __graft_entry__.smoke() and bench.py's CPU legs
    for path in (ROOT / "scripts").glob("*.py"):
        for line in path.read_text().splitlines():
            code = line.split("#", 1)[0]
            assert not re.search(r"^\s*(from|import)\s+oracle\b", code), (path, line)
            assert "libwax_oracle" not in code, (path, line)
    needed = subprocess.run(["readelf", "-d", str(build.build())], capture_output=True, text=True).stdout
    assert "oracle" not in needed
    undefined = subprocess.run(["nm", "-D", "--undefined-only", str(build.build())], capture_output=True, text=True).stdout
    assert "wax_oracle" not in undefined


def test_header_is_valid_c_and_cxx_mirror_links(tmp_path):
    """gcc -std=c11 on a C probe and g++ -std=c++17 on the C++ mirror probe, linked against the built .so."""
    from wax_b200 import build
    lib = build.build()
    env_rpath = f"-Wl,-rpath,{lib.parent}"
    c_exe, cpp_exe = tmp_path / "c_probe", tmp_path / "cpp_probe"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", f"-I{ROOT / 'include'}", str(ROOT / "tests" / "c_abi_probe.c"),
                    f"-L{lib.parent}", "-lwaxvs_cuda", env_rpath, "-o", str(c_exe)], check=True, capture_output=True)
    out = subprocess.run([str(c_exe)], capture_output=True, text=True)
    assert out.returncode == 0 and "sm_90a" in out.stdout, (out.returncode, out.stdout, out.stderr)
    subprocess.run(["g++", "-std=c++17", "-Wall", str(ROOT / "tests" / "cpp_mirror_probe.cpp"), f"-L{lib.parent}",
                    "-lwaxvs_cuda", env_rpath, "-o", str(cpp_exe)], check=True, capture_output=True)
    out = subprocess.run([str(cpp_exe)], capture_output=True, text=True)
    assert out.returncode == 0 and "dimensions must be > 0" in out.stdout, (out.returncode, out.stdout, out.stderr)
