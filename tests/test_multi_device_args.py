"""The argument checks of a multi-device wax_vs_create (n_devices >= 2), which run before any device query, and the C++
mirror's device-list constructor (compiled and linked as test_abi.py does for the mirror)."""
import ctypes as C
import subprocess
from pathlib import Path

import pytest

from wax_b200 import _lib as L
from wax_b200 import build

ROOT = Path(__file__).resolve().parents[1]


def _create(devices, n=None):
    h = C.c_void_p()
    n = len(devices) if n is None else n
    arr = (C.c_int32 * len(devices))(*devices) if devices is not None else None
    rc = L.lib().wax_vs_create(64, 0, arr, n, C.byref(h))
    assert not h.value
    return rc, L.last_error()


@pytest.mark.parametrize("devices, code, reason", [
    ([0] * 17, L.ERR_ARGUMENT, "17 devices: a multi-device handle takes at most 16"),
    ([0, -1], L.ERR_ARGUMENT, "device ordinal -1 is negative"),
    ([-3, 0, 0], L.ERR_ARGUMENT, "device ordinal -3 is negative"),
])
def test_create_refuses_bad_device_lists_before_any_device_query(devices, code, reason):
    assert _create(devices) == (code, reason)


def test_create_refuses_a_null_device_list():
    assert _create(None, n=2) == (L.ERR_NULL, "devices is NULL")


def test_dimension_and_metric_checks_come_first():
    h = C.c_void_p()
    assert L.lib().wax_vs_create(0, 0, (C.c_int32 * 17)(*[0] * 17), 17, C.byref(h)) == L.ERR_ARGUMENT
    assert L.last_error() == "dimensions must be > 0"


def test_cxx_mirror_device_list_constructor_links(tmp_path):
    lib = build.build()
    src = tmp_path / "probe.cpp"
    src.write_text(f'''#include <cstdio>
#include "{ROOT / "wax_b200" / "host" / "cuda_vector_engine.hpp"}"
int main() {{
    try {{
        wax::CUDAVectorEngine bad(wax::VectorMetric::cosine, 64, std::vector<int32_t>{{0, -1}});
        return 1;
    }} catch (const wax::WaxError &e) {{
        std::printf("%s\\n", e.what());
    }}
    return 0;
}}
''')
    exe = tmp_path / "probe"
    subprocess.run(["g++", "-std=c++17", "-Wall", str(src), f"-L{lib.parent}", "-lwaxvs_cuda", f"-Wl,-rpath,{lib.parent}",
                    "-o", str(exe)], check=True, capture_output=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and "device ordinal -1 is negative" in out.stdout, (out.returncode, out.stdout, out.stderr)
