"""b200_alltoall argument checks that need no GPU."""
import ctypes

from ray_b200 import _native


def test_alltoall_rejects_a_null_communicator(native_lib):
    ptrs = (ctypes.c_void_p * 2)()
    counts = (ctypes.c_size_t * 2)(4, 4)
    rc = native_lib.b200_alltoall(None, ptrs, counts, ptrs, counts, _native.F32, None)
    assert rc == _native.ERR_INVALID


def test_alltoall_kernel_is_in_the_library(native_lib):
    import subprocess

    import pytest

    sass = subprocess.run(["cuobjdump", "-sass", str(_native.LIB_PATH)], capture_output=True, text=True)
    if sass.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    assert "alltoall_kernel" in sass.stdout
