"""The undecided list that the device's interval proofs share (UndecidedList in derp_host.cuh), probed through
derp_test_undecided_list: a kernel appends the items 0 .. n - 1, and the list relaunches it once when they overflow its
starting capacity.  The library's own calls start at 2^20 entries, which no test workload fills."""
import ctypes as C

import numpy as np
import pytest

from facebook360_dep_b200 import capi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    lib = capi.load_cuda().lib
    lib.derp_test_undecided_list.restype = C.c_int
    lib.derp_test_undecided_list.argtypes = [C.c_int, C.c_int, C.c_uint64, C.c_void_p]
    return lib


@pytest.mark.parametrize("n, start_capacity, launches", [
    (0, 1024, 1),         # nothing listed
    (1000, 1024, 1),      # below the capacity
    (1024, 1024, 1),      # exactly full
    (100_000, 1, 2),      # overflow: one relaunch with a list of n entries
])
def test_collects_every_item(lib, n, start_capacity, launches):
    out = np.full(max(n, 1), np.iinfo(np.uint64).max, np.uint64)
    got = lib.derp_test_undecided_list(0, n, start_capacity, out.ctypes.data)
    assert got == launches, (got, lib.derp_last_error())
    assert np.array_equal(np.sort(out[:n]), np.arange(n, dtype=np.uint64))
