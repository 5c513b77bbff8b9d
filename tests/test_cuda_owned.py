"""The owning device buffer of csrc/cuda_owned.h, which holds every buffer of the decoder and the channelizer, driven
through build/host_emul.so.  reserve() must record a pointer and a capacity only once an allocation has succeeded: a
failed one leaves the buffer empty, and the next reserve tries again instead of reporting success with a null pointer.
A request of 2**50 bytes is refused without allocating anything, so this is safe on a shared GPU."""
import ctypes as C

import numpy as np
import pytest

from conftest import have_gpu
from gr_lora_b200 import build as B

HUGE = 1 << 50


@pytest.fixture(scope="module")
def reserve():
    """reserve(sizes) -> [(cudaError_t, pointer or None, capacity)] after each reserve on one fresh buffer."""
    L = C.CDLL(str(B.build_host_emul()))
    L.lb_emul_buffer_reserve.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]

    def run(sizes):
        n = len(sizes)
        sz = np.array(sizes, np.uint64)
        rc, ptr, cap = np.zeros(n, np.int32), np.zeros(n, np.uint64), np.zeros(n, np.uint64)
        L.lb_emul_buffer_reserve(sz.ctypes.data, n, rc.ctypes.data, ptr.ctypes.data, cap.ctypes.data)
        return [(int(r), int(p) or None, int(c)) for r, p, c in zip(rc, ptr, cap)]
    return run


def test_failed_reserve_leaves_buffer_empty(reserve):
    for rc, ptr, cap in reserve([HUGE, HUGE]):      # the second, identical request tries again and fails the same way
        assert rc != 0
        assert ptr is None and cap == 0


def test_every_reserve_fails_without_gpu(reserve):
    if have_gpu():
        pytest.skip("a CUDA device is present")
    for rc, ptr, cap in reserve([1, 4096, HUGE, 4096]):
        assert rc != 0
        assert ptr is None and cap == 0


@pytest.mark.gpu
def test_reserve_grows_only_past_capacity(reserve):
    huge, r4k, r1k, r8k, huge2 = reserve([HUGE, 4096, 1024, 8192, HUGE])
    assert huge[0] != 0 and huge[1:] == (None, 0)
    assert r4k[0] == 0 and r4k[1] is not None and r4k[2] == 4096
    assert r1k == r4k                                # within capacity: the same buffer
    assert r8k[0] == 0 and r8k[1] is not None and r8k[2] == 8192
    assert huge2[0] != 0 and huge2[1:] == (None, 0)  # a failed growth has freed the old buffer and left the buffer empty
