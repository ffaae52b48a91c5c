"""Per-thread error state without a CUDA device: two threads that call at once each get kind Cuda and their own "CUDA device unavailable"
message, a host-side refusal on one thread leaves the other's message alone, and pco_b200_thread_release on a thread whose device set-up
failed is harmless - the next call fails loudly again.  The device set-up caches "no device" as a permanent outcome; these checks keep it
cached and loud."""
import ctypes as C
import threading

import numpy as np
import pytest

CUDA, INVALID_TYPE = 6, 5


@pytest.fixture(scope="module")
def L():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from pcodec_b200 import _lib

    return _lib.lib()


def _compress(L, nums, dtype_byte):
    dst = np.zeros(4096, np.uint8)
    nw = C.c_size_t()
    return L.pco_b200_compress_ex(nums.ctypes.data_as(C.c_void_p), C.c_size_t(nums.size), C.c_ubyte(dtype_byte), None, C.c_int(0),
                                  dst.ctypes.data_as(C.c_void_p), C.c_size_t(dst.size), C.byref(nw), None, C.c_size_t(0), None, C.c_uint32(0), None)


def _message(L):
    return L.pco_b200_last_error_message().decode()


def _run(workers, timeout=60):
    """Runs each worker on its own thread; they meet at a barrier first so their calls overlap.  Returns their results."""
    barrier = threading.Barrier(len(workers))
    out = [None] * len(workers)
    errors = []

    def run(i, fn):
        try:
            barrier.wait(timeout)
            out[i] = fn(barrier)
        except BaseException as ex:  # noqa: BLE001
            errors.append(ex)

    threads = [threading.Thread(target=run, args=(i, fn)) for i, fn in enumerate(workers)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout)
    assert not any(t.is_alive() for t in threads), "a worker thread is still running"
    assert not errors, errors
    return out


def test_two_threads_each_get_their_own_cuda_error(L):
    nums = np.arange(1000, dtype=np.uint32)

    def worker(barrier):
        rc = _compress(L, nums, 1)
        barrier.wait(60)  # both calls have failed before either thread reads its message
        return rc, _message(L)

    for rc, msg in _run([worker, worker]):
        assert rc == CUDA
        assert msg.startswith("CUDA device unavailable ("), msg


def test_host_refusal_leaves_the_other_threads_message_alone(L):
    nums = np.arange(1000, dtype=np.uint32)

    def refused(barrier):
        rc = _compress(L, nums, 99)  # unknown dtype: refused on the host, before the device is looked at
        barrier.wait(60)
        return rc, _message(L)

    def no_device(barrier):
        rc = _compress(L, nums, 1)
        barrier.wait(60)
        return rc, _message(L)

    (rc_a, msg_a), (rc_b, msg_b) = _run([refused, no_device])
    assert rc_a == INVALID_TYPE and msg_a == "unknown number type byte: 99", msg_a
    assert rc_b == CUDA and msg_b.startswith("CUDA device unavailable ("), msg_b


def test_release_after_a_failed_set_up_is_harmless(L):
    nums = np.arange(1000, dtype=np.uint64)

    def worker(barrier):
        first = _compress(L, nums, 2), _message(L)
        L.pco_b200_thread_release()
        L.pco_b200_thread_release()
        second = _compress(L, nums, 2), _message(L)
        L.pco_b200_thread_release()
        return first, second

    for first, second in _run([worker, worker]):
        assert first[0] == second[0] == CUDA
        assert first[1] == second[1] and first[1].startswith("CUDA device unavailable ("), (first, second)
