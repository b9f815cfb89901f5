"""b2q_rpm_append_masked_cursor validates its arguments on the host, before any launch: null pointers, n < 1 and capacity < n are -1."""
import ctypes as C


def test_masked_append_rejects_bad_arguments_without_a_launch():
    from paddlerobotics_b200 import _lib
    lib = _lib.load()
    p = C.c_void_p(256)                     # never dereferenced: every call below is rejected first
    ring, rows = [p] * 5, [p] * 5
    call = lambda valid, n, cap, state: lib.b2q_rpm_append_masked_cursor(*ring, *rows, valid, n, 49, 12, cap, state, None)
    assert call(None, 4, 8, p) == -1
    assert call(p, 4, 8, None) == -1
    assert call(p, 0, 8, p) == -1
    assert call(p, 9, 8, p) == -1
    assert lib.b2q_rpm_append_masked_cursor(None, *ring[1:], *rows, p, 4, 49, 12, 8, p, None) == -1
    assert lib.b2q_rpm_append_masked_cursor(*ring, None, *rows[1:], p, 4, 49, 12, 8, p, None) == -1
