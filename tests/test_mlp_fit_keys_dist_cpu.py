"""ctr_mlp_fit_keys_dist without a GPU: its argument refusals come before it touches the model or the feature store (so
before any device or collective work), each with its own message through ctr_mlp_last_error(NULL), and both float64
wrappers carry fit_keys_dist.  The export list matching the header is test_abi_cpu.py's."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g

_lp = C.POINTER(C.c_int64)


def _call(L, m, h, arrays, n):
    u, i, t, y = arrays
    it = C.c_int32(-1); used = C.c_int64(-1)
    rc = L.ctr_mlp_fit_keys_dist(m, h, u, i, t, y, C.c_int64(n), C.byref(it), None, C.byref(used))
    return rc, L.ctr_mlp_last_error(None).decode(), it.value, used.value


@pytest.fixture(scope="module")
def L():
    return g.load_library()


def test_argument_refusals_come_first(L):
    keys = np.arange(4, dtype=np.int64)
    lab = np.ones(4, np.float32)
    kp, yp = keys.ctypes.data_as(_lp), lab.ctypes.data_as(C.POINTER(C.c_float))
    full = (kp, kp, kp, yp)
    bad = "bad fit_keys_dist arguments"
    for arrays, n in [((None, kp, kp, yp), 4), ((kp, None, kp, yp), 4), ((kp, kp, None, yp), 4), ((kp, kp, kp, None), 4),
                      (full, -1), (full, 2 ** 31), (full, 2 ** 40), ((None, None, None, None), 1)]:
        rc, msg, it, used = _call(L, None, None, arrays, n)
        assert rc == g.EINVAL and bad in msg, (n, msg)
        assert it == -1 and used == -1                                      # nothing written
    # good arguments (n = 0 with null arrays included): the null model or feature store is the refusal
    fake = C.c_void_p(8)                                                    # never dereferenced: the model is null
    for m, h, arrays, n in [(None, None, full, 4), (None, fake, full, 4), (None, None, (None,) * 4, 0)]:
        rc, msg, it, used = _call(L, m, h, arrays, n)
        assert rc == g.EINVAL and "null model or feature store" in msg, (m, h, n, msg)
        assert it == -1 and used == -1


def test_both_float64_wrappers_have_fit_keys_dist():
    for cls in (g.engine.MLPClassifier, g.engine.MLPRegressor):
        assert callable(getattr(cls, "fit_keys_dist", None)), cls
        assert cls.fit_keys_dist is g.engine._Mlp64.fit_keys_dist
    assert "ctr_mlp_fit_keys_dist" in g.EXPORTS
