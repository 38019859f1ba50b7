"""FluidSimulation.splats() on a stubbed library: how records are packed for fluid_splats, and which
inputs are refused before the library is called."""
import ctypes as C

import numpy as np
import pytest

import webgl_fluid_simulation_b200 as pkg
from webgl_fluid_simulation_b200.sim import FluidSimulation


class StubLib:
    """Records every fluid_* call; fluid_splats copies the block it is handed, as the library does."""

    def __init__(self):
        self.calls = []

    def fluid_splats(self, h, ptr, n):
        block = np.ctypeslib.as_array(ptr, shape=(n * 7,)).reshape(n, 7).copy() if n else np.zeros((0, 7), np.float32)
        self.calls.append(("fluid_splats", h, block, n))
        return 0

    def fluid_set_param_f64(self, h, key, value):
        self.calls.append(("fluid_set_param_f64", key, value))
        return 0

    def fluid_last_error(self, h):
        return b""


def bare():
    s = object.__new__(FluidSimulation)
    s.config = pkg.default_config()
    s.canvas = {"width": 800, "height": 600}
    s._L = StubLib()
    s._h = C.c_void_p(0x1234)
    s._pushed = {}
    return s


def splats_calls(s):
    return [c for c in s._L.calls if c[0] == "fluid_splats"]


def test_records_are_packed_in_order_as_c_contiguous_float32():
    s = bare()
    rng = np.random.default_rng(3)
    recs = rng.standard_normal((300, 7)).astype(np.float32)
    s.splats(recs[:, ::1])
    s.splats(np.asfortranarray(recs))                    # any memory layout: packed row by row
    s.splats(recs.tolist())                              # any array-like
    calls = splats_calls(s)
    assert len(calls) == 3
    for _, h, block, n in calls:
        assert h is s._h and n == 300
        assert block.dtype == np.float32 and np.array_equal(block.view(np.uint32), recs.view(np.uint32))


def test_config_is_pushed_before_the_call():
    s = bare()
    s.splats(np.zeros((2, 7)))
    names = [c[0] for c in s._L.calls]
    assert "fluid_set_param_f64" in names and names[-1] == "fluid_splats"
    assert names.index("fluid_set_param_f64") < names.index("fluid_splats")


def test_float64_narrows_exactly_as_c_float():
    s = bare()
    rng = np.random.default_rng(4)
    vals = np.concatenate([rng.standard_normal(60) * 10.0 ** rng.integers(-45, 39, 60),
                           [0.1, 1 / 3, -0.0, 1e-46, 3.4e38, 3.5e38, -1e39, np.inf, -np.inf, 1 + 2 ** -24, 1 + 3 * 2 ** -25]])
    vals = np.resize(vals, 77).reshape(11, 7)
    with np.errstate(over="ignore"):                     # 3.5e38 and -1e39 round to infinities, as in C
        s.splats(vals)
    block = splats_calls(s)[0][2]
    want = np.array([[C.c_float(float(v)).value for v in row] for row in vals], np.float32)
    assert np.array_equal(block.view(np.uint32), want.view(np.uint32))


def test_zero_records_still_calls_with_n_zero():
    s = bare()
    s.splats(np.zeros((0, 7)))
    assert [c[3] for c in splats_calls(s)] == [0]


@pytest.mark.parametrize("shape", [(5, 6), (5, 8), (7,), (0,), (2, 7, 1), (1, 1, 7), ()])
def test_bad_shapes_are_refused_before_any_library_call(shape):
    s = bare()
    with pytest.raises(ValueError):
        s.splats(np.zeros(shape))
    assert s._L.calls == []
