"""splats() with CUDA arrays, against a stand-in library that records the calls: CUDA arrays reach
fluid_splats_device / fluid_splats_batch_device with their pointers and n, then fluid_sync; numpy arrays take the
host entry points as before; mixed, mistyped and misshapen inputs raise ValueError before any call.  The arrays
are stand-ins with a version-3 __cuda_array_interface__ whose "stream" is None, so no driver call is made."""
import ctypes as C

import numpy as np
import pytest

from webgl_fluid_simulation_b200 import sim


class Recorder:
    def __init__(self, members=1):
        self.B = members
        self.calls = []

    def fluid_members(self, h):
        return self.B

    def fluid_set_param(self, h, key, v):
        return 0

    def fluid_set_param_f64(self, h, key, v):
        return 0

    def fluid_splats(self, h, recs, n):
        self.calls.append(("splats", np.ctypeslib.as_array(recs, (n, 7)).copy(), n))
        return 0

    def fluid_splats_batch(self, h, members, recs, n):
        self.calls.append(("splats_batch", np.ctypeslib.as_array(members, (n,)).copy(),
                           np.ctypeslib.as_array(recs, (n, 7)).copy(), n))
        return 0

    def fluid_splats_device(self, h, recs, n):
        self.calls.append(("splats_device", recs.value, n))
        return 0

    def fluid_splats_batch_device(self, h, members, recs, n):
        self.calls.append(("splats_batch_device", members.value, recs.value, n))
        return 0

    def fluid_sync(self, h):
        self.calls.append(("sync",))
        return 0

    def fluid_last_error(self, h):
        return b""

    def take(self):
        c, self.calls = self.calls, []
        return c


class CudaArray:
    """What a producer with nothing pending would hand over: a version-3 interface, "stream": None."""

    def __init__(self, ptr, shape, typestr, strides=None):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False),
                                         "strides": strides, "version": 3, "stream": None}


def sim_stand_in():
    s = object.__new__(sim.FluidSimulation)
    s.config = sim.default_config()
    s.canvas = {"width": 256, "height": 256}
    s._L = Recorder()
    s._h = C.c_void_p(1)
    s._pushed = {}
    s._push_config()
    s._L.take()
    return s


def batch_stand_in(B):
    b = object.__new__(sim.FluidBatch)
    b.config = sim.default_config()
    b.canvas = {"width": 256, "height": 256}
    b._L = Recorder(B)
    b._h = C.c_void_p(1)
    b._pushed = {}
    b.member_config = [{} for _ in range(B)]
    b._push_config()
    b._L.take()
    return b


@pytest.mark.parametrize("n", [0, 1, 300])
def test_simulation_cuda_records_reach_the_device_call(n):
    s = sim_stand_in()
    s.splats(CudaArray(0x7000_0000, (n, 7), "<f4"))
    assert s._L.take() == [("splats_device", 0x7000_0000, n), ("sync",)]


def test_simulation_numpy_records_take_the_host_call():
    s = sim_stand_in()
    recs = np.arange(21, dtype=np.float64).reshape(3, 7)
    s.splats(recs)
    (name, got, n), = s._L.take()
    assert (name, n) == ("splats", 3)
    assert np.array_equal(got, recs.astype(np.float32))


@pytest.mark.parametrize("n", [0, 1, 5000])
def test_batch_cuda_arrays_reach_the_device_call(n):
    b = batch_stand_in(4)
    b.splats(CudaArray(0x5000_0000, (n,), "<i4"), CudaArray(0x6000_0000, (n, 7), "<f4"))
    assert b._L.take() == [("splats_batch_device", 0x5000_0000, 0x6000_0000, n), ("sync",)]


def test_batch_numpy_arrays_take_the_host_call():
    b = batch_stand_in(4)
    members, recs = np.array([3, 0, 3]), np.ones((3, 7))
    b.splats(members, recs)
    (name, m, r, n), = b._L.take()
    assert (name, n) == ("splats_batch", 3)
    assert m.tolist() == [3, 0, 3] and np.array_equal(r, np.ones((3, 7), np.float32))


def test_batch_mixed_host_and_device_is_refused():
    b = batch_stand_in(4)
    with pytest.raises(ValueError):
        b.splats(np.zeros(2, np.int32), CudaArray(0x6000_0000, (2, 7), "<f4"))
    with pytest.raises(ValueError):
        b.splats(CudaArray(0x5000_0000, (2,), "<i4"), np.zeros((2, 7), np.float32))
    assert b._L.take() == []


@pytest.mark.parametrize("shape,typestr,strides", [
    ((4, 7), "<f8", None),             # float64
    ((4, 6), "<f4", None),             # not 7 floats a record
    ((28,), "<f4", None),              # flat
    ((4, 7), "<f4", (56, 4)),          # rows not adjacent
    ((4, 7), "<f4", (4, 16)),          # column-major
])
def test_bad_record_arrays_are_refused(shape, typestr, strides):
    s = sim_stand_in()
    with pytest.raises(ValueError):
        s.splats(CudaArray(0x7000_0000, shape, typestr, strides))
    b = batch_stand_in(4)
    with pytest.raises(ValueError):
        b.splats(CudaArray(0x5000_0000, (shape[0],), "<i4"), CudaArray(0x6000_0000, shape, typestr, strides))
    assert s._L.take() == [] and b._L.take() == []


@pytest.mark.parametrize("shape,typestr", [((4,), "<i8"), ((4,), "<f4"), ((3,), "<i4"), ((5,), "<i4")])
def test_bad_member_arrays_are_refused(shape, typestr):
    b = batch_stand_in(4)
    with pytest.raises(ValueError):
        b.splats(CudaArray(0x5000_0000, shape, typestr), CudaArray(0x6000_0000, (4, 7), "<f4"))
    assert b._L.take() == []
