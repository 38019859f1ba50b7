"""FluidBatch's push rule for per-member values, against a stand-in library that records the calls: a key whose
values agree across members goes through fluid_set_param_f64 as on a FluidSimulation, other keys through
fluid_set_param_members, and only when a key's values changed since the last push."""
import ctypes as C

import numpy as np
import pytest

from webgl_fluid_simulation_b200 import sim
from webgl_fluid_simulation_b200._lib import PARAM

NAME = {v: k for k, v in PARAM.items()}


class Recorder:
    def __init__(self, members):
        self.B = members
        self.calls = []

    def fluid_members(self, h):
        return self.B

    def fluid_set_param_f64(self, h, key, v):
        self.calls.append(("f64", NAME[key], v))
        return 0

    def fluid_set_param_members(self, h, key, values, n):
        self.calls.append(("members", NAME[key], np.ctypeslib.as_array(values, (n,)).tolist()))
        return 0

    def fluid_step(self, h, dt):
        self.calls.append(("step", dt))
        return 0

    def fluid_step_members(self, h, dt, n):
        self.calls.append(("step_members", np.ctypeslib.as_array(dt, (n,)).tolist()))
        return 0

    def fluid_last_error(self, h):
        return b""

    def take(self):
        c, self.calls = self.calls, []
        return c


def stand_in(B):
    b = object.__new__(sim.FluidBatch)
    b.config = sim.default_config()
    b.canvas = {"width": 256, "height": 128}
    b._L = Recorder(B)
    b._h = C.c_void_p(1)
    b._pushed = {}
    b.member_config = [{} for _ in range(B)]
    b._push_config()
    return b


def test_first_push_is_a_fluid_simulation_push():
    b = stand_in(3)
    calls = b._L.take()
    assert all(c[0] == "f64" for c in calls)
    assert {c[1] for c in calls} == {"DENSITY_DISSIPATION", "VELOCITY_DISSIPATION", "PRESSURE", "PRESSURE_ITERATIONS",
                                     "CURL", "SPLAT_RADIUS", "ASPECT"}
    b._push_config()
    assert b._L.take() == []


def test_overrides_push_members_and_removal_pushes_the_shared_value():
    b = stand_in(3)
    b._L.take()
    b.member_config[1]["CURL"] = 5.0
    b.step(0.016)
    assert b._L.take() == [("members", "CURL", [30.0, 5.0, 30.0]), ("step", pytest.approx(0.016))]
    b.step(0.016)
    assert b._L.take() == [("step", pytest.approx(0.016))]             # unchanged: nothing pushed
    b.config["CURL"] = 10.0                                              # the shared value moves the other members
    b.step(0.016)
    assert b._L.take()[0] == ("members", "CURL", [10.0, 5.0, 10.0])
    del b.member_config[1]["CURL"]
    b.step(0.016)
    assert b._L.take()[0] == ("f64", "CURL", 10.0)
    for m in range(3):                                                   # overrides that agree: one f64 push
        b.member_config[m]["PRESSURE"] = 0.5
    b._push_config()
    assert b._L.take() == [("f64", "PRESSURE", 0.5)]
    b.member_config[2]["PRESSURE"] = -0.0
    b.member_config[1]["PRESSURE"] = -0.0
    b.member_config[0]["PRESSURE"] = 0.0                                 # -0.0 and 0.0 are different values
    b._push_config()
    assert b._L.take() == [("members", "PRESSURE", [0.0, -0.0, -0.0])]


def test_step_takes_one_dt_or_one_per_member():
    b = stand_in(2)
    b._L.take()
    b.step([0.1, 1 / 60])
    assert b._L.take() == [("step_members", [np.float32(0.1), np.float32(1 / 60)])]
    b.step(np.array([0.0, 0.5], np.float64))
    assert b._L.take() == [("step_members", [0.0, 0.5])]
    for bad in ([0.1], [0.1, 0.2, 0.3], [[0.1, 0.2]], []):
        with pytest.raises(ValueError):
            b.step(bad)
    assert b._L.take() == []


def test_misuse_raises():
    b = stand_in(2)
    b.member_config[0]["PRESSURE_ITERATIONS"] = 5
    with pytest.raises(ValueError):
        b._push_config()
    b.member_config[0].clear()
    b.member_config = [{}]
    with pytest.raises(ValueError):
        b.step(0.016)
