"""fluid_resize (initFramebuffers on a live simulation, S:982-1010 + resizeDoubleFBO S:1116-1126) on fp32
and half-storage handles: a field whose size did not change is kept bit for bit, and a resize whose new
fields do not fit in device memory leaves the handle exactly as it was."""
import numpy as np
import pytest

from conftest import bits_equal
from sim_harness import make, special
from sim_harness import pkg  # noqa: F401 -- a fixture

pytestmark = pytest.mark.gpu
DT = 0.016666
FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
FLUID_ERR_NOMEM = -6


def resize(s, sizes):
    s._sizes = sizes
    s.initFramebuffers()
    assert s._dims("velocity")[:2] == sizes[:2] and s._dims("dye")[:2] == sizes[2:]


def assert_zero(s, names):
    for n in names:
        assert not s.readField(n).view(np.uint32).any(), n      # +0.0 in every cell


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "half"])
def test_resize_keeps_a_same_size_field_bit_for_bit(pkg, half):
    rng = np.random.default_rng(11)
    s = make(pkg, 36, 20, 54, 30, pkg.FLAG_HALF_STORAGE if half else 0)
    # a step first: pressure, divergence and curl hold values and the pairs have been swapped
    s.writeField("velocity", (rng.standard_normal((20, 36, 2)) * 50).astype(np.float32))
    s.writeField("dye", rng.random((30, 54, 4), dtype=np.float32))
    s.step(DT)
    assert s.readField("curl").any()

    # only the dye grid changes: velocity is kept as it is
    s.writeField("velocity", special((rng.standard_normal((20, 36, 2)) * 50).astype(np.float32), rng))
    v = s.readField("velocity")
    resize(s, (36, 20, 97, 31))
    assert bits_equal(s.readField("velocity"), v)
    assert_zero(s, ("pressure", "divergence", "curl"))

    # only the sim grid changes: dye is kept as it is
    s.step(DT)
    s.writeField("dye", special(rng.uniform(-1, 2, (31, 97, 4)).astype(np.float32), rng))
    d = s.readField("dye")
    resize(s, (23, 41, 97, 31))
    assert bits_equal(s.readField("dye"), d)
    assert_zero(s, ("pressure", "divergence", "curl"))
    s.close()


def test_resize_that_does_not_fit_changes_nothing(pkg):
    """An fp32 81920^2 dye buffer is 100 GiB, more than the whole card, so the new fields cannot be
    allocated.  The call fails with FLUID_ERR_NOMEM, every field reads back as before, and the handle
    goes on stepping and rendering exactly like a twin that never attempted the resize."""
    sizes = (64, 64, 128, 128)
    rng = np.random.default_rng(12)
    v = (rng.standard_normal((64, 64, 2)) * 50).astype(np.float32)
    d = rng.random((128, 128, 4), dtype=np.float32)
    s, twin = make(pkg, *sizes), make(pkg, *sizes)
    for x in (s, twin):
        x.writeField("velocity", v); x.writeField("dye", d)
        x.step(DT)
    before = {n: s.readField(n) for n in FIELDS}

    assert s._L.fluid_resize(s._h, 64, 64, 81920, 81920) == FLUID_ERR_NOMEM
    assert s._dims("velocity")[:2] == (64, 64) and s._dims("dye")[:2] == (128, 128)
    for n in FIELDS:
        assert bits_equal(s.readField(n), before[n]), n

    for x in (s, twin):
        x.splat(0.3, 0.6, 150.0, -80.0, (0.2, 0.5, 0.9))
        x.step(DT)
    for n in FIELDS:
        assert bits_equal(s.readField(n), twin.readField(n)), n
    assert bits_equal(s.render(96, 80), twin.render(96, 80))
    s.close(); twin.close()
