"""arena_model.py without a GPU: the layout against offsets worked out by hand, and the checker on numpy
arenas -- one flipped byte in padding, in a neighbouring slot's first row, in an input slot and in the flag
words is reported where it is; a change inside an allowed extent is not."""
import numpy as np
import pytest

import arena_model as A

MiB = 1 << 20
PAR0 = {"velocity": 0, "dye": 0, "pressure": 0}


def test_layout_4096_fp32():
    """Every extent a multiple of 2 MiB: no padding anywhere, slots back to back."""
    L = A.layout(4096, 4096, 4096, 4096)
    assert (L.v, L.dye, L.p) == ((0, 128 * MiB), (256 * MiB, 512 * MiB), (768 * MiB, 832 * MiB))
    assert (L.div, L.curl, L.flags, L.bytes) == (896 * MiB, 960 * MiB, 1024 * MiB, 1024 * MiB + 1024)
    assert [L.extent(f) for f in ("velocity", "dye", "pressure")] == [128 * MiB, 256 * MiB, 64 * MiB]


def test_layout_1024x512_has_no_padding():
    L = A.layout(1024, 512, 1024, 512)
    assert L.extent("pressure") == 2 * MiB and L.extent("velocity") == 4 * MiB and L.extent("dye") == 8 * MiB
    assert (L.v, L.dye, L.p, L.div, L.curl, L.flags) == ((0, 4 * MiB), (8 * MiB, 16 * MiB), (24 * MiB, 26 * MiB),
                                                        28 * MiB, 30 * MiB, 32 * MiB)
    for name, field, lo in L.slots():
        assert A.describe(L, lo + L.extent(field) - 1).startswith(name)      # last byte of a slot is its field


def test_layout_1000x524_less_than_a_row_of_padding():
    """2,096,000 bytes of pressure in a 2 MiB slot: 1152 bytes of padding, less than one 4000-byte row."""
    L = A.layout(1000, 524, 1000, 524)
    assert L.extent("pressure") == 2_096_000 and L.p[1] - L.p[0] - L.extent("pressure") == 1152
    assert L.v[1] - L.extent("velocity") == 2304 and L.dye[1] - L.dye[0] - L.extent("dye") == 4608
    assert (L.v, L.dye, L.p, L.div, L.curl, L.flags) == ((0, 4 * MiB), (8 * MiB, 16 * MiB), (24 * MiB, 26 * MiB),
                                                        28 * MiB, 30 * MiB, 32 * MiB)
    assert A.describe(L, L.p[0] + L.extent("pressure")) == "padding of pressure[0] +0"
    assert A.describe(L, L.p[1]) == "pressure[1] row 0 column 0 byte 0"


def test_layout_half_storage():
    """fp16: 4 / 8 / 2 bytes per cell.  100 x 60 / 150 x 90: every field fits one 2 MiB slot; 1024^2 pressure
    fills its slot exactly."""
    L = A.layout(100, 60, 150, 90, half=True)
    assert (L.extent("velocity"), L.extent("dye"), L.extent("pressure")) == (24000, 108000, 12000)
    assert (L.v, L.dye, L.p, L.div, L.curl, L.flags, L.bytes) == (
        (0, 2 * MiB), (4 * MiB, 6 * MiB), (8 * MiB, 10 * MiB), 12 * MiB, 14 * MiB, 16 * MiB, 16 * MiB + 1024)
    L = A.layout(1024, 1024, 1024, 1024, half=True)
    assert L.extent("pressure") == 2 * MiB and (L.p[0], L.div, L.flags) == (24 * MiB, 28 * MiB, 32 * MiB)
    assert A.describe(L, L.v[0] + 3 * 4096 + 4 * 5 + 2) == "velocity[0] row 3 column 5 byte 2"


def test_may_change_follows_the_parity():
    L = A.layout(1000, 524, 1000, 524)
    ext = L.extent("velocity")
    assert A.may_change("vorticity", L, PAR0) == [(L.v[1], L.v[1] + ext)]
    assert A.may_change("vorticity", L, dict(PAR0, velocity=1)) == [(L.v[0], L.v[0] + ext)]
    assert A.may_change("write", L, dict(PAR0, dye=1), field="dye") == [(L.dye[1], L.dye[1] + L.extent("dye"))]
    assert A.may_change("write", L, PAR0, field="curl") == [(L.curl, L.curl + L.extent("curl"))]
    assert A.may_change("render", L, PAR0) == []


def flipped(a, off):
    b = a.copy()
    b[off] ^= 0x40
    return b


@pytest.mark.parametrize("W,H,Wd,Hd", [(1000, 524, 1000, 524), (1024, 512, 1024, 512)])
def test_checker_reports_a_flipped_byte_where_it_is(W, H, Wd, Hd):
    L = A.layout(W, H, Wd, Hd)
    rng = np.random.default_rng(W)
    a = rng.integers(0, 256, L.bytes, dtype=np.uint8)
    allowed = A.may_change("gradient_subtract", L, PAR0)           # velocity[1]
    cases = [(L.p[1], "pressure[1] row 0 column 0 byte 0"),      # the neighbour's first row (past pressure[0])
             (L.v[0] + 8 * W + 8 * 7 + 3, "velocity[0] row 1 column 7 byte 3"),    # an input slot
             (L.flags + 5, "flag words +5"),
             (L.div + L.extent("divergence") - 2, f"divergence row {H - 1} column {W - 1} byte 2")]
    if L.p[1] - L.p[0] > L.extent("pressure"):
        cases.append((L.p[0] + L.extent("pressure") + 17, "padding of pressure[0] +17"))
    else:                                                           # no padding: the byte past velocity[1] is dye[0]'s
        cases.append((L.v[1] + L.extent("velocity"), "dye[0] row 0 column 0 byte 0"))
    for off, where in cases:
        n, rep = A.changes_outside(a, flipped(a, off), allowed, L)
        assert n == 1 and rep == [f"{off}: {where}"], (off, rep)


def test_checker_accepts_changes_inside_an_allowed_extent():
    L = A.layout(1000, 524, 1000, 524)
    a = np.zeros(L.bytes, np.uint8)
    b = a.copy()
    lo, hi = A.may_change("curl_vorticity_divergence", L, PAR0)[0]
    b[lo] = b[hi - 1] = 1
    b[L.curl:L.curl + L.extent("curl")] = 7
    assert A.changes_outside(a, b, A.may_change("curl_vorticity_divergence", L, PAR0), L) == (0, [])
    b[hi] = 1                                                     # one byte past velocity[1]: its padding
    assert A.changes_outside(a, b, A.may_change("curl_vorticity_divergence", L, PAR0), L) == (
        1, [f"{hi}: padding of velocity[1] +0"])


def test_fresh_arena_image():
    """make_arena's image: zeros, dye alpha 1.0 in both dye slots, padding zero."""
    L = A.layout(36, 20, 54, 30)
    a = A.fresh(L)
    for k in (0, 1):
        d = a[L.dye[k]:L.dye[k] + L.extent("dye")].view(np.float32).reshape(30, 54, 4)
        assert np.all(d[..., 3] == 1) and not d[..., :3].any()
    mask = np.ones(L.bytes, bool)
    for k in (0, 1):
        mask[L.dye[k]:L.dye[k] + L.extent("dye")] = False
    assert not a[mask].any()
