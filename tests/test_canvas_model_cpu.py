"""The canvas rule of fluid_render_canvas (tests/canvas_model.py) on hand cases, and inputs on which every
wrong rule the model knows changes at least one byte."""
import numpy as np
import pytest

import canvas_model as CM

F = np.float32
BACK_RGB = (10 / 255, 20 / 255, 30 / 255)
BLACK = (0.0, 0.0, 0.0)


def one(texel):
    """A 1 x 1 fragment."""
    return np.asarray(texel, F).reshape(1, 1, 4)


def test_checkerboard_bytes_are_derived_in_fp32():
    """The dark square 0.8 stores 204; the light one is 1 * 0.1f + 0.8f = 0.90000004f, times 255 = 229.50002f,
    which rounds to 230."""
    v = np.unique(CM.checkerboard(64, 48, 64 / 48))
    assert v.tolist() == [F(0.8), F(F(1) * F(0.1)) + F(0.8)]
    assert v[1] == F(0.90000004) and v[1] * F(255) == F(229.50002)
    d8 = CM.destination_bytes(64, 48, BLACK, True, 64 / 48)
    assert np.unique(d8).tolist() == [204, 230]


def test_checkerboard_matches_the_display_model():
    """The fp32 checkerboard is the one render() draws (display_model.background_colour)."""
    import display_model as M
    from oracle import oracle as O
    for w, h in ((128, 128), (807, 640), (64, 48)):
        ours = CM.background(w, h, BLACK, True, w / h)
        theirs = M.background_colour(w, h, BLACK, O.BG_CHECKERBOARD, w / h)
        assert np.array_equal(ours.view(np.uint32), np.ascontiguousarray(theirs, F).view(np.uint32))


def test_clamp_before_blending_on_the_dark_square():
    """c.r = 1.2, a = 1.5 over the dark square: the fp32 frame gives 1.2 + 0.8 * (1 - 1.5) = 0.8, byte 204; the
    canvas clamps first: 1 + 0.8 * 0 = 1, byte 255."""
    frag = one([1.2, 0.0, 1.5, 1.5])
    assert CM.destination_bytes(1, 1, BLACK, True, 1.0)[0, 0, 0] == 204
    got = CM.canvas(frag, BLACK, True, 1.0)
    assert got[0, 0].tolist() == [255, 0, 255, 255]
    assert CM.canvas(frag, BLACK, True, 1.0, mutant="no_clamp")[0, 0, 0] == 204


@pytest.mark.parametrize("transparent,back", [(False, BACK_RGB), (False, BLACK), (True, BLACK)])
def test_alpha_above_one_hides_every_background(transparent, back):
    """Any clamp(a) = 1 leaves nothing of the destination: the bytes are u8(c), alpha 255."""
    rng = np.random.default_rng(3)
    frag = rng.random((6, 5, 4), dtype=F) * F(0.9)
    frag[..., 3] = F(1) + rng.random((6, 5), dtype=F) * F(9)
    got = CM.canvas(frag, back, transparent, 5 / 6)
    assert np.array_equal(got, np.concatenate([CM.u8(frag[..., :3]), np.full((6, 5, 1), 255, np.uint8)], -1)[::-1])


def test_non_finite_fragments():
    """NaN clamps to 0 and +inf to 1, in the colour and in alpha; -inf to 0."""
    back = BACK_RGB
    d8 = CM.destination_bytes(1, 1, back, False, 1.0)[0, 0]
    nan, inf = np.nan, np.inf
    assert CM.canvas(one([nan, nan, nan, nan]), back, False, 1.0)[0, 0].tolist() == d8.tolist() + [255]
    assert CM.canvas(one([inf, 0, 0, inf]), back, False, 1.0)[0, 0].tolist() == [255, 0, 0, 255]
    assert CM.canvas(one([-inf, nan, 1.0, 1.0]), back, False, 1.0)[0, 0].tolist() == [0, 0, 255, 255]
    half = CM.canvas(one([-inf, 0.25, 0.5, 0.5]), back, False, 1.0)[0, 0]
    d = d8.astype(F) / F(255)
    assert half.tolist() == [CM.u8(F(0) + d[0] * F(0.5)), CM.u8(F(0.25) + d[1] * F(0.5)),
                             CM.u8(F(0.5) + d[2] * F(0.5)), 255]


def exact_ties():
    """fp32 x in [0, 1] whose product x * 255 is exactly m + 0.5."""
    out = []
    for m in range(255):
        x = F((m + 0.5) / 255)
        for _ in range(4):
            x = np.nextafter(x, F(0))
        for _ in range(9):
            if x * F(255) == F(m + 0.5):
                out.append((x, m))
            x = np.nextafter(x, F(1))
    return out


def test_exact_ties_round_to_even():
    """clamp(x) * 255 = m + 0.5 exactly stores the even one of m, m + 1."""
    ties = exact_ties()
    assert len(ties) > 20
    for x, m in ties:
        want = m if m % 2 == 0 else m + 1
        assert CM.u8(x) == want, (x, m)
        got = CM.canvas(one([x, 0, 1, 1]), BACK_RGB, False, 1.0)[0, 0, 0]    # clamp(a) = 1: out = c
        assert got == want
        assert CM.canvas(one([x, 0, 1, 1]), BACK_RGB, False, 1.0, mutant="truncate")[0, 0, 0] == m


def test_rows_are_stored_top_first():
    frag = np.zeros((3, 2, 4), F)
    frag[0] = [1, 0, 0, 1]                                       # the bottom row is red
    got = CM.canvas(frag, BLACK, False, 1.0)
    assert got[2, 0].tolist() == [255, 0, 0, 255] and got[0, 0].tolist() == [0, 0, 0, 255]


def discriminating_fragment(back, transparent, seed=5):
    """A fragment holding the hand cases, seeded values up to 10 (alpha > 1 too), non-finite texels and
    and along its top row fused-rule witnesses for each texel's destination."""
    rng = np.random.default_rng(seed)
    h, w = 16, 24
    frag = rng.random((h, w, 4), dtype=F) ** 2
    frag[: h // 2] *= F(10)
    frag[..., 3] = np.fmax(frag[..., 0], np.fmax(frag[..., 1], frag[..., 2]))
    frag[0, 0] = [1.2, 0.0, 1.5, 1.5]
    frag[0, 1] = [np.nan, 0.2, np.inf, np.inf]
    frag[0, 2] = [-np.inf, 0.3, 0.4, 0.4]
    d8 = CM.destination_bytes(w, h, back, transparent, w / h)
    row = h - 1                                                  # witnesses per destination value of the row
    for i in range(w):
        r, g, a = CM.fused_witnesses(F(d8[row, i, 0]) / F(255), 1, rng)[0]
        frag[row, i] = [r, g, a, a]
    return frag


def test_integer_back_colours_are_their_own_bytes():
    """BACK_COLOR / 255 of an integer colour stores that integer, so an unquantised destination shows only
    over the checkerboard or a fractional colour."""
    k = np.arange(256)
    assert np.array_equal(CM.u8(np.asarray(k / 255, F)), k)


@pytest.mark.parametrize("transparent,back", [(False, (0.3, 0.55, 0.7)), (True, BLACK), (True, BACK_RGB)])
def test_every_wrong_rule_changes_a_byte(transparent, back):
    """On these inputs each mutant differs from the rule somewhere: no clamp before blending, truncation,
    an unquantised destination, a fused d * (1 - a) + c, bottom row first."""
    frag = discriminating_fragment(back, transparent)
    want = CM.canvas(frag, back, transparent, frag.shape[1] / frag.shape[0])
    for m in CM.MUTANTS:
        got = CM.canvas(frag, back, transparent, frag.shape[1] / frag.shape[0], mutant=m)
        assert np.count_nonzero(got != want) > 0, m


def test_fused_witnesses_are_half_representable_and_discriminate():
    rng = np.random.default_rng(1)
    for d8 in (10, 20, 30, 204, 230):
        d = F(d8) / F(255)
        wit = CM.fused_witnesses(d, 4, rng)
        assert np.array_equal(wit.astype(np.float16).astype(F), wit)
        for r, _, a in wit:
            k = F(1) - a
            assert r <= a and CM.u8(r + d * k) != CM.u8(F(np.float64(d) * np.float64(k) + np.float64(r)))
