"""The numpy restatement of draw_lincomb (tests/lincomb_np.py) equals the unmodified reference's draw_lincomb bit for bit
(tests/golden/lincomb.npz, stored as colour-table indices) on every case without tied |coef|, and the colour table is what
cv2.applyColorMap does to uint8."""
import os

import numpy as np
import pytest

import lincomb_np as ln

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'lincomb.npz')


@pytest.mark.parametrize('name', ln.GOLDEN_CASES)
def test_oracle_equals_golden(name):
    proto, coef = ln.case_inputs(name)
    lut = ln.winter_lut()
    want = lut[np.load(GOLDEN)[name]]                     # the golden holds the colour-table index of every pixel
    got = ln.lincomb(proto, coef, lut)
    assert got.shape == want.shape and np.array_equal(got, want), np.argwhere(got != want)[:5]


def test_golden_covers_the_cases():
    g = np.load(GOLDEN)
    assert sorted(g.files) == sorted(ln.GOLDEN_CASES)
    assert {ln.CASES[n][0] for n in g.files} == {138, 136, 69, 16}
    assert any(ln.has_tie(ln.case_inputs(n)[1]) for n in ln.CASES) and not any(ln.has_tie(ln.case_inputs(n)[1]) for n in g.files)
    assert (ln.case_inputs('p69_neg')[1][0] < 0).all()


def test_tie_order_is_lower_channel_first():
    proto, coef = ln.case_inputs('p16_tie')
    order = np.argsort(-np.abs(coef[0]), kind='stable')
    assert order[:5].tolist() == [3, 9, 10, 20, 31]


def test_lut_is_apply_color_map():
    import cv2
    img = np.random.RandomState(0).randint(0, 256, size=(37, 53), dtype=np.uint8)
    assert np.array_equal(ln.winter_lut()[img], cv2.applyColorMap(img, cv2.COLORMAP_WINTER))
