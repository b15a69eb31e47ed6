"""CPU: the numpy restatement of draw_img (oracle/draw_np.py) equals the reference's draw_img (tests/golden/draw.npz) exactly:
the returned image, total_obj and every crop handed to cv2.imwrite, and their file names; plus the blend formula against
cv2.addWeighted for every (colour, pixel) pair."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import draw_np as dn

cv2 = pytest.importorskip('cv2')

CASES = dn.golden_cases()


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_oracle_equals_reference_golden(case):
    from yolact_minimal_b200.config import COLORS
    g = load_golden('draw.npz')
    ids, scores, boxes, masks, img, cfg, name, fps = dn.case_inputs(case)
    src = img.copy()
    out, writes = dn.draw(ids, scores, boxes, masks, src, cfg, COLORS, img_name=name, fps=fps)
    want = g[f'{name}/image']
    assert out.dtype == np.uint8 and out.shape == want.shape and np.array_equal(out, want)
    if cfg.hide_mask and not cfg.real_time or ids is None:
        assert out is src
    paths = list(g[f'{name}/paths']) if f'{name}/paths' in g.files else []
    assert [p for p, _ in writes] == paths
    for k, (_, a) in enumerate(writes):
        w = g[f'{name}/write{k}']
        assert a.shape == w.shape and np.array_equal(a, w), (name, k)


def test_golden_cases_cover_the_quirks():
    g = load_golden('draw.npz')
    sizes = {dn.SIZES[c[2]] for c in CASES}
    assert sizes == {(96, 128), (128, 96), (37, 70)}
    assert {c[4] for c in CASES} == {81, 21}
    many = dn.case_inputs([c for c in CASES if c[0] == 's1_many_cutout'][0])
    ids, boxes, masks = many[0], many[2], many[3]
    assert (ids == 79).sum() >= 2 and len(set(ids.tolist())) < len(ids)
    assert (boxes[:, 2] > 96).any() and (masks != 0).sum(0).max() > 10
    assert sum(g[k].nbytes for k in g.files) < 4 << 20


def test_blend_equals_cv2_add_weighted_for_all_pairs():
    c, p = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing='ij')
    assert np.array_equal(dn.blend(c, p), cv2.addWeighted(c, 0.4, p, 0.6, 0))
