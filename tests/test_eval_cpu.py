"""CPU: the mAP oracle (oracle/eval_np.py) reproduces what the reference's utils/common_utils.py computed for the inputs of
eval_np.eval_set (tests/golden/eval.npz, minted by tests/golden/make_golden_eval.py) exactly -- data points in push order, gt
counts, emptiness, every get_ap() and the calc_map rows -- and the package's common_utils imports and runs its host-only parts
without a GPU."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import eval_np as ev


def _oracle(seed, C, thr, dense=True):
    o = ev.EvalOracle(C, thr)
    for im in ev.eval_set(seed, num_classes=C):
        o.add_synth(im, dense=dense)
    return o


@pytest.mark.parametrize('seed', [1, 2, 3])
def test_oracle_equals_reference_golden(seed):
    g = load_golden('eval.npz')
    C, thr = int(g['num_classes']), [float(x) for x in g['iou_thres']]
    assert thr == [x / 100 for x in range(50, 100, 5)]
    o = _oracle(seed, C, thr)
    p = f'seed{seed}/'
    offs, k = g[p + 'point_offset'], 0
    for typ in range(2):
        for t in range(len(thr)):
            for c in range(C):
                pts = o.points[typ][t][c]
                lo, hi = offs[k], offs[k + 1]
                assert [s for s, _ in pts] == list(g[p + 'point_score'][lo:hi]), (typ, t, c)
                assert [bool(b) for _, b in pts] == list(g[p + 'point_tp'][lo:hi]), (typ, t, c)
                assert o.num_gt[typ, t, c] == g[p + 'num_gt'][typ, t, c]
                assert o.is_empty(typ, t, c) == g[p + 'is_empty'][typ, t, c]
                assert o.get_ap(typ, t, c) == g[p + 'ap'][typ, t, c], (typ, t, c)
                k += 1
    ap, nonempty = o.ap_array()
    box_row, mask_row = ev.map_rows(ap, nonempty, thr)
    assert box_row[1:] == list(g[p + 'box_row']) and mask_row[1:] == list(g[p + 'mask_row'])


def test_golden_cases_cover_the_contract():
    """The fixtures exercise what the contract singles out: TPs decided by the double threshold test, NaN IoUs, ties,
    a class with only detections and one with only gts, an image with no detections."""
    g = load_golden('eval.npz')
    C, thr = int(g['num_classes']), [float(x) for x in g['iou_thres']]
    ims = ev.eval_set(1, num_classes=C)
    assert any(len(im['ids']) == 0 for im in ims)
    im = ims[1]                                               # 480 x 640: gt * size is exact
    biou = ev.box_iou(im['boxes_px'], im['gt'], im['h'], im['w'])
    miou = ev.mask_iou_rects(im['det_rects'], im['gt_rects'])
    j = len(im['gt']) - 2                                     # the 20 x 15 px gt of class C-3
    assert biou[0, j] == np.float32(0.55) and float(biou[0, j]) > 0.55 and not biou[0, j] > np.float32(0.55)
    assert miou[0, j] == np.float32(0.6) and biou[1, j] == np.float32(0.8) and miou[1, j] == np.float32(0.55)
    assert np.isnan(biou[2, j + 1]) and np.isnan(miou[2, j + 1])
    dense = ev.mask_iou_dense(ev.rect_masks(im['det_rects'], im['h'], im['w']), ev.rect_masks(im['gt_rects'], im['h'], im['w']))
    assert np.array_equal(dense, miou, equal_nan=True)
    # the 0.55 box pair is a TP at threshold .55 only because the comparison is in double
    t55 = thr.index(0.55)
    assert g['seed1/num_gt'][0, t55, C - 3] > 0 and not g['seed1/is_empty'][0, 0, C - 1] and not g['seed1/is_empty'][0, 0, C - 2]
    assert g['seed1/ap'][0, 0, C - 1] == 0 and g['seed1/num_gt'][0, 0, C - 1] == 0
    scores = g['seed1/point_score']
    assert len(np.unique(scores)) < len(scores)


def test_common_utils_host_parts_without_gpu(tmp_path, monkeypatch):
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils import common_utils as cu
    g = load_golden('eval.npz')
    # MakeJson.add_bbox == the reference's records
    mj = cu.MakeJson()
    im = ev.eval_set(1, num_classes=int(g['num_classes']))[3]
    ids, scores = list(im['ids'].astype(int)), list(im['scores'].astype(float))
    for j in range(6):
        mj.add_bbox(1000 + j, ids[j] * 9 % 80, im['boxes_px'][j, :], scores[j])
    assert [r['image_id'] for r in mj.bbox_data] == list(g['json/image_id'])
    assert [r['category_id'] for r in mj.bbox_data] == list(g['json/category_id'])
    assert [r['bbox'] for r in mj.bbox_data] == g['json/bbox'].tolist()
    assert [r['score'] for r in mj.bbox_data] == list(g['json/score'])
    # unbound ap_data: empty objects, calc_map of nothing; push / add_gt_positives refuse
    thr = [x / 100 for x in range(50, 100, 5)]
    ap_data = {'box': [[cu.APDataObject() for _ in range(3)] for _ in thr], 'mask': [[cu.APDataObject() for _ in range(3)] for _ in thr]}
    table, box_row, mask_row = cu.calc_map(ap_data, thr, 3, step=12000)
    assert box_row == ['box'] + [0] * 11 and mask_row == ['mask'] + [0] * 11 and '12k' in table and '95' in table
    with pytest.raises(_lib.YolactB200Error):
        ap_data['box'][0][0].push(0.5, True)
    with pytest.raises(_lib.YolactB200Error):
        ap_data['box'][0][0].add_gt_positives(1)
    with pytest.raises(_lib.YolactB200Error):
        cu.MapEvaluator(80, [0.5] * 17)
    # ProgressBar, save_best / save_latest
    bar = cu.ProgressBar(10, 4)
    assert bar.get_bar(1) == '██' + '░' * 8 and bar.get_bar(9) == '█' * 10
    monkeypatch.chdir(tmp_path)
    (tmp_path / 'weights').mkdir()

    class Net:
        def state_dict(self):
            return {}
    cu.save_best(Net(), 30.5, 'res50_coco', 1000)
    cu.save_best(Net(), 29.0, 'res50_coco', 2000)              # worse: kept
    cu.save_best(Net(), 31.25, 'res50_coco', 3000)
    cu.save_latest(Net(), 'res50_coco', 10)
    cu.save_latest(Net(), 'res50_coco', 20)
    assert sorted(p.name for p in (tmp_path / 'weights').iterdir()) == ['best_31.25_res50_coco_3000.pth', 'latest_res50_coco_20.pth']
