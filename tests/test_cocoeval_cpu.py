"""CPU: COCO's own mAP (oracle/cocoeval_np.py, the restatement the GPU path is checked against) on cases whose answers are derived
by hand from COCOeval's rules; CocoEvaluator's host tables; COCOeval.summarize's stats and lines; COCOValDetection(coco_eval=True)
and its PackedValBatch fields; and, where pycocotools is importable, the oracle against COCOeval itself."""
import pickle
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import cocoeval_np as ce
from yolact_minimal_b200.config import COCO_LABEL_MAP
from yolact_minimal_b200.utils import cocoeval as cev

P1 = 1 / (1 + np.spacing(1))          # one true positive: tp / (fp + tp + eps) with fp + tp = 1, 0.9999999999999998


def gt(img, box, k=0, crowd=0, area=None):
    x, y, w, h = box
    return {'image_id': img, 'category': k, 'bbox': [float(v) for v in box], 'area': float(w * h if area is None else area),
            'iscrowd': crowd, 'rect': (x, y, x + w, y + h)}


def dt(img, box, score, k=0):
    x, y, w, h = box
    return {'image_id': img, 'category': k, 'bbox': [float(v) for v in box], 'score': float(np.float32(score)), 'rect': (x, y, x + w, y + h)}


def both(gts, dts, imgs=(1,), K=1):
    return [ce.evaluate(gts, dts, list(imgs), K, t) for t in ('bbox', 'segm')]


def test_thresholds_are_linspace():
    assert np.array_equal(cev.IOU_THRS, ce.IOU_THRS) and np.array_equal(cev.REC_THRS, ce.REC_THRS)
    assert cev.REC_THRS[35] != 0.35 and cev.IOU_THRS[8] == 0.8999999999999999 and cev.IOU_THRS[5] == 0.75
    assert cev.MAX_DETS == ce.MAX_DETS and cev.AREA_RNG == ce.AREA_RNG


def test_one_exact_detection():
    for prec, rec in both([gt(1, (10, 10, 10, 10))], [dt(1, (10, 10, 10, 10), .9)]):
        assert (prec[:, :, 0, :2] == P1).all() and (prec[:, :, 0, 2:] == -1).all()
        assert (rec[:, 0, :2] == 1).all() and (rec[:, 0, 2:] == -1).all()
        s, _ = cev.summarize(prec, rec)
        # AP, AP50, AP75, APs: the mean of 0.9999999999999998s (printed 1.000); AR1/10/100, ARs: exactly 1; medium / large: -1
        assert np.allclose(s[[0, 1, 2, 3]], 1, rtol=0, atol=1e-15) and (s[[6, 7, 8, 9]] == 1).all()
        assert (s[[4, 5, 10, 11]] == -1).all()


def test_false_positive_first():
    gts, dts = [gt(1, (10, 10, 10, 10))], [dt(1, (50, 50, 10, 10), .9), dt(1, (10, 10, 10, 10), .8)]
    for prec, rec in both(gts, dts):
        assert (prec[:, :, 0, :2, 1:] == 0.5).all()              # 1 / (2 + eps): 2 + eps rounds to 2
        assert (prec[:, :, 0, :2, 0] == 0).all()                 # maxDets 1: the false positive alone
        s, _ = cev.summarize(prec, rec)
        assert s[0] == 0.5 and s[6] == 0 and s[7] == 1
    # a crowd gt containing the 0.9 detection: that detection matches it and is ignored
    for prec, rec in both(gts + [gt(1, (45, 45, 20, 20), crowd=1)], dts):
        assert (prec[:, :, 0, 0, 1:] == P1).all()
        assert np.allclose(cev.summarize(prec, rec)[0][0], 1, rtol=0, atol=1e-15)


def test_area_exactly_1024_is_small_and_medium():
    for prec, rec in both([gt(1, (0, 0, 32, 32))], [dt(1, (0, 0, 32, 32), .9)]):
        assert (rec[:, 0, :3] == 1).all() and (rec[:, 0, 3] == -1).all()
        assert (prec[:, :, 0, :3] == P1).all()


def test_unmatched_detection_outside_the_range_is_ignored():
    gts = [gt(1, (10, 10, 10, 10))]
    dts = [dt(1, (100, 100, 50, 50), .9), dt(1, (10, 10, 10, 10), .8)]      # the 0.9 one: area 2500, medium
    for prec, _ in both(gts, dts):
        assert (prec[:, :, 0, 0, 1:] == 0.5).all()               # all: a false positive first
        assert (prec[:, :, 0, 1, 1:] == P1).all()                # small: ignored


def test_equal_ious_go_to_the_later_gt():
    # det 1 has IoU .5 with both gts; taking the later one leaves the earlier one to det 2 (IoU 1), so both match at .5
    gts = [gt(1, (10, 10, 10, 20)), gt(1, (10, 10, 20, 10))]
    dts = [dt(1, (10, 10, 10, 10), .9), dt(1, (10, 10, 10, 20), .8)]
    prec, rec = ce.evaluate(gts, dts, [1], 1, 'bbox')
    assert rec[0, 0, 0, 2] == 1 and rec[1, 0, 0, 2] == 0.5


def test_break_prefers_a_non_ignored_gt():
    # the crowd gt comes first in the file and has IoU 1 (crowd: / the detection's area); the plain gt has IoU 100/120
    gts = [gt(1, (10, 10, 10, 12), crowd=1), gt(1, (10, 10, 10, 10))]
    prec, rec = ce.evaluate(gts, [dt(1, (10, 10, 10, 12), .9)], [1], 1, 'bbox')
    assert (rec[:7, 0, 0, 2] == 1).all() and (rec[7:, 0, 0, 2] == 0).all()    # 100/120 = .833 passes .5 ... .8


def test_more_than_100_detections_of_a_class():
    dts = [dt(1, (200 + 3 * i, 0, 2, 2), 1 - i / 1000) for i in range(150)]
    dts[120] = dt(1, (10, 10, 10, 10), 1 - 120 / 1000)           # the only match is ranked 120: dropped
    dts[50] = dt(1, (40, 40, 10, 10), 1 - 50 / 1000)
    gts = [gt(1, (10, 10, 10, 10)), gt(1, (40, 40, 10, 10))]
    for prec, rec in both(gts, dts):
        assert (rec[:, 0, 0, 2] == 0.5).all() and (rec[:, 0, 0, 1] == 0).all()
        assert (prec[:, 0, 0, 0, 2] == 1 / 51).all()             # the 51st of the 100 kept detections


def test_equal_scores_follow_image_id():
    gts = [gt(1, (10, 10, 10, 10))]
    dts = [dt(2, (10, 10, 10, 10), .5), dt(1, (10, 10, 10, 10), .5)]    # image 2 produced first
    for prec, _ in both(gts, dts, imgs=(2, 1)):
        assert (prec[:, :, 0, 0] == P1).all()                    # image 1's true positive comes first


def test_npig_counts_images_never_added():
    gts = [gt(1, (10, 10, 10, 10)), gt(3, (10, 10, 10, 10))]
    for prec, rec in both(gts, [dt(1, (10, 10, 10, 10), .9)], imgs=(1, 3)):
        assert (rec[:, 0, 0, 2] == 0.5).all()
        assert (prec[:, :51, 0, 0, 2] == P1).all() and (prec[:, 51:, 0, 0, 2] == 0).all()


def test_iou_of_exactly_point_nine():
    prec, rec = ce.evaluate([gt(1, (0, 0, 10, 10))], [dt(1, (0, 0, 10, 9), .9)], [1], 1, 'bbox')
    assert 90 / 100 == 0.9 and rec[8, 0, 0, 2] == 1 and rec[9, 0, 0, 2] == 0


def test_recall_on_the_rec_thr_boundary():
    # 7 of 20 gts found: recall 7/20 = 0.35 < recThrs[35] = 0.35000000000000003, so sample 35 lies past the last detection
    gts = [gt(1, (40 * i, 0, 10, 10)) for i in range(20)]
    dts = [dt(1, (40 * i, 0, 10, 10), .9 - i / 100) for i in range(7)]
    for prec, rec in both(gts, dts):
        assert (rec[:, 0, 0, 2] == 0.35).all()
        assert (prec[:, 1:35, 0, 0, 2] == 1).all() and (prec[:, 35:, 0, 0, 2] == 0).all() and (prec[:, 0, 0, 0, 2] == 1).all()


def test_summarize_lines():
    prec, rec = ce.evaluate([gt(1, (10, 10, 10, 10))], [dt(1, (10, 10, 10, 10), .9)], [1], 1, 'bbox')
    _, lines = cev.summarize(prec, rec)
    assert lines == [
        ' Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets=100 ] = 1.000',
        ' Average Precision  (AP) @[ IoU=0.50      | area=   all | maxDets=100 ] = 1.000',
        ' Average Precision  (AP) @[ IoU=0.75      | area=   all | maxDets=100 ] = 1.000',
        ' Average Precision  (AP) @[ IoU=0.50:0.95 | area= small | maxDets=100 ] = 1.000',
        ' Average Precision  (AP) @[ IoU=0.50:0.95 | area=medium | maxDets=100 ] = -1.000',
        ' Average Precision  (AP) @[ IoU=0.50:0.95 | area= large | maxDets=100 ] = -1.000',
        ' Average Recall     (AR) @[ IoU=0.50:0.95 | area=   all | maxDets=  1 ] = 1.000',
        ' Average Recall     (AR) @[ IoU=0.50:0.95 | area=   all | maxDets= 10 ] = 1.000',
        ' Average Recall     (AR) @[ IoU=0.50:0.95 | area=   all | maxDets=100 ] = 1.000',
        ' Average Recall     (AR) @[ IoU=0.50:0.95 | area= small | maxDets=100 ] = 1.000',
        ' Average Recall     (AR) @[ IoU=0.50:0.95 | area=medium | maxDets=100 ] = -1.000',
        ' Average Recall     (AR) @[ IoU=0.50:0.95 | area= large | maxDets=100 ] = -1.000']


# ------------------------------------------------------------------------------------------------------------------ host side
class _StubCOCO:
    def __init__(self, anns, h, w):
        self.anns, self.h, self.w = anns, h, w
        self.imgToAnns = {k: v for k, v in anns.items()}

    def getAnnIds(self, imgIds):
        return [(imgIds, i) for i in range(len(self.anns[imgIds]))]

    def loadAnns(self, ids):
        return [self.anns[k][i] for k, i in ids]

    def loadImgs(self, img_id):
        return [{'file_name': f'{img_id}.jpg'}]

    def annToMask(self, a):
        m = np.zeros((self.h, self.w), np.uint8)
        x, y, w, h = (int(v) for v in a['bbox'])
        m[max(y, 0):y + h, max(x, 0):x + w] = 1
        return m


H, W = 60, 70
ANNS = [dict(bbox=[10.5, 10.25, 20.125, 14.0], area=250.3, category_id=3, iscrowd=0),
        dict(bbox=[5.0, 5.0, 30.0, 30.0], area=812.0, category_id=4, iscrowd=1),
        dict(bbox=[1.0 / 3, 5.0, 30.0, 30.0], area=1024.0, category_id=90, iscrowd=0)]


def _dataset(coco_eval, anns=None):
    from yolact_minimal_b200.utils.coco import COCOValDetection
    cfg = SimpleNamespace(val_imgs='/nonexistent', val_ann=None, continuous_id=COCO_LABEL_MAP, val_num=-1, img_size=550)
    ds = COCOValDetection(cfg, coco=_StubCOCO(anns or {7: ANNS, 3: ANNS[:1]}, H, W), coco_eval=coco_eval)
    ds.load_image = lambda name: np.full((H, W, 3), int(name.split('.')[0]), np.uint8)
    return ds


def test_loader_coco_eval_rows():
    from yolact_minimal_b200.utils.coco import val_collate
    from yolact_minimal_b200.utils.mask_utils import pack_masks_host
    plain, full = _dataset(False), _dataset(True)
    for i in range(len(plain)):
        a, b = plain[i], full[i]
        assert len(a) == 5 and len(b) == 6
        for x, y in zip(a[:3], b[:3]):
            assert x.dtype == y.dtype and np.array_equal(x, y)
        assert a[3:] == b[3:5]
    cls, box, area, crowd, bits = full[0][5]
    assert list(cls) == [2, 3, 79] and list(crowd) == [0, 1, 0]
    assert box.dtype == np.float64 and [list(r) for r in box] == [a['bbox'] for a in ANNS] and box[2, 0] == 1.0 / 3
    assert area.dtype == np.float64 and list(area) == [250.3, 812.0, 1024.0]
    assert np.array_equal(bits, pack_masks_host(np.stack([full.coco.annToMask(a) for a in ANNS])))
    packed = val_collate([full[0], full[1]])
    assert packed.ann_offset == [0, 3, 4] and packed.ann_cls.tolist() == [2, 3, 79, 2]
    assert packed.ann_box.dtype.is_floating_point and packed.ann_box.shape == (4, 4) and packed.ann_area.tolist()[:3] == [250.3, 812.0, 1024.0]
    assert packed.ann_mask_off == [0, bits.size, bits.size + bits.size // 3] and packed.ann_masks.numel() == packed.ann_mask_off[-1]
    again = pickle.loads(pickle.dumps(packed))
    assert again.ann_cls.tolist() == packed.ann_cls.tolist() and again.ann_offset == packed.ann_offset
    # the default batch carries none of it and pickles as before
    plain_packed = val_collate([plain[0], plain[1]])
    assert plain_packed.ann_cls is None and 'ann_cls' not in vars(plain_packed)


def test_evaluator_host_tables():
    coco = _StubCOCO({7: ANNS, 3: ANNS[:1], 11: [dict(bbox=[0, 0, 1, 1], area=9216.0, category_id=3, iscrowd=0)]}, H, W)
    ev = cev.CocoEvaluator(coco, COCO_LABEL_MAP)
    assert ev.rank == {3: 0, 7: 1, 11: 2} and ev.num_classes == 80
    want = np.zeros((80, 4), np.int64)
    want[2] = [3, 2, 1, 1]                 # 250.3 twice (small), 9216 (medium and large)
    want[79] = [1, 1, 1, 0]                # 1024: small and medium
    assert np.array_equal(ev.npig, want)   # the crowd annotation is not counted


# ------------------------------------------------------------------------------------------------------------ against pycocotools
def test_oracle_equals_pycocotools():
    pytest.importorskip('pycocotools')
    from pycocotools.coco import COCO
    from pycocotools.cocoeval import COCOeval
    from pycocotools import mask as mask_util
    rng = np.random.RandomState(0)
    h, w, K = 80, 96, 3
    gts, dts, images, anns, res = [], [], [], [], {'bbox': [], 'segm': []}
    for img in range(1, 13):
        images.append({'id': img, 'height': h, 'width': w})
        for _ in range(rng.randint(0, 6)):
            x, y = rng.randint(0, w - 8), rng.randint(0, h - 8)
            bw, bh = rng.randint(1, w - x), rng.randint(1, h - y)
            g = gt(img, (x, y, bw, bh), k=rng.randint(K), crowd=int(rng.rand() < .2), area=float(rng.choice([bw * bh, 1024, 9216])))
            gts.append(g)
            m = np.zeros((h, w), np.uint8, order='F')
            m[y:y + bh, x:x + bw] = 1
            anns.append({'id': len(anns) + 1, 'image_id': img, 'category_id': g['category'] + 1, 'bbox': g['bbox'], 'area': g['area'],
                         'iscrowd': g['iscrowd'], 'segmentation': mask_util.encode(m)})
        for _ in range(rng.randint(0, 30)):
            x, y = rng.randint(0, w - 4), rng.randint(0, h - 4)
            d = dt(img, (x, y, rng.randint(1, w - x), rng.randint(1, h - y)), rng.choice([.3, .5, .7, rng.rand()]), k=rng.randint(K))
            dts.append(d)
            m = np.zeros((h, w), np.uint8, order='F')
            m[y:y + d['rect'][3] - y, x:x + d['rect'][2] - x] = 1
            res['bbox'].append({'image_id': img, 'category_id': d['category'] + 1, 'bbox': d['bbox'], 'score': d['score']})
            res['segm'].append({'image_id': img, 'category_id': d['category'] + 1, 'segmentation': mask_util.encode(m), 'score': d['score']})
    coco = COCO()
    coco.dataset = {'images': images, 'annotations': anns, 'categories': [{'id': k + 1} for k in range(K)]}
    coco.createIndex()
    for t in ('bbox', 'segm'):
        E = COCOeval(coco, coco.loadRes(res[t]), t)
        E.evaluate()
        E.accumulate()
        prec, rec = ce.evaluate(gts, dts, [im['id'] for im in images], K, t)
        assert np.array_equal(E.eval['precision'], prec) and np.array_equal(E.eval['recall'], rec), t
