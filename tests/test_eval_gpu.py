"""GPU: box and mask mAP on the device (csrc/eval.cu behind utils/common_utils.py) equals the reference bit for bit.
  * drop-in: eval.py's loop body with the package's prep_metrics / calc_map on the golden cases, float and packed masks
  * MapEvaluator fed in batches of 1, 3 and all images gives identical AP arrays (tie order across batches, zero-detection skip)
  * ~500 images x 100 detections at 480x640 == the oracle, also when the record buffers have to grow
  * Yolact -> nms -> after_nms(mask_dtype='bits') -> prep_metrics == the oracle fed the same after_nms outputs
  * one add() is a fixed number of launches; misuse is refused with YolactB200Error."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import eval_np as ev

pytestmark = pytest.mark.gpu

THR = [x / 100 for x in range(50, 100, 5)]


def _rect_bits(rects, h, w, dev):
    from yolact_minimal_b200.utils.mask_utils import pack_masks
    r = torch.from_numpy(np.asarray(rects, np.int64).reshape(-1, 4)).to(dev)
    ys = torch.arange(h, device=dev)[None, :, None]
    xs = torch.arange(w, device=dev)[None, None, :]
    m = (xs >= r[:, 0, None, None]) & (xs < r[:, 2, None, None]) & (ys >= r[:, 1, None, None]) & (ys < r[:, 3, None, None])
    return pack_masks(m.to(torch.uint8))


def _rect_float(rects, h, w, dev):
    from yolact_minimal_b200.utils.mask_utils import unpack_masks
    return unpack_masks(_rect_bits(rects, h, w, dev), w).float()


def _batch(images, dev, D=None):
    """eval_set images -> MapEvaluator.add arguments (detect_batched-style records padded to D)."""
    B = len(images)
    D = D or max(1, max(len(im['ids']) for im in images))
    count = np.array([len(im['ids']) for im in images], np.int32)
    cls = np.zeros((B, D), np.int32)
    score = np.zeros((B, D), np.float32)
    boxes = np.zeros((B, D, 4), np.int32)
    for b, im in enumerate(images):
        d = len(im['ids'])
        cls[b, :d], score[b, :d], boxes[b, :d] = im['ids'], im['scores'], im['boxes_px']
    t = lambda a: torch.from_numpy(a).to(dev)
    det = {'count': t(count), 'cls': t(cls), 'score': t(score)}
    masks = [_rect_bits(im['det_rects'], im['h'], im['w'], dev) for im in images]
    gt = t(np.concatenate([im['gt'] for im in images]).reshape(-1, 5))
    gt_masks = [_rect_bits(im['gt_rects'], im['h'], im['w'], dev) for im in images]
    off = np.concatenate([[0], np.cumsum([len(im['gt']) for im in images])]).tolist()
    return det, t(boxes), masks, gt, off, gt_masks, [(im['h'], im['w']) for im in images]


def _oracle_ap(images, C):
    o = ev.EvalOracle(C, THR)
    for im in images:
        o.add_synth(im)
    return o.ap_array()


def _ap_data(cu, C):
    return {'box': [[cu.APDataObject() for _ in range(C)] for _ in THR], 'mask': [[cu.APDataObject() for _ in range(C)] for _ in THR]}


@pytest.mark.parametrize('packed', [False, True])
@pytest.mark.parametrize('seed', [1, 2, 3])
def test_drop_in_equals_reference_golden(cuda, seed, packed):
    from yolact_minimal_b200.utils import common_utils as cu
    g = load_golden('eval.npz')
    C = int(g['num_classes'])
    ap_data = _ap_data(cu, C)
    for im in ev.eval_set(seed, num_classes=C):
        if len(im['ids']) == 0:                                  # eval.py:53
            continue
        h, w = im['h'], im['w']
        ids_p, class_p = list(im['ids'].astype(int)), list(im['scores'].astype(float))
        boxes_p = torch.from_numpy(im['boxes_px']).to(cuda)
        masks_p = _rect_bits(im['det_rects'], h, w, cuda) if packed else _rect_float(im['det_rects'], h, w, cuda)
        gt = torch.from_numpy(im['gt']).to(cuda)
        gt_before = gt.clone()
        gt_masks = _rect_float(im['gt_rects'], h, w, cuda)
        cu.prep_metrics(ap_data, ids_p, class_p, boxes_p, masks_p, gt, gt_masks, h, w, THR)
        assert torch.equal(gt, gt_before)                        # not scaled in place
    p = f'seed{seed}/'
    for typ, name in enumerate(('box', 'mask')):
        for t in range(len(THR)):
            for c in range(C):
                o = ap_data[name][t][c]
                assert o.get_ap() == g[p + 'ap'][typ, t, c], (name, t, c)
                assert o.is_empty() == g[p + 'is_empty'][typ, t, c], (name, t, c)
    _, box_row, mask_row = cu.calc_map(ap_data, THR, C, step=None)
    assert box_row[1:] == list(g[p + 'box_row']) and mask_row[1:] == list(g[p + 'mask_row'])


def test_batch_invariance(cuda):
    from yolact_minimal_b200.utils.common_utils import MapEvaluator
    C = 12
    images = ev.eval_set(7, num_images=11, num_classes=C, dets_per_image=40, empty_image=4)
    res = []
    for bs in (1, 3, len(images)):
        m = MapEvaluator(C, THR)
        for i in range(0, len(images), bs):
            m.add(*_batch(images[i:i + bs], cuda, D=40))
        res.append(m.ap())
    for ap, ne in res[1:]:
        assert np.array_equal(ap.view(np.uint64), res[0][0].view(np.uint64)) and np.array_equal(ne, res[0][1])
    ap, ne = _oracle_ap(images, C)
    assert np.array_equal(res[0][0], ap) and np.array_equal(res[0][1], ne)


def test_scale_and_growth_match_oracle(cuda):
    from yolact_minimal_b200.utils.common_utils import MapEvaluator
    C = 80
    images = ev.eval_set(11, num_images=500, num_classes=C, dets_per_image=100, sizes=((480, 640),), max_gt=13, empty_image=17)
    want_ap, want_ne = _oracle_ap(images, C)
    assert want_ne.sum() > 60 and (want_ap > 0).sum() > 200
    for capacity in (1 << 16, 8):                                # 8 records: the buffers grow on almost every batch
        m = MapEvaluator(C, THR, capacity=capacity)
        for i in range(0, len(images), 64):
            m.add(*_batch(images[i:i + 64], cuda, D=100))
        ap, ne = m.ap()
        assert np.array_equal(ap, want_ap) and np.array_equal(ne, want_ne), capacity
        assert m.num_records() == sum(len(im['ids']) for im in images)


def test_end_to_end_res50(cuda):
    from oracle import forward_torch as ft, synth
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    from yolact_minimal_b200.utils import common_utils as cu
    from yolact_minimal_b200.utils.mask_utils import unpack_masks
    from yolact_minimal_b200.utils.output_utils import nms, after_nms
    S, C = 128, 80
    cfg = make_config('res50_coco', S)
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict('res50', seed=0), strict=True)
    net = net.to(cuda).eval()
    ap_data = _ap_data(cu, C)
    o = ev.EvalOracle(C, THR)
    seen = 0
    for k, (h, w) in enumerate(((96, 128), (128, 100), (77, 128))):
        img = torch.from_numpy(synth.image_batch(20 + k, 1, S)).to(cuda)
        with torch.no_grad():
            class_p, box_p, coef_p, proto_p = net(img)
        ids_p, class_p, box_p, coef_p, proto_p = nms(class_p, box_p, coef_p, proto_p, net.anchors, cfg)
        ids_p, class_p, boxes_p, masks_p = after_nms(ids_p, class_p, box_p, coef_p, proto_p, h, w, mask_dtype='bits')
        if ids_p is None:
            continue
        ids_l = list(ids_p.cpu().numpy().astype(int))
        cls_l = list(class_p.cpu().numpy().astype(float))
        # synthetic gts: the classes and (shifted) boxes of some detections, plus one unrelated gt
        bx = boxes_p.cpu().numpy().astype(np.float64)
        sel = list(range(0, len(ids_l), 3))
        gpx = np.clip(bx[sel] + np.array([2, -1, 3, 1]), 0, [w, h, w, h])
        gpx = np.concatenate([gpx, [[5, 5, 40, 30]]])
        gcls = np.array([ids_l[i] for i in sel] + [7], np.float64)
        gt_np = np.concatenate([gpx[:, [0]] / w, gpx[:, [1]] / h, gpx[:, [2]] / w, gpx[:, [3]] / h, gcls[:, None]], 1).astype(np.float32)
        grects = np.floor(gpx).astype(np.int64)
        gt = torch.from_numpy(gt_np).to(cuda)
        gt_masks = _rect_float(grects, h, w, cuda)
        cu.prep_metrics(ap_data, ids_l, cls_l, boxes_p, masks_p, gt, gt_masks, h, w, THR)
        dm = unpack_masks(masks_p, w).cpu().numpy()
        o.add_image(ids_l, cls_l, ev.box_iou(boxes_p.cpu().numpy(), gt_np, h, w),
                    ev.mask_iou_dense(dm, ev.rect_masks(grects, h, w)), gt_np[:, 4].astype(np.int32))
        seen += 1
    assert seen >= 1
    ap, ne = o.ap_array()
    got = cu.evaluator_of(ap_data).ap()
    assert np.array_equal(got[0], ap) and np.array_equal(got[1], ne)
    _, box_row, mask_row = cu.calc_map(ap_data, THR, C, step=None)
    assert (box_row, mask_row) == ev.map_rows(ap, ne, THR)


def test_launch_count_is_fixed(cuda):
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils.common_utils import MapEvaluator
    deltas = []
    for C, n in ((8, 2), (30, 9)):
        images = ev.eval_set(5, num_images=n, num_classes=C)
        args = _batch(images, cuda)
        m = MapEvaluator(C, THR)
        before = _lib.launch_count()
        m.add(*args)
        deltas.append(_lib.launch_count() - before)
    assert deltas == [1, 1]


def test_misuse_is_refused(cuda):
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils import common_utils as cu
    im = ev.eval_set(1)[1]
    h, w = im['h'], im['w']
    args = lambda **kw: dict(dict(ids_p=list(im['ids']), classes_p=list(im['scores'].astype(float)),
                                  boxes_p=torch.from_numpy(im['boxes_px']).to(cuda), masks_p=_rect_float(im['det_rects'], h, w, cuda),
                                  gt=torch.from_numpy(im['gt']).to(cuda), gt_masks=_rect_float(im['gt_rects'], h, w, cuda),
                                  height=h, width=w, iou_thres=THR), **kw)
    with pytest.raises(_lib.YolactB200Error):                    # CPU tensors
        cu.prep_metrics(_ap_data(cu, 8), **args(boxes_p=torch.from_numpy(im['boxes_px'])))
    with pytest.raises(_lib.YolactB200Error):
        cu.prep_metrics(_ap_data(cu, 8), **args(gt_masks=_rect_float(im['gt_rects'], h, w, cuda).cpu()))
    with pytest.raises(_lib.YolactB200Error):                    # packed masks of another image size
        cu.prep_metrics(_ap_data(cu, 8), **args(masks_p=_rect_bits(im['det_rects'], h, w + 64, cuda)))
    with pytest.raises(_lib.YolactB200Error):
        cu.prep_metrics(_ap_data(cu, 8), **args(gt_masks=_rect_float(im['gt_rects'], h - 1, w, cuda)))
    thr17 = [0.5 + i / 100 for i in range(17)]
    ap17 = {'box': [[cu.APDataObject() for _ in range(8)] for _ in thr17], 'mask': [[cu.APDataObject() for _ in range(8)] for _ in thr17]}
    with pytest.raises(_lib.YolactB200Error):                    # more than 16 thresholds
        cu.prep_metrics(ap17, **args(iou_thres=thr17))
    ap_data = _ap_data(cu, 8)
    cu.prep_metrics(ap_data, **args())
    with pytest.raises(_lib.YolactB200Error):
        ap_data['box'][0][0].push(0.9, True)
    # the C entry points refuse NULL pointers and more than 16 thresholds
    import ctypes
    L = _lib.lib()
    p = _lib.EvalParams(8, 17)
    assert L.yb_eval_match(ctypes.byref(p), 1, 4, *([None] * 6), 0, None, None, None, 0, None, None, 0, None, None, None, 0, None, None, 0,
                           None) != 0
    p = _lib.EvalParams(8, 10)
    assert L.yb_eval_match(ctypes.byref(p), 1, 4, *([None] * 6), 0, None, None, None, 0, None, None, 0, None, None, None, 0, None, None, 0,
                           None) != 0
    assert L.yb_eval_ap(ctypes.byref(p), None, None, None, 0, None, None, 0, None, None, None) != 0
