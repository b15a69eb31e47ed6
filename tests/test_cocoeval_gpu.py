"""GPU: COCO's own mAP on the device (csrc/cocoeval.cu behind utils/cocoeval.CocoEvaluator) equals oracle/cocoeval_np.py bit for bit.
  * 500 images x 100 detections, 80 classes, crowd gts, area-boundary gts, score ties, images added out of id order, images of the
    annotation set never added; and D = 256 with more than 100 detections of one class in an image
  * B = 1, 7 and 64 give identical arrays
  * add() never synchronises and is one library launch whatever B and the detections are; misuse raises YolactB200Error
  * evaluate(net, cfg) with cfg.coco_gpu == the oracle fed the per-image loop's detections (tests/val_loop.py's path)."""
import numpy as np
import pytest
import torch

from oracle import cocoeval_np as ce

pytestmark = pytest.mark.gpu

IDENTITY = {k + 1: k + 1 for k in range(80)}


def _rect_masks(rects, h, w):
    from yolact_minimal_b200.utils.mask_utils import pack_masks_host
    m = np.zeros((len(rects), h, w), np.uint8)
    for i, (x1, y1, x2, y2) in enumerate(rects):
        m[i, max(y1, 0):max(y2, 0), max(x1, 0):max(x2, 0)] = 1
    return pack_masks_host(m)


def make_set(seed, n, K=80, D=100, sizes=((96, 128), (128, 96)), max_gt=9, classes_per_image=6, hot=None, extra_images=5):
    """Synthetic images: gts with float boxes and rectangle masks (some crowd, areas on the range boundaries), detections near them
    with coarse float32 scores (ties), some of zero area; `hot` = a class given D // 2 detections in every image."""
    rng = np.random.RandomState(seed)
    ids = rng.permutation(np.arange(1, 4 * (n + extra_images)))[:n + extra_images].tolist()
    images = []
    for b, img_id in enumerate(ids):
        h, w = sizes[b % len(sizes)]
        cls_pool = rng.randint(0, K, size=classes_per_image)
        if hot is not None:
            cls_pool[0] = hot
        gts = []
        for _ in range(rng.randint(1, max_gt + 1)):
            x1, y1 = rng.randint(0, w - 2), rng.randint(0, h - 2)
            x2, y2 = rng.randint(x1 + 1, w + 1), rng.randint(y1 + 1, h + 1)
            box = [x1 + rng.choice([0, .25, .5]), y1 + rng.choice([0, .125]), x2 - x1 - rng.choice([0, .5]), y2 - y1 + 0.0]
            area = float(rng.choice([(x2 - x1) * (y2 - y1), 1024.0, 9216.0, rng.uniform(0, 15000)]))
            gts.append({'cls': int(rng.choice(cls_pool)), 'bbox': box, 'area': area, 'crowd': int(rng.rand() < .15),
                        'rect': (x1, y1, x2, y2)})
        d = rng.randint(D // 2, D + 1) if hot is None else D
        dets = []
        for i in range(d):
            k = hot if hot is not None and i < D // 2 + D // 4 else int(rng.choice(cls_pool))
            if gts and rng.rand() < .6:
                gx1, gy1, gx2, gy2 = gts[rng.randint(len(gts))]['rect']
                j = rng.randint(-3, 4, size=4)
                x1, y1 = int(np.clip(gx1 + j[0], 0, w - 1)), int(np.clip(gy1 + j[1], 0, h - 1))
                x2, y2 = int(np.clip(gx2 + j[2], x1, w)), int(np.clip(gy2 + j[3], y1, h))
            else:
                x1, y1 = rng.randint(0, w), rng.randint(0, h)
                x2, y2 = rng.randint(x1, w + 1), rng.randint(y1, h + 1)
            mrect = (x1, y1, x2, max(y1, y2 - rng.randint(0, 2)))        # the mask need not equal the box
            dets.append({'cls': k, 'score': np.float32(rng.randint(1, 30) / 30), 'box': (x1, y1, x2, y2), 'rect': mrect})
        images.append({'id': img_id, 'h': h, 'w': w, 'gts': gts, 'dets': dets, 'added': b < n})
    return images


class _Coco:
    def __init__(self, images):
        self.imgToAnns = {im['id']: [{'category_id': g['cls'] + 1, 'area': g['area'], 'iscrowd': g['crowd']} for g in im['gts']]
                          for im in images}


class _Batch:
    """What CocoEvaluator.add reads of a PackedValBatch."""

    def __init__(self, ims):
        self.ids, self.sizes = [im['id'] for im in ims], [(im['h'], im['w']) for im in ims]
        g = [im['gts'] for im in ims]
        self.ann_offset = np.concatenate([[0], np.cumsum([len(x) for x in g])]).astype(int).tolist()
        self.ann_cls = torch.tensor([a['cls'] for x in g for a in x], dtype=torch.int32)
        self.ann_box = torch.tensor([a['bbox'] for x in g for a in x], dtype=torch.float64).reshape(-1, 4)
        self.ann_area = torch.tensor([a['area'] for x in g for a in x], dtype=torch.float64)
        self.ann_crowd = torch.tensor([a['crowd'] for x in g for a in x], dtype=torch.int32)
        bits = [_rect_masks([a['rect'] for a in im['gts']], im['h'], im['w']) for im in ims]
        self.ann_mask_off = np.concatenate([[0], np.cumsum([x.size for x in bits])]).astype(int).tolist()
        self.ann_masks = torch.from_numpy(np.concatenate([x.reshape(-1) for x in bits]))

    def __len__(self):
        return len(self.ids)


def batch_args(ims, dev, D):
    B = len(ims)
    count = np.array([len(im['dets']) for im in ims], np.int32)
    cls = np.zeros((B, D), np.int32)
    score = np.zeros((B, D), np.float32)
    boxes = np.zeros((B, D, 4), np.int32)
    for b, im in enumerate(ims):
        for i, d in enumerate(im['dets']):
            cls[b, i], score[b, i], boxes[b, i] = d['cls'], d['score'], d['box']
    t = lambda a: torch.from_numpy(a).to(dev)
    masks = [t(_rect_masks([d['rect'] for d in im['dets']] or [(0, 0, 0, 0)], im['h'], im['w'])) for im in ims]
    return {'count': t(count), 'cls': t(cls), 'score': t(score)}, t(boxes), masks, _Batch(ims)


def oracle(images, K=80):
    gts = [{'image_id': im['id'], 'category': g['cls'], 'bbox': g['bbox'], 'area': g['area'], 'iscrowd': g['crowd'], 'rect': g['rect']}
           for im in images for g in im['gts']]
    dts = []
    for im in images:
        if not im['added']:
            continue
        for d in im['dets']:
            x1, y1, x2, y2 = d['box']
            if (y2 - y1) * (x2 - x1) > 0:
                dts.append({'image_id': im['id'], 'category': d['cls'], 'bbox': [x1, y1, x2 - x1, y2 - y1], 'score': float(d['score']),
                            'rect': d['rect']})
    ids = [im['id'] for im in images]
    return {t: ce.evaluate(gts, dts, ids, K, t) for t in ('bbox', 'segm')}


def run(images, dev, B, D, order=None):
    from yolact_minimal_b200.utils.cocoeval import CocoEvaluator
    ev = CocoEvaluator(_Coco(images), IDENTITY, dev, capacity=8)
    added = [im for im in images if im['added']]
    if order is not None:
        added = [added[i] for i in order]
    for i in range(0, len(added), B):
        ev.add(*batch_args(added[i:i + B], dev, D))
    return ev


def check(ev, want):
    from yolact_minimal_b200.utils.cocoeval import summarize
    got = ev.accumulate()
    for t in ('bbox', 'segm'):
        assert np.array_equal(got[t]['precision'], want[t][0]), t
        assert np.array_equal(got[t]['recall'], want[t][1]), t
    stats = ev.summarize()
    for i, t in enumerate(('bbox', 'segm')):
        assert np.array_equal(stats[i], summarize(*want[t])[0]), t
    return got


def test_scale_matches_oracle(cuda):
    images = make_set(1, 500)
    want = oracle(images)
    p = want['bbox'][0]
    assert (p > 0).sum() > 1000 and (want['segm'][0] > 0).sum() > 1000
    order = np.random.RandomState(0).permutation(500)                        # added out of image-id order
    check(run(images, cuda, 64, 100, order), want)


def test_more_than_100_detections_of_a_class(cuda):
    images = make_set(2, 24, D=256, hot=3, sizes=((64, 80),))
    want = oracle(images)
    assert (want['bbox'][1] == -1).any() and want['bbox'][1][0, 3, 0, 2] > 0
    check(run(images, cuda, 7, 256), want)


def test_batch_sizes_give_identical_results(cuda):
    images = make_set(3, 60)
    want = oracle(images)
    res = [run(images, cuda, B, 100).accumulate() for B in (1, 7, 64)]
    for r in res:
        for t in ('bbox', 'segm'):
            assert np.array_equal(r[t]['precision'], want[t][0]) and np.array_equal(r[t]['recall'], want[t][1])


def test_add_no_sync_fixed_launches(cuda):
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils.cocoeval import CocoEvaluator
    images = make_set(4, 40)
    ev = CocoEvaluator(_Coco(images), IDENTITY, cuda)
    batches = [batch_args(images[a:b], cuda, D) for a, b, D in ((0, 1, 100), (1, 8, 100), (8, 40, 160), (0, 3, 120))]
    for bt in batches:                                                         # pin the host tables outside the checked region
        for name in ('ann_cls', 'ann_box', 'ann_area', 'ann_crowd', 'ann_masks'):
            setattr(bt[3], name, getattr(bt[3], name).pin_memory())
    ev.add(*batches[0])                                                        # warm-up: state, workspace
    deltas = []
    torch.cuda.set_sync_debug_mode('error')
    try:
        for bt in batches[1:]:
            before = _lib.launch_count()
            ev.add(*bt)
            deltas.append(_lib.launch_count() - before)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert deltas == [1, 1, 1]
    ev.accumulate()


def test_misuse_is_refused(cuda):
    import ctypes
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils.cocoeval import CocoEvaluator
    images = make_set(5, 4, extra_images=0)
    ev = CocoEvaluator(_Coco(images), IDENTITY, cuda)
    det, boxes, masks, packed = batch_args(images[:2], cuda, 100)
    with pytest.raises(_lib.YolactB200Error):                                 # CPU tensors
        ev.add({k: v.cpu() for k, v in det.items()}, boxes, masks, packed)
    with pytest.raises(_lib.YolactB200Error):                                 # an image id outside the annotation set
        packed.ids = [packed.ids[0], 10 ** 9]
        ev.add(det, boxes, masks, packed)
    det, boxes, masks, packed = batch_args(images[:2], cuda, 100)
    with pytest.raises(_lib.YolactB200Error):                                 # a batch without annotations
        packed.ann_cls = None
        ev.add(det, boxes, masks, packed)
    det, boxes, masks, packed = batch_args(images[:2], cuda, 100)
    with pytest.raises(_lib.YolactB200Error):                                 # inconsistent shapes
        ev.add(det, boxes[:1], masks, packed)
    with pytest.raises(_lib.YolactB200Error):                                 # masks of another image size
        ev.add(det, boxes, [masks[1], masks[0]], packed)
    L = _lib.lib()
    p = _lib.CocoEvalParams()
    assert L.yb_cocoeval_match(ctypes.byref(p), 1, 4, *([None] * 6), 0, *([None] * 7), 0, None, None, 0, None, 0, None, None, 0, None) != 0
    p = ev.params
    assert L.yb_cocoeval_match(ctypes.byref(p), 1, 4, *([None] * 6), 0, *([None] * 7), 0, None, None, 0, None, 0, None, None, 0, None) != 0
    assert L.yb_cocoeval_accumulate(ctypes.byref(p), None, 0, None, None, None, 0, None, None, None) != 0
    big = _lib.CocoEvalParams()
    ctypes.memmove(ctypes.byref(big), ctypes.byref(p), ctypes.sizeof(p))
    big.num_images = 1 << 26                                                   # 7 class bits + 26 image bits > 32
    ws = torch.empty(1024, dtype=torch.uint8, device=cuda)
    assert L.yb_cocoeval_accumulate(ctypes.byref(big), None, 0, ws.data_ptr(), ws.data_ptr(), ws.data_ptr(), ws.numel(), ws.data_ptr(),
                                    ws.data_ptr(), None) == -3


# ------------------------------------------------------------------------------------------------------------------------ evaluate
def test_evaluate_coco_gpu_equals_oracle_on_per_image_loop(cuda, tmp_path):
    from oracle import forward_torch as ft
    from test_val_batch_gpu import _eval_set
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.eval import evaluate
    from yolact_minimal_b200.modules.yolact import Yolact
    from yolact_minimal_b200.utils.augmentations import val_aug
    from yolact_minimal_b200.utils.coco import COCOValDetection
    from yolact_minimal_b200.utils.cocoeval import summarize
    from yolact_minimal_b200.utils.mask_utils import unpack_masks
    from yolact_minimal_b200.utils.output_utils import after_nms, nms
    cfg = make_config('res101_coco', 550, mode='val')
    cfg.precision, cfg.max_batch = 'fp16', 64
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict('res101', seed=0), strict=True)
    net = net.to(cuda).eval()
    cfg.val_imgs = str(tmp_path)
    coco = _eval_set(tmp_path, net, cfg, n=20)
    for k, (_, h, w, anns) in coco.images.items():
        for i, a in enumerate(anns):
            a['area'] = [a['bbox'][2] * a['bbox'][3], 1024.0, 300.25][i % 3]
    ds = COCOValDetection(cfg, coco=coco, coco_eval=True)
    # the per-image loop's detections (val_aug, net(img[None]), nms, after_nms), kept as eval.py's JSON keeps them
    gts, dts = [], []
    for i in range(len(ds)):
        img, _, _, (h, w), img_id, (cls, box, area, crowd, bits) = ds[i]
        gm = unpack_masks(torch.from_numpy(bits).to(cuda), w).cpu().numpy()
        for j in range(len(cls)):
            gts.append({'image_id': img_id, 'category': int(cls[j]), 'bbox': list(box[j]), 'area': float(area[j]), 'iscrowd': int(crowd[j]),
                        'mask': gm[j]})
        with torch.no_grad():
            out = net(val_aug(img, cfg.img_size, cuda)[None])
        ids_p, class_p, box_p, coef_p, proto_p = nms(*out, net.anchors, cfg)
        ids_p, class_p, boxes_p, masks_p = after_nms(ids_p, class_p, box_p, coef_p, proto_p, h, w)
        if ids_p is None:
            continue
        bx, ms = boxes_p.cpu().numpy(), masks_p.cpu().numpy()
        for j, (k, s) in enumerate(zip(ids_p.cpu().numpy(), class_p.cpu().numpy())):
            x1, y1, x2, y2 = (int(v) for v in bx[j])
            if (y2 - y1) * (x2 - x1) > 0:
                dts.append({'image_id': img_id, 'category': int(k), 'bbox': [x1, y1, x2 - x1, y2 - y1], 'score': float(s), 'mask': ms[j] > 0})
    ids = list(coco.imgToAnns.keys())
    want = [summarize(*ce.evaluate(gts, dts, ids, 80, t))[0] for t in ('bbox', 'segm')]
    assert want[0][0] > 0 and want[1][0] > 0
    cfg.coco_gpu, cfg.val_bs = True, 8
    box_stats, mask_stats = evaluate(net, cfg, dataset=ds, num_workers=0)
    assert np.array_equal(box_stats, want[0]) and np.array_equal(mask_stats, want[1])
