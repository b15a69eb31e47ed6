"""GPU: batched COCO evaluation (yolact_minimal_b200.eval.evaluate) and its two batched stages, bit for bit:
  * val_aug_batch image b == yb_val_aug on image b (B in {1, 7, 64}, mixed sizes, S in {544, 550});
  * after_nms_batched == yb_mask_assemble(mask_f32 = 2) per image on the first count[b] detections, masks and boxes; rows past
    count[b] are zero boxes and write no mask word (sentinels around every image's range and at the buffer's tail stay);
  * host-packed gt masks == yb_pack_mask_bits;
  * evaluate() == the reference's per-image loop (tests/val_loop.py), tables compared with ==, at res101 550 fp16, and at
    res50_pascal (21 classes, identity category ids);
  * library launches per batch do not depend on B or the detections, and the per-batch body never synchronises."""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SIZES = [(550, 550), (480, 640), (640, 480), (427, 640), (300, 200), (1, 97), (600, 700), (33, 33), (640, 427)]


def _images(seed, B):
    rng = np.random.RandomState(seed)
    return [rng.randint(0, 256, size=(*SIZES[(seed + i) % len(SIZES)], 3), dtype=np.uint8) for i in range(B)]


@pytest.mark.parametrize('S', [544, 550])
@pytest.mark.parametrize('B', [1, 7, 64])
def test_val_aug_batch_equals_val_aug(cuda, B, S):
    from yolact_minimal_b200.utils.augmentations import pack_images, val_aug, val_aug_batch
    imgs = _images(B + S, B)
    buf, items = pack_images(imgs)
    for pinned in (False, True):
        out = val_aug_batch(buf.pin_memory() if pinned else buf, items, S, cuda)
        assert out.shape == (B, 3, S, S)
        for b, im in enumerate(imgs):
            assert torch.equal(out[b], val_aug(im, S, cuda)), (b, im.shape)


# ------------------------------------------------------------------------------------------------------------------- mask assembly
def _per_image(proto, coef, box, h, w, crop):
    """yb_mask_assemble(mask_f32 = 2) on one image's first n detections -> (packed masks [n,h,wd], boxes_px [n,4])."""
    from yolact_minimal_b200 import _lib
    L = _lib.lib()
    n, K = coef.shape
    P = proto.shape[0]
    masks = torch.zeros(max(n, 1), h, (w + 31) // 32, dtype=torch.int32, device=proto.device)
    boxes = torch.zeros(max(n, 1), 4, dtype=torch.int32, device=proto.device)
    ws = torch.empty(max(int(L.yb_mask_workspace_bytes(n, P)), 1), dtype=torch.uint8, device=proto.device)
    _lib.check(L.yb_mask_assemble(proto.data_ptr(), coef.contiguous().data_ptr(), box.contiguous().data_ptr(), n, P, K, h, w, crop, 2,
                                  ws.data_ptr(), ws.numel(), masks.data_ptr(), boxes.data_ptr(), torch.cuda.current_stream().cuda_stream),
               'yb_mask_assemble')
    return masks[:n], boxes[:n]


SENTINEL = 0x5A5A5A5A


def _check_batched(det, proto, sizes, crop, gap=3):
    """after_nms_batched's result, and a direct call with `gap` sentinel words between the images and at the tail, against the
    per-image entry point."""
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils.output_utils import after_nms_batched
    boxes_px, views = after_nms_batched(det, proto, sizes, crop=crop)
    count = det['count'].cpu().tolist()
    B, D, K = det['coef'].shape
    P = proto.shape[1]
    # direct call: gaps between the images' ranges, prefilled with sentinels
    n_words = [D * h * ((w + 31) // 32) for h, w in sizes]
    off = [gap]
    for n in n_words:
        off.append(off[-1] + n + gap)
    off[-1] -= gap
    off = np.asarray(off, np.int64)
    total = int(off[-1]) + gap
    out = torch.full((total,), SENTINEL, dtype=torch.int32, device=proto.device)
    bpx = torch.full((B, D, 4), 7, dtype=torch.int32, device=proto.device)
    hw = np.asarray(sizes, np.int32)
    L = _lib.lib()
    ws = torch.empty(int(L.yb_mask_assemble_batch_workspace_bytes(B, D, P)), dtype=torch.uint8, device=proto.device)
    _lib.check(L.yb_mask_assemble_batch(proto.data_ptr(), det['coef'].contiguous().data_ptr(), det['box'].contiguous().data_ptr(),
                                        det['count'].data_ptr(), B, D, P, K, hw.ctypes.data, off.ctypes.data, total, int(crop),
                                        ws.data_ptr(), ws.numel(), out.data_ptr(), bpx.data_ptr(), torch.cuda.current_stream().cuda_stream),
               'yb_mask_assemble_batch')
    assert torch.equal(bpx, boxes_px)
    for b, (h, w) in enumerate(sizes):
        n = min(max(count[b], 0), D)
        want_m, want_b = _per_image(proto[b], det['coef'][b, :n], det['box'][b, :n], h, w, int(crop))
        wd = (w + 31) // 32
        assert views[b].shape == (D, h, wd)
        assert torch.equal(views[b][:n], want_m), b
        assert torch.equal(boxes_px[b, :n], want_b), b
        assert not boxes_px[b, n:].any(), b                                  # zero box past count
        mine = out[int(off[b]):int(off[b]) + n_words[b]].view(D, h, wd)
        assert torch.equal(mine[:n], want_m), b
        assert bool((mine[n:] == SENTINEL).all()), b                          # nothing written past count
        lo = 0 if b == 0 else int(off[b - 1]) + n_words[b - 1]
        assert bool((out[lo:int(off[b])] == SENTINEL).all()), b               # the gap before the image
    assert bool((out[int(off[B]):] == SENTINEL).all())                       # the tail
    return views


def _hand_record(cuda, B, D, K, counts, seed):
    rng = np.random.RandomState(seed)
    box = rng.uniform(-0.2, 1.2, size=(B, D, 4)).astype(np.float32)
    box[:, ::5, 2] = box[:, ::5, 0]                                          # zero width
    box[:, 1::5] = box[:, 1::5, ::-1]                                        # reversed corners
    box[:, 2::5] = rng.uniform(1.5, 3.0, size=box[:, 2::5].shape)            # far out of range
    coef = rng.normal(0, 1, size=(B, D, K)).astype(np.float32)
    cls = np.zeros((B, D), np.int32)
    score = np.zeros((B, D), np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    return {'count': t(np.asarray(counts, np.int32)), 'cls': t(cls), 'score': t(score), 'box': t(box), 'coef': t(coef)}


@pytest.mark.parametrize('crop', [True, False])
def test_after_nms_batched_hand_records(cuda, crop):
    B, D, K, P = 5, 100, 32, 69
    proto = torch.from_numpy(np.random.RandomState(3).uniform(0, 1.5, size=(B, P, P, K)).astype(np.float32)).to(cuda)
    det = _hand_record(cuda, B, D, K, [0, 1, D, 37, 17], 4)
    _check_batched(det, proto, [(480, 640), (640, 480), (1, 97), (550, 550), (427, 640)], crop)


def test_after_nms_batched_real_records(cuda):
    from oracle import forward_torch as ft, synth
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    from yolact_minimal_b200.utils.output_utils import detect_batched
    S, B = 256, 4
    cfg = make_config('res50_coco', S)
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict('res50', seed=0), strict=True)
    net = net.to(cuda).eval()
    with torch.no_grad():
        cls, box, coef, proto = net(torch.from_numpy(synth.image_batch(31, B, S)).to(cuda))
    det = detect_batched(cls, box, coef, net.anchors, cfg)
    assert int(det['count'].sum()) > 0
    for crop in (True, False):
        _check_batched(det, proto, [(480, 640), (200, 256), (640, 427), (97, 1)], crop)


def test_host_packed_gt_equals_device_packing(cuda):
    from yolact_minimal_b200.utils.mask_utils import pack_masks, pack_masks_host
    rng = np.random.RandomState(0)
    for w in (1, 31, 32, 33, 640):
        m = (rng.rand(3, 11, w) > 0.5).astype(np.uint8)
        assert np.array_equal(pack_masks_host(m), pack_masks(torch.from_numpy(m).to(cuda)).cpu().numpy()), w


# ------------------------------------------------------------------------------------------------------------------------ evaluate
class _StubCOCO:
    """The pycocotools.coco.COCO methods COCOValDetection uses, over in-memory annotations of several images."""

    def __init__(self, images):
        self.images = images                                     # img_id -> (file_name, h, w, anns)
        self.imgToAnns = {k: v[3] for k, v in images.items()}

    def getAnnIds(self, imgIds):
        return [(imgIds, i) for i in range(len(self.images[imgIds][3]))]

    def loadAnns(self, ids):
        return [self.images[k][3][i] for k, i in ids]

    def loadImgs(self, img_id):
        return [{'file_name': self.images[img_id][0]}]

    def annToMask(self, a):
        h, w = a['_hw']
        m = np.zeros((h, w), np.uint8)
        x, y, bw, bh = (int(v) for v in a['bbox'])
        m[max(y, 0):y + bh, max(x, 0):x + bw] = 1
        return m


EVAL_SIZES = [(480, 640), (640, 480), (427, 640), (550, 550), (300, 200), (64, 97), (640, 427)]


def _eval_set(tmp_path, net, cfg, n=45):
    """n synthetic PNG images on disk; gts from a first detection pass (shifted boxes of some detections, an unrelated box, one
    crowd annotation), as in test_eval_gpu.py's end-to-end case.  Category ids are the config's: COCO's for the COCO configs, the
    identity map of cfg.continuous_id otherwise."""
    import cv2
    from yolact_minimal_b200.utils.augmentations import val_aug
    from yolact_minimal_b200.utils.output_utils import after_nms, nms
    cat_id = {label - 1: cid for cid, label in cfg.continuous_id.items()}
    nfg = cfg.num_classes - 1
    rng = np.random.RandomState(9)
    images = {}
    dev = next(net.parameters()).device
    for k in range(n):
        h, w = EVAL_SIZES[k % len(EVAL_SIZES)]
        # smooth blobs plus noise: enough structure for the synthetic net to fire
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([128 + 100 * np.sin(xx / (7 + k % 5) + c) * np.cos(yy / (11 + c)) for c in range(3)], -1)
        img = np.clip(base + rng.normal(0, 20, size=(h, w, 3)), 0, 255).astype(np.uint8)
        name = f'{k:03d}.png'
        cv2.imwrite(str(tmp_path / name), img)
        with torch.no_grad():
            out = net(val_aug(img, cfg.img_size, dev)[None])
        ids_p, class_p, box_p, coef_p, proto_p = nms(*out, net.anchors, cfg)
        ids_p, class_p, boxes_p, _ = after_nms(ids_p, class_p, box_p, coef_p, proto_p, h, w)
        anns = []
        if ids_p is not None:
            bx = boxes_p.cpu().numpy().astype(np.float64)
            ids = ids_p.cpu().numpy()
            for i in range(0, len(ids), 3):
                x1, y1, x2, y2 = np.clip(bx[i] + [2, -1, 3, 1], 0, [w, h, w, h])
                anns.append(dict(bbox=[x1, y1, x2 - x1, y2 - y1], category_id=cat_id[int(ids[i])], iscrowd=0))
        anns.append(dict(bbox=[5.0, 5.0, 35.0, 25.0], category_id=cat_id[(7 * k) % nfg], iscrowd=0))
        anns.append(dict(bbox=[1.0, 2.0, 20.0, 20.0], category_id=cat_id[k % nfg], iscrowd=1))
        for a in anns:
            a['_hw'] = (h, w)
        images[1000 + k] = (name, h, w, anns)
    return _StubCOCO(images)


def _synthetic_net(dev, config, arch):
    """An eval-mode Yolact of `config` at 550 fp16 with synthetic weights of its class count."""
    import time
    from oracle import forward_torch as ft
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    cfg = make_config(config, 550, mode='val')
    cfg.precision, cfg.max_batch = 'fp16', 64
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict(arch, num_classes=cfg.num_classes, seed=0), strict=True)
    net = net.to(dev).eval()
    print(f'\n{config}: net built in {time.time() - t0:.1f} s, peak memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB')
    return net, cfg


@pytest.fixture(scope='module')
def res101(cuda):
    return _synthetic_net(cuda, 'res101_coco', 'res101')


@pytest.fixture(scope='module')
def pascal(cuda):
    """res50_pascal: 21 classes, category ids 1..20 through the identity continuous_id."""
    return _synthetic_net(cuda, 'res50_pascal', 'res50')


def _evaluate_equals_per_image_loop(net, cfg, tmp_path, traditional, val_bss):
    import time
    from val_loop import per_image_evaluate
    from yolact_minimal_b200.eval import evaluate
    from yolact_minimal_b200.utils.coco import COCOValDetection
    t0 = time.time()
    cfg.traditional_nms = traditional
    cfg.val_imgs = str(tmp_path)
    coco = _eval_set(tmp_path, net, cfg)
    ds = COCOValDetection(cfg, coco=coco)
    want = per_image_evaluate(net, cfg, (ds[i] for i in range(len(ds))))
    assert want[1][1] > 0 and want[2][1] > 0                                 # the case has matches in both types
    for val_bs in val_bss:
        for workers in (0, 2):
            cfg.val_bs = val_bs
            got = evaluate(net, cfg, dataset=ds, num_workers=workers)
            assert got == want, (val_bs, workers, got[1:], want[1:])
    print(f'{type(cfg).__name__} traditional={traditional}: {time.time() - t0:.1f} s, peak memory '
          f'{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB')


@pytest.mark.parametrize('traditional', [False, True])
def test_evaluate_equals_per_image_loop(res101, tmp_path, traditional):
    _evaluate_equals_per_image_loop(*res101, tmp_path, traditional, (1, 8, 64))


@pytest.mark.parametrize('traditional', [False, True])
def test_pascal_evaluate_equals_per_image_loop(pascal, tmp_path, traditional):
    net, cfg = pascal
    assert cfg.num_classes == 21 and cfg.continuous_id == {i: i for i in range(1, 21)}
    _evaluate_equals_per_image_loop(net, cfg, tmp_path, traditional, (1, 8))


def _batch_body(net, cfg, packed, ev, dev):
    from yolact_minimal_b200.utils.augmentations import val_aug_batch
    from yolact_minimal_b200.utils.output_utils import after_nms_batched, detect_batched
    with torch.no_grad():
        images = val_aug_batch(packed.buffer, packed.items, cfg.img_size, dev)
        class_p, box_p, coef_p, proto_p = net(images)
    det = detect_batched(class_p, box_p, coef_p, net.anchors, cfg)
    boxes_px, masks = after_nms_batched(det, proto_p, packed.sizes)
    gt, gt_masks = packed.gt_to(dev)
    ev.add(det, boxes_px, masks, gt, packed.gt_offset, gt_masks, packed.sizes)


def test_launches_fixed_and_no_sync(res101, tmp_path):
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.eval import iou_thres
    from yolact_minimal_b200.utils.coco import COCOValDetection, val_collate
    from yolact_minimal_b200.utils.common_utils import MapEvaluator
    net, cfg = res101
    cfg.traditional_nms = False
    cfg.val_imgs = str(tmp_path)
    ds = COCOValDetection(cfg, coco=_eval_set(tmp_path, net, cfg, n=12))
    dev = next(net.parameters()).device
    ev = MapEvaluator(len(cfg.class_names), iou_thres, device=dev)
    batches = [val_collate([ds[i] for i in idx]).pin_memory() for idx in ([0], [1, 2, 3], list(range(3, 12)), [5, 6])]
    _batch_body(net, cfg, batches[0], ev, dev)                               # warm-up: anchors upload, workspaces
    deltas = []
    torch.cuda.set_sync_debug_mode('error')
    try:
        for p in batches[1:]:
            before = _lib.launch_count()
            _batch_body(net, cfg, p, ev, dev)
            deltas.append(_lib.launch_count() - before)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(set(deltas)) == 1, deltas
    assert ev.num_records() > 0
