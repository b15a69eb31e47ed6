"""GPU: draw_img's overlay and cutout on the device (csrc/draw.cu behind utils/output_utils.py) equal the reference bit for bit.
  * draw_img on every golden case, for CUDA float32 / uint8 / packed-bit masks and numpy bool masks (after_nms_numpy's form),
    including the arrays handed to cv2.imwrite by cfg.cutout
  * the blend of all 65 536 (colour, pixel) pairs through the C ABI equals cv2.addWeighted
  * 1080x1920 with 100 overlapping detections, every mask format, equals the oracle
  * hide_mask draws into the caller's array; ids_p=None returns it; crops follow numpy's slicing of odd boxes
  * detect.py's loop body (:61-82) with the package's imports on a synthetic res50
  * the overlay is one kernel launch; misuse is refused."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import draw_np as dn

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip('cv2')

CASES = dn.golden_cases()
KINDS = ('f32', 'u8', 'bits', 'np_bool')


def _masks(masks, kind, dev):
    from yolact_minimal_b200.utils.mask_utils import pack_masks
    if kind == 'np_bool':
        return np.asarray(masks) != 0
    m = torch.from_numpy(np.ascontiguousarray(masks, np.float32)).to(dev)
    return {'f32': lambda: m, 'u8': lambda: m.to(torch.uint8), 'bits': lambda: pack_masks(m)}[kind]()


def _dets(ids, scores, boxes, masks, kind, dev):
    """after_nms-like outputs: CUDA tensors (ids int64, scores float32, boxes int32), or numpy arrays for 'np_bool'."""
    m = _masks(masks, kind, dev)
    if kind == 'np_bool':
        return ids, scores, boxes, m
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return t(ids), t(scores), t(boxes), m


def _capture(monkeypatch):
    writes = []
    monkeypatch.setattr(cv2, 'imwrite', lambda path, arr, *a: writes.append((path, np.array(arr))) or True)
    return writes


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_draw_img_equals_reference_golden(cuda, case, kind, monkeypatch):
    from yolact_minimal_b200.utils.output_utils import draw_img
    g = load_golden('draw.npz')
    ids, scores, boxes, masks, img, cfg, name, fps = dn.case_inputs(case)
    writes = _capture(monkeypatch)
    src = img.copy()
    if ids is None:
        res = draw_img(None, None, None, None, src, cfg, img_name=name, fps=fps)
    else:
        res = draw_img(*_dets(ids, scores, boxes, masks, kind, cuda), src, cfg, img_name=name, fps=fps)
    want = g[f'{name}/image']
    assert isinstance(res, np.ndarray) and res.dtype == np.uint8 and np.array_equal(res, want)
    if ids is None or (cfg.hide_mask and not cfg.real_time):
        assert res is src
    elif not cfg.hide_mask:
        assert res is not src and np.array_equal(src, img)        # the caller's image is untouched
    paths = list(g[f'{name}/paths']) if f'{name}/paths' in g.files else []
    assert [p for p, _ in writes] == paths
    for k, (_, a) in enumerate(writes):
        w = g[f'{name}/write{k}']
        assert a.dtype == np.uint8 and a.shape == w.shape and np.array_equal(a, w), (name, k)


def test_blend_all_pairs_through_the_abi(cuda):
    """Pixel (y, x) gets semantic index y (8 bit-plane masks with weights 2^k) and image value x: all 65 536 pairs per channel."""
    from yolact_minimal_b200 import _lib
    L = _lib.lib()
    v = np.arange(256)
    ids = torch.tensor([(1 << k) - 1 for k in range(8)], dtype=torch.int32, device=cuda)
    masks = torch.from_numpy(((v[None, :, None] >> np.arange(8)[:, None, None]) & 1).repeat(256, 2).astype(np.uint8)).to(cuda)
    img_np = np.ascontiguousarray(np.stack([np.broadcast_to(v[None, :], (256, 256)), np.broadcast_to(255 - v[None, :], (256, 256)),
                                            np.broadcast_to((v[None, :] * 7) % 256, (256, 256))], -1).astype(np.uint8))
    pal_np = np.stack([v, (v * 3 + 11) % 256, 255 - v], 1).astype(np.uint8)
    img, pal = torch.from_numpy(img_np).to(cuda), torch.from_numpy(pal_np).to(cuda)
    out = torch.empty_like(img)
    s = torch.cuda.current_stream().cuda_stream
    _lib.check(L.yb_draw_masks(img.data_ptr(), 256, 256, masks.data_ptr(), 0, 8, ids.data_ptr(), pal.data_ptr(), 256, out.data_ptr(), s))
    want = cv2.addWeighted(np.ascontiguousarray(np.broadcast_to(pal_np[:, None, :], (256, 256, 3))), 0.4, img_np, 0.6, 0)
    assert np.array_equal(out.cpu().numpy(), want)
    assert np.array_equal(want[..., 0], dn.blend(v[:, None].repeat(256, 1), v[None, :].repeat(256, 0)))


def _big_case(dev, h=1080, w=1920, n=100, seed=7):
    """n overlapping rectangle / ellipse masks built on the device, and a random image."""
    rng = np.random.default_rng(seed)
    cx, cy = rng.uniform(0, w, n), rng.uniform(0, h, n)
    rx, ry = rng.uniform(40, w / 2, n), rng.uniform(30, h / 2, n)
    ys = torch.arange(h, device=dev, dtype=torch.float32)[None, :, None]
    xs = torch.arange(w, device=dev, dtype=torch.float32)[None, None, :]
    t = lambda a: torch.from_numpy(a.astype(np.float32)).to(dev)[:, None, None]
    ell = ((xs - t(cx)) / t(rx)) ** 2 + ((ys - t(cy)) / t(ry)) ** 2 <= 1
    rect = ((xs - t(cx)).abs() <= t(rx)) & ((ys - t(cy)).abs() <= t(ry))
    masks = torch.where(torch.from_numpy(np.arange(n) % 2 == 0).to(dev)[:, None, None], ell, rect).to(torch.float32)
    ids = rng.integers(0, 80, n)
    ids[:7] = 79
    boxes = np.stack([cx - rx, cy - ry, cx + rx, cy + ry], 1).clip(0, max(h, w)).astype(np.int32)
    scores = np.sort(rng.uniform(0.05, 1, n).astype(np.float32))[::-1].copy()
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    return ids.astype(np.int64), scores, boxes, masks, img


def test_1080p_100_detections_every_format(cuda):
    from yolact_minimal_b200.config import COLORS
    from yolact_minimal_b200.utils.mask_utils import pack_masks
    from yolact_minimal_b200.utils.output_utils import blend_masks, draw_img
    ids, scores, boxes, masks, img = _big_case(cuda)
    masks_np = masks.to(torch.uint8).cpu().numpy()
    assert masks_np.sum(0).max() > 20
    want = dn.overlay(img, ids, masks_np, 81, COLORS)
    img_d, ids_d = torch.from_numpy(img).to(cuda), torch.from_numpy(ids).to(cuda)
    for m in (masks, masks.to(torch.uint8), masks.bool(), pack_masks(masks)):
        assert np.array_equal(blend_masks(img_d, ids_d, m, 81).cpu().numpy(), want), m.dtype
    cfg = dn.draw_cfg(81)
    want_img, _ = dn.draw(ids, scores, boxes, masks_np, img, cfg, COLORS)
    got = draw_img(ids_d, torch.from_numpy(scores).to(cuda), torch.from_numpy(boxes).to(cuda), pack_masks(masks), img, cfg)
    assert np.array_equal(got, want_img)


def test_none_and_hide_mask_return_the_callers_array(cuda):
    from yolact_minimal_b200.utils.output_utils import draw_img
    ids, scores, boxes, masks, img, cfg, name, fps = dn.case_inputs(CASES[1])
    src = img.copy()
    assert draw_img(None, None, None, None, src, cfg) is src and np.array_equal(src, img)
    cfg.hide_mask = True
    res = draw_img(*_dets(ids, scores, boxes, masks, 'bits', cuda), src, cfg)
    assert res is src and not np.array_equal(src, img)            # boxes and labels drawn into the caller's array


def test_cutout_follows_numpy_slicing(cuda, monkeypatch):
    """Boxes with negative, reversed, out-of-image and empty extents: each crop is numpy's slice of the matte."""
    from yolact_minimal_b200.config import COLORS
    from yolact_minimal_b200.utils.output_utils import draw_img
    h, w = 53, 77
    ids, scores, _, masks = dn.detections(5, h, w, True, 81)
    n = len(ids)
    rng = np.random.default_rng(3)
    boxes = rng.integers(-90, 100, (n, 4)).astype(np.int32)
    boxes[0] = (10, 5, 10, 40)
    boxes[1] = (0, 0, w, h)
    boxes[2] = (-3, -60, 200, -1)
    img = dn.test_image(5, h, w)
    cfg = dn.draw_cfg(81, cutout=True, hide_bbox=True)
    _, want = dn.draw(ids, scores, boxes, masks, img.copy(), cfg, COLORS, img_name='odd')
    for kind in KINDS:
        writes = _capture(monkeypatch)
        draw_img(*_dets(ids, scores, boxes, masks, kind, cuda), img.copy(), cfg, img_name='odd')
        assert [p for p, _ in writes] == [p for p, _ in want]
        for (_, a), (_, b) in zip(writes, want):
            assert a.shape == b.shape and np.array_equal(a, b), kind


def test_detect_loop_res50(cuda, monkeypatch, tmp_path):
    """detect.py:61-82 with nms, after_nms, draw_img from the package: the written image == the oracle's drawing of the same
    after_nms outputs on the host."""
    from oracle import forward_torch as ft, synth
    from yolact_minimal_b200.config import COLORS, make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    from yolact_minimal_b200.utils.output_utils import nms, after_nms, draw_img
    monkeypatch.chdir(tmp_path)
    (tmp_path / 'results' / 'images').mkdir(parents=True)
    S = 128
    cfg = make_config('res50_coco', S)
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict('res50', seed=0), strict=True)
    net = net.to(cuda).eval()
    drawn = 0
    for k, (img_h, img_w) in enumerate(((96, 128), (150, 101))):
        img = torch.from_numpy(synth.image_batch(40 + k, 1, S)).to(cuda)
        img_origin = dn.test_image(k, img_h, img_w)
        img_name = f'synthetic_{k}.jpg'
        with torch.no_grad():
            class_p, box_p, coef_p, proto_p = net(img)
        ids_p, class_p, box_p, coef_p, proto_p = nms(class_p, box_p, coef_p, proto_p, net.anchors, cfg)
        ids_p, class_p, boxes_p, masks_p = after_nms(ids_p, class_p, box_p, coef_p, proto_p, img_h, img_w, cfg, img_name=img_name)
        img_numpy = draw_img(ids_p, class_p, boxes_p, masks_p, img_origin, cfg, img_name=img_name)
        assert cv2.imwrite(f'results/images/{img_name}', img_numpy)
        if ids_p is None:
            assert img_numpy is img_origin
            continue
        want, _ = dn.draw(ids_p.cpu().numpy(), class_p.cpu().numpy(), boxes_p.cpu().numpy(), masks_p.cpu().numpy(), img_origin,
                          cfg, COLORS, img_name=img_name)
        assert np.array_equal(img_numpy, want)
        drawn += 1
    assert drawn >= 1
    assert sorted(p.name for p in (tmp_path / 'results' / 'images').iterdir()) == ['synthetic_0.jpg', 'synthetic_1.jpg']


def test_overlay_is_one_launch(cuda, monkeypatch):
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils.output_utils import blend_masks, draw_img
    ids, scores, boxes, masks, img, cfg, name, fps = dn.case_inputs(CASES[1])
    for kind in ('f32', 'u8', 'bits'):
        d = _dets(ids, scores, boxes, masks, kind, cuda)
        img_d = torch.from_numpy(img).to(cuda)
        before = _lib.launch_count()
        blend_masks(img_d, d[0], d[3], 81)
        assert _lib.launch_count() - before == 1
        before = _lib.launch_count()
        draw_img(*d, img, cfg)
        assert _lib.launch_count() - before == 1
    writes = _capture(monkeypatch)
    cfg.cutout = True
    d = _dets(ids, scores, boxes, masks, 'bits', cuda)
    before = _lib.launch_count()
    draw_img(*d, img, cfg, img_name='x')
    assert _lib.launch_count() - before == 3 and len(writes) == len(ids) + 1       # overlay, total_obj, crops


def test_misuse_is_refused(cuda):
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils.output_utils import blend_masks, draw_img
    ids, scores, boxes, masks, img, cfg, name, fps = dn.case_inputs(CASES[3])
    h, w = img.shape[:2]
    d = _dets(ids, scores, boxes, masks, 'f32', cuda)
    with pytest.raises(_lib.YolactB200Error):                    # CPU tensors
        draw_img(d[0].cpu(), *d[1:], img, cfg)
    with pytest.raises(_lib.YolactB200Error):
        draw_img(*d[:3], d[3].cpu(), img, cfg)
    bits = _masks(masks, 'bits', cuda)
    with pytest.raises(_lib.YolactB200Error):                    # packed masks of another image width
        draw_img(*d[:3], torch.cat([bits, bits], 2), img, cfg)
    with pytest.raises(_lib.YolactB200Error):                    # one mask short
        draw_img(*d[:3], d[3][1:], img, cfg)
    with pytest.raises(_lib.YolactB200Error):                    # float64 masks
        draw_img(*d[:3], d[3].double(), img, cfg)
    with pytest.raises(ValueError):                              # not a uint8 HWC image
        draw_img(*d, img.astype(np.float32), cfg)
    with pytest.raises(ValueError):                              # more colours than the palette has
        blend_masks(torch.from_numpy(img).to(cuda), d[0], d[3], 200)
    L = _lib.lib()
    img_d = torch.from_numpy(img).to(cuda)
    out = torch.empty_like(img_d)
    ids32 = d[0].to(torch.int32)
    pal = torch.zeros(300, 3, dtype=torch.uint8, device=cuda)
    m = d[3]
    args = lambda **kw: [kw.get(k, v) for k, v in (('img', img_d.data_ptr()), ('h', h), ('w', w), ('masks', m.data_ptr()), ('fmt', 1),
                                                   ('n', len(ids)), ('ids', ids32.data_ptr()), ('pal', pal.data_ptr()), ('nc', 80),
                                                   ('out', out.data_ptr()), ('stream', None))]
    assert L.yb_draw_masks(*args()) == 0
    torch.cuda.synchronize()
    for bad in (dict(img=None), dict(out=None), dict(masks=None), dict(ids=None), dict(pal=None), dict(h=0), dict(w=-1),
                dict(fmt=3), dict(fmt=-1), dict(nc=0), dict(nc=1025), dict(n=-1), dict(n=4097), dict(masks=m.data_ptr() + 4)):
        assert L.yb_draw_masks(*args(**bad)) != 0, bad
    yyxx = torch.zeros(len(ids), 4, dtype=torch.int32, device=cuda)
    off = torch.zeros(len(ids) + 1, dtype=torch.int64, device=cuda)
    cargs = [img_d.data_ptr(), h, w, m.data_ptr(), 1, len(ids), ids32.data_ptr(), 80, yyxx.data_ptr(), off.data_ptr(), out.data_ptr(),
             pal.data_ptr(), None]
    assert L.yb_draw_cutout(*cargs) == 0
    torch.cuda.synchronize()
    for k in (0, 8, 9, 10, 11):
        bad = list(cargs)
        bad[k] = None
        assert L.yb_draw_cutout(*bad) != 0, k
    assert L.yb_draw_cutout(*cargs[:7], 0, *cargs[8:]) != 0                   # num_colors 0
