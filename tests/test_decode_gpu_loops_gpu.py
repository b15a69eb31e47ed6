"""GPU: with decode_gpu the detect and evaluate loops decode their JPEG inputs on the device and give what the default path gives:
  * `detect --decode_gpu` writes the same files, byte for byte, at det_bs 1 and 8, on tests/test_detect_batch_gpu.py's folder plus
    a 4:4:4 file with restart markers and a progressive file (read by cv2 in the worker), with the default options and hide_mask
    (which draws on the decoded pixels copied back to the host);
  * `evaluate(..., decode_gpu)` returns the same (table, box_row, mask_row) on tests/test_val_batch_gpu.py's evaluation set
    re-encoded as JPEG (4:2:0, 4:2:2 and 4:4:4, with and without restart markers, some files progressive)."""
import os
import shutil

import pytest

import jpeg_decode_corpus
from test_detect_batch_gpu import folder, res101  # noqa: F401  (fixtures)
from test_val_batch_gpu import _eval_set

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def res101_val(cuda):
    """test_val_batch_gpu.py's network: res101 at 550, fp16, max_batch 64, in val mode."""
    from oracle import forward_torch as ft
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    cfg = make_config('res101_coco', 550, mode='val')
    cfg.precision, cfg.max_batch = 'fp16', 64
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict('res101', seed=0), strict=True)
    return net.to(cuda).eval(), cfg


def _files(d):
    out = {}
    for name in sorted(os.listdir(d)):
        with open(os.path.join(d, name), 'rb') as f:
            out[name] = f.read()
    return out


@pytest.mark.parametrize('det_bs', [1, 8])
@pytest.mark.parametrize('opt', ['default', 'hide_mask'])
def test_detect_decode_gpu_files_equal_default_path(res101, folder, tmp_path, monkeypatch, opt, det_bs):  # noqa: F811
    import cv2
    from yolact_minimal_b200.detect import detect_images
    net, cfg = res101
    path, mid = folder
    images = tmp_path / 'images'
    shutil.copytree(path, images)
    src = cv2.imread(os.path.join(path, '000.jpg'))
    (images / '100_prog.jpg').write_bytes(jpeg_decode_corpus.encode(src, 90, '420', progressive=True))
    (images / '101_rst.jpg').write_bytes(jpeg_decode_corpus.encode(src[:301, :333], 95, '444', rst=2))
    base = dict(visual_thre=mid, hide_mask=opt == 'hide_mask', hide_bbox=False, hide_score=False, cutout=False, save_lincomb=False,
                no_crop=False, traditional_nms=False, real_time=False, image=str(images), jpeg_gpu=False)
    for k, v in base.items():
        setattr(cfg, k, v)
    got = {}
    try:
        for decode_gpu in (False, True):
            d = tmp_path / str(decode_gpu)
            os.makedirs(d / 'results' / 'images')
            monkeypatch.chdir(d)
            cfg.decode_gpu = decode_gpu
            detect_images(net, cfg, det_bs, num_workers=0 if det_bs == 1 else 2)
            got[decode_gpu] = _files(d / 'results' / 'images')
    finally:
        cfg.decode_gpu = False
    want = got[False]
    assert len(want) == 13
    assert sorted(got[True]) == sorted(want)
    for name in want:
        assert got[True][name] == want[name], name


def test_evaluate_decode_gpu_equals_default_path(res101_val, tmp_path):
    import cv2
    from yolact_minimal_b200.eval import evaluate
    from yolact_minimal_b200.utils.augmentations import EncodedImage
    from yolact_minimal_b200.utils.coco import COCOValDetection
    net, cfg = res101_val
    cfg.traditional_nms = False
    cfg.val_imgs = str(tmp_path)
    coco = _eval_set(tmp_path, net, cfg, n=21)
    for k, name in enumerate(sorted(p for p in os.listdir(tmp_path) if p.endswith('.png'))):
        img = cv2.imread(str(tmp_path / name))
        layout = ('420', '422', '444')[k % 3]
        data = jpeg_decode_corpus.encode(img, 92, layout, rst=k % 4, progressive=k % 7 == 3)
        (tmp_path / name).write_bytes(data)                   # the file names stay, the contents are JPEG
    rows = {}
    try:
        for decode_gpu in (False, True):
            cfg.decode_gpu = decode_gpu
            ds = COCOValDetection(cfg, coco=coco, decode_gpu=decode_gpu)
            if decode_gpu:
                kinds = [isinstance(ds[i][0], EncodedImage) for i in range(len(ds))]
                assert 0 < kinds.count(False) < kinds.count(True)
            for val_bs in (1, 8):
                cfg.val_bs = val_bs
                rows[(decode_gpu, val_bs)] = evaluate(net, cfg, dataset=ds, num_workers=2)
    finally:
        cfg.decode_gpu = False
    want = rows[(False, 1)]
    assert want[1][1] > 0
    for key, got in rows.items():
        assert got == want, key
