"""GPU: `detect --jpeg_gpu` writes every file byte for byte as the default path (cv2.imwrite) does, on the folder set-up of
tests/test_detect_batch_gpu.py (mixed sizes, a uniform image and a visual_thre that leaves some images with nothing visible), at
det_bs 1 and 8, for the default options, hide_mask, save_lincomb, cutout and no_crop."""
import os

import pytest

from test_detect_batch_gpu import folder, res101  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

OPTIONS = {'default': {}, 'hide_mask': {'hide_mask': True}, 'save_lincomb': {'save_lincomb': True}, 'cutout': {'cutout': True},
           'no_crop': {'no_crop': True}}


def _files(d):
    out = {}
    for name in sorted(os.listdir(d)):
        with open(os.path.join(d, name), 'rb') as f:
            out[name] = f.read()
    return out


@pytest.mark.parametrize('det_bs', [1, 8])
@pytest.mark.parametrize('opt', list(OPTIONS))
def test_jpeg_gpu_files_equal_default_path(res101, folder, tmp_path, monkeypatch, opt, det_bs):  # noqa: F811
    from yolact_minimal_b200.detect import detect_images
    net, cfg = res101
    path, mid = folder
    base = dict(visual_thre=mid, hide_mask=False, hide_bbox=False, hide_score=False, cutout=False, save_lincomb=False, no_crop=False,
                traditional_nms=False, real_time=False, image=path)
    for k, v in {**base, **OPTIONS[opt]}.items():
        setattr(cfg, k, v)
    got = {}
    try:
        for jpeg_gpu in (False, True):
            d = tmp_path / str(jpeg_gpu)
            os.makedirs(d / 'results' / 'images')
            monkeypatch.chdir(d)
            cfg.jpeg_gpu = jpeg_gpu
            detect_images(net, cfg, det_bs, num_workers=0)
            got[jpeg_gpu] = _files(d / 'results' / 'images')
    finally:
        cfg.jpeg_gpu = False
    want = got[False]
    assert len([n for n in want if n[0].isdigit() and '_' not in n]) >= 8
    if opt == 'save_lincomb':
        assert any(n.startswith('lincomb_') for n in want)
    if opt == 'cutout':
        assert any(n.endswith('_total_obj.jpg') for n in want)
    assert sorted(got[True]) == sorted(want)
    for name in want:
        assert got[True][name] == want[name], name
