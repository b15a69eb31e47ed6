"""GPU: batched detection (python -m yolact_minimal_b200.detect) and its two new kernels, bit for bit:
  * yb_draw_masks_batch image b == yb_draw_masks on image b's first min(count[b], D) masks; count <= 0 copies the image; bytes
    between and after the output images are never written;
  * yb_draw_lincomb == the numpy restatement (tests/lincomb_np.py) and the reference's golden, on hand cases (ties included) and
    on a res101 550 fp16 forward; images with count 0 are not written; after_nms(save_lincomb) writes the golden image;
  * detect's images and video frames == the per-image loop (tests/detect_loop.py) under every option set, at det_bs 1, 3 and 8;
  * the enqueue of a batch never synchronises, and its library launches do not depend on B or the detections."""
import os

import numpy as np
import pytest
import torch

import lincomb_np as ln

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'lincomb.npz')   # colour-table indices
SENT = 0xA5


# ------------------------------------------------------------------------------------------------------------- batched overlay
@pytest.mark.parametrize('seed', [0, 1])
def test_draw_masks_batch_equals_per_image(cuda, seed):
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils.augmentations import VAL_ITEM_DTYPE
    from yolact_minimal_b200.utils.output_utils import _palette, blend_masks
    rng = np.random.RandomState(seed)
    D, num_classes = 100, 81
    sizes = [(1, 97), (33, 33), (480, 640), (427, 640), (1080, 1920), (50, 45), (70, 130)]
    counts = [0, 1, 37, D, D + 5, -3, 12]
    B, gap = len(sizes), 7
    imgs = [rng.randint(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in sizes]
    items = np.zeros(B, VAL_ITEM_DTYPE)
    src = np.full(sum(im.nbytes + gap for im in imgs) + gap, SENT, np.uint8)
    o = gap
    for b, im in enumerate(imgs):
        items[b] = (o, *im.shape[:2])
        src[o:o + im.nbytes] = im.reshape(-1)
        o += im.nbytes + gap
    words = [D * h * ((w + 31) // 32) for h, w in sizes]
    off = np.concatenate([[3], 3 + np.cumsum([n + 5 for n in words])]).astype(np.int64)
    bits = torch.from_numpy(rng.randint(-2 ** 31, 2 ** 31, size=int(off[-1]) + 5, dtype=np.int64).astype(np.int32)).to(cuda)
    for b in range(B):                                      # sparser masks, and some empty ones
        v = bits[int(off[b]):int(off[b]) + words[b]]
        v &= torch.from_numpy(rng.randint(-2 ** 31, 2 ** 31, size=words[b], dtype=np.int64).astype(np.int32)).to(cuda)
        v.view(D, -1)[::9] = 0
    ids = torch.from_numpy(rng.randint(0, num_classes - 1, size=(B, D)).astype(np.int32)).to(cuda)
    count = torch.tensor(counts, dtype=torch.int32, device=cuda)
    src_d = torch.from_numpy(src).to(cuda)
    out = torch.full_like(src_d, SENT)
    pal, nc = _palette(num_classes, cuda)
    L = _lib.lib()
    ws = torch.empty(int(L.yb_draw_masks_batch_workspace_bytes(B)), dtype=torch.uint8, device=cuda)
    _lib.check(L.yb_draw_masks_batch(src_d.data_ptr(), src_d.numel(), items.ctypes.data, B, bits.data_ptr(), off.ctypes.data, bits.numel(),
                                     D, ids.data_ptr(), count.data_ptr(), pal.data_ptr(), nc, ws.data_ptr(), ws.numel(), out.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream), 'yb_draw_masks_batch')
    got = out.cpu().numpy()
    mask = np.ones(len(src), bool)
    for b, (h, w) in enumerate(sizes):
        a = int(items[b]['img_off'])
        mask[a:a + h * w * 3] = False
        mine = got[a:a + h * w * 3].reshape(h, w, 3)
        n = min(max(counts[b], 0), D)
        if n == 0:
            assert np.array_equal(mine, imgs[b]), b                           # copied unchanged
            continue
        m = bits[int(off[b]):int(off[b]) + words[b]].view(D, h, (w + 31) // 32)[:n]
        want = blend_masks(torch.from_numpy(imgs[b]).to(cuda), ids[b, :n], m, num_classes).cpu().numpy()
        assert np.array_equal(mine, want), (b, sizes[b], n)
    assert (got[mask] == SENT).all()                                          # gaps and tail untouched


# ----------------------------------------------------------------------------------------------------------------------- lincomb
def _lincomb_raw(proto, coef, count, cuda):
    """yb_draw_lincomb into an output prefilled with SENT."""
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils.output_utils import _winter_lut
    B, P = proto.shape[0], proto.shape[1]
    out = torch.full((B, 4 * P, 8 * P, 3), SENT, dtype=torch.uint8, device=cuda)
    _lib.check(_lib.lib().yb_draw_lincomb(proto.data_ptr(), coef.data_ptr(), None if count is None else count.data_ptr(), B,
                                          coef.shape[1], P, 32, _winter_lut(proto.device).data_ptr(), out.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream), 'yb_draw_lincomb')
    return out.cpu().numpy()


@pytest.mark.parametrize('name', list(ln.CASES))
def test_lincomb_equals_oracle_and_golden(cuda, name):
    from yolact_minimal_b200.utils.output_utils import lincomb_batched
    proto, coef = ln.case_inputs(name)
    want = ln.lincomb(proto, coef, ln.winter_lut())
    if name in ln.GOLDEN_CASES:
        assert np.array_equal(want, ln.winter_lut()[np.load(GOLDEN)[name]])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    # image 1: the same case with count 0 (not written); image 2: count 2
    proto3, coef3 = t(np.stack([proto] * 3)), t(np.stack([coef] * 3))
    got = _lincomb_raw(proto3, coef3, t(np.array([1, 0, 2], np.int32)), cuda)
    assert np.array_equal(got[0], want) and np.array_equal(got[2], want)
    assert (got[1] == SENT).all()
    assert np.array_equal(_lincomb_raw(proto3, coef3, None, cuda)[1], want)               # NULL count: every image
    assert np.array_equal(lincomb_batched(proto3[:1], {'coef': coef3[:1]})[0].cpu().numpy(), want)


@pytest.fixture(scope='module')
def res101(cuda):
    from oracle import forward_torch as ft
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    cfg = make_config('res101_coco', 550, mode='detect')
    cfg.precision, cfg.max_batch = 'fp16', 8
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict('res101', seed=0), strict=True)
    return net.to(cuda).eval(), cfg


def _scene(k, h, w, rng):
    """Smooth blobs plus noise: enough structure for the synthetic net to fire (as tools/bench_val.py's images)."""
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([128 + 100 * np.sin(xx / (7 + k % 5) + c) * np.cos(yy / (11 + c)) for c in range(3)], -1)
    return np.clip(base + rng.normal(0, 20, size=(h, w, 3)), 0, 255).astype(np.uint8)


def test_lincomb_of_a_forward(res101, cuda):
    from yolact_minimal_b200.utils.augmentations import val_aug
    from yolact_minimal_b200.utils.output_utils import detect_batched, lincomb_batched
    net, cfg = res101
    rng = np.random.RandomState(0)
    imgs = torch.stack([val_aug(_scene(k, 480, 640, rng), 550, cuda) for k in range(3)])
    with torch.no_grad():
        class_p, box_p, coef_p, proto_p = net(imgs)
    det = detect_batched(class_p, box_p, coef_p, net.anchors, cfg)
    count = det['count'].cpu().numpy()
    assert count.max() > 0
    got = lincomb_batched(proto_p, det).cpu().numpy()
    for b in range(3):
        if count[b] > 0:
            want = ln.lincomb(proto_p[b].float().cpu().numpy(), det['coef'][b].cpu().numpy(), ln.winter_lut())
            assert np.array_equal(got[b], want), b
        else:
            assert not got[b].any(), b


def test_after_nms_save_lincomb_writes_golden(cuda, monkeypatch):
    import cv2
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.utils.output_utils import after_nms
    writes = {}
    monkeypatch.setattr(cv2, 'imwrite', lambda path, arr, *a: writes.__setitem__(path, np.array(arr)) or True)
    cfg = make_config('res101_coco', 550, save_lincomb=True)
    for name in ln.GOLDEN_CASES:
        proto, coef = ln.case_inputs(name)
        t = lambda a: torch.from_numpy(a).to(cuda)
        d = coef.shape[0]
        box = t(np.tile(np.array([[0.1, 0.1, 0.6, 0.7]], np.float32), (d, 1)))
        r = after_nms(t(np.arange(d)), t(np.linspace(0.9, 0.5, d).astype(np.float32)), box, t(coef), t(proto), 60, 80, cfg,
                      img_name=f'{name}.jpg')
        assert r[0] is not None
        assert np.array_equal(writes.pop(f'results/images/lincomb_{name}.jpg'), ln.winter_lut()[np.load(GOLDEN)[name]]), name
    assert not writes


# ------------------------------------------------------------------------------------------------------------------- end to end
SIZES = [(480, 640), (640, 480), (427, 640), (300, 200), (97, 131), (550, 550), (33, 65)]
N_IMAGES = 11


@pytest.fixture(scope='module')
def folder(res101, tmp_path_factory):
    """N_IMAGES synthetic JPEGs of mixed sizes, and visual_thre values that leave some images with nothing visible."""
    import cv2
    from detect_loop import _one
    d = tmp_path_factory.mktemp('detect_images')
    rng = np.random.RandomState(5)
    for k in range(N_IMAGES):
        h, w = SIZES[k % len(SIZES)]
        img = _scene(k, h, w, rng) if k != 4 else np.full((h, w, 3), 128, np.uint8)
        cv2.imwrite(str(d / f'{k:03d}.jpg'), img)
    # the per-image best score at visual_thre 0 picks a threshold between the images' best scores
    net, cfg = res101
    best = []
    from yolact_minimal_b200.utils.augmentations import val_aug
    from yolact_minimal_b200.utils.output_utils import nms
    for k in range(N_IMAGES):
        img = cv2.imread(str(d / f'{k:03d}.jpg'))
        with torch.no_grad():
            out = net(val_aug(img, cfg.img_size, next(net.parameters()).device)[None])
        r = nms(*out, net.anchors, cfg)
        best.append(0.0 if r[0] is None else float(r[1][0]))
    best = sorted(best)
    assert best[-1] > 0, best
    mid = float(np.float32((best[len(best) // 3] + best[len(best) // 3 + 1]) / 2))
    return str(d), mid


def _capture(monkeypatch):
    import cv2
    writes = {}

    def imwrite(path, arr, *a):
        assert path not in writes, path
        writes[path] = np.array(arr)
        return True
    monkeypatch.setattr(cv2, 'imwrite', imwrite)
    return writes


OPTIONS = {'default': {}, 'thre0': {'visual_thre': 0.0}, 'thre03': {'visual_thre': 0.3}, 'hide_mask': {'hide_mask': True},
           'hide_bbox_score': {'hide_bbox': True, 'hide_score': True}, 'cutout': {'cutout': True},
           'save_lincomb': {'save_lincomb': True}, 'no_crop': {'no_crop': True}, 'traditional_nms': {'traditional_nms': True}}


@pytest.mark.parametrize('opt', list(OPTIONS))
def test_images_equal_per_image_loop(res101, folder, monkeypatch, opt):
    import glob

    import cv2
    from detect_loop import per_image_detect
    from yolact_minimal_b200.detect import detect_images
    net, cfg = res101
    path, mid = folder
    base = dict(visual_thre=mid, hide_mask=False, hide_bbox=False, hide_score=False, cutout=False, save_lincomb=False, no_crop=False,
                traditional_nms=False, real_time=False, image=path)
    for k, v in {**base, **OPTIONS[opt]}.items():
        setattr(cfg, k, v)
    writes = _capture(monkeypatch)
    per_image_detect(net, cfg, sorted(glob.glob(path + '/*.jpg')))
    want = dict(writes)
    assert len([p for p in want if p.startswith('results/images/0')]) >= N_IMAGES
    if opt == 'default':
        drawn = [p for p in want if not np.array_equal(want[p], cv2.imread(os.path.join(path, p.split('/')[-1])))]
        assert 0 < len(drawn) < N_IMAGES, drawn                                 # some images drawn, some with nothing visible
    if opt == 'save_lincomb':
        assert any('lincomb_' in p for p in want)
    if opt == 'cutout':
        assert any(p.endswith('_total_obj.jpg') for p in want)
    for det_bs, workers in ((1, 0), (3, 2), (8, 0)):
        writes.clear()
        detect_images(net, cfg, det_bs, num_workers=workers)
        assert sorted(writes) == sorted(want), (det_bs, set(writes) ^ set(want))
        for p in want:
            assert np.array_equal(writes[p], want[p]), (det_bs, p)


class _Writer:
    frames = []

    def __init__(self, *a, **k):
        pass

    def write(self, f):
        _Writer.frames.append(np.array(f))

    def release(self):
        pass


@pytest.mark.parametrize('opt', ['default', 'hide_mask'])
def test_video_equals_per_frame_loop(res101, folder, tmp_path, monkeypatch, opt):
    import cv2
    from detect_loop import per_frame_detect
    from yolact_minimal_b200.detect import detect_video
    net, cfg = res101
    _, mid = folder
    video = str(tmp_path / 'clip.avi')
    vw = cv2.VideoWriter(video, cv2.VideoWriter_fourcc(*'MJPG'), 10, (320, 240))
    rng = np.random.RandomState(2)
    for k in range(10):
        vw.write(_scene(k % 3, 240, 320, rng))
    vw.release()
    assert round(cv2.VideoCapture(video).get(cv2.CAP_PROP_FRAME_COUNT)) == 10
    for k, v in dict(visual_thre=mid, hide_mask=opt == 'hide_mask', hide_bbox=False, hide_score=False, cutout=False, save_lincomb=False,
                     no_crop=False, traditional_nms=False, real_time=False, video=video).items():
        setattr(cfg, k, v)
    _capture(monkeypatch)
    _Writer.frames = []
    per_frame_detect(net, cfg, video, _Writer())
    want = _Writer.frames
    assert len(want) == 10
    monkeypatch.setattr(cv2, 'VideoWriter', _Writer)
    for det_bs in (1, 3, 8):
        _Writer.frames = []
        detect_video(net, cfg, det_bs)
        assert len(_Writer.frames) == 10
        for i, (a, b) in enumerate(zip(_Writer.frames, want)):
            assert np.array_equal(a, b), (det_bs, i)


def test_enqueue_never_syncs_and_launches_are_fixed(res101, folder, monkeypatch):
    import cv2
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.detect import _HostBuffers, enqueue, finish
    from yolact_minimal_b200.utils.coco import DetectImages, detect_collate
    net, cfg = res101
    path, mid = folder
    for k, v in dict(visual_thre=mid, hide_mask=False, hide_bbox=False, hide_score=False, cutout=False, save_lincomb=True, no_crop=False,
                     traditional_nms=False, real_time=False, image=path).items():
        setattr(cfg, k, v)
    monkeypatch.setattr(cv2, 'imwrite', lambda *a: True)
    ds = DetectImages(cfg)
    batches = [detect_collate([ds[i] for i in idx]).pin_memory() for idx in ([0], [1, 2, 3], list(range(3, 11)), [4], [5, 6])]
    hosts = (_HostBuffers(), _HostBuffers())
    finish(enqueue(net, cfg, batches[0], hosts[0]), cfg, lambda *a: None)          # warm-up: anchors, palette, colour table
    deltas = []
    for i, p in enumerate(batches[1:]):
        torch.cuda.set_sync_debug_mode('error')
        try:
            before = _lib.launch_count()
            pending = enqueue(net, cfg, p, hosts[i % 2])
            deltas.append(_lib.launch_count() - before)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        finish(pending, cfg, lambda *a: None)
    assert len(set(deltas)) == 1, deltas
