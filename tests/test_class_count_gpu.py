"""GPU: one class bound, 2 .. YB_MAX_CLASSES = 129 (background included), at every entry point.

  * yb_net_create and yb_train_create accept 129 and refuse 130 (and 1000) with YB_ERR_UNSUPPORTED, at create time;
  * a 129-class net runs its forward (k_head_finalize holds five logits per lane) and its detections equal the oracle's, with
    Fast-NMS and traditional NMS;
  * yb_detect refuses 130 classes, and 129 classes with max_det = 256 (the final top-k's keys would need 257 KiB of shared
    memory), before anything is launched or written; 129 classes with max_det = 100 run;
  * yb_losses accepts 129 and refuses 130 (YB_ERR_INVALID) without writing an output.
The op-by-op check of the 129-class forward, and its equality with yb_net_forward, are in test_forward_ops_gpu.py."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import synth, forward_torch as ft, postprocess_np as pp
from test_postprocess_gpu import _cfg, _run, _check_image
from test_traditional_nms_gpu import _raw_detect

pytestmark = pytest.mark.gpu

YB_ERR_INVALID, YB_ERR_UNSUPPORTED = -1, -3


def test_create_bound(cuda):
    from yolact_minimal_b200 import _lib
    L = _lib.lib()
    for nc, want in ((1, YB_ERR_INVALID), (2, 0), (129, 0), (130, YB_ERR_UNSUPPORTED), (1000, YB_ERR_UNSUPPORTED)):
        cfg = _lib.NetConfig(50, 128, nc, 3, 32)
        h = ctypes.c_void_p()
        assert L.yb_net_create(ctypes.byref(cfg), ctypes.byref(h)) == want, nc
        if want == 0:
            L.yb_net_destroy(h)
        elif nc > 2:
            assert b'num_classes' in L.yb_last_error()
        t = ctypes.c_void_p()
        assert L.yb_train_create(ctypes.byref(cfg), 2, 1, ctypes.byref(t)) == (YB_ERR_UNSUPPORTED if want else 0), nc
        if want == 0:
            L.yb_train_destroy(t)


def test_forward_and_detect_at_129(cuda):
    """Yolact at 129 classes, fp32, against the fp32 torch forward (smoke()'s tolerance), then its detections against the oracle."""
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    S, arch, NC = 128, 'res50', 129
    sd = ft.synth_state_dict(arch, num_classes=NC, seed=0)
    img = synth.image_batch(11, 2, S)
    ref = [t.numpy() for t in ft.forward(torch.from_numpy(img), sd, arch, num_classes=NC)]
    cfg = make_config(arch + '_coco', S)
    cfg.num_classes, cfg.precision = NC, 'fp32'
    net = Yolact(cfg)
    net.load_state_dict(sd, strict=True)
    net = net.to(cuda).eval()
    with torch.no_grad():
        out = [t.cpu().numpy() for t in net(torch.from_numpy(img).to(cuda))]
    assert out[0].shape == (2, ref[0].shape[1], NC)
    for name, m, r in zip(('cls', 'box', 'coef', 'proto'), out, ref):
        assert np.abs(m - r).max() < 1e-3, name
    assert np.allclose(out[0].sum(-1), 1, atol=1e-5)
    anchors = pp.make_anchors(S)
    cls, box, coef = (np.ascontiguousarray(o) for o in out[:3])
    for traditional in (False, True):
        r = _run(cuda, cls, box, coef, anchors, _cfg(traditional, S=S, classes=NC))
        for b in range(2):
            _check_image(r, b, pp.nms(cls[b], box[b], anchors, traditional=traditional, img_size=S), coef[b])


def test_detect_refuses_before_launching(cuda):
    """A refused yb_detect launches no kernel and leaves every output and workspace byte as it was; max_det = 100 at 129 classes,
    next to the refused max_det = 256, runs and equals the oracle."""
    from yolact_minimal_b200 import _lib
    S = 128
    anchors = pp.make_anchors(S)
    A = anchors.shape[0]
    for C, max_det in ((129, 256), (130, 100)):
        cls, box, coef = synth.head_outputs(61, A, C, 'stress')
        for traditional in (0, 1):
            before = _lib.launch_count()
            st, ws, out = _raw_detect(cuda, cls[None], box[None], coef[None], anchors, S, 0xA5, max_det=max_det, traditional=traditional)
            assert st == YB_ERR_UNSUPPORTED, (C, max_det, traditional, st)
            assert _lib.launch_count() == before
            assert bool((ws == 0xA5).all())
            for k, v in out.items():
                assert bool((v == 0xA5).all()), k
    cls, box, coef = synth.head_outputs(61, A, 129, 'stress')
    for traditional in (0, 1):
        st, _, out = _raw_detect(cuda, cls[None], box[None], coef[None], anchors, S, 0xA5, max_det=100, traditional=traditional)
        assert st == 0
        o = pp.nms(cls, box, anchors, traditional=bool(traditional), img_size=S)
        d = len(o[0])
        assert d == 100 and out['count'].view(torch.int32).item() == d
        assert np.array_equal(out['cls'].view(torch.int32).cpu().numpy()[:d], o[0])
        assert np.array_equal(out['anchor'].view(torch.int32).cpu().numpy()[:d], o[3])


def test_losses_bound(cuda):
    """yb_losses at 129 classes runs; at 130 it returns YB_ERR_INVALID and leaves its sentinel-filled outputs alone."""
    import train_checks as tc
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    S, B = 128, 2
    cfg = make_config('res50_coco', S, mode='train', train_bs=B)
    a = Yolact(cfg).anchors
    anchors = (a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)).reshape(-1, 4).astype(np.float32)
    A, P, Hs = anchors.shape[0], S // 4, S // 8
    for C in (129, 130):
        tg, mk = synth.train_targets(9, B, S, n=4, num_classes=C - 1)
        args = [synth.normal(21, 1, (B, A, C)).astype(np.float32), np.zeros((B, A, 4), np.float32), np.zeros((B, A, 32), np.float32),
                np.zeros((B, P, P, 32), np.float32), np.zeros((B, C - 1, Hs, Hs), np.float32)]
        r = tc.run_native_losses(cuda, cfg, anchors, tg, mk, *args, sentinel=-7, check=False)
        if C == 129:
            assert r['status'] == 0 and np.isfinite(r['losses']).all() and (r['d_cls'] != -7).all()
        else:
            assert r['status'] == YB_ERR_INVALID
            for k in ('losses', 'labels', 'd_cls', 'd_seg'):
                assert (r[k] == -7).all(), k
