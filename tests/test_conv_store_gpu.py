"""GPU: the tensor-core convolution writes only the rows of the images in its launch.

An engine finalized for 4 images runs a batch of 4, then a batch of 3 other images into a caller's `proto` buffer that is
allocated for 4 images and filled with a sentinel.  The proto layer's dense fp32 rows are staged in shared memory and copied
out with 16-byte stores of the valid rows only, so the sentinel must survive past image 3, while images 0-2 are written.
(Image 3 of a stage output cannot be checked the same way: the engine's arena gives a stage output's slot to earlier tensors of
the forward, whose batch-3 images legitimately cover those bytes.)"""
import pytest
import torch

from oracle import synth, forward_torch as ft

pytestmark = pytest.mark.gpu

SENTINEL = 1234.5


def test_proto_rows_past_the_batch_untouched(cuda):
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    arch, S = 'res50', 128
    cfg = make_config(arch + '_coco', S)
    cfg.precision, cfg.max_batch = 'fp16', 4
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict(arch, seed=0), strict=True)
    net = net.to(cuda).eval()
    with torch.no_grad():
        net(torch.from_numpy(synth.image_batch(31, 4, S)).to(cuda))
    eng = net.engine(4)

    img = torch.from_numpy(synth.image_batch(32, 3, S)).to(cuda)
    A, P, C, K = eng.num_anchors, eng.proto_size, eng.cfg.num_classes, eng.cfg.coef_dim
    cls = torch.empty(3, A, C, dtype=torch.float32, device=cuda)
    box = torch.empty(3, A, 4, dtype=torch.float32, device=cuda)
    coef = torch.empty(3, A, K, dtype=torch.float32, device=cuda)
    proto = torch.full((4, P, P, K), SENTINEL, dtype=torch.float32, device=cuda)
    with torch.cuda.device(cuda):
        _lib.check(eng.L.yb_net_forward(eng.h, img.data_ptr(), 3, cls.data_ptr(), box.data_ptr(), coef.data_ptr(), proto.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream), 'yb_net_forward')
    torch.cuda.synchronize()

    assert bool((proto[3] == SENTINEL).all()), 'proto rows past the batch were written'
    assert not bool((proto[:3] == SENTINEL).any()), 'proto rows of the batch were not written'
