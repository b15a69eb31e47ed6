"""GPU: the staged epilogue of the tensor-core convolution (shared-memory segments stored by TMA, the residual loaded by TMA) at
the shapes tests/test_conv_gpu.py does not reach: a residual at every tile width, whose segments are 64-, 32- and 16-column TMA
boxes (176 = 64 + 64 + 32 + 16), BN = 16 without one, ragged last tiles, and a launch of fewer rows than one warpgroup's 64.
Each shape runs in every launch form and is checked as tests/test_conv_gpu.py checks its shapes: against a float64 PyTorch
reference on the same 16-bit-rounded operands, and ('auto') against the CUDA-core kernel."""
import pytest
import torch

from test_conv_gpu import conv_case, reference, run_conv

pytestmark = pytest.mark.gpu

# (B, Cin, H, Cout, k, stride, relu, residual)
SHAPES = [
    (2, 64, 17, 64, 1, 1, 1, 1),       # residual, BN = 64
    (1, 128, 20, 128, 3, 1, 1, 1),     # residual, BN = 128, ragged last tile (484 rows)
    (2, 64, 11, 16, 3, 1, 1, 0),       # BN = 16
    (1, 64, 13, 176, 1, 1, 1, 1),      # residual, BN = 176: segments of 64, 64, 32 and 16 columns
    (2, 64, 9, 32, 3, 1, 0, 1),        # residual, BN = 32
    (3, 128, 7, 48, 1, 1, 1, 1),       # residual, BN = 16, three N tiles
    (1, 256, 23, 192, 3, 1, 1, 1),     # residual, BN = 192, ragged last tile (625 rows)
    (2, 128, 35, 256, 1, 2, 1, 1),     # stride 2 + residual, BN = 256
    (5, 64, 6, 64, 3, 1, 1, 1),        # residual, many small images per tile, ragged last tile (320 rows)
    (1, 64, 3, 16, 1, 1, 0, 1),        # residual, 25 rows: the second consumer warpgroup has no valid row
]


@pytest.mark.parametrize('form', ['auto', 'single', 'pair'])
@pytest.mark.parametrize('precision', ['bf16', 'fp16'])
@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: 'B%d_Cin%d_H%d_Cout%d_k%d_s%d_relu%d_res%d' % s)
def test_conv_staged_epilogue(cuda, shape, precision, form, monkeypatch):
    """`form` forces the launch form: one CTA per 128-row tile, or a CTA pair; 'auto' is the per-layer choice of the engine."""
    if form != 'auto':
        monkeypatch.setenv('YOLACT_B200_PAIR', '1' if form == 'pair' else '0')
    B, Cin, H, Cout, k, stride, relu, res = shape
    x, w, b, r = conv_case(6, B, Cin, H, Cout, k, stride, res)
    prec, rnd, eps = (1, torch.bfloat16, 2.0 ** -8) if precision == 'bf16' else (2, torch.float16, 2.0 ** -11)
    ref = reference(cuda, x, w, b, r, k, stride, relu, rnd)
    y_tc = run_conv(cuda, x, w, b, r, k, stride, relu, prec, 1)
    scale = max(1.0, float(ref.abs().max()))
    err = float((y_tc - ref).abs().max())
    assert err < 1.5 * eps * scale, (err, scale)          # only the final 16-bit rounding of the output
    if form == 'auto':
        y_simt = run_conv(cuda, x, w, b, r, k, stride, relu, prec, 0)
        assert float((y_tc - y_simt).abs().max()) < 1.5 * eps * scale       # same math on CUDA cores
