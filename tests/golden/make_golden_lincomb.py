#!/usr/bin/env python
"""Golden vectors of draw_lincomb (TEST INFRASTRUCTURE).  Runs only where a read-only checkout of the reference is named by
$YOLACT_REFERENCE; it writes tests/golden/lincomb.npz and touches no other fixture.

    python tests/golden/make_golden_lincomb.py

It imports the UNMODIFIED reference utils/output_utils.py the way make_golden_draw.py does, aliases np.float = float so the
reference's arr_run line (dead code: arr_run is never written) runs under numpy >= 1.24, captures the array its cv2.imwrite call
receives, and runs draw_lincomb(proto, coef, name) on the inputs of tests/lincomb_np.case_inputs() for the cases without tied
|coef| (the reference orders ties by numpy's unstable argsort).  It stores the colour-table index of every pixel (a third of
the image's bytes): COLORMAP_WINTER's 256 entries are distinct, and the image is checked to be the table applied to them.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import lincomb_np as ln  # noqa: E402
from make_golden_draw import import_reference  # noqa: E402


def main():
    import torch
    rou = import_reference()
    np.float = float
    writes = []
    rou.cv2.imwrite = lambda path, arr, *a: writes.append((path, np.array(arr))) or True
    lut = ln.winter_lut()
    out = {}
    for name in ln.GOLDEN_CASES:
        proto, coef = ln.case_inputs(name)
        assert not ln.has_tie(coef), name
        writes.clear()
        rou.draw_lincomb(torch.from_numpy(proto), torch.from_numpy(coef), f'{name}.jpg')
        (path, img), = writes
        assert path == f'results/images/lincomb_{name}.jpg', path
        assert img.dtype == np.uint8 and img.shape == (4 * proto.shape[0], 8 * proto.shape[0], 3)
        if name == 'p136_zero':                              # 0 / 0 -> NaN -> byte 0 on x86-64
            P = proto.shape[0]
            i = int(np.argsort(-np.abs(coef[0]), kind='stable').tolist().index(ln.ZERO_CHANNEL))
            r, c = divmod(i, 8)
            assert (img[r * P:(r + 1) * P, c * P:(c + 1) * P] == lut[0]).all()
        idx = ln.lut_index(img, lut)
        assert np.array_equal(lut[idx], img)
        out[name] = idx
    np.savez_compressed(os.path.join(HERE, 'lincomb.npz'), **out)
    print('wrote', os.path.join(HERE, 'lincomb.npz'), len(out), 'arrays')


if __name__ == '__main__':
    main()
