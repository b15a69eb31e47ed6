#!/usr/bin/env python
"""Golden vectors of draw_img (TEST INFRASTRUCTURE).  Runs only where a read-only checkout of the reference is named by
$YOLACT_REFERENCE; it writes tests/golden/draw.npz and touches no other fixture.

    python tests/golden/make_golden_draw.py

It imports the UNMODIFIED reference utils/output_utils.py (with a stub cython_nms module in sys.modules: draw_img does not use
it), replaces its module-global COLORS with the package's palette (yolact_minimal_b200.config.COLORS), captures the arrays its
cv2.imwrite calls receive, and runs draw_img on the inputs of oracle/draw_np.golden_cases() -- numpy arrays, float32 masks, as
detect.py hands over after_nms' outputs.  The tests rebuild the inputs from the case table.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ['YOLACT_REFERENCE']
sys.path.insert(0, ROOT)

from oracle import draw_np as dn  # noqa: E402
from yolact_minimal_b200.config import COLORS  # noqa: E402


def import_reference():
    scratch = '/tmp/yolact_ref_cwd'
    os.makedirs(scratch, exist_ok=True)
    os.chdir(scratch)                                        # config.py mkdirs in CWD on import (config.py:6-15)
    stub = types.ModuleType('cython_nms')
    stub.nms = None
    sys.modules['cython_nms'] = stub
    sys.path.insert(0, REF)
    from utils import output_utils as rou
    rou.COLORS = COLORS.astype(np.int64)                     # the package's palette, in the reference table's dtype
    return rou


def main():
    rou = import_reference()
    writes = []
    rou.cv2.imwrite = lambda path, arr, *a: writes.append((path, np.array(arr))) or True
    out = {}
    for case in dn.golden_cases():
        ids, scores, boxes, masks, img, cfg, name, fps = dn.case_inputs(case)
        writes.clear()
        src = img.copy()                                     # hide_mask draws into the caller's array
        res = rou.draw_img(ids, scores, boxes, masks, src, cfg, img_name=name, fps=fps)
        out[f'{name}/image'] = np.asarray(res)
        assert res.dtype == np.uint8
        if writes:
            out[f'{name}/paths'] = np.array([p for p, _ in writes])
            for k, (_, a) in enumerate(writes):
                assert a.size == 0 or (np.array_equal(a, np.round(a)) and a.min() >= 0 and a.max() <= 255)
                out[f'{name}/write{k}'] = a.astype(np.uint8)
    np.savez_compressed(os.path.join(HERE, 'draw.npz'), **out)
    print('wrote', os.path.join(HERE, 'draw.npz'), len(out), 'arrays')


if __name__ == '__main__':
    main()
