"""Mints tests/golden/jpeg.npz: what cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, q]) writes for every image of the JPEG
test corpus (tests/jpeg_corpus.py) at q 95, 100 and 50, so the numpy oracle and the CUDA encoder are pinned to one libjpeg-turbo
build even where another cv2 is installed.  Per case '{name}@{q}': the file's SHA-256 and length; files of at most 64x64 pixels
are stored whole.

    python tests/golden/make_golden_jpeg.py
"""
import hashlib
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import jpeg_corpus  # noqa: E402


def main():
    out = {'cv2_version': np.array(cv2.__version__)}
    for name, img in jpeg_corpus.corpus():
        for q in jpeg_corpus.QUALITIES:
            data = cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()
            key = f'{name}@{q}'
            out[f'sha256/{key}'] = np.frombuffer(hashlib.sha256(data).digest(), np.uint8)
            out[f'len/{key}'] = np.array(len(data), np.int64)
            if img.shape[0] * img.shape[1] <= 64 * 64:
                out[f'bytes/{key}'] = np.frombuffer(data, np.uint8)
    np.savez_compressed(os.path.join(HERE, 'jpeg.npz'), **out)


if __name__ == '__main__':
    main()
