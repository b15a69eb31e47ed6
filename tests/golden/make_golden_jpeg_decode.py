"""Writes tests/golden/jpeg_decode.npz: for every file of tests/jpeg_decode_corpus.py, the sha256 of the file cv2 wrote and of the
pixels cv2.imread returned, and for the small ones the file and the pixels themselves.  This pins the expected decode to one
libjpeg-turbo build (3.1.2 in the cv2 that minted it), as jpeg.npz pins the encoder.

    python tests/golden/make_golden_jpeg_decode.py
"""
import hashlib
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import jpeg_decode_corpus  # noqa: E402


def main():
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for name, data in jpeg_decode_corpus.corpus():
            img = jpeg_decode_corpus.cv2_decode(data, d)
            out[f'file_sha256/{name}'] = np.frombuffer(hashlib.sha256(data).digest(), np.uint8)
            out[f'pixels_sha256/{name}'] = np.frombuffer(hashlib.sha256(img.tobytes()).digest(), np.uint8)
            out[f'shape/{name}'] = np.array(img.shape, np.int64)
            if len(data) <= 4096:
                out[f'file/{name}'] = np.frombuffer(data, np.uint8)
                out[f'pixels/{name}'] = img
    np.savez_compressed(os.path.join(HERE, 'jpeg_decode.npz'), **out)


if __name__ == '__main__':
    main()
