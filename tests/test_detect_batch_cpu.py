"""Host side of batched detection: DetectImages follows the reference's sorted glob of *.jpg, detect_collate packs the images
back to back with their yb_val_aug_item table, and yb_draw_masks_batch / yb_draw_lincomb refuse malformed arguments before any
device work (fake device pointers are never touched)."""
import types

import numpy as np

from yolact_minimal_b200 import _lib


def test_detect_images_and_collate(tmp_path):
    import cv2
    from yolact_minimal_b200.utils.coco import DetectImages, detect_collate
    rng = np.random.RandomState(0)
    imgs = {'b.jpg': (30, 41), 'a.jpg': (7, 97), 'c.jpg': (64, 32)}
    for name, (h, w) in imgs.items():
        cv2.imwrite(str(tmp_path / name), rng.randint(0, 256, size=(h, w, 3), dtype=np.uint8))
    (tmp_path / 'd.png').write_bytes(b'')
    ds = DetectImages(types.SimpleNamespace(image=str(tmp_path)))
    assert len(ds) == 3
    samples = [ds[i] for i in range(3)]
    assert [s[1] for s in samples] == ['a.jpg', 'b.jpg', 'c.jpg']
    packed = detect_collate(samples)
    assert packed.names == ['a.jpg', 'b.jpg', 'c.jpg'] and packed.sizes == [(7, 97), (30, 41), (64, 32)] and len(packed) == 3
    for b, (img, _) in enumerate(samples):
        assert np.array_equal(packed.image(b), img)
        assert np.array_equal(packed.image(b), cv2.imread(str(tmp_path / packed.names[b])))


def test_malformed_arguments_refused_before_launch():
    from yolact_minimal_b200.utils.augmentations import VAL_ITEM_DTYPE
    L = _lib.lib()
    fake, out_far = 1 << 40, 1 << 41

    def draw(items, off, src_bytes=10 ** 6, words=10 ** 9, D=100, nc=80, ws=1 << 20, out=out_far, count=fake):
        items, off = np.asarray(items, VAL_ITEM_DTYPE), np.asarray(off, np.int64)
        return L.yb_draw_masks_batch(fake, src_bytes, items.ctypes.data, len(items), fake, off.ctypes.data, words, D, fake, count, fake, nc,
                                     fake, ws, out, None)

    need = lambda h, w: 100 * h * ((w + 31) // 32)
    items = [(0, 480, 640), (480 * 640 * 3, 1, 97)]
    off = [0, need(480, 640), need(480, 640) + need(1, 97)]
    assert draw(items, [0, need(480, 640) - 1, 10 ** 7]) == -1                       # image 0's masks overlap image 1's
    assert draw(items, off, words=off[-1] - 1) == -1                                 # past the mask buffer
    assert draw([(0, 480, 640), (480 * 640 * 3 - 1, 1, 97)], off, src_bytes=480 * 640 * 3 + 289) == -1   # image past src
    assert draw([(0, 0, 640), (0, 1, 97)], off) == -1
    assert draw(items, off, out=fake + 5) == -1                                      # out overlaps src
    assert draw(items, off, ws=8) == -1
    assert draw(items, off, D=0) == -3 and draw(items, off, D=5000) == -3
    assert draw(items, off, nc=0) == -1
    assert draw(items, off, count=None) == -1                                        # the count is required

    def lincomb(K=32, B=2, P=138, count=fake):
        return L.yb_draw_lincomb(fake, fake, count, B, 100, P, K, fake, fake, None)

    assert lincomb(K=16) == -3 and lincomb(K=64) == -3                              # the 4 x 8 grid needs 32 channels
    assert lincomb(B=0) == -1 and lincomb(P=0) == -1
    assert L.yb_draw_lincomb(None, fake, fake, 2, 100, 138, 32, fake, fake, None) == -1
