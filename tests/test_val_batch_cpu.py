"""CPU: the host side of batched evaluation -- COCOValDetection's annotation rules (the reference's utils/coco.py:69-119 in 'val'
mode), cfg.val_num, the host bit-packing of gt masks, the PackedValBatch layout and its pickle round trip, and the C entry points
refusing malformed tables before anything is launched."""
import ctypes
import pickle
from types import SimpleNamespace

import numpy as np
import pytest

from yolact_minimal_b200 import _lib
from yolact_minimal_b200.config import COCO_LABEL_MAP


class _StubCOCO:
    """The pycocotools.coco.COCO methods COCOValDetection uses; image id k has annotation list anns[k] on an h x w image."""

    def __init__(self, anns, h, w):
        self.anns, self.h, self.w = anns, h, w
        self.imgToAnns = {k: v for k, v in enumerate(anns)}

    def getAnnIds(self, imgIds):
        return [(imgIds, i) for i in range(len(self.anns[imgIds]))]

    def loadAnns(self, ids):
        return [self.anns[k][i] for k, i in ids]

    def loadImgs(self, img_id):
        return [{'file_name': f'{img_id}.jpg'}]

    def annToMask(self, a):
        m = np.zeros((self.h, self.w), np.uint8)
        x, y, w, h = (int(v) for v in a['bbox'])
        m[max(y, 0):y + h, max(x, 0):x + w] = 1
        return m


H, W = 120, 161
ANNS = [dict(bbox=[10.5, 10.25, 50.0, 40.0], category_id=3, iscrowd=0),
        dict(bbox=[5.0, 5.0, 30.0, 30.0], category_id=4, iscrowd=1),      # crowd: dropped
        dict(bbox=[-1.0, 5.0, 30.0, 30.0], category_id=5, iscrowd=0),     # x < 0: kept in val
        dict(bbox=[20.0, 30.0, 3.5, 30.0], category_id=90, iscrowd=0),    # w < 4: kept in val
        dict(bbox=[60.0, 40.0, 101.0, 80.0], category_id=7, iscrowd=0)]


def _cfg(val_num=-1):
    return SimpleNamespace(val_imgs='/nonexistent', val_ann=None, continuous_id=COCO_LABEL_MAP, val_num=val_num, img_size=550)


def _dataset(anns_per_image, val_num=-1):
    from yolact_minimal_b200.utils.coco import COCOValDetection
    ds = COCOValDetection(_cfg(val_num), coco=_StubCOCO(anns_per_image, H, W))
    ds.load_image = lambda name: np.full((H, W, 3), int(name.split('.')[0]) + 1, np.uint8)
    return ds


def _pack_ref(m):
    """numpy restatement of the packed layout: bit x & 31 of word x >> 5 is pixel x."""
    n, h, w = m.shape
    words = np.zeros((n, h, (w + 31) // 32), np.uint64)
    for x in range(w):
        words[..., x >> 5] |= m[..., x].astype(np.uint64) << np.uint64(x & 31)
    return words.astype(np.uint32).view(np.int32)


def test_val_annotation_rules():
    ds = _dataset([ANNS])
    img, gt, bits, (h, w), img_id = ds[0]
    assert img.shape == (H, W, 3) and img.dtype == np.uint8 and (h, w) == (H, W) and img_id == 0
    kept = [a for a in ANNS if not a['iscrowd']]
    # the reference: np.array([x, y, x + w, y + h]) per annotation, / (w, h, w, h) in float64, hstack the labels, float32 in val_collate
    boxes = np.array([np.array([a['bbox'][0], a['bbox'][1], a['bbox'][0] + a['bbox'][2], a['bbox'][1] + a['bbox'][3]]) for a in kept])
    labels = np.array([COCO_LABEL_MAP[a['category_id']] - 1 for a in kept])
    ref = np.hstack((boxes / np.array([W, H, W, H]), np.expand_dims(labels, axis=1)))
    assert gt.dtype == np.float32 and np.array_equal(gt, ref.astype(np.float32))
    assert list(gt[:, 4]) == [2, 4, 79, 6]
    masks = np.stack([ds.coco.annToMask(a) for a in kept])
    assert bits.dtype == np.int32 and np.array_equal(bits, _pack_ref(masks))


def test_no_object_left_raises():
    ds = _dataset([ANNS, [ANNS[1]]])
    ds[0]
    with pytest.raises(RuntimeError):
        ds[1]


def test_val_num():
    assert len(_dataset([ANNS] * 5)) == 5
    assert len(_dataset([ANNS] * 5, val_num=3)) == 3
    assert len(_dataset([ANNS] * 5, val_num=9)) == 5


def test_train_dataset_still_refuses_val():
    from yolact_minimal_b200.utils.coco import COCODetection
    with pytest.raises(ValueError):
        COCODetection(SimpleNamespace(train_imgs='', continuous_id=COCO_LABEL_MAP), mode='val', coco=_StubCOCO([ANNS], H, W))


@pytest.mark.parametrize('w', [1, 31, 32, 33, 640])
def test_host_packing(w):
    from yolact_minimal_b200.utils.mask_utils import pack_masks_host
    m = (np.random.RandomState(w).rand(3, 7, w) > 0.5).astype(np.uint8)
    assert np.array_equal(pack_masks_host(m), _pack_ref(m))


def _check_layout(packed, samples):
    buf = packed.buffer.numpy()
    assert len(packed) == len(samples) and packed.sizes == [s[3] for s in samples] and packed.ids == [s[4] for s in samples]
    off = g = words = 0
    for b, (img, gt, bits, (h, w), _) in enumerate(samples):
        it = packed.items[b]
        assert (it['img_off'], it['h'], it['w']) == (off, h, w)
        assert np.array_equal(buf[off:off + img.nbytes], img.reshape(-1))
        assert packed.gt_offset[b] == g and packed.gt_mask_off[b] == words
        assert np.array_equal(packed.gt.numpy()[g:g + len(gt)], gt)
        assert np.array_equal(packed.gt_masks.numpy()[words:words + bits.size], bits.reshape(-1))
        off, g, words = off + img.nbytes, g + len(gt), words + bits.size
    assert packed.buffer.numel() == off and packed.gt_offset[-1] == g and packed.gt_mask_off[-1] == words
    assert packed.items.dtype.itemsize == ctypes.sizeof(_lib.ValAugItem) == 16


def test_packed_batch_layout_and_pickle():
    from yolact_minimal_b200.utils.coco import val_collate
    ds = _dataset([ANNS, ANNS[:1], ANNS[2:]])
    samples = [ds[i] for i in range(3)]
    packed = val_collate(samples)
    _check_layout(packed, samples)
    _check_layout(pickle.loads(pickle.dumps(packed)), samples)


def test_malformed_tables_refused_before_launch():
    """The host checks run before any device work: fake device pointers are never touched."""
    from yolact_minimal_b200.utils.augmentations import VAL_ITEM_DTYPE
    L = _lib.lib()
    fake = ctypes.c_void_p(1 << 40)

    def val_aug(items, src_bytes=1000, S=550, ws=4096):
        items = np.asarray(items, VAL_ITEM_DTYPE)
        return L.yb_val_aug_batch(fake, src_bytes, items.ctypes.data, len(items), S, fake, ws, fake, None)

    ok = [(0, 10, 10), (300, 10, 10)]
    bad = [[(0, 10, 10), (701, 10, 10)],          # ends past src
           [(-3, 10, 10)], [(0, 0, 10)], [(0, 10, -1)], [(0, 70000, 1)]]
    for items in bad:
        assert val_aug(items) == -1, items
    assert val_aug(ok, S=0) == -1 and val_aug(ok, S=9000) == -1 and val_aug(ok, ws=10) == -1 and val_aug(ok, src_bytes=0) == -1
    assert L.yb_val_aug_batch(fake, 1000, None, 1, 550, fake, 4096, fake, None) == -1

    def masks(hw, off, words=10 ** 9, B=None, D=100, ws=1 << 40):
        hw, off = np.asarray(hw, np.int32), np.asarray(off, np.int64)
        B = len(hw) if B is None else B
        return L.yb_mask_assemble_batch(fake, fake, fake, fake, B, D, 138, 32, hw.ctypes.data, off.ctypes.data, words, 1, fake, ws,
                                        fake, fake, None)

    need = lambda h, w: 100 * h * ((w + 31) // 32)
    good_off = [0, need(480, 640), need(480, 640) + need(1, 97)]
    assert masks([(480, 640), (1, 97)], [0, need(480, 640) - 1, 10 ** 7]) == -1      # image 0 overlaps image 1
    assert masks([(480, 640), (1, 97)], good_off, words=good_off[-1] - 1) == -1        # past the output
    assert masks([(480, 640), (1, 97)], [-1] + good_off[1:]) == -1
    assert masks([(480, 0), (1, 97)], good_off) == -1
    assert masks([(480, 640), (1, 97)], good_off, ws=100) == -1
    assert masks([(480, 640), (1, 97)], good_off, D=0) == -1
    assert L.yb_mask_assemble_batch(fake, fake, fake, None, 2, 100, 138, 32, None, None, 0, 1, fake, 1, fake, fake, None) == -1
