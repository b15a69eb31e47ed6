"""CPU: the train_aug host planner against goldens minted from the reference's own train_aug (cv2), the numpy oracle
of the pixel path within the minted bounds, the collate's refill and packing, and the dataset's annotation rules."""
import os
import random

import numpy as np
import pytest

from oracle import augment_np as an
from yolact_minimal_b200.utils.augmentations import train_aug_plan

HERE = os.path.dirname(os.path.abspath(__file__))
SUB = 23


def golden():
    return np.load(os.path.join(HERE, 'golden', 'train_aug.npz'))


def cases():
    g = golden()
    for c in g['cases']:
        name, h, w, n, kind, S, a, b = str(c).split(':')
        yield name, int(h), int(w), int(n), kind, int(S), range(int(a), int(b))


def sample(name, h, w, n, kind):
    names = [c[0] for c in cases()]
    return an.synthetic_sample(1 + names.index(name), h, w, n, kind)


CASE_NAMES = ['wide', 'tall', 'square', 's544', 'one', 'many', 'tiny', 'zero']


@pytest.mark.parametrize('case', CASE_NAMES)
def test_planner_matches_reference(case):
    """Same random seed -> the reference's boxes (float64, bit for bit), labels, surviving mask indices, None-ness and
    post-call random state;
    after train_collate's float32 conversion the targets are identical."""
    g = golden()
    name, h, w, n, kind, S, seeds = next(c for c in cases() if c[0] == case)
    _, _, boxes, labels = sample(name, h, w, n, kind)
    for seed in seeds:
        key = f'{name}/{seed}'
        random.seed(seed)
        plan = train_aug_plan(h, w, boxes, labels, S)
        assert np.array_equal(np.asarray(random.getstate()[1], dtype=np.int64), g[key + '/state']), key
        assert (plan is None) == bool(g[key + '/none']), key
        if plan is None:
            continue
        assert np.array_equal(plan.boxes, g[key + '/boxes']), key
        assert np.array_equal(plan.labels, g[key + '/labels']), key
        ref_t = np.hstack((g[key + '/boxes'], g[key + '/labels'][:, None])).astype(np.float32)
        assert np.array_equal(np.hstack((plan.boxes, plan.labels[:, None])).astype(np.float32), ref_t)
        assert np.array_equal(plan.keep, g[key + '/keep']), key
        assert len(plan.keep) == len(g[key + '/mask_sum'])


@pytest.mark.parametrize('case', CASE_NAMES)
def test_oracle_pixels_within_minted_bound(case):
    """oracle/augment_np fed the plan vs the reference's pixels; uint8-path masks exact."""
    g = golden()
    tol_img, tol_mask = float(g['img_err']) * 1.01 + 1e-7, float(g['mask_err']) * 1.01 + 1e-7
    name, h, w, n, kind, S, seeds = next(c for c in cases() if c[0] == case)
    img, masks, boxes, labels = sample(name, h, w, n, kind)
    for seed in seeds:
        key = f'{name}/{seed}'
        random.seed(seed)
        plan = train_aug_plan(h, w, boxes, labels, S)
        if plan is None:
            continue
        o_img, o_masks = an.train_aug_pixels(img, masks, plan)
        assert o_img.shape == (3, S, S) and o_masks.shape == (len(plan.keep), S, S)
        assert np.abs(o_img[:, ::SUB, ::SUB] - g[key + '/img_sub']).max() <= tol_img, key
        assert np.abs(o_masks[:, ::SUB, ::SUB] - g[key + '/mask_sub']).max() <= (0 if plan.mask_u8 else tol_mask), key
        np.testing.assert_allclose(o_img.astype(np.float64).sum(axis=(1, 2)), g[key + '/img_sum'], atol=tol_img * S * S / 50, err_msg=key)
        np.testing.assert_allclose(o_masks.astype(np.float64).sum(axis=(1, 2)), g[key + '/mask_sum'], atol=tol_mask * S * S / 50 + 1e-6,
                                   err_msg=key)


def test_hsv_round_trip_within_minted_bound():
    g = golden()
    bgr, sat, hue = an.hsv_triples(7, 1 << 18)
    mine = an.hsv_round_trip(bgr, sat, hue)
    assert (mine < 0).any()                     # S > 1 drives channels negative before the clip
    assert np.abs(mine[::8] - g['hsv/sub']).max() <= float(g['hsv/err']) * 1.01 + 1e-6


def test_crop_gives_up_after_1000_tries():
    """Only zero-area boxes: no window keeps one (0/0 is NaN), so a crop draws 1000 (x, y) pairs and the plan is None.
    The golden 'zero' case pins the post-call random state against the reference."""
    boxes = np.array([[10.0, 10.0, 10.0, 50.0]])
    for seed in range(20):
        random.seed(seed)
        assert train_aug_plan(100, 200, boxes, [3], 550) is None


def test_mirror_and_plan_fields():
    boxes = np.array([[10.0, 20.0, 110.0, 220.0]])
    for seed in range(200):
        random.seed(seed)
        p = train_aug_plan(300, 400, boxes, [5], 550)
        if p is not None and p.mirror and p.crop == (0, 0, 400, 300):
            # mirror x1' = w - x2, x2' = w - x1, then pad y, scale, to_train_size offset
            x1, x2 = (400 - 110.0) * (p.resize / p.square), (400 - 10.0) * (p.resize / p.square)
            if p.resize < 550:
                x1, x2 = x1 + p.train_off[0], x2 + p.train_off[0]
                assert p.boxes[0, 0] == np.clip(x1, 0, 549) / 550 and p.boxes[0, 2] == np.clip(x2, 0, 549) / 550
                assert p.square == 400 and p.pad[0] == 0 and not p.mask_u8
                return
    pytest.fail('no seed mirrored without a crop and padded')


class _StubCOCO:
    """The pycocotools.coco.COCO methods COCODetection uses, over an in-memory annotation list."""

    def __init__(self, anns, h, w):
        self.anns, self.h, self.w = anns, h, w
        self.imgToAnns = {1: anns}

    def getAnnIds(self, imgIds):
        return list(range(len(self.anns)))

    def loadAnns(self, ids):
        return [self.anns[i] for i in ids]

    def loadImgs(self, img_id):
        return [{'file_name': 'x.jpg'}]

    def annToMask(self, a):
        m = np.zeros((self.h, self.w), np.uint8)
        x, y, w, h = (int(v) for v in a['bbox'])
        m[max(y, 0):y + h, max(x, 0):x + w] = 1
        return m


def test_dataset_annotation_rules():
    from types import SimpleNamespace
    from yolact_minimal_b200.utils.coco import COCODetection
    h, w = 120, 160
    anns = [dict(bbox=[10.0, 10.0, 50.0, 40.0], category_id=3, iscrowd=0),
            dict(bbox=[5.0, 5.0, 30.0, 30.0], category_id=4, iscrowd=1),      # crowd: dropped
            dict(bbox=[-1.0, 5.0, 30.0, 30.0], category_id=5, iscrowd=0),     # x < 0: dropped
            dict(bbox=[20.0, 30.0, 3.5, 30.0], category_id=6, iscrowd=0),     # w < 4: dropped
            dict(bbox=[60.0, 40.0, 80.0, 60.0], category_id=7, iscrowd=0)]
    cfg = SimpleNamespace(train_imgs='/nonexistent', train_ann=None, continuous_id={k: k + 10 for k in range(1, 91)}, img_size=550)
    ds = COCODetection(cfg, coco=_StubCOCO(anns, h, w))
    img = np.full((h, w, 3), 7, np.uint8)
    ds.load_image = lambda name: img
    random.seed(3)
    img_u8, masks, plan = ds[0]
    random.seed(3)
    ref = train_aug_plan(h, w, np.array([[10.0, 10.0, 60.0, 50.0], [60.0, 40.0, 140.0, 100.0]]), np.array([12, 16]), 550)
    assert masks.shape == (2, h, w) and masks.dtype == np.uint8 and img_u8 is not None
    assert np.array_equal(plan.boxes, ref.boxes) and np.array_equal(plan.labels, ref.labels)
    with pytest.raises(ValueError):
        COCODetection(cfg, mode='val', coco=_StubCOCO(anns, h, w))
    only_bad = COCODetection(cfg, coco=_StubCOCO(anns[2:4], h, w))
    only_bad.load_image = lambda name: img
    assert only_bad[0] is None


def _plan(h, w, n, seed):
    _, _, boxes, labels = an.synthetic_sample(seed, h, w, n)
    for s in range(100):
        random.seed(s)
        p = train_aug_plan(h, w, boxes, labels, 550)
        if p is not None:
            return p
    raise AssertionError


def check_packed(packed, order):
    """The packed buffer, item table, keep table and targets hold `order`'s samples back to back."""
    assert len(packed) == len(order)
    buf = packed.buffer.numpy()
    off = rows = 0
    for i, (img, masks, plan) in enumerate(order):
        it = packed.items[i]
        assert (it['img_off'], it['mask_off'], it['h'], it['w'], it['num_masks']) == \
            (off, off + img.nbytes, img.shape[0], img.shape[1], masks.shape[0])
        assert np.array_equal(buf[off:off + img.nbytes], img.reshape(-1))
        assert np.array_equal(buf[it['mask_off']:it['mask_off'] + masks.nbytes], masks.reshape(-1))
        assert it['out_mask'] == it['keep_begin'] == rows and it['num_keep'] == len(plan.keep)
        assert np.array_equal(packed.keep[rows:rows + it['num_keep']], plan.keep)
        assert (it['crop_x'], it['crop_y'], it['crop_w'], it['crop_h']) == plan.crop and it['resize'] == plan.resize
        assert it['mask_u8'] == plan.mask_u8 and it['mirror'] == plan.mirror
        assert it['hue_delta'] == np.float32(plan.hue) and it['saturation_scale'] == np.float32(plan.saturation)
        assert np.array_equal(packed.targets[i].numpy(), np.hstack((plan.boxes, plan.labels[:, None])).astype(np.float32))
        off += img.nbytes + masks.nbytes
        rows += len(plan.keep)
    assert packed.buffer.numel() == off and packed.keep.shape == (rows,)


def two_samples():
    a = an.synthetic_sample(1, 30, 40, 3)
    b = an.synthetic_sample(2, 50, 20, 2)
    return (a[0], a[1], _plan(30, 40, 3, 1)), (b[0], b[1], _plan(50, 20, 2, 2))


def test_collate_refills_and_packs():
    from yolact_minimal_b200.utils.coco import train_collate
    sa, sb = two_samples()
    packed = train_collate([None, sa, None, sb, None])
    check_packed(packed, [sa, sb, sa, sb, sa])            # valid ones, then valid[0], valid[1], valid[2]
    import pickle
    check_packed(pickle.loads(pickle.dumps(packed)), [sa, sb, sa, sb, sa])


class _ListDataset:
    def __init__(self, samples):
        self.samples = samples

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        return self.samples[i]


@pytest.mark.parametrize('pin', [False, pytest.param(True, marks=pytest.mark.gpu)])
def test_collate_through_dataloader_workers(pin):
    """train_collate runs in DataLoader workers; the packed batch crosses the process boundary (and the pin thread)."""
    import torch
    from yolact_minimal_b200.utils.coco import train_collate
    if pin and not torch.cuda.is_available():
        pytest.skip('pinning needs a CUDA device')
    sa, sb = two_samples()
    ds = _ListDataset([sa, None, sb, sb, None, sa])
    loader = torch.utils.data.DataLoader(ds, batch_size=3, num_workers=2, collate_fn=train_collate, timeout=120, pin_memory=pin)
    batches = list(loader)
    assert len(batches) == 2
    check_packed(batches[0], [sa, sb, sa])
    check_packed(batches[1], [sb, sa, sb])
    assert all(b.buffer.is_pinned() == pin for b in batches)
