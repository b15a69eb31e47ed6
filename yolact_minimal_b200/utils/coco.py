"""COCO training data for the GPU augmentation: the reference's utils/coco.py:47-133 COCODetection in 'train'
mode and its train_collate (:14-28), with train_aug's pixel work left to the GPU.

Each worker reads the image and decodes the instance masks as the reference does, applies the same annotation
rules, and draws the train_aug plan on the host (utils.augmentations.train_aug_plan); it returns the raw uint8
image, the raw uint8 masks and the plan.  train_collate packs a batch into one uint8 buffer plus the kernel's
tables, and utils.augmentations.TrainAugLoader (or train_aug_batch) augments it on the device.
"""
import os.path as osp

import numpy as np

from .augmentations import PackedTrainBatch, train_aug_plan


def train_collate(batch):
    """A sample that came back None is replaced by repeating the valid ones, as the reference does
    (valid_batch.append(valid_batch[i])); the batch is packed for yb_train_aug."""
    valid = [s for s in batch if s is not None]
    for i in range(len(batch) - len(valid)):
        valid.append(valid[i])
    return PackedTrainBatch(valid)


class COCODetection:
    """COCODetection(cfg, mode='train'): returns (img_u8 [h,w,3] BGR, masks_u8 [n,h,w], TrainAugPlan) or None.
    `coco` may be passed in (any object with the pycocotools.coco.COCO methods used here); by default it is
    pycocotools' COCO on cfg.train_ann."""

    def __init__(self, cfg, mode='train', coco=None):
        if mode != 'train':
            raise ValueError(f"COCODetection(mode='{mode}'): this class feeds the GPU training augmentation only; use the "
                             "reference's utils/coco.py COCODetection for 'val' and 'detect' (val_aug here runs on the GPU, "
                             "not in DataLoader workers)")
        self.mode, self.cfg = mode, cfg
        self.image_path = cfg.train_imgs
        if coco is None:
            from pycocotools.coco import COCO
            coco = COCO(cfg.train_ann)
        self.coco = coco
        self.ids = list(self.coco.imgToAnns.keys())
        self.continuous_id = cfg.continuous_id

    def __len__(self):
        return len(self.ids)

    def load_image(self, file_name):
        import cv2
        img_path = osp.join(self.image_path, file_name)
        assert osp.exists(img_path), f'Image path does not exist: {img_path}'
        return cv2.imread(img_path)

    def __getitem__(self, index):
        img_id = self.ids[index]
        target = [a for a in self.coco.loadAnns(self.coco.getAnnIds(imgIds=img_id)) if not a['iscrowd']]
        img = self.load_image(self.coco.loadImgs(img_id)[0]['file_name'])
        height, width, _ = img.shape
        assert len(target) > 0, 'No annotation in this image!'
        boxes, masks, labels = [], [], []
        for a in target:
            x, y, w, h = a['bbox']
            if x < 0 or y < 0 or w < 4 or h < 4:      # wrong boxes are ignored when training
                continue
            boxes.append([x, y, x + w, y + h])
            masks.append(self.coco.annToMask(a))
            labels.append(self.continuous_id[a['category_id']] - 1)
        if not boxes:
            print(f'No valid object in image: {img_id}. Use a repeated image in this batch.')
            return None
        masks = np.ascontiguousarray(np.stack(masks, axis=0).astype(np.uint8, copy=False))
        assert masks.shape == (len(boxes), height, width), 'Unmatched annotations.'
        plan = train_aug_plan(height, width, np.array(boxes, dtype=np.float64), np.array(labels), self.cfg.img_size)
        if plan is None:
            return None
        return np.ascontiguousarray(img), masks, plan
