"""COCO data for the GPU augmentations: the reference's utils/coco.py:47-133 COCODetection and its collates.

'train' (COCODetection, train_collate :14-28): each worker reads the image and decodes the instance masks as the
reference does, applies the same annotation rules, and draws the train_aug plan on the host
(utils.augmentations.train_aug_plan); it returns the raw uint8 image, the raw uint8 masks and the plan.  train_collate
packs a batch into one uint8 buffer plus the kernel's tables, and utils.augmentations.TrainAugLoader (or
train_aug_batch) augments it on the device.

'val' (COCOValDetection, val_collate :31-35): each worker returns the raw uint8 image, the gts and the gt masks
bit-packed on the host; val_collate packs a batch into a PackedValBatch, and yolact_minimal_b200.eval.evaluate runs
val_aug on the device for the whole batch (utils.augmentations.val_aug_batch).

'detect' (DetectImages, detect_collate :38-40): each worker reads one image of the folder; detect_collate packs a batch into a
PackedDetectBatch, and yolact_minimal_b200.detect runs val_aug, the network and the drawing on the device for the whole batch.
"""
import glob
import os.path as osp

import numpy as np

from .augmentations import EncodedImage, PackedTrainBatch, PackedValBatch, pack_any, read_image, train_aug_plan
from .mask_utils import pack_masks_host


def _imread(image_path, file_name, decode_gpu=False):
    img_path = osp.join(image_path, file_name)
    assert osp.exists(img_path), f'Image path does not exist: {img_path}'
    return read_image(img_path, decode_gpu)


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
        return _imread(self.image_path, file_name)

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


def val_collate(batch):
    """Packs a batch of COCOValDetection samples for val_aug_batch and MapEvaluator.add (or CocoEvaluator.add)."""
    return PackedValBatch(batch)


class COCOValDetection:
    """The reference's COCODetection(cfg, mode='val') for batched evaluation on the GPU.  Its annotation rules
    (utils/coco.py:69-119): crowd annotations are dropped, no box is filtered out, labels are continuous_id - 1, gt boxes
    are divided by (w, h, w, h) in float64 and then rounded to float32 (as val_collate's torch.tensor does); an image with no
    annotation left raises RuntimeError.  len() honours cfg.val_num.

    Returns (img_u8 [h,w,3] BGR, gt float32 [n,5], gt masks bit-packed int32 [n,h,ceil(w/32)] (mask_utils.pack_masks layout),
    (h, w), COCO image id); val_aug runs on the device for a whole batch.  `coco` may be passed in (any object with the
    pycocotools.coco.COCO methods used here); by default it is pycocotools' COCO on cfg.val_ann.

    With coco_eval=True each sample also carries every annotation of the image in file order, crowd ones included, for
    utils.cocoeval.CocoEvaluator: (class int32 [m] (continuous_id - 1), bbox float64 [m,4] (the annotation's x,y,w,h), area
    float64 [m], iscrowd int32 [m], masks bit-packed int32 [m,h,ceil(w/32)] (annToMask)).  The images visited, their order, len()
    and the RuntimeError rule stay the same.

    With decode_gpu=True the image is the file's bytes (utils.augmentations.EncodedImage, (h, w) from yb_jpeg_header) when
    yb_jpeg_decode_batch decodes it, and the batch is decoded on the device (PackedValBatch.to_device); a file it refuses is read
    by cv2.imread here, as without the flag."""

    def __init__(self, cfg, coco=None, coco_eval=False, decode_gpu=False):
        self.cfg = cfg
        self.coco_eval = bool(coco_eval)
        self.decode_gpu = bool(decode_gpu)
        self.image_path = cfg.val_imgs
        if coco is None:
            from pycocotools.coco import COCO
            coco = COCO(cfg.val_ann)
        self.coco = coco
        self.ids = list(self.coco.imgToAnns.keys())
        self.continuous_id = cfg.continuous_id

    def __len__(self):
        return len(self.ids) if self.cfg.val_num == -1 else min(self.cfg.val_num, len(self.ids))

    def load_image(self, file_name):
        return _imread(self.image_path, file_name, self.decode_gpu)

    def __getitem__(self, index):
        img_id = self.ids[index]
        anns = self.coco.loadAnns(self.coco.getAnnIds(imgIds=img_id))
        target = [a for a in anns if not a['iscrowd']]
        img = self.load_image(self.coco.loadImgs(img_id)[0]['file_name'])
        height, width, _ = img.shape
        if not target:
            raise RuntimeError('Error, no valid object in this image.')
        boxes = np.array([[a['bbox'][0], a['bbox'][1], a['bbox'][0] + a['bbox'][2], a['bbox'][1] + a['bbox'][3]] for a in target])
        labels = np.array([self.continuous_id[a['category_id']] - 1 for a in target])
        all_masks = [self.coco.annToMask(a) for a in (anns if self.coco_eval else target)]
        masks = np.stack([m for m, a in zip(all_masks, anns) if not a['iscrowd']] if self.coco_eval else all_masks, axis=0)
        assert masks.shape == (boxes.shape[0], height, width), 'Unmatched annotations.'
        boxes = boxes / np.array([width, height, width, height])
        gt = np.hstack((boxes, np.expand_dims(labels, axis=1))).astype(np.float32)
        sample = (img if isinstance(img, EncodedImage) else np.ascontiguousarray(img), gt, pack_masks_host(masks), (height, width), img_id)
        if not self.coco_eval:
            return sample
        ann = (np.array([self.continuous_id[a['category_id']] - 1 for a in anns], np.int32),
               np.array([a['bbox'] for a in anns], np.float64).reshape(-1, 4), np.array([a['area'] for a in anns], np.float64),
               np.array([int(a['iscrowd']) for a in anns], np.int32), pack_masks_host(np.stack(all_masks, axis=0)))
        return sample + (ann,)


class PackedDetectBatch:
    """A batch of images for yolact_minimal_b200.detect: `buffer` / `items` the raw uint8 BGR images back to back and their
    yb_val_aug_item table (pack_images), `names` their file names, `sizes` their (h, w).  With DataLoader(pin_memory=True) the
    loader's pin thread page-locks the buffer.
    With images given as JPEG files (EncodedImage) `buffer` is None until the device buffer is copied back, and `mixed`
    (utils.augmentations.MixedImages) holds the files and the pixels of the others; to_device decodes them."""

    def __init__(self, images, names):
        self.buffer, self.items, self.mixed = pack_any(images)
        self.names = list(names)
        self.sizes = [(int(h), int(w)) for _, h, w in self.items.tolist()]

    def __len__(self):
        return len(self.items)

    def pin_memory(self):
        if self.mixed is not None:
            self.mixed.pin_memory()
        else:
            self.buffer = self.buffer.pin_memory()
        return self

    def to_device(self, device):
        """-> (CUDA uint8 buffer of the images in `items`' layout, device int32 status of the files decoded there (entry k is image
        mixed.encoded[k]) or None).  No host sync."""
        if self.mixed is not None:
            return self.mixed.to_device(device)
        return self.buffer.to(device, non_blocking=self.buffer.is_pinned()), None

    def image(self, b):
        """Image b as a numpy view [h,w,3] of the (host) buffer."""
        off, h, w = self.items[b].tolist()
        return self.buffer.numpy()[off:off + h * w * 3].reshape(h, w, 3)


def detect_collate(batch):
    """Packs a batch of DetectImages samples."""
    return PackedDetectBatch([s[0] for s in batch], [s[1] for s in batch])


class DetectImages:
    """The reference's COCODetection(cfg, mode='detect') images (utils/coco.py:56-67): the sorted glob(cfg.image + '/*.jpg').
    Returns (img_u8 [h,w,3] BGR, file name); val_aug runs on the device for a whole batch.  With decode_gpu=True the image is the
    file's bytes (EncodedImage) when yb_jpeg_decode_batch decodes it, and cv2.imread's pixels otherwise."""

    def __init__(self, cfg, decode_gpu=False):
        self.image_path = glob.glob(cfg.image + '/*.jpg')
        self.image_path.sort()
        self.decode_gpu = bool(decode_gpu)

    def __len__(self):
        return len(self.image_path)

    def __getitem__(self, index):
        img_name = self.image_path[index]
        img = read_image(img_name, self.decode_gpu)
        if img is None:
            raise RuntimeError(f'cannot read image {img_name}')
        return img if isinstance(img, EncodedImage) else np.ascontiguousarray(img), img_name.split(osp.sep)[-1]
