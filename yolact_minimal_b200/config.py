"""Configuration surface kept from the reference (config.py:70-253) so that its train.py /
eval.py / detect.py keep working against this package: `get_config(args, mode)` returns an
object whose CLASS NAME selects the backbone (modules/yolact.py:98-106 dispatches on
`cfg.__class__.__name__`) and whose attributes are the ones the hot path reads
(SURVEY.md 8(b) "cfg fields read by the hot path").

Differences from the reference, all deliberate:
  * importing this module has no side effects (the reference creates ten directories in CWD,
    config.py:6-15); call `make_output_dirs()` if a script wants them;
  * `img_size` may be any integer >= 64: the FPN here interpolates to the lateral size, so the
    multiple-of-32 assertion (config.py:75) is only enforced when `strict_img_size=True`.
"""
import os

import numpy as np
import torch
import torch.distributed as dist

def _coco_names():
    multi = ('traffic light', 'fire hydrant', 'stop sign', 'parking meter', 'sports ball', 'baseball bat',
             'baseball glove', 'tennis racket', 'wine glass', 'hot dog', 'potted plant', 'dining table',
             'cell phone', 'teddy bear', 'hair drier')
    s = ('person bicycle car motorcycle airplane bus train truck boat traffic_light fire_hydrant stop_sign '
         'parking_meter bench bird cat dog horse sheep cow elephant bear zebra giraffe backpack umbrella handbag '
         'tie suitcase frisbee skis snowboard sports_ball kite baseball_bat baseball_glove skateboard surfboard '
         'tennis_racket bottle wine_glass cup fork knife spoon bowl banana apple sandwich orange broccoli carrot '
         'hot_dog pizza donut cake chair couch potted_plant bed dining_table toilet tv laptop mouse remote '
         'keyboard cell_phone microwave oven toaster sink refrigerator book clock vase scissors teddy_bear '
         'hair_drier toothbrush')
    names = tuple(n.replace('_', ' ') for n in s.split())
    assert len(names) == 80 and all(m in names for m in multi)
    return names


COCO_CLASSES = _coco_names()
# COCO category ids have gaps (91 ids, 80 used); map id -> 1-based contiguous label.
_MISSING = (12, 26, 29, 30, 45, 66, 68, 69, 71, 83)
COCO_LABEL_MAP = {cid: i + 1 for i, cid in enumerate(c for c in range(1, 91) if c not in _MISSING)}
PASCAL_CLASSES = ('aeroplane', 'bicycle', 'bird', 'boat', 'bottle', 'bus', 'car', 'cat', 'chair', 'cow', 'diningtable',
                  'dog', 'horse', 'motorbike', 'person', 'pottedplant', 'sheep', 'sofa', 'train', 'tvmonitor')
CUSTOM_CLASSES = ('dog', 'person', 'bear', 'sheep')

# BGR mean / std used by the reference's normalisation (config.py:66-67)
norm_mean = np.array([103.94, 116.78, 123.68], dtype=np.float32)
norm_std = np.array([57.38, 57.12, 58.40], dtype=np.float32)

# Per-class drawing colours of utils/output_utils.draw_img (row 0: background; row id + 1: class id).  The package's own table,
# not the reference's.
COLORS = np.array([[0, 0, 0]] + [[(37 * i + 90) % 256, (91 * i + 30) % 256, (173 * i + 200) % 256]
                                 for i in range(80)], dtype='uint8')


def make_output_dirs():
    for d in ('results/images', 'results/videos', 'weights', 'tensorboard_log'):
        os.makedirs(d, exist_ok=True)


class _BaseConfig:
    backbone_weight = 'weights/backbone_res101.pth'
    class_names = COCO_CLASSES
    anchor_scales_544 = (24, 48, 96, 192, 384)
    strict_img_size = False

    def __init__(self, args):
        self.mode = args.mode
        self.cuda = args.cuda
        self.gpu_id = args.gpu_id
        if self.strict_img_size:
            assert args.img_size % 32 == 0, f'Img_size must be divisible by 32, got {args.img_size}.'
        assert args.img_size >= 64, f'img_size must be >= 64, got {args.img_size}.'
        self.img_size = args.img_size
        self.class_names = type(self).class_names
        self.num_classes = len(self.class_names) + 1
        self.continuous_id = (COCO_LABEL_MAP if self.class_names is COCO_CLASSES
                              else {i + 1: i + 1 for i in range(self.num_classes - 1)})
        self.scales = [int(self.img_size / 544 * s) for s in self.anchor_scales_544]      # config.py:80
        self.aspect_ratios = [1, 1 / 2, 2]
        train = self.mode == 'train'
        self.weight = (args.resume if getattr(args, 'resume', None) else self.backbone_weight) if train else args.weight
        self.data_root = os.environ.get('YOLACT_DATA_ROOT', '/home/feiyu/Data/')
        if train:
            self.train_imgs = self.data_root + 'coco2017/train2017/'
            self.train_ann = self.data_root + 'coco2017/annotations/instances_train2017.json'
            self.train_bs = args.train_bs
            self.bs_per_gpu = args.bs_per_gpu
            self.val_interval = args.val_interval
            self.bs_factor = self.train_bs / 8                                               # config.py:96-101
            self.lr = 0.001 * self.bs_factor
            self.warmup_init = self.lr * 0.1
            self.warmup_until = 500
            self.lr_steps = tuple(int(s / self.bs_factor) for s in (0, 280000, 560000, 620000, 680000))
            self.pos_iou_thre, self.neg_iou_thre = 0.5, 0.4
            self.conf_alpha, self.bbox_alpha, self.mask_alpha, self.semantic_alpha = 1, 1.5, 6.125, 1
            self.masks_to_train = 100
        if self.mode in ('train', 'val'):
            self.val_imgs = self.data_root + 'coco2017/val2017/'
            self.val_ann = self.data_root + 'coco2017/annotations/instances_val2017.json'
            self.val_bs = 1
            self.val_num = args.val_num
            self.coco_api = args.coco_api
        self.traditional_nms = args.traditional_nms
        self.nms_score_thre = 0.05                                                           # config.py:122-125
        self.nms_iou_thre = 0.5
        self.top_k = 200
        self.max_detections = 100
        self._customise(args)
        if self.mode == 'detect':
            for k, v in vars(args).items():
                setattr(self, k, v)

    def _customise(self, args):
        pass

    def print_cfg(self):
        print('\n' + '-' * 30 + type(self).__name__ + '-' * 30)
        for k, v in vars(self).items():
            if k not in ('continuous_id', 'data_root', 'cfg'):
                print(f'{k}: {v}')
        print()


class res101_coco(_BaseConfig):
    pass


class res50_coco(_BaseConfig):
    backbone_weight = 'weights/backbone_res50.pth'


class swin_tiny_coco(_BaseConfig):
    backbone_weight = 'weights/swin_tiny.pth'

    def _customise(self, args):
        if self.mode == 'train':
            self.lr = 0.00005 * self.bs_factor


class res50_pascal(_BaseConfig):
    backbone_weight = 'weights/backbone_res50.pth'
    class_names = PASCAL_CLASSES

    def _customise(self, args):
        self.use_square_anchors = False
        if self.mode == 'train':
            self.train_imgs = self.data_root + 'pascal_sbd/img'
            self.train_ann = self.data_root + 'pascal_sbd/pascal_sbd_train.json'
            self.lr_steps = tuple(int(s / self.bs_factor) for s in (0, 60000, 100000, 120000))
            self.scales = [int(self.img_size / 544 * s) for s in (32, 64, 128, 256, 512)]
        if self.mode in ('train', 'val'):
            self.val_imgs = self.data_root + 'pascal_sbd/img'
            self.val_ann = self.data_root + 'pascal_sbd/pascal_sbd_val.json'


class _CustomMixin:
    class_names = CUSTOM_CLASSES

    def _customise(self, args):
        if self.mode == 'train':
            self.train_imgs, self.train_ann = 'custom_dataset/', 'custom_dataset/custom_ann.json'
            self.warmup_until = 100
            self.lr_steps = (0, 1200, 1600, 2000)
        if self.mode in ('train', 'val'):
            self.val_imgs = self.val_ann = ''


class res101_custom(_CustomMixin, _BaseConfig):
    pass


class res50_custom(_CustomMixin, _BaseConfig):
    backbone_weight = 'weights/backbone_res50.pth'


def get_config(args, mode):
    """config.py:222-253.  Fills args.cuda / args.mode / args.gpu_id (/ args.bs_per_gpu), brings
    up the NCCL process group in train mode on GPU, and instantiates the class named args.cfg."""
    args.cuda = torch.cuda.is_available()
    args.mode = mode
    if args.cuda:
        args.gpu_id = os.environ.get('CUDA_VISIBLE_DEVICES') or '0'
        if mode == 'train':
            local_rank = getattr(args, 'local_rank', None)
            if local_rank is None:
                local_rank = int(os.environ.get('LOCAL_RANK', 0))
            torch.cuda.set_device(local_rank)
            if not dist.is_initialized():
                dist.init_process_group(backend='nccl', init_method='env://')
            num_gpus = int(os.environ['WORLD_SIZE'])
            assert args.train_bs % num_gpus == 0, 'Total training batch size must be divisible by GPU number.'
            args.bs_per_gpu = args.train_bs // num_gpus
    else:
        args.gpu_id = None
        if mode == 'train':
            args.bs_per_gpu = args.train_bs
    cls = globals().get(args.cfg)
    if not (isinstance(cls, type) and issubclass(cls, _BaseConfig)):
        raise KeyError(f'unknown config {args.cfg!r}')
    cfg = cls(args)
    if not args.cuda or mode != 'train' or dist.get_rank() == 0:
        if getattr(args, 'verbose', True):
            cfg.print_cfg()
    return cfg


def make_config(name='res101_coco', img_size=544, mode='detect', **overrides):
    """Convenience constructor without argparse (tests, bench, smoke)."""
    import types
    ns = types.SimpleNamespace(cfg=name, img_size=img_size, weight=None, traditional_nms=False, visual_thre=0.0,
                               save_lincomb=False, no_crop=False, image=None, video=None, hide_mask=False,
                               hide_bbox=False, hide_score=False, cutout=False, real_time=False, val_num=-1,
                               coco_api=False, resume=None, train_bs=8, val_interval=-1, verbose=False)
    for k, v in overrides.items():
        setattr(ns, k, v)
    # like get_config, minus the process-group initialisation and the printing
    ns.cuda, ns.mode = torch.cuda.is_available(), mode
    ns.gpu_id = (os.environ.get('CUDA_VISIBLE_DEVICES') or '0') if ns.cuda else None
    if mode == 'train' and not hasattr(ns, 'bs_per_gpu'):
        ns.bs_per_gpu = ns.train_bs
    cls = globals().get(name)
    if not (isinstance(cls, type) and issubclass(cls, _BaseConfig)):
        raise KeyError(f'unknown config {name!r}')
    return cls(ns)
