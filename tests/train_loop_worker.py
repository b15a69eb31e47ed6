"""torchrun worker for tests/test_train_loop_gpu.py: `python -m yolact_minimal_b200.train`'s train() at 128x128 on a stub COCO
(synthetic PNG images, box-shaped masks) in a scratch directory, with shortened lr_steps.

    worker.py OUT.json CFG_NAME WORKDIR MODE        MODE: 'run' (train, evaluate, resume) or 'ranks' (train; compare the ranks)
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(160, 200), (200, 160), (128, 128), (150, 190)]


class StubCOCO:
    """The pycocotools.coco.COCO methods COCODetection / COCOValDetection use, over in-memory annotations."""

    def __init__(self, images):
        self.images = images                                     # img_id -> (file_name, h, w, anns)
        self.imgToAnns = {k: v[3] for k, v in images.items()}

    def getAnnIds(self, imgIds):
        return [(imgIds, i) for i in range(len(self.images[imgIds][3]))]

    def loadAnns(self, ids):
        return [self.images[k][3][i] for k, i in ids]

    def loadImgs(self, img_id):
        return [{'file_name': self.images[img_id][0]}]

    def annToMask(self, a):
        h, w = a['_hw']
        m = np.zeros((h, w), np.uint8)
        x, y, bw, bh = (int(v) for v in a['bbox'])
        m[max(y, 0):y + bh, max(x, 0):x + bw] = 1
        return m


def make_coco(img_dir, n, seed):
    import cv2
    from yolact_minimal_b200.config import COCO_LABEL_MAP
    coco_id = {label - 1: cid for cid, label in COCO_LABEL_MAP.items()}
    rng = np.random.RandomState(seed)
    images = {}
    for k in range(n):
        h, w = SIZES[k % len(SIZES)]
        yy, xx = np.mgrid[0:h, 0:w]
        img = np.stack([128 + 60 * np.sin(xx / (9 + k % 3) + c) * np.cos(yy / (13 + c)) for c in range(3)], -1)
        anns = []
        for j in range(2 + k % 3):
            bw, bh = rng.randint(24, w // 2), rng.randint(24, h // 2)
            x, y = rng.randint(0, w - bw), rng.randint(0, h - bh)
            img[y:y + bh, x:x + bw] = (40 * j + 20, 200 - 50 * j, 90 + 30 * j)
            anns.append(dict(bbox=[float(x), float(y), float(bw), float(bh)], category_id=coco_id[(3 * j + k) % 5], iscrowd=0, _hw=(h, w)))
        name = f'{seed}_{k:03d}.png'
        cv2.imwrite(os.path.join(img_dir, name), np.clip(img + rng.normal(0, 8, size=img.shape), 0, 255).astype(np.uint8))
        images[1000 + k] = (name, h, w, anns)
    return StubCOCO(images)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out')
    ap.add_argument('cfg')
    ap.add_argument('workdir')
    ap.add_argument('mode')
    a = ap.parse_args()
    from yolact_minimal_b200.config import get_config, make_config, make_output_dirs
    from yolact_minimal_b200.eval import evaluate
    from yolact_minimal_b200.modules.yolact import Yolact
    from yolact_minimal_b200.train import parse_args, train
    from yolact_minimal_b200.utils.coco import COCODetection, COCOValDetection

    world = int(os.environ['WORLD_SIZE'])
    args = parse_args(['--cfg', a.cfg, '--train_bs', str(2 * world), '--img_size', '128', '--val_interval', '4', '--val_bs', '3'])
    args.verbose = False
    cfg = get_config(args, mode='train')
    cfg.val_bs = args.val_bs
    rank = dist.get_rank()
    os.chdir(a.workdir)
    img_dir = os.path.join(a.workdir, 'imgs')
    if rank == 0:
        make_output_dirs()
        os.makedirs(img_dir, exist_ok=True)
        torch.manual_seed(0)
        torch.save(Yolact(cfg).backbone.state_dict(), cfg.backbone_weight)   # the initial backbone train() loads
        make_coco(img_dir, 8, 1)
        make_coco(img_dir, 6, 2)
    dist.barrier()
    cfg.train_imgs = cfg.val_imgs = img_dir
    train_coco = _load(img_dir, 8, 1)
    val_coco = _load(img_dir, 6, 2)
    dataset = COCODetection(cfg, coco=train_coco)
    val_dataset = COCOValDetection(cfg, coco=val_coco)
    cfg.warmup_until, cfg.warmup_init = 2, cfg.lr * 0.1
    res = {'world': world}
    torch.manual_seed(1 + rank)
    if a.mode == 'ranks':
        cfg.val_interval, cfg.lr_steps = -1, (0, 4, 7)
        log = train(cfg, dataset, num_workers=1)
        net = log.net
        flat = {'params': torch.cat([p.detach().reshape(-1) for p in net.parameters()]),
                'buffers': torch.cat([b.detach().reshape(-1).double() for n, b in net.named_buffers() if 'running' in n])}
        for k, t in flat.items():
            got = [torch.zeros_like(t) for _ in range(world)]
            dist.all_gather(got, t.contiguous())
            res[k + '_equal'] = all(torch.equal(got[0], g) for g in got)
            res[k + '_numel'] = t.numel()
        res['params_finite'] = bool(torch.isfinite(flat['params']).all())
    else:
        cfg.lr_steps = (0, 5, 9)
        log = train(cfg, dataset, val_dataset, num_workers=1)
        res['lrs'] = {str(k): v for k, v in log.lrs.items()}
        res['evals'] = [(s, list(b), list(m)) for s, b, m in log.evals]
        res['files'] = sorted(os.listdir('weights'))
        res['cfg_lr'] = cfg.lr
        # a fresh module loaded from latest_* evaluates to the in-loop rows of the same weights
        vcfg = make_config(a.cfg, 128, mode='val')
        vcfg.val_bs, vcfg.val_imgs = 3, img_dir
        fresh = Yolact(vcfg)
        fresh.load_weights(f'weights/latest_{a.cfg}_9.pth', True)
        fresh = fresh.cuda().eval()
        _, box_row, mask_row = evaluate(fresh, vcfg, 8, dataset=COCOValDetection(vcfg, coco=val_coco))
        res['fresh_eval'] = (8, list(box_row), list(mask_row))
        # resume from latest_*: the parsed step, the rule's learning rates, weights from the checkpoint
        cfg.lr_steps, cfg.val_interval = (0, 5, 11, 13), -1
        log2 = train(cfg, dataset, resume=f'weights/latest_{a.cfg}_9.pth', num_workers=1)
        res['resume_start'] = log2.start_step
        res['resume_lrs'] = {str(k): v for k, v in log2.lrs.items()}
        res['files_after_resume'] = sorted(os.listdir('weights'))
    if rank == 0:
        json.dump(res, open(a.out, 'w'))
    dist.barrier()
    dist.destroy_process_group()


def _load(img_dir, n, seed):
    """The stub annotations of make_coco(img_dir, n, seed) without writing the images again."""
    import cv2
    real_imwrite = cv2.imwrite
    cv2.imwrite = lambda *a, **k: True
    try:
        return make_coco(img_dir, n, seed)
    finally:
        cv2.imwrite = real_imwrite


if __name__ == '__main__':
    main()
