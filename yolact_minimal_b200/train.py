"""The reference's train.py (train.py:21-200) as a module whose whole training step runs in this library:

    torchrun --nproc_per_node=8 -m yolact_minimal_b200.train --cfg res101_coco --train_bs 64 --img_size 550 --val_bs 32

A step is the training engine's forward and backward (csrc/train.cu) writing every gradient into its flat fp32 buffer, ONE
all-reduce of that buffer when there is more than one rank, and the optimizer step as one launch (csrc/optim.cu: torch's foreach
SGD / AdamW bit for bit).  There is no autograd, no DistributedDataParallel and no copy of the gradient.  What DDP does for the
reference is done here explicitly: the parameters and buffers are broadcast from rank 0 once at the start, the BatchNorm buffers
before each forward (broadcast_buffers=True, train.py:76), and the summed gradient is scaled by 1 / world inside the optimizer.

The arguments, the learning-rate rule (train.py:103-109, quirks included), the optimizer choice (train.py:60-65), the log line,
the evaluation every --val_interval steps and the checkpoint names (save_best / save_latest) are the reference's.  Differences
(DESIGN.md §13): --resume accepts swin_tiny_coco checkpoints; --val_bs is the batched evaluation's batch size; the log line keeps
t_t and the ETA but not the per-phase times, which would need a host synchronisation per phase; the losses are read on the host
only at the logged steps.
"""
import argparse
import datetime
import os
import re
import time

import torch
import torch.distributed as dist
from torch.utils.data import DataLoader
from torch.utils.data.distributed import DistributedSampler

from . import train_native
from .optim import NativeOptimizer


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description='Yolact Training Script')
    parser.add_argument('--local_rank', type=int, default=None)
    parser.add_argument('--cfg', default='res101_coco', help='The configuration name to use.')
    parser.add_argument('--train_bs', type=int, default=8, help='total training batch size')
    parser.add_argument('--img_size', default=544, type=int, help='The image size for training.')
    parser.add_argument('--resume', default=None, type=str, help='The path of the weight file to resume training with.')
    parser.add_argument('--val_interval', default=4000, type=int,
                        help='The validation interval during training, pass -1 to disable.')
    parser.add_argument('--val_num', default=-1, type=int, help='The number of images for test, set to -1 for all.')
    parser.add_argument('--traditional_nms', default=False, action='store_true', help='Whether to use traditional nms.')
    parser.add_argument('--coco_api', action='store_true', help='Whether to use cocoapi to evaluate results.')
    parser.add_argument('--val_bs', default=1, type=int, help='Images per batch of the evaluation on the GPU.')
    return parser.parse_args(argv)


def parse_resume(path):
    """(cfg name, step) of a checkpoint written by save_best / save_latest, e.g. 'weights/best_30.5_res101_coco_392000.pth' or
    'weights/latest_swin_tiny_coco_1000.pth'.  The reference's pattern (train.py:51) matches res* names only."""
    m = re.search(r'((?:res\d+|swin_tiny)_[a-z]+)_(\d+)\.pth$', os.path.basename(path))
    if m is None:
        raise ValueError(f'cannot read a configuration name and a step from {path!r}')
    return m.group(1), int(m.group(2))


def learning_rate(cfg, step, lr):
    """train.py:103-109: the learning rate of `step`, given the one in force before it (cfg.lr at the start of a run, resumed or
    not).  Step 0 is in lr_steps, so it runs at cfg.lr; a run resumed after the warm-up keeps cfg.lr until the next listed step."""
    if cfg.warmup_until > 0 and step <= cfg.warmup_until:
        lr = (cfg.lr - cfg.warmup_init) * (step / cfg.warmup_until) + cfg.warmup_init
    if step in cfg.lr_steps:
        lr = cfg.lr * 0.1 ** cfg.lr_steps.index(step)
    return lr


def optimizer_settings(cfg_name):
    """train.py:60-65: SGD for res* configs, AdamW for swin_tiny_coco."""
    if 'res' in cfg_name:
        return dict(kind='sgd', momentum=0.9, weight_decay=5e-4)
    if cfg_name == 'swin_tiny_coco':
        return dict(kind='adamw', weight_decay=0.05)
    raise ValueError('Unrecognized cfg.')


def optimizer_params(net, names):
    """The module's parameters in the engine's gradient order (`names`: its kind-0 tensors); every parameter exactly once."""
    params = dict(net.named_parameters())
    if sorted(names) != sorted(params):
        missing, extra = sorted(set(params) - set(names)), sorted(set(names) - set(params))
        raise ValueError(f'the engine\'s parameters differ from the module\'s: missing {missing[:5]}, unknown {extra[:5]}')
    return [params[n] for n in names]


class NativeTrainer:
    """One training step of `net` on the native engine and optimizer; `world` ranks all-reduce the gradient."""

    def __init__(self, net, cfg_name, world=1):
        self.net, self.world = net, world
        self.settings = optimizer_settings(cfg_name)
        self.opt = self.names = self.bn_flat = None

    def _first(self, eng):
        self.names = list(eng.param_names)
        self.opt = NativeOptimizer(optimizer_params(self.net, self.names), **self.settings)
        if self.world > 1:
            tensors = dict(self.net.named_buffers())
            self.bn = [tensors[n] for n, _, k in eng.names if k == 1]
            self.bn_flat = torch.cat([b.reshape(-1) for b in self.bn]) if self.bn else None

    def broadcast_buffers(self):
        """broadcast_buffers=True: every rank takes rank 0's BatchNorm statistics, in one flat tensor."""
        if self.bn_flat is None:
            return
        parts = list(self.bn_flat.split([b.numel() for b in self.bn]))
        torch._foreach_copy_(parts, [b.reshape(-1) for b in self.bn])
        dist.broadcast(self.bn_flat, 0)
        torch._foreach_copy_([b.reshape(-1) for b in self.bn], parts)

    def step(self, images, targets, masks, lr):
        """Forward, backward, all-reduce and optimizer step; returns the four losses of this rank (device tensor, no sync)."""
        eng, args, nbt = train_native.prepare_step(self.net, images, targets, masks)
        if self.opt is None:
            self._first(eng)
        elif eng.param_names != self.names:
            raise RuntimeError('two training engines of one module disagree on the gradient order')
        self.broadcast_buffers()
        losses = eng.forward(*args)
        eng.backward_into_grad_flat()
        if nbt:
            torch._foreach_add_(nbt, 1)
        if self.world > 1:
            dist.all_reduce(eng.grad_flat)
        self.opt.step(eng.grad_flat, lr, 1.0 / self.world)
        return losses


def broadcast_module(net):
    """What DDP's constructor does: every parameter and buffer takes rank 0's value."""
    with torch.no_grad():
        for t in list(net.parameters()) + list(net.buffers()):
            dist.broadcast(t.data, 0)


class TrainLog:
    """What a run did, for callers and tests: the trained module, the learning rate of each step, the logged losses and each
    in-loop evaluation (step, box_row, mask_row)."""

    def __init__(self, net, start_step):
        self.net, self.start_step, self.lrs, self.evals, self.losses = net, start_step, {}, [], {}


def train(cfg, dataset=None, val_dataset=None, resume=None, num_workers=None):
    """train.py:44-200 on the native training step.  `dataset` replaces COCODetection(cfg) and `val_dataset` evaluation's
    COCOValDetection(cfg) (tests build both on a stub `coco`); `resume` is the --resume path.  Returns a TrainLog."""
    from .eval import evaluate
    from .modules.yolact import Yolact
    from .utils.augmentations import TrainAugLoader
    from .utils.coco import COCODetection, train_collate
    from .utils.common_utils import save_best, save_latest

    cfg_name = cfg.__class__.__name__
    settings = optimizer_settings(cfg_name)
    world = dist.get_world_size() if dist.is_initialized() else 1
    main_gpu = not dist.is_initialized() or dist.get_rank() == 0
    dev = torch.device('cuda', torch.cuda.current_device())

    net = Yolact(cfg)
    net.train()
    if resume:
        name, start_step = parse_resume(resume)
        assert name == cfg_name, 'Resume weight is not compatible with current cfg.'
        net.load_weights(resume, cfg.cuda)
    else:
        net.backbone.init_backbone(cfg.weight)
        start_step = 0
    net = net.to(dev)
    if world > 1:
        broadcast_module(net)
    trainer = NativeTrainer(net, cfg_name, world)

    dataset = COCODetection(cfg, mode='train') if dataset is None else dataset
    sampler = DistributedSampler(dataset, shuffle=True, num_replicas=world, rank=dist.get_rank() if world > 1 else 0)
    workers = cfg.bs_per_gpu // 2 if num_workers is None else num_workers
    data_loader = DataLoader(dataset, cfg.bs_per_gpu, num_workers=workers, sampler=sampler, pin_memory=True, collate_fn=train_collate)
    loader = TrainAugLoader(data_loader, cfg.img_size, dev)

    writer = None
    if main_gpu:
        try:
            from tensorboardX import SummaryWriter
            writer = SummaryWriter(f'tensorboard_log/{cfg_name}')
        except ImportError:
            pass
        print(f'Number of all parameters: {sum(p.numel() for p in net.parameters())}\n')
        print(f'Optimizer: {settings["kind"]} on the native step, {world} rank(s)\n')

    log = TrainLog(net, start_step)
    map_tables = []
    epoch_seed, step, lr = 0, start_step, cfg.lr
    training = True
    t_last = None

    def finish():
        save_latest(net, cfg_name, step)
        print('\nValidation results during training:\n')
        for table in map_tables:
            print(table, '\n')

    try:
        while training:
            epoch_seed += 1
            sampler.set_epoch(epoch_seed)
            for images, targets, masks in loader:
                lr = learning_rate(cfg, step, lr)
                log.lrs[step] = lr
                losses = trainer.step(images, targets, masks, lr)

                if step % 10 == 0 and step != start_step:
                    all_loss = losses.clone()
                    if world > 1:
                        dist.all_reduce(all_loss)
                    l_c, l_b, l_m, l_s = (all_loss / world).tolist()             # the only host synchronisation of a step
                    now = time.perf_counter()
                    t_t = (now - t_last) / 10 if t_last is not None else 0.0
                    t_last = now
                    log.losses[step] = (l_c, l_b, l_m, l_s)
                    if main_gpu:
                        if writer is not None:
                            for tag, v in (('class', l_c), ('box', l_b), ('mask', l_m), ('semantic', l_s), ('total', l_c + l_b + l_m + l_s)):
                                writer.add_scalar(f'loss/{tag}', v, global_step=step)
                        eta = str(datetime.timedelta(seconds=(cfg.lr_steps[-1] - step) * t_t)).split('.')[0]
                        print(f'step: {step} | lr: {lr:.2e} | l_class: {l_c:.3f} | l_box: {l_b:.3f} | l_mask: {l_m:.3f} | '
                              f'l_semantic: {l_s:.3f} | t_t: {t_t:.3f} | ETA: {eta}')

                if cfg.val_interval > 0 and step % cfg.val_interval == 0 and step != start_step:
                    if main_gpu:
                        net.eval()
                        net.refresh_engine()             # the optimizer wrote the weights through raw pointers: no _version bump
                        table, box_row, mask_row = evaluate(net, cfg, step, dataset=val_dataset)
                        map_tables.append(table)
                        log.evals.append((step, box_row, mask_row))
                        net.train()
                        if writer is not None:
                            writer.add_scalar('mAP/box_map', box_row[1], global_step=step)
                            writer.add_scalar('mAP/mask_map', mask_row[1], global_step=step)
                        save_best(net, mask_row[1], cfg_name, step)
                    t_last = None

                step += 1
                if step >= cfg.lr_steps[-1]:
                    training = False
                    trainer.broadcast_buffers()                  # every rank ends with the statistics rank 0 saves
                    if main_gpu:
                        finish()
                        print('Training completed.')
                    break
    except KeyboardInterrupt:
        if main_gpu:
            finish()
    return log


def main(argv=None):
    from .config import get_config, make_output_dirs
    args = parse_args(argv)
    cfg = get_config(args, mode='train')
    cfg.val_bs = args.val_bs
    if not dist.is_initialized() or dist.get_rank() == 0:
        make_output_dirs()
    try:
        train(cfg, resume=args.resume)
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


if __name__ == '__main__':
    main()
