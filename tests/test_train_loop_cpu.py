"""CPU: the host side of `python -m yolact_minimal_b200.train` -- the learning-rate rule against the reference's train.py:103-109
executed on a torch.optim param group, the arguments, checkpoint-name parsing, the optimizer choice and the parameter order the
native optimizer is built in."""
import random

import pytest
import torch

from yolact_minimal_b200.config import make_config
from yolact_minimal_b200.train import learning_rate, optimizer_params, optimizer_settings, parse_args, parse_resume


def _reference_lrs(cfg, steps):
    """train.py:103-109 verbatim on a real param group, created with lr=cfg.lr as train.py:61 does, over increasing `steps`."""
    optimizer = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=cfg.lr, momentum=0.9, weight_decay=5e-4)
    out = {}
    for step in steps:
        if cfg.warmup_until > 0 and step <= cfg.warmup_until:  # warm up learning rate.
            for param_group in optimizer.param_groups:
                param_group['lr'] = (cfg.lr - cfg.warmup_init) * (step / cfg.warmup_until) + cfg.warmup_init

        if step in cfg.lr_steps:  # learning rate decay.
            for param_group in optimizer.param_groups:
                param_group['lr'] = cfg.lr * 0.1 ** cfg.lr_steps.index(step)
        out[step] = optimizer.param_groups[0]['lr']
    return out


def _steps(cfg, start):
    """Every step at which the rule can change the rate (the warm-up and the listed steps), their neighbours and a few between."""
    s = set(range(0, cfg.warmup_until + 2))
    for x in cfg.lr_steps:
        s.update((x - 1, x, x + 1))
    s.update(x // 2 + 7 for x in cfg.lr_steps)
    return sorted(x for x in s if x >= start)


@pytest.mark.parametrize('name', ['res101_coco', 'swin_tiny_coco', 'res101_custom'])
@pytest.mark.parametrize('train_bs', [8, 16])
def test_learning_rate_follows_the_reference_rule(name, train_bs):
    cfg = make_config(name, 550, mode='train', train_bs=train_bs)
    for start in (0, cfg.warmup_until // 3, cfg.warmup_until + 57, cfg.lr_steps[1] + 3, cfg.lr_steps[2]):
        steps = _steps(cfg, start)
        want = _reference_lrs(cfg, steps)
        lr = cfg.lr
        for step in steps:
            lr = learning_rate(cfg, step, lr)
            assert lr == want[step], (name, train_bs, start, step)
    got = {}
    lr = cfg.lr
    for step in _steps(cfg, 0):
        got[step] = lr = learning_rate(cfg, step, lr)
    # the quirks, pinned: step 0 is listed, so it runs at cfg.lr, not warmup_init
    assert got[0] == cfg.lr and got[1] == (cfg.lr - cfg.warmup_init) * (1 / cfg.warmup_until) + cfg.warmup_init
    assert got[cfg.warmup_until] == cfg.lr and got[cfg.warmup_until + 1] == cfg.lr
    for i, x in enumerate(cfg.lr_steps):
        assert got[x] == cfg.lr * 0.1 ** i
    # a run resumed past the warm-up keeps cfg.lr until the next listed step
    start = cfg.lr_steps[1] + 3
    lr = cfg.lr
    for step in range(start, start + 5):
        lr = learning_rate(cfg, step, lr)
        assert lr == cfg.lr
    assert learning_rate(cfg, cfg.lr_steps[2], lr) == cfg.lr * 0.1 ** 2


def test_arguments_are_the_reference_ones_plus_val_bs():
    a = parse_args([])
    assert (a.local_rank, a.cfg, a.train_bs, a.img_size, a.resume, a.val_interval, a.val_num, a.traditional_nms, a.coco_api,
            a.val_bs) == (None, 'res101_coco', 8, 544, None, 4000, -1, False, False, 1)
    a = parse_args(['--cfg', 'swin_tiny_coco', '--train_bs', '16', '--img_size', '550', '--resume', 'weights/latest_swin_tiny_coco_20.pth',
                    '--val_interval', '-1', '--val_num', '500', '--traditional_nms', '--coco_api', '--local_rank', '3', '--val_bs', '32'])
    assert (a.local_rank, a.cfg, a.train_bs, a.img_size, a.resume, a.val_interval, a.val_num, a.traditional_nms, a.coco_api,
            a.val_bs) == (3, 'swin_tiny_coco', 16, 550, 'weights/latest_swin_tiny_coco_20.pth', -1, 500, True, True, 32)


def test_resume_names():
    assert parse_resume('weights/latest_res101_coco_35000.pth') == ('res101_coco', 35000)
    assert parse_resume('weights/best_30.5_res101_coco_392000.pth') == ('res101_coco', 392000)
    assert parse_resume('/results/run/weights/best_0.0_res50_pascal_12.pth') == ('res50_pascal', 12)
    assert parse_resume('weights/latest_res101_custom_1200.pth') == ('res101_custom', 1200)
    assert parse_resume('weights/latest_swin_tiny_coco_1000.pth') == ('swin_tiny_coco', 1000)
    assert parse_resume('weights/best_28.1_swin_tiny_coco_4000.pth') == ('swin_tiny_coco', 4000)
    for bad in ('weights/backbone_res101.pth', 'weights/latest_res101_coco.pth', 'weights/swin_tiny.pth'):
        with pytest.raises(ValueError):
            parse_resume(bad)


def test_optimizer_choice():
    assert optimizer_settings('res101_coco') == dict(kind='sgd', momentum=0.9, weight_decay=5e-4)
    assert optimizer_settings('res50_pascal')['kind'] == 'sgd'
    assert optimizer_settings('swin_tiny_coco') == dict(kind='adamw', weight_decay=0.05)
    with pytest.raises(ValueError):
        optimizer_settings('swin_tiny_custom')


@pytest.mark.parametrize('name', ['res50_coco', 'swin_tiny_coco'])
def test_optimizer_parameters_follow_the_engine_order(name):
    from yolact_minimal_b200.modules.yolact import Yolact
    net = Yolact(make_config(name, 128, mode='train', train_bs=2))
    named = dict(net.named_parameters())
    names = list(named)
    random.Random(0).shuffle(names)
    got = optimizer_params(net, names)
    assert len(got) == len(names) and all(g is named[n] for g, n in zip(got, names))
    assert sum(p.numel() for p in got) == sum(p.numel() for p in net.parameters())
    with pytest.raises(ValueError):
        optimizer_params(net, names[1:])
    with pytest.raises(ValueError):
        optimizer_params(net, names + ['backbone.not_a_parameter'])
