"""Shared by tests/golden/make_golden_train_swin.py and the Swin training tests: the golden step's shape and seed, the engine's
stochastic-depth draws restated in numpy, and the fixed gradient sample stored per parameter."""
import zlib

import numpy as np
import torch

S, B = 128, 2
SEED_STEP = 0            # torch.manual_seed before the step: Yolact.forward in train mode draws the engine's seed from it


def step_seed(torch_seed):
    """The seed train_native.training_step hands the engine after torch.manual_seed(torch_seed)."""
    g = torch.Generator().manual_seed(torch_seed)
    return int(torch.randint(0, 2 ** 31 - 1, (1,), generator=g).item())


def _hash32(x):
    x = np.uint64(x) & np.uint64(0xffffffff)
    x ^= x >> np.uint64(16); x = (x * np.uint64(0x7feb352d)) & np.uint64(0xffffffff)
    x ^= x >> np.uint64(15); x = (x * np.uint64(0x846ca68b)) & np.uint64(0xffffffff)
    x ^= x >> np.uint64(16)
    return x


def swin_drop_masks(seed, batch, blocks=12):
    """csrc/swin_train.cu k_drop_path_masks: mask[b][blk][branch] = floor(keep + U), U = hash32(seed ^ hash32(salt + i)) >> 8 / 2^24,
    i = (b * 12 + blk) * 2 + branch, keep = 1 - 0.2 blk / 11 in fp32."""
    out = np.zeros((batch, blocks, 2), np.float32)
    for i in range(batch * blocks * 2):
        blk = (i // 2) % blocks
        keep = np.float32(1) - np.float32(np.float32(0.2) * np.float32(blk)) / np.float32(blocks - 1)
        u = _hash32(np.uint64(seed) ^ _hash32(0x5d2f1a97 + i))
        out.reshape(-1)[i] = np.floor(np.float32(keep + np.float32(int(u >> np.uint64(8))) * np.float32(1 / 16777216)))
    return out


def grad_sample(name, g):
    """Every element of a gradient of <= 4096 elements, otherwise 512 elements at indices fixed by the parameter's name."""
    flat = np.asarray(g, np.float32).reshape(-1)
    return flat.copy() if flat.size <= 4096 else flat[sample_index(name, flat.size)]


def sample_index(name, n):
    return np.sort(np.random.default_rng(zlib.crc32(name.encode())).choice(n, 512, replace=False))
