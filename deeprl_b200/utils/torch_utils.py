"""Device selection, tensor conversion, seeding and small helpers with the reference's names
(``deep_rl/utils/torch_utils.py:12-58``)."""
import os

import numpy as np
import torch

from .config import Config


def select_device(gpu_id):
    """torch_utils.py:12-17: ``gpu_id >= 0`` selects ``cuda:<id>``, negative selects the CPU."""
    Config.DEVICE = torch.device("cuda:%d" % gpu_id) if gpu_id >= 0 else torch.device("cpu")
    if gpu_id >= 0:
        torch.cuda.set_device(gpu_id)


def tensor(x):
    """torch_utils.py:20-25: tensors pass through untouched; everything else becomes float32 on
    ``Config.DEVICE``."""
    if isinstance(x, torch.Tensor):
        return x
    return torch.from_numpy(np.asarray(x, dtype=np.float32)).to(Config.DEVICE)


def range_tensor(end):
    return torch.arange(end, dtype=torch.long, device=Config.DEVICE)


def to_np(t):
    return t.detach().cpu().numpy()


def random_seed(seed=None):
    """torch_utils.py:36-38: numpy is seeded first, torch's seed is derived FROM numpy."""
    np.random.seed(seed)
    torch.manual_seed(np.random.randint(int(1e6)))


def philox_seed():
    """The key of a device Philox stream, drawn from torch's (seeded) generator: one draw per call."""
    return int(torch.randint(0, 2 ** 62, (1,)).item())


def set_one_thread():
    os.environ["OMP_NUM_THREADS"] = "1"
    os.environ["MKL_NUM_THREADS"] = "1"
    torch.set_num_threads(1)


def huber(x, k=1.0):
    ax = x.abs()
    return torch.where(ax < k, 0.5 * x.pow(2), k * (ax - 0.5 * k))


def epsilon_greedy(epsilon, x):
    """torch_utils.py:51-58 (same order of numpy draws: randint, then rand)."""
    if x.ndim == 1:
        return np.random.randint(len(x)) if np.random.rand() < epsilon else np.argmax(x)
    if x.ndim == 2:
        explore = np.random.randint(x.shape[1], size=x.shape[0])
        greedy = np.argmax(x, axis=-1)
        dice = np.random.rand(x.shape[0])
        return np.where(dice < epsilon, explore, greedy)
    raise ValueError("epsilon_greedy expects a 1-D or 2-D array")
