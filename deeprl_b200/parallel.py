"""One learner per GPU (SURVEY.md 8e): the only exchange step of the path is the gradient all-reduce.

Replay, sum tree and loss kernels are rank-local (each rank owns an independent ring + tree, its own envs and its
own Philox stream seeded with the rank); parameters start identical (rank-0 broadcast) and stay identical because
every rank applies the same clipped update to the same summed gradient.  The collective is NCCL on GPUs
(``backend="nccl"``); the same host logic runs over ``gloo`` on CPU tensors for the world_size-2 tests.
"""
import os

import torch
import torch.distributed as dist


def env_world():
    return int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))


def init(backend=None):
    """Initialise torch.distributed from the torchrun environment (no-op for a single process)."""
    world, rank, local = env_world()
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        kw = dict(device_id=torch.device("cuda", local)) if backend == "nccl" else {}
        dist.init_process_group(backend, **kw)
    return world, rank, local


def broadcast_parameters(flat, src=0):
    """Make the flat parameter arena identical on every rank."""
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.broadcast(flat, src)
    return flat


def allreduce_gradients(flat_grad, async_op=False):
    """SUM the flat gradient arena (or a slice of it) over ranks; the 1/world factor is folded into the clip kernel's
    grad_scale.  ``async_op``: returns the work handle (the learner all-reduces fc4's slice beside the convolution backward and
    waits for it before the optimizer kernels; inside a CUDA-graph capture the handle's wait() becomes a graph dependency)."""
    if dist.is_initialized() and dist.get_world_size() > 1:
        return dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, async_op=async_op)
    return None


def leave():
    """End of a multi-rank run whose collectives were captured in CUDA graphs: the process group's destructor can hang then
    (measured), so the ranks synchronise, flush and exit directly."""
    import sys
    if dist.is_initialized() and dist.get_world_size() > 1:
        if torch.cuda.is_available():
            torch.cuda.synchronize()
        dist.barrier()
        if torch.cuda.is_available():
            torch.cuda.synchronize()
        sys.stdout.flush(), sys.stderr.flush()
        os._exit(0)


def grad_scale():
    return 1.0 / dist.get_world_size() if dist.is_initialized() else 1.0


def max_over_ranks(value, device):
    """Device-side max over ranks of a host scalar (timings are reported as the slowest rank's)."""
    t = torch.tensor([float(value)], device=device)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def agree(value, device, what):
    """The same integer on every rank, or a B2RLError naming the disagreement (one all-reduce of [v, -v] with MAX)."""
    t = torch.tensor([int(value), -int(value)], dtype=torch.int64, device=device)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    hi, lo = int(t[0]), -int(t[1])
    if hi != lo:
        from ._lib import B2RLError
        raise B2RLError("%s differs between ranks (%d .. %d)" % (what, lo, hi))
    return hi


class ExchangeRegions:
    """The device memory the data-parallel PPO kernel exchanges gradients through (csrc/ppo_phases.h, "data parallel"): this
    rank's region (cudaMalloc'd and zero-filled once) and every peer's, mapped into this process with CUDA IPC.
    ``table`` holds the device addresses in rank order (``table[rank]`` is this rank's own region)."""

    def __init__(self, nbytes, device):
        import ctypes
        from . import _lib
        world, rank = dist.get_world_size(), dist.get_rank()
        dev = torch.device(device).index
        self.own = ctypes.c_void_p()
        _lib.call("b2rl_ipc_alloc", int(nbytes), ctypes.addressof(self.own))
        handle = ctypes.create_string_buffer(64)
        _lib.call("b2rl_ipc_get_handle", self.own, handle)
        infos = [None] * world
        dist.all_gather_object(infos, (dev, bytes(handle.raw)))
        self.opened, table = [], []
        for p, (pdev, raw) in enumerate(infos):
            if p == rank:
                table.append(self.own.value)
                continue
            ok = ctypes.c_int32(0)
            _lib.call("b2rl_peer_access_ok", dev, pdev, ctypes.addressof(ok))
            if not ok.value:
                raise _lib.B2RLError("PPO data-parallel exchange: device %d (rank %d) has no peer access to device %d (rank %d)"
                                     % (dev, rank, pdev, p))
            ptr = ctypes.c_void_p()
            _lib.call("b2rl_ipc_open_handle", ctypes.create_string_buffer(raw, 64), ctypes.addressof(ptr))
            self.opened.append(ptr)
            table.append(ptr.value)
        self.table = (ctypes.c_void_p * world)(*table)
        dist.barrier()                 # every peer has mapped every region before any rank publishes into one

    def close(self):
        from . import _lib
        for ptr in self.opened:
            _lib.call("b2rl_ipc_close", ptr)
        self.opened = []
        if self.own:
            _lib.call("b2rl_ipc_free", self.own)
            self.own = None


def rank_seed(base_seed):
    """Rank-local RNG stream for the replay shard / envs."""
    _, rank, _ = env_world()
    return int(base_seed) * 1000003 + rank
