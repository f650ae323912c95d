#!/usr/bin/env python
"""bench.py -- gradient-updates/s of the DQN hot path (BASELINE.json metric) on N H100s.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl b2rl|reference] [--workload dqn|per|c51|qr|ppo]
                  [--replay async|sync] [--repeats R] [--no-extras]

A "step" is ONE gradient update of ``DQNAgent.step`` (DQN_agent.py:101-138) at batch 512: the 4 env transitions
that ``sgd_update_frequency = 4`` implies are fed to the ring, a batch is sampled from a 1M-transition ring of
84x84 uint8 frames (7.06 GB, larger than L2, random indices every step), target / online NatureConvBody forward,
fused loss, backward, global-norm clip, RMSprop(centered) step.  Weights are random-init, frames synthetic.

Timing: W untimed warm-up steps, then R (default 5) timed regions of EXACTLY K steps each, every region bracketed by a
barrier + torch.cuda.synchronize() and timed with CUDA events on the launching stream, max over ranks per region;
``ms_per_step`` / ``value`` are the MEDIAN region (all regions are in ``repeat_ms``).

  value      whole-job updates/s with the env transitions already in HBM (graph replays back to back)
  e2e        same metric through host buffers: per step the 4 transitions are copied host->device from pinned
             memory inside the timed region and the loss is read back device->host
  e2e_agent  the same update driven through the reference's own seam, ``DQNAgent.step()`` with ``config.cuda_graph``
             (actor env steps + host feed + one graph replay per step)
  roofline   the replay gather kernel (HBM): SURVEY 8d algorithmic bytes per launch / CUDA-event time per launch;
             ``roofline_tensor``: the dominant wgmma kernel (conv1 forward) and the whole step against the bf16 peaks
  extra_workloads   PER / C51 / QR-DQN / PPO (BASELINE configs[2..4]) measured in the same run
  cpu_baseline / --impl reference   the oracle port of the reference's CPU path (oracle/agents.py, torch-CPU) timed on the
             host cores with the reference's own ``set_one_thread()`` and with 32 threads (median of >= 20 updates where
             the time budget allows); the reference is pure Python, /root/reference does not exist on the GPU box

Multi-GPU: launched by torchrun, one rank per GPU; each rank owns a replay shard and a full batch-512 update,
gradients are all-reduced (NCCL) every step: weak scaling, value = ranks x updates/s.
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

B, HIST, FRAME, CAP, ACTIONS = 512, 4, 84 * 84, 1_000_000, 4
# SURVEY 8d: per sampled transition read 5 unique frames, write 2 x 4 frames in the output dtype
ALGO_BYTES = 5 * FRAME + 2 * 4 * FRAME                    # SURVEY 8d: 91 728 algorithmic bytes per sampled transition
FLOPS_PER_UPDATE = {"dqn": 34.9e9, "per": 34.9e9 + 512 * 18.69e6}    # SURVEY 8d (+ one more forward for double-Q)


def peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        return {}


class ClockSampler:
    FIELDS = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index=0):
        self.rows, self.stop, self.index = [], threading.Event(), index
        self.t = threading.Thread(target=self.run, daemon=True)

    def run(self):
        while not self.stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.FIELDS,
                                      "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=5).stdout
                self.rows.append([x.strip() for x in out.strip().split(",")])
            except Exception:
                pass
            self.stop.wait(0.2)

    def __enter__(self):
        self.t.start()
        return self

    def __exit__(self, *a):
        self.stop.set()
        self.t.join(timeout=5)

    def summary(self):
        sm = [float(r[0]) for r in self.rows if len(r) >= 7 and r[0].replace(".", "").isdigit()]
        mx = [float(r[1]) for r in self.rows if len(r) >= 7 and r[1].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = sorted({n for r in self.rows if len(r) >= 7 for n, v in zip(names, r[3:7]) if v.lower().startswith("active")})
        return dict(sm_mhz=float(np.median(sm)) if sm else None, sm_max_mhz=max(mx) if mx else None, reasons=reasons,
                    samples=len(sm))


# --------------------------------------------------------------------------------------------- product arm
def synthetic_ring(rl, replay_cls, device, seed, capacity=None):
    """SURVEY 8d synthetic inputs, generated on the device in chunks."""
    capacity = CAP if capacity is None else capacity
    pos = 123_457 if capacity > 200_000 else capacity // 3
    g = torch.Generator(device=device).manual_seed(seed)
    frames = torch.empty((capacity, FRAME), dtype=torch.uint8, device=device)
    step = 50_000
    for s in range(0, capacity, step):
        n = min(step, capacity - s)
        frames[s:s + n] = torch.randint(0, 256, (n, FRAME), dtype=torch.uint8, device=device, generator=g)
    action = torch.randint(0, ACTIONS, (capacity,), device=device, generator=g).int()
    u = torch.rand(capacity, device=device, generator=g)
    reward = torch.where(u < 0.05, -1.0, torch.where(u > 0.95, 1.0, 0.0)).double()
    mask = (torch.rand(capacity, device=device, generator=g) > 1e-3).int()
    rp = replay_cls(capacity, B, n_step=1, discount=0.99, history_length=HIST, device=device, seed=seed)
    rp.item_shape, rp.item_dtype = (84, 84), np.dtype(np.uint8)
    if replay_cls.__name__ == "PrioritizedReplay":
        pr = (torch.randn(capacity, device=device, generator=g).abs() + 0.01).sqrt()
        rp.load_synthetic(frames, action, reward, mask, pos=pos, priorities=pr)
    else:
        rp.load_synthetic(frames, action, reward, mask, pos=pos)
    return rp


def build_learner(rl, workload, device, rank, world, prefetch=True):
    from deeprl_b200.learner import GraphedDQNLearner
    torch.manual_seed(0)                                   # identical initial parameters on every rank
    body = lambda: rl.NatureConvBody(in_channels=HIST)
    if workload in ("dqn", "per"):
        mk = (lambda: rl.DuelingNet(ACTIONS, body())) if workload == "per" else (lambda: rl.VanillaNet(ACTIONS, body()))
        topt = lambda p: torch.optim.RMSprop(p, lr=0.00025, alpha=0.95, eps=0.01, centered=True)     # examples.py:67-68
        kind = "dqn"
    elif workload == "c51":
        mk = lambda: rl.CategoricalNet(ACTIONS, 51, body())
        topt = lambda p: torch.optim.Adam(p, lr=0.00025, eps=0.01 / 32)                               # examples.py:204
        kind = "c51"
    else:
        mk = lambda: rl.QuantileNet(ACTIONS, 200, body())
        topt = lambda p: torch.optim.Adam(p, lr=0.00005, eps=0.01 / 32)                               # examples.py:139
        kind = "qr"
    net, tgt = mk(), mk()
    tgt.load_state_dict(net.state_dict())
    if rl.Config.DENSE_BACKEND != "tcgen05":               # cuDNN prefers channels_last weights; the wgmma path packs its own
        net = net.to(memory_format=torch.channels_last)
        tgt = tgt.to(memory_format=torch.channels_last)
    opt = rl.ops.FlatOptimizer.from_torch(topt(net.parameters()))
    replay_cls = rl.PrioritizedReplay if workload == "per" else rl.UniformReplay
    rp = synthetic_ring(rl, replay_cls, device, seed=rank)
    return GraphedDQNLearner(net, tgt, opt, rp, kind=kind, double_q=(workload == "per"), gradient_clip=5.0,
                             feeds_per_update=4, compute_dtype=torch.bfloat16, world_size=world,
                             target_sync_every=0, prefetch=prefetch)


def time_gather_kernel(rl, rp, iters=64, reps=5):
    """Average duration per launch of the replay gather kernel alone, for the raw uint8 variant (SURVEY 8d accounting)
    and the fused bf16 space-to-depth variant the step uses.  ``iters`` launches, each with its own fresh random index
    vector into the 7 GB ring (every launch misses L2), are captured in one CUDA graph so that the host launch rate does
    not enter; CUDA events bracket the graph replay on the launching stream; best of ``reps`` replays / iters."""
    res = {}
    bufs_u8 = rp._buffers(B, torch.uint8, "nchw", tag=7)
    bufs_bf = rp._buffers(B, torch.bfloat16, "s2d", tag=7)
    idxs = [torch.randint(8, CAP - 8, (B,), device=rp.device) for _ in range(iters)]
    idxs = [torch.where((i > 123_440) & (i < 123_470), i + 100, i) for i in idxs]            # keep clear of the ring seam
    for name, fn in (("u8", lambda i: rp.gather(i, B, bufs_u8)),
                     ("bf16_s2d", lambda i: rp.gather(i, B, bufs_bf, torch.bfloat16, None, "s2d"))):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for i in idxs[:3]:
                fn(i)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in idxs:
                fn(i)
        best = 1e9
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            g.replay()
            b.record()
            torch.cuda.synchronize()
            best = min(best, a.elapsed_time(b) / iters)
        res[name] = float(best)
    return res


@contextlib.contextmanager
def stdout_to_stderr():
    """Route file descriptor 1 to stderr for the duration (library banners), so that stdout carries the one JSON line."""
    sys.stdout.flush()
    saved = os.dup(1)
    os.dup2(2, 1)
    try:
        yield
    finally:
        sys.stdout.flush()
        os.dup2(saved, 1)
        os.close(saved)


def timed_regions(step, K, repeats, barrier, world, dev, clocks=None):
    """``repeats`` timed regions of exactly K calls of ``step`` each (barrier + synchronize on both sides, CUDA events on
    the launching stream, max over ranks).  Returns the list of region times in ms."""
    import torch.distributed as dist
    out = []
    for _ in range(repeats):
        barrier()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(K):
            step()
        t1.record()
        barrier()
        ms = torch.tensor([t0.elapsed_time(t1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        out.append(float(ms))
    return out


def median(xs):
    return float(np.median(np.asarray(xs, dtype=np.float64)))


def measure_learner(rl, workload, dev, rank, world, K, W, repeats, barrier, prefetch, full, dump=None):
    """Build + capture + time one workload.  ``full``: also the end-to-end (host buffers) figure.  ``dump``: directory that
    receives what the last timed update computed (see dump_outputs)."""
    import gc
    learner = build_learner(rl, workload, dev, rank, world, prefetch=prefetch)
    if world > 1:                                          # parameters identical on every rank
        rl.parallel.broadcast_parameters(learner.opt.flat, 0)
        learner.tgt.load_state_dict(learner.net.state_dict())
    learner.capture(warmup=3, with_h2d=False)
    for _ in range(W):
        learner.update()
    reg = timed_regions(learner.update, K, repeats, barrier, world, dev)
    if dump and rank == 0:
        dump_outputs(learner, dump)
    res = dict(value=round(world * K / (median(reg) * 1e-3), 1), ms_per_step=round(median(reg) / K, 4),
               repeat_ms=[round(x, 4) for x in reg], loss=float(learner.loss),
               replay="async_replay=True" if learner.prefetch else ("async_replay=False, K1 (conv1 reads the uint8 ring)" if learner.ring
                                                                   else "async_replay=False"))
    # launches of OUR kernels per update (count one eager update; graph replays do not pass through the C ABI)
    rl._lib.reset_launch_count()
    learner._main(), learner._allreduce(), learner._opt()
    torch.cuda.synchronize()
    res["gpu_launches_per_step"] = int(rl._lib.launch_count())
    if full:
        learner.capture(warmup=1, with_h2d=True)
        rng = np.random.RandomState(rank)
        host = [(rng.randint(0, 256, (4, FRAME)).astype(np.uint8), rng.randint(0, ACTIONS, 4).astype(np.int32),
                 rng.choice([-1.0, 0.0, 1.0], 4), (rng.rand(4) > 1e-3).astype(np.int32)) for _ in range(16)]
        it = [0]
        last = [None]

        def e2e_step():
            last[0] = learner.update_from_host(*host[it[0] % 16], beta=0.4 + 0.6 * (it[0] % 1000) / 1000)
            it[0] += 1
        for _ in range(W):
            e2e_step()
        ereg = timed_regions(e2e_step, K, repeats, barrier, world, dev)
        res["e2e"] = dict(value=round(world * K / (median(ereg) * 1e-3), 1), unit="updates/s", h2d_bytes_per_step=learner.h2d_bytes,
                          d2h_bytes_per_step=4, ms_per_step=round(median(ereg) / K, 4), repeat_ms=[round(x, 4) for x in ereg])
        res["last_e2e_loss"] = last[0]
    return learner, res


def dump_outputs(learner, out_dir):
    """What the timed update hands its caller after the last timed step, as float32 .npy files: the parameter arena of the
    online network (every weight and bias after the optimizer step, 6.7 MB for DQN) and the loss of that update."""
    os.makedirs(out_dir, exist_ok=True)
    torch.cuda.synchronize()
    np.save(os.path.join(out_dir, "params.npy"), learner.opt.flat.detach().float().cpu().numpy())
    np.save(os.path.join(out_dir, "loss.npy"), np.atleast_1d(learner.loss.detach().float().cpu().numpy()))


def dump_ppo_outputs(ag, out_dir):
    """What the last timed PPO iteration leaves its caller, as float32 .npy files: every network parameter in
    ``named_parameters()`` order, and the state normaliser's running mean / variance."""
    os.makedirs(out_dir, exist_ok=True)
    torch.cuda.synchronize()
    flat = torch.cat([p.detach().float().reshape(-1) for p in ag.network.parameters()])
    np.save(os.path.join(out_dir, "params.npy"), flat.cpu().numpy())
    rms = ag.config.state_normalizer.rms
    f32 = lambda x: x.detach().float().cpu().numpy() if torch.is_tensor(x) else np.asarray(x, dtype=np.float32)
    np.save(os.path.join(out_dir, "state_mean.npy"), f32(rms.mean))
    np.save(os.path.join(out_dir, "state_var.npy"), f32(rms.var))


def leave(world):
    """End of a multi-rank run (deeprl_b200.parallel.leave: barrier, flush, exit without the process group's destructor)."""
    if world > 1:
        from deeprl_b200 import parallel
        parallel.leave()


def free(*objs):
    import gc
    for o in objs:
        del o
    gc.collect()
    torch.cuda.empty_cache()


def time_kernel_graph(fn, iters=20, reps=5):
    """Average duration of ``fn`` (one kernel launch) when ``iters`` launches run back to back in a CUDA graph."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    best = 1e9
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b) / iters)
    return float(best)


def tensor_roofline(rl, learner, pk, value, world, workload):
    """The dominant wgmma kernel family (conv1 forward: the largest share of the step's kernel time) timed alone, and the
    whole step's dense flops against the sustained bf16 peak."""
    from deeprl_b200.network import nature_tc
    dev = learner.dev
    body = learner.net.body
    pkd = body._packed
    x0 = torch.randint(0, 256, (B * 441, 64), device=dev).to(torch.bfloat16)
    x1 = torch.empty((B * 100, 128), dtype=torch.bfloat16, device=dev)
    b1 = body.conv1.bias.detach()
    us = time_kernel_graph(lambda: nature_tc.conv_gemm(0, x0, pkd.w1f, 32, 4, 2, 21, 1, x1, bias=b1, relu=True, out_map=1, G=21,
                                                       V=20, block_n=32)) * 1e3
    flops = 2.0 * B * 441 * 32 * 256
    ach = flops / (us * 1e-6) / 1e12
    burst = pk.get("bf16_tflops", 989.0)
    sust = pk.get("bf16_tflops_sustained", 989.0)
    step_flops = FLOPS_PER_UPDATE.get(workload)
    return dict(bound="tensor", kernel="conv_slab_wgmma_kernel<32> (conv1 forward, 2x2 taps x 64 channels, N = 32)",
                achieved=round(ach, 1), peak=burst, unit="TFLOP/s", frac=round(ach / burst, 4), us_per_launch=round(us, 2),
                flops_per_launch=flops, peak_source="MEASURED_PEAKS.json bf16_tflops (burst: kernel timed alone)" if "bf16_tflops" in pk
                else "fallback 989 (H100 SXM data sheet, dense bf16)",
                whole_step=(dict(flops_per_update=step_flops, achieved_tflops=round(step_flops * value / world / 1e12, 1),
                                 peak=sust, frac=round(step_flops * value / world / (sust * 1e12), 4),
                                 peak_source="bf16_tflops_sustained (kernels timed inside a long step)") if step_flops else None))


def agent_e2e(rl, steps=48):
    """Updates/s through the reference's own seam: ``DQNAgent.step()`` (DQN_agent.py:101-138) with ``config.cuda_graph``:
    per step the actor plays sgd_update_frequency = 4 env steps on the host (batch-1 forward each, itself a captured launch
    sequence), the transitions are fed to the HBM ring and ONE captured update runs.  Batch 512, 100k-transition ring, SyntheticAtari-v0."""
    c = rl.Config()
    c.merge(dict(tag=None))
    c.task_fn = lambda: rl.Task("SyntheticAtari-v0", seed=2)
    c.eval_env = rl.Task("SyntheticAtari-v0", seed=2)
    c.optimizer_fn = lambda p: torch.optim.RMSprop(p, lr=0.00025, alpha=0.95, eps=0.01, centered=True)
    c.network_fn = lambda: rl.VanillaNet(c.action_dim, rl.NatureConvBody(in_channels=4))
    c.random_action_prob = rl.LinearSchedule(1.0, 0.01, 1e6)
    c.batch_size = B
    c.replay_fn = lambda: rl.ReplayWrapper(rl.UniformReplay, dict(memory_size=100_000, batch_size=B, n_step=1, discount=0.99,
                                                                  history_length=4), async_=False)
    c.state_normalizer, c.reward_normalizer = rl.ImageNormalizer(), rl.SignNormalizer()
    c.discount, c.history_length, c.double_q, c.n_step = 0.99, 4, False, 1
    c.target_network_update_freq, c.exploration_steps, c.sgd_update_frequency, c.gradient_clip = 10_000, 700, 4, 5
    c.async_actor = False
    c.cuda_graph = True
    ag = rl.DQNAgent(c)
    while ag.total_steps <= c.exploration_steps + 40:       # exploration phase + graph capture + a few captured updates
        ag.step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        ag.step()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    ok = getattr(ag, "_learner", None) is not None
    ag.close()
    return dict(value=round(steps / dt, 1), unit="updates/s", steps=steps, graph_path=bool(ok),
                note="DQNAgent.step() through run_steps' seam: 4 host env steps, each with the actor's batch-1 forward as one captured "
                     "launch sequence (GraphedQActor: pinned frame upload -> wgmma network -> pinned q download), + feed + one "
                     "captured update per step; wall clock")


def run_b2rl(args):
    import torch.distributed as dist
    import deeprl_b200 as rl
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: the hot path has no CPU fallback (use --impl reference for the CPU arm)")
    torch.cuda.set_device(local)
    rl.select_device(local)
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda", local)
    if world > 1:
        with stdout_to_stderr():                           # NCCL prints its version banner on stdout at communicator creation
            dist.init_process_group("nccl", device_id=dev)
            dist.barrier()
            torch.cuda.synchronize()
    K, W, R = args.steps, max(args.warmup, 3), max(args.repeats, 1)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    if args.quick:                                        # A/B runs: the resident-input number only
        learner, res = measure_learner(rl, args.workload, dev, rank, world, K, W, 1, barrier, args.replay == "async", False,
                                       dump=args.dump_outputs)
        if rank == 0:
            print(json.dumps(dict(quick=True, value=res["value"], ms_per_step=res["ms_per_step"], loss=res["loss"],
                                  launches=res["gpu_launches_per_step"])), flush=True)
        leave(world)
        return

    with ClockSampler(local) as clocks:
        learner, main = measure_learner(rl, args.workload, dev, rank, world, K, W, R, barrier, args.replay == "async", True,
                                        dump=args.dump_outputs)
    # ---- the other replay mode (async_replay on / off), resident inputs
    pk = peaks()
    roof = roof_t = None
    if rank == 0:
        gt = time_gather_kernel(rl, learner.replay)
        roof_t = tensor_roofline(rl, learner, pk, main["value"], world, args.workload)
    free(learner)
    learner = None
    _, other = measure_learner(rl, args.workload, dev, rank, world, K, W, min(R, 3), barrier, args.replay != "async", False)
    free(_)
    extras = {}
    if not args.no_extras:
        for w in ("dqn", "per", "c51", "qr"):
            if w == args.workload:
                continue
            lw, rw = measure_learner(rl, w, dev, rank, world, K, W, min(R, 3), barrier, args.replay == "async", True)
            free(lw)
            extras[w] = dict(metric="gradient-updates/sec", value=rw["value"], unit="updates/s", ms_per_step=rw["ms_per_step"],
                             repeat_ms=rw["repeat_ms"], e2e=rw["e2e"], gpu_launches_per_step=rw["gpu_launches_per_step"],
                             config=WORKLOADS[w], replay=rw["replay"])
    if world > 1:
        barrier()
    if rank != 0:
        leave(world)                                       # (its barrier waits for rank 0 to print the line)
        return
    single = world == 1                                    # PPO, the agent-API run and the CPU baseline are N=1 measurements
    if not args.no_extras and single:
        try:
            extras["ppo"] = ppo_result(rl, args, quiet=True)
        except Exception as e:                             # noqa: BLE001 -- an extra must never take the headline line down
            extras["ppo"] = dict(error=str(e).splitlines()[0][:200])
    # ---- roofline of the replay gather kernel, timed alone (burst peak applies)
    hbm = pk.get("hbm_gbs", 3350.0)
    ach = B * ALGO_BYTES / (gt["bf16_s2d"] * 1e-3) / 1e9
    ach_u8 = B * ALGO_BYTES / (gt["u8"] * 1e-3) / 1e9
    roof = dict(bound="hbm", kernel="gather_cvt_kernel<bf16, space-to-depth> (replay sample: frame-stack gather -> exact u8->bf16 -> "
                                    "conv1 input layout; the kernel the step launches with async_replay)",
                achieved=round(ach, 1), peak=hbm, unit="GB/s", frac=round(ach / hbm, 4),
                peak_source="MEASURED_PEAKS.json hbm_gbs (burst: kernel timed alone)" if "hbm_gbs" in pk else "fallback 3350 (H100 SXM data sheet)",
                us_per_launch=round(gt["bf16_s2d"] * 1e3, 2), algorithmic_bytes_per_launch=B * ALGO_BYTES,
                algorithmic_bytes_definition="SURVEY 8d: 512 samples x (5 unique frames read + 2 x 4 frames written) x 7056 B = 91 728 B "
                                             "per sample (this variant writes bf16, i.e. twice the write bytes, most of which stay in L2)",
                raw_u8_variant=dict(kernel="gather_raw_tma_kernel (uint8 stacks: exactly the SURVEY 8d bytes; UniformReplay.sample())",
                                    achieved=round(ach_u8, 1), frac=round(ach_u8 / hbm, 4), us_per_launch=round(gt["u8"] * 1e3, 2)))
    ag = cpu = None
    if single:
        try:
            ag = agent_e2e(rl)
        except Exception as e:                             # noqa: BLE001
            ag = dict(error=str(e).splitlines()[0][:200])
        cpu = cpu_baseline(args.workload)                  # (selects the CPU device: last)
    line = dict(
        metric="gradient-updates/sec (DQN batch 512, 84x84x4 synthetic)", value=main["value"], unit="updates/s",
        n_gpus=world, steps=K, warmup=W, repeats=R, ms_per_step=main["ms_per_step"], repeat_ms=main["repeat_ms"],
        higher_is_better=True, scaling="weak", vs_baseline=None, dtype="bf16", data="synthetic",
        config=dict(workload=WORKLOADS[args.workload], batch=B, replay_capacity=CAP, replay_bytes=CAP * FRAME, actions=ACTIONS,
                    feeds_per_update=4, l2_policy="inputs larger than L2: 7.06 GB ring, fresh random indices every step",
                    parallelism="dp%d (rank-local replay shard, NCCL all-reduce of 6.7 MB fp32 gradients per step)" % world,
                    dense=("wgmma GEMM kernels (csrc/gemm.cu): bf16 operands, fp32 accumulation in registers, fp32 master weights"
                           if rl.Config.DENSE_BACKEND == "tcgen05" else "cuDNN/cuBLAS bf16 (fp32 accumulate, fp32 master weights)"),
                    replay=main["replay"], cuda_graph=True, timing="median of %d regions of %d steps" % (R, K)),
        e2e=main["e2e"], e2e_agent=ag, gpu_launches=int(main["gpu_launches_per_step"] * K),
        gpu_launches_per_step=main["gpu_launches_per_step"],
        other_replay_mode=dict(replay=other["replay"], value=other["value"], ms_per_step=other["ms_per_step"],
                               repeat_ms=other["repeat_ms"], gpu_launches_per_step=other["gpu_launches_per_step"]),
        clocks=clocks.summary(), roofline=roof, roofline_tensor=roof_t, cpu_baseline=cpu, loss=main["loss"],
        last_e2e_loss=main.get("last_e2e_loss"), extra_workloads=extras,
        tensor_frac_of_sustained=(roof_t["whole_step"]["frac"] if roof_t and roof_t.get("whole_step") else None),
    )
    print(json.dumps(line), flush=True)
    leave(world)


WORKLOADS = {"dqn": "DQN synthetic 84x84x4 uint8 frames, 1M-transition uniform Replay, batch 512, NatureConvBody, 1 H100 (BASELINE configs[1])",
             "per": "Prioritized Dueling Double-DQN, 1M sum-tree PrioritizedReplay, batch 512 (BASELINE configs[2])",
             "c51": "C51 51 atoms, batch 512 (BASELINE configs[4])", "qr": "QR-DQN 200 quantiles, batch 512 (BASELINE configs[4])"}


# --------------------------------------------------------------------------------------------- PPO (BASELINE configs[3])
def ppo_result(rl, args, quiet=False):
    """PPO on synthetic HalfCheetah-shaped states (17-dim obs, 6-dim action): 2048-step x 16-worker rollout, GAE(0.95),
    10 epochs x 64-sample minibatches (examples.py:496-522).  One "step" = one PPO iteration (rollout + GAE + advantage
    normalisation + 5 120 minibatch updates); the envs step on the host (north_star), everything else on the device."""
    dtype0 = rl.Config.COMPUTE_DTYPE
    rl.Config.COMPUTE_DTYPE = torch.float32
    try:
        torch.manual_seed(0), np.random.seed(0)
        c = rl.Config()
        c.merge(dict(tag=None))
        c.num_workers = 16
        c.task_fn = lambda: rl.Task("SyntheticCheetah-v0", num_envs=16, seed=0)
        c.eval_env = rl.Task("SyntheticCheetah-v0", seed=0)
        c.network_fn = lambda: rl.GaussianActorCriticNet(c.state_dim, c.action_dim, actor_body=rl.FCBody(c.state_dim, gate=torch.tanh),
                                                         critic_body=rl.FCBody(c.state_dim, gate=torch.tanh))
        c.actor_opt_fn = lambda p: torch.optim.Adam(p, 3e-4)
        c.critic_opt_fn = lambda p: torch.optim.Adam(p, 1e-3)
        c.discount, c.use_gae, c.gae_tau, c.gradient_clip = 0.99, True, 0.95, 0.5
        c.rollout_length, c.optimization_epochs, c.mini_batch_size, c.ppo_ratio_clip, c.target_kl = 2048, 10, 64, 0.2, 0.01
        c.state_normalizer = rl.MeanStdNormalizer()
        c.graph_minibatch = args.replay != "sync" or quiet    # --replay sync (stand-alone): the eager minibatch loop
        ag = rl.PPOAgent(c)
        sgd = [0.0]
        if c.graph_minibatch:                                 # time the minibatch phase on its own as well
            inner = ag._graphed_epochs

            def timed_epochs(entries):
                torch.cuda.synchronize()
                t = time.perf_counter()
                inner(entries)
                torch.cuda.synchronize()
                sgd[0] += time.perf_counter() - t
            ag._graphed_epochs = timed_epochs
        K, W = (1 if quiet else max(1, args.steps)), 1
        for _ in range(W):
            ag.step()
        torch.cuda.synchronize()
        rl._lib.reset_launch_count()
        sgd[0] = 0.0
        t0 = time.perf_counter()
        for _ in range(K):
            ag.step()
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / K
        if not quiet and getattr(args, "dump_outputs", None):
            dump_ppo_outputs(ag, args.dump_outputs)
        mb = c.optimization_epochs * (c.rollout_length * c.num_workers // c.mini_batch_size)
        res = dict(
            metric="PPO minibatch updates/sec (17-dim obs, 2048 x 16 rollout, GAE 0.95, 10 epochs x 64)", value=round(mb / dt, 1),
            unit="updates/s", n_gpus=1, steps=K, warmup=W, ms_per_step=round(dt * 1e3, 1), higher_is_better=True, scaling="weak",
            vs_baseline=None, dtype="f32", data="synthetic",
            config=dict(workload="PPO synthetic HalfCheetah-shape 17-dim obs, 2048-step x 16-worker rollout, GAE 0.95, 10 epochs x 64 "
                                 "minibatch (BASELINE configs[3]); one step = one PPO iteration incl. the host env rollout",
                        minibatch_updates_per_iteration=mb, env_steps_per_iteration=c.rollout_length * c.num_workers,
                        timing="wall clock around whole iterations (host envs + eager launches), torch.cuda.synchronize on both sides"),
            env_steps_per_s=round(c.rollout_length * c.num_workers / dt, 1),
            minibatch_phase=(dict(updates_per_s=round(mb * K / sgd[0], 1), seconds_per_iteration=round(sgd[0] / K, 3),
                                  form=("ONE persistent-kernel launch for all %d minibatch updates (PersistentPPOLearner: weights in shared "
                                        "memory, KL gate on the device)" % mb if type(ag._graph).__name__ == "PersistentPPOLearner"
                                        else "one CUDA-graph replay per minibatch (GraphedPPOLearner), KL gate on the device"))
                             if c.graph_minibatch else dict(form="eager loop (PPOAgent._minibatch)")),
            gpu_launches=int(rl._lib.launch_count() + (K * mb * ag._graph.launches_per_update if c.graph_minibatch else 0)),
            gpu_launches_per_minibatch=(round(ag._graph.launches_per_update, 4) if c.graph_minibatch else None))
        ag.close()
        return res
    finally:
        rl.Config.COMPUTE_DTYPE = dtype0


def run_ppo(args):
    import deeprl_b200 as rl
    if not torch.cuda.is_available():
        raise SystemExit("bench.py --workload ppo needs a CUDA device")
    rl.select_device(0)
    print(json.dumps(ppo_result(rl, args)), flush=True)


# --------------------------------------------------------------------------------------------- CPU arm (oracle port)
def make_cpu_agent(workload, capacity=20_000):
    """The reference's CPU path as restated in oracle/ (pinned against the reference by tests/test_oracle_golden.py):
    python-list replay with per-sample np.array stacking, float64 ImageNormalizer, torch-CPU networks, torch.optim."""
    from oracle import agents, nets  # noqa: F401
    from oracle.replay import PrioritizedReplay, UniformReplay
    import deeprl_b200 as rl
    rl.select_device(-1)
    torch.manual_seed(0)
    body = rl.NatureConvBody(in_channels=HIST)
    if workload == "per":
        net, head = rl.DuelingNet(ACTIONS, body), "dueling"
    elif workload == "c51":
        net, head = rl.CategoricalNet(ACTIONS, 51, body), "categorical"
    elif workload == "qr":
        net, head = rl.QuantileNet(ACTIONS, 200, body), "quantile"
    else:
        net, head = rl.VanillaNet(ACTIONS, body), "vanilla"
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    if workload in ("dqn", "per"):
        opt = lambda p: torch.optim.RMSprop(p, lr=0.00025, alpha=0.95, eps=0.01, centered=True)
    else:
        opt = lambda p: torch.optim.Adam(p, lr=0.00025, eps=0.01 / 32)
    orc = agents.DQNFamilyOracle(sd, head, "nature", ACTIONS, opt, 0.99, 1, double_q=(workload == "per"), gradient_clip=5,
                                 state_coef=1.0 / 255, atoms=np.linspace(-10, 10, 51) if workload == "c51" else None,
                                 v_min=-10, v_max=10, num_quantiles=200 if workload == "qr" else None,
                                 replay_beta=lambda: 0.4)
    cls = PrioritizedReplay if workload == "per" else UniformReplay
    rp = cls(capacity, B, 1, 0.99, HIST)
    rng = np.random.RandomState(0)
    for i in range(capacity):
        rp.feed(dict(state=[rng.randint(0, 256, (84, 84)).astype(np.uint8)], action=[int(rng.randint(ACTIONS))],
                     reward=[float(rng.choice([-1.0, 0.0, 1.0], p=[0.05, 0.9, 0.05]))], mask=[int(rng.rand() > 1e-3)]))
    return orc, rp, rng


def cpu_step(orc, rp, rng, workload):
    for _ in range(4):                                     # the 4 feeds per update (sgd_update_frequency)
        rp.feed(dict(state=[rng.randint(0, 256, (84, 84)).astype(np.uint8)], action=[int(rng.randint(ACTIONS))],
                     reward=[0.0], mask=[1]))
    if workload == "per":
        tr = rp.sample()
        orc.update(tr, rp)
    else:
        tr, _, _ = rp.sample()
        orc.update(tr)


def cpu_time_updates(workload, threads, seconds, min_updates=5, max_updates=20):
    """Median seconds per batch-512 update of the oracle port with ``threads`` torch threads: 1 warm-up, then updates until
    ``max_updates`` or until ``seconds`` have passed (but at least ``min_updates``)."""
    torch.set_num_threads(threads)
    orc, rp, rng = make_cpu_agent(workload)
    cpu_step(orc, rp, rng, workload)                       # warm-up
    ts, t_all = [], time.perf_counter()
    while len(ts) < max_updates and (len(ts) < min_updates or time.perf_counter() - t_all < seconds):
        t0 = time.perf_counter()
        cpu_step(orc, rp, rng, workload)
        ts.append(time.perf_counter() - t0)
    return ts


def cpu_baseline(workload, seconds=30.0):
    """The reference's torch-CPU path (oracle port) with its own default ``set_one_thread()`` (examples.py:623) and with 32
    threads (one NUMA node's worth; all 128+ threads of the box oversubscribe MKL-DNN and run 5-10x slower)."""
    cores = os.cpu_count() or 1
    cap = min(32, cores)
    one = cpu_time_updates(workload, 1, seconds)
    many = cpu_time_updates(workload, cap, seconds)
    v1, vn = 1.0 / float(np.median(one)), 1.0 / float(np.median(many))
    best_threads = cap if vn >= v1 else 1
    return dict(value=round(max(v1, vn), 4), unit="updates/s", cores=best_threads, kind="port", host_cores=cores,
                one_thread=dict(value=round(v1, 4), updates=len(one), median_s=round(float(np.median(one)), 3)),
                capped_threads=dict(threads=cap, value=round(vn, 4), updates=len(many), median_s=round(float(np.median(many)), 3)),
                sample="median of %d (1 thread, the reference's set_one_thread()) and %d (%d threads) full batch-512 updates (4 feeds + "
                       "sample + fwd/bwd + clip + optimizer) of the oracle port of the reference's torch-CPU path, replay capacity 20k "
                       "(its sampling cost does not depend on capacity); value = the faster of the two (%d thread(s))"
                       % (len(one), len(many), cap, best_threads))


def run_reference(args):
    if args.workload == "ppo":
        print(json.dumps(dict(impl="reference", unavailable="the CPU reference arm times the DQN-family update only")), flush=True)
        return
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    cpu = cpu_baseline(args.workload, seconds=60.0)
    v = cpu["value"]
    K = cpu["one_thread"]["updates"] + cpu["capped_threads"]["updates"]
    print(json.dumps(dict(
        impl="reference", metric="gradient-updates/sec (DQN batch 512, 84x84x4 synthetic)", value=round(v, 4),
        unit="updates/s", n_gpus=int(os.environ.get("WORLD_SIZE", "1")), steps=K, warmup=2, ms_per_step=round(1e3 / v, 2),
        higher_is_better=True, scaling="weak", vs_baseline=None, dtype="f32", data="synthetic",
        config=dict(workload="same as the b2rl arm: %s" % args.workload, batch=B, device="host CPU",
                    timing="median seconds per update, bounded sample (requested steps %d)" % args.steps),
        cpu_baseline=cpu,
        e2e=dict(value=round(v, 4), unit="updates/s", h2d_bytes_per_step=0, d2h_bytes_per_step=0))), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5, help="timed regions of --steps updates each; the median is reported")
    ap.add_argument("--impl", default="b2rl", choices=["b2rl", "reference"])
    ap.add_argument("--workload", default="dqn", choices=["dqn", "per", "c51", "qr", "ppo"])
    ap.add_argument("--replay", default="async", choices=["async", "sync"],
                    help="async_replay of the reference's launchers (examples.py:16 default True; :646 runs False); the other "
                         "mode is timed as well and reported under other_replay_mode")
    ap.add_argument("--quick", action="store_true", help="developer A/B runs: print the resident-input value only")
    ap.add_argument("--no-extras", action="store_true", help="skip the extra workloads (PER / C51 / QR / PPO)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed update computed (parameters, loss) as DIR/<name>.npy")
    a = ap.parse_args()
    if a.impl == "reference":
        run_reference(a)
    elif a.workload == "ppo":
        run_ppo(a)
    else:
        run_b2rl(a)
