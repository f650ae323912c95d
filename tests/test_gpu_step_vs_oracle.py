"""The assembled update that bench.py times (GraphedDQNLearner: bf16 wgmma body, K1 conv1 from the uint8 ring, fused loss,
fused backward epilogues, two-launch tail) against the oracle's fp32 restatement of ``DQNAgent.step``'s update
(DQN_agent.py:115-134; oracle/agents.py DQNFamilyOracle, pinned against the real reference by tests/test_oracle_golden.py)
on the SAME batch (the indices the learner sampled), the same weights, target network and optimizer state, at batch 512.

Tolerances are those of bf16 operands with fp32 accumulation: loss 2e-2 relative, gradient / parameter-delta cosine."""
import os
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import bench
    import deeprl_b200 as rl
    rl.select_device(0)
    rl.Config.COMPUTE_DTYPE = torch.bfloat16
    bench.CAP = 30_000
    return bench, rl


def cosine(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


@pytest.mark.parametrize("workload", ["dqn", "per", "c51", "qr"])
@pytest.mark.parametrize("prefetch", [False, True])
def test_learner_update_matches_oracle_update(env, workload, prefetch):
    bench, rl = env
    from oracle import agents
    dev = torch.device("cuda", 0)
    lr = bench.build_learner(rl, workload, dev, 0, 1, prefetch=prefetch)
    rp = lr.replay
    for _ in range(2):                                   # creates buffers, fills the prefetch slot
        lr._main(), lr._opt()
    # a clean optimizer state on both sides; remember parameters / target before the update under test
    lr.opt.s1.zero_(), lr.opt.s2.zero_(), lr.opt.step_dev.zero_()
    lr.refresh_packed()
    sd0 = {k: v.detach().float().cpu().clone() for k, v in lr.net.state_dict().items()}
    tgt0 = {k: v.detach().float().cpu().clone() for k, v in lr.tgt.state_dict().items()}
    flat0 = lr.opt.flat.clone()
    # ---- the update under test; the batch it trains on is the one in the buffer set of this parity
    parity = lr._parity if prefetch else 0
    lr._main()
    torch.cuda.synchronize()
    t = lr._batch[parity] if prefetch else None
    key = [k for k in rp._bufs if k[0] == bench.B and k[3] == parity and k[1] == torch.bfloat16][0]
    bufs = rp._bufs[key]
    idx = bufs["idx"].clone()
    grad = lr.opt.grad.clone()                           # kernel A wrote the reference-layout gradients here
    loss_dev = float(lr.loss)
    lr._opt()
    torch.cuda.synchronize()
    delta = (lr.opt.flat - flat0)
    # ---- the same batch for the oracle: uint8 stacks straight from the ring
    hl = rp.history_length
    rows = idx.view(-1, 1) + torch.arange(-(hl - 1), 1, device=dev).view(1, -1)
    frames = rp.frames.view(-1, 84, 84)
    tr = types.SimpleNamespace(state=frames[rows.view(-1)].view(-1, hl, 84, 84).cpu().numpy(),
                               next_state=frames[(rows + rp.n_step).view(-1)].view(-1, hl, 84, 84).cpu().numpy(),
                               action=bufs["action"].cpu().numpy(), reward=bufs["reward"].cpu().numpy(),
                               mask=bufs["mask"].cpu().numpy())
    head = {"dqn": "vanilla", "per": "dueling", "c51": "categorical", "qr": "quantile"}[workload]
    if workload in ("dqn", "per"):
        opt_fn = lambda p: torch.optim.RMSprop(p, lr=0.00025, alpha=0.95, eps=0.01, centered=True)
    elif workload == "c51":
        opt_fn = lambda p: torch.optim.Adam(p, lr=0.00025, eps=0.01 / 32)
    else:
        opt_fn = lambda p: torch.optim.Adam(p, lr=0.00005, eps=0.01 / 32)
    beta = float(lr.d_beta[0])
    orc = agents.DQNFamilyOracle(sd0, head, "nature", bench.ACTIONS, opt_fn, 0.99, 1, double_q=(workload == "per"), gradient_clip=5,
                                 state_coef=1.0 / 255, atoms=np.linspace(-10, 10, 51) if workload == "c51" else None, v_min=-10,
                                 v_max=10, num_quantiles=200 if workload == "qr" else None, replay_beta=lambda: beta)
    for k, v in tgt0.items():
        orc.target_sd[k].copy_(v)
    if workload == "per":
        tr.sampling_prob = bufs["prob"].cpu().numpy()
        tr.idx = bufs["tree_idx"].cpu().numpy()
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    before = {k: v.detach().clone() for k, v in orc.sd.items()}
    loss_orc = float(orc.update(tr))
    # ---- loss
    np.testing.assert_allclose(loss_dev, loss_orc, rtol=2e-2)
    # ---- gradients (the oracle's .grad is clipped in place; direction is what is compared) and parameter deltas
    names = [n for n, _ in lr.net.named_parameters()]
    base = lr.opt.flat.data_ptr()
    g_dev, g_orc, d_dev, d_orc = [], [], [], []
    for n, p in lr.net.named_parameters():
        off = (p.data_ptr() - base) // 4
        gd = grad[off:off + p.numel()].float().cpu()
        go = orc.sd[n].grad.flatten()
        dd = delta[off:off + p.numel()].float().cpu()
        do = (orc.sd[n].detach() - before[n]).flatten()
        if go.norm() > 1e-8:
            assert cosine(gd, go) > 0.98, "gradient direction of %s: %.5f" % (n, cosine(gd, go))
        g_dev.append(gd), g_orc.append(go), d_dev.append(dd), d_orc.append(do)
    assert cosine(torch.cat(g_dev), torch.cat(g_orc)) > 0.995
    assert cosine(torch.cat(d_dev), torch.cat(d_orc)) > 0.98
    # magnitudes: the clipped global norm and the size of the step
    n_dev = float(torch.cat(g_dev).norm()) * min(1.0, 5.0 / (float(torch.cat(g_dev).norm()) + 1e-6))
    np.testing.assert_allclose(n_dev, float(torch.cat(g_orc).norm()), rtol=5e-2)
    np.testing.assert_allclose(float(torch.cat(d_dev).norm()), float(torch.cat(d_orc).norm()), rtol=5e-2)
    assert names
