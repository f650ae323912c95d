"""The update schedule of GraphedDQNLearner (``learner.update_plan``) for the configurations the learner supports: which
replay read conv1 takes (K1 or the materialising gather), which head and forward layout run, where the async-replay
prefetch branch forks and where it joins the main stream.  Every row states the schedule the learner captures for that
configuration; no GPU is needed."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deeprl_b200.learner import update_plan  # noqa: E402

# defaults of every row: world 1, bf16, a K1-capable NatureConvBody, the fused tail available, narrow 16-byte aligned heads,
# no switch set
BEST = dict(k1_body=True, dual_body=True, tail=True, narrow_head=True, world=1, one_graph=True)
FP32 = dict(k1_body=False, dual_body=False, tail=False)
K1_OFF = {"B2RL_K1": "0"}
FUSED = {"B2RL_FUSED_HEAD": "1"}

# (case, update_plan arguments, ring, head, forward, prefetch, join)
ROWS = [
    ("dqn", dict(kind="dqn"), True, "separate", "two-branch", None, None),
    ("dqn-async", dict(kind="dqn", prefetch=True), True, "separate", "two-branch", "after-ring-read", "opt"),
    ("per-async", dict(kind="dqn", per=True, prefetch=True), False, "separate", "two-branch", "start", "main"),
    ("per", dict(kind="dqn", per=True), True, "separate", "two-branch", None, None),
    ("k1-off-async", dict(prefetch=True, env=K1_OFF), False, "separate", "two-branch", "gather-after-bwd", "opt"),
    ("prefetch-at-dgrad", dict(prefetch=True, env={**K1_OFF, "B2RL_PREFETCH_AT": "dgrad"}),
     False, "separate", "two-branch", "gather-after-dgrad", "opt"),
    ("prefetch-late-off", dict(prefetch=True, env={**K1_OFF, "B2RL_PREFETCH_LATE": "0"}),
     False, "separate", "two-branch", "start", "main"),
    ("fused-head-async", dict(prefetch=True, env=FUSED), False, "fused-two", "two-branch", "gather-after-bwd", "main"),
    ("fused-head-one", dict(prefetch=True, env={"B2RL_FUSED_HEAD": "one"}),
     False, "fused-one", "two-branch", "gather-after-bwd", "main"),
    ("fused-head-no-tail", dict(prefetch=True, env={**FUSED, "B2RL_TAIL": "0"}),
     False, "separate", "two-branch", "gather-after-bwd", "opt"),
    ("fused-head-sync", dict(env=FUSED), True, "fused-two", "two-branch", None, None),
    ("c51-fused-switch", dict(kind="c51", prefetch=True, env=FUSED), True, "separate", "two-branch", "after-ring-read", "opt"),
    ("dual-async", dict(prefetch=True, dual=True), False, "separate", "dual", "gather-after-bwd", "opt"),
    ("dual", dict(dual=True), False, "separate", "dual", None, None),
    ("single-stream", dict(prefetch=True, env={"B2RL_SINGLE_STREAM": "1"}),
     True, "separate", "one-stream", "after-ring-read", "opt"),
    ("c51-dist-head-off", dict(kind="c51", env={"B2RL_DIST_HEAD": "0"}), True, "separate", "two-branch", None, None),
    ("c51-dist-head-off-async", dict(kind="c51", prefetch=True, env={"B2RL_DIST_HEAD": "0"}),
     True, "separate", "two-branch", "after-ring-read", "opt"),
    ("world2-gather", dict(world=2, prefetch=True, env=K1_OFF), False, "separate", "two-branch", "gather-after-bwd", "opt"),
    ("world2-nccl-outside", dict(world=2, prefetch=True, env={**K1_OFF, "B2RL_NCCL_IN_GRAPH": "0"}),
     False, "separate", "two-branch", "start", "main"),
    ("world2-capture-failed", dict(world=2, prefetch=True, one_graph=False, env=K1_OFF),
     False, "separate", "two-branch", "start", "main"),
    ("world2-k1-split", dict(world=2, prefetch=True, one_graph=False), True, "separate", "two-branch", "after-ring-read", "main"),
    ("fp32", dict(**FP32), False, "separate", "two-branch", None, None),
    ("fp32-async", dict(prefetch=True, **FP32), False, "separate", "two-branch", "gather-after-bwd", "opt"),
    ("fp32-per-async", dict(per=True, prefetch=True, **FP32), False, "separate", "two-branch", "start", "main"),
]


@pytest.mark.parametrize("case,args,ring,head,forward,prefetch,join", ROWS, ids=[r[0] for r in ROWS])
def test_update_plan(case, args, ring, head, forward, prefetch, join):
    p = update_plan(**{**BEST, **args})
    assert (p.ring, p.head, p.forward, p.prefetch, p.join) == (ring, head, forward, prefetch, join)
    assert p.tail == (args.get("tail", True) and args.get("env", {}).get("B2RL_TAIL") != "0")
    assert p.repack_online == (not p.tail)                 # without the fused tail the online operands are re-packed
    assert p.single_stream == (forward == "one-stream")
    assert p.dist_head == (args.get("kind") in ("c51", "qr") and p.tail and args.get("env", {}).get("B2RL_DIST_HEAD") != "0")
    assert p.one_graph == (args.get("one_graph", True) and
                           (args.get("world", 1) == 1 or args.get("env", {}).get("B2RL_NCCL_IN_GRAPH") != "0"))


def test_fused_head_switch_needs_the_fused_tail_and_narrow_heads():
    """The fused head needs the tail's bias-gradient buffer and heads under 32 outputs; without them the separate kernels
    run, but the switch still keeps the materialising gather under async replay."""
    for kw in (dict(tail=False), dict(narrow_head=False)):
        p = update_plan(**{**BEST, "prefetch": True, "env": FUSED, **kw})
        assert (p.ring, p.head, p.prefetch, p.join) == (False, "separate", "gather-after-bwd", "opt")
    p = update_plan(**{**BEST, "env": FUSED, "narrow_head": False})
    assert p.ring and p.head == "separate"


def test_prefetch_at_dgrad_on_the_fused_head_forks_after_the_backward_pass():
    """The fused head's backward has no dgrad hook: B2RL_PREFETCH_AT=dgrad leaves its gather after the backward pass."""
    p = update_plan(**{**BEST, "prefetch": True, "env": {**FUSED, "B2RL_PREFETCH_AT": "dgrad"}})
    assert (p.head, p.prefetch, p.join) == ("fused-two", "gather-after-bwd", "main")


def test_single_stream_and_dual_switches():
    """B2RL_SINGLE_STREAM keeps the dual forward (its weight gradients move to the main stream) and does not apply to the
    fused head, whose body forwards always fork."""
    p = update_plan(**{**BEST, "dual": True, "env": {"B2RL_SINGLE_STREAM": "1"}})
    assert p.forward == "dual" and p.single_stream
    p = update_plan(**{**BEST, "env": {**FUSED, "B2RL_SINGLE_STREAM": "1"}})
    assert p.head == "fused-two" and p.forward == "two-branch" and not p.single_stream
    p = update_plan(**{**BEST, "dual": True, "dual_body": False})
    assert not p.ring and p.forward == "two-branch"        # dual requested on bodies without it: no K1 either


def test_per_async_prioritized_keeps_whole_branch_at_start_under_every_switch():
    for env in ({}, K1_OFF, {"B2RL_PREFETCH_AT": "dgrad"}, FUSED):
        p = update_plan(**{**BEST, "per": True, "prefetch": True, "env": env})
        assert not p.ring and (p.prefetch, p.join) == ("start", "main")
