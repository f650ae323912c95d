"""The coverage predicates (component/coverage.py) return the same reason, byte for byte, for every row of one table: per
predicate the accepted configuration (``None`` on a faked CUDA device), one row per condition in check order, and rows that
fail two conditions, which pin the order.  ``q_actor_unsupported`` is pinned by its decision (``None`` or not).

The expected strings were not written by hand: they are what this table gave when run against the predicates as they were
in component/actor.py before they moved here, with ``torch.Tensor.is_cuda`` forced for the rows on a "CUDA device" and the
C ABI's shared-memory sizes stubbed as here.  The real sizes are checked against the kernels by the GPU refusal tests
(``test_unsupported_configurations_are_refused``)."""
import contextlib
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SMEM_FITS = 64 * 1024
GLOBALS = dict(dtype=torch.bfloat16, backend="tcgen05", fused_bwd=True, conv_slab=2)   # the accepted rows' settings


@contextlib.contextmanager
def _settings(rl, smem, **change):
    """The module-level switches the captured predicates read, and ``_lib.lib()`` as a stub whose every
    ``*_smem_bytes`` returns ``smem``."""
    from deeprl_b200 import _lib
    from deeprl_b200.network import nature_tc
    g = dict(GLOBALS, **change)
    saved = (rl.Config.COMPUTE_DTYPE, rl.Config.DENSE_BACKEND, nature_tc.FUSED_BWD, _lib.CONV_SLAB, _lib.lib)
    rl.Config.COMPUTE_DTYPE, rl.Config.DENSE_BACKEND = g["dtype"], g["backend"]
    nature_tc.FUSED_BWD, _lib.CONV_SLAB = g["fused_bwd"], g["conv_slab"]
    _lib.lib = lambda: types.SimpleNamespace(**{k: (lambda *a: smem) for k in (
        "b2rl_a2c_smem_bytes", "b2rl_nstep_dqn_smem_bytes", "b2rl_dqn_replay_smem_bytes", "b2rl_dist_dqn_smem_bytes",
        "b2rl_rainbow_smem_bytes")})
    try:
        yield
    finally:
        rl.Config.COMPUTE_DTYPE, rl.Config.DENSE_BACKEND, nature_tc.FUSED_BWD, _lib.CONV_SLAB, _lib.lib = saved


def _config(rl, base, change):
    c = rl.Config()
    for k, v in dict(base, **change).items():
        setattr(c, k, v)
    return c


def _agent(cls, config, network, optimizer=None, flat=True, replay=None):
    ag = cls.__new__(cls)
    ag.config, ag.network = config, network
    ag.optimizer = optimizer if optimizer is not None else torch.optim.RMSprop(network.parameters(), 1e-3)
    ag._flat = object() if flat else None
    ag.replay = replay
    return ag


def _wrapper(rl, replay_cls=None, async_=True, primed=False, history_length=4):
    w = rl.ReplayWrapper.__new__(rl.ReplayWrapper)
    w.replay_cls, w.async_, w._primed = replay_cls or rl.UniformReplay, async_, primed
    w.replay_kwargs = dict(memory_size=100, batch_size=32, history_length=history_length)
    return w


def cases(rl):
    """(predicate, label, on CUDA, smem bytes, settings change, make): ``make()`` returns the predicate's arguments."""
    nets = {}

    def net(key, build):                                  # the networks are built once (the predicates only read them)
        if key not in nets:
            torch.manual_seed(0)
            nets[key] = build()
        return nets[key]

    uint8 = [np.zeros((4, 84, 84), np.uint8)] * 2
    rms = lambda n, **k: torch.optim.RMSprop(n.parameters(), 1e-3, **k)
    adam = lambda n, **k: torch.optim.Adam(n.parameters(), 1e-3, **k)
    sgd = lambda n: torch.optim.SGD(n.parameters(), 1e-3)
    rows = []

    def add(pred, label, make, cuda=True, smem=SMEM_FITS, **change):
        rows.append((pred, label, cuda, smem, change, make))

    # ---- nstep_q_graph_unsupported(config, network, optimizer, states)
    vnat = lambda A=4, **k: net(("vnat", A, tuple(k.items())), lambda: rl.VanillaNet(A, rl.NatureConvBody(**k)))

    def nq(network=None, opt=None, states=uint8, **kw):
        n = network or vnat()
        c = _config(rl, dict(cuda_graph=True, state_normalizer=rl.ImageNormalizer()), kw)
        return lambda: (c, n, (opt or rms)(n), states)

    P = "nstep_q_graph_unsupported"
    add(P, "accepted", nq())
    add(P, "no_cuda_graph", nq(cuda_graph=False))
    add(P, "device_nstep_dqn", nq(device_nstep_dqn=True))
    add(P, "dueling", nq(net("dnat", lambda: rl.DuelingNet(4, rl.NatureConvBody()))))
    add(P, "fc_body", nq(net("vfc", lambda: rl.VanillaNet(4, rl.FCBody(16)))))
    add(P, "noisy_body", nq(vnat(noisy_linear=True)))
    add(P, "noisy_config", nq(noisy_linear=True))
    add(P, "channels", nq(vnat(in_channels=1)))
    add(P, "fp32", nq(), dtype=torch.float32)
    add(P, "library", nq(), backend="library")
    add(P, "fused_bwd_off", nq(), fused_bwd=False)
    add(P, "conv_slab_off", nq(), conv_slab=0)
    add(P, "actions", nq(vnat(32)))
    add(P, "normalizer", nq(state_normalizer=rl.MeanStdNormalizer()))
    add(P, "float_frames", nq(states=[np.zeros((4, 84, 84), np.float32)]))
    add(P, "frame_shape", nq(states=[np.zeros((1, 84, 84), np.uint8)]))
    add(P, "sgd", nq(opt=sgd))
    add(P, "rmsprop_momentum", nq(opt=lambda n: rms(n, momentum=0.9)))
    add(P, "adam_amsgrad", nq(opt=lambda n: adam(n, amsgrad=True)))
    add(P, "cpu", nq(), cuda=False)
    add(P, "no_cuda_graph+device_flag", nq(cuda_graph=False, device_nstep_dqn=True))
    add(P, "fc_body+noisy_config", nq(net("vfc", None), noisy_linear=True))
    add(P, "fp32+cpu", nq(), cuda=False, dtype=torch.float32)
    add(P, "normalizer+float_frames", nq(states=[np.zeros((4, 84, 84), np.float32)], state_normalizer=rl.MeanStdNormalizer()))
    add(P, "sgd+cpu", nq(opt=sgd), cuda=False)

    # ---- a2c_graph_unsupported / ppo_graph_unsupported(config, network, optimizer, states)
    acnat = lambda A=4, **k: net(("acnat", A, tuple(k.items())), lambda: rl.CategoricalActorCriticNet(
        None, A, phi_body=rl.NatureConvBody(**{a: b for a, b in k.items() if a != "actor_fc"}),
        actor_body=rl.FCBody(512) if k.get("actor_fc") else None))

    def ac(network=None, opt=None, states=uint8, **kw):
        n = network or acnat()
        c = _config(rl, dict(cuda_graph=True, state_normalizer=rl.ImageNormalizer(), shared_repr=True, rollout_length=128,
                             num_workers=8, mini_batch_size=256), kw)
        return lambda: (c, n, (opt or rms)(n), states)

    acfc = lambda: net("acfc", lambda: rl.CategoricalActorCriticNet(None, 4, phi_body=rl.FCBody(16)))
    for P in ("a2c_graph_unsupported", "ppo_graph_unsupported"):
        add(P, "accepted", ac())
        add(P, "no_cuda_graph", ac(cuda_graph=False))
        add(P, "device_a2c", ac(device_a2c=True))
        add(P, "vanilla", ac(vnat()))
        add(P, "fc_phi_body", ac(acfc()))
        add(P, "actor_body", ac(acnat(actor_fc=True)))
        add(P, "noisy_body", ac(acnat(noisy_linear=True)))
        add(P, "noisy_config", ac(noisy_linear=True))
        add(P, "channels", ac(acnat(in_channels=1)))
        add(P, "fp32", ac(), dtype=torch.float32)
        add(P, "library", ac(), backend="library")
        add(P, "fused_bwd_off", ac(), fused_bwd=False)
        add(P, "actions", ac(acnat(32)))
        add(P, "normalizer", ac(state_normalizer=rl.MeanStdNormalizer()))
        add(P, "float_frames", ac(states=[np.zeros((4, 84, 84), np.float32)]))
        add(P, "sgd", ac(opt=sgd))
        add(P, "adam_weight_decay", ac(opt=lambda n: adam(n, weight_decay=1e-4)))
        add(P, "cpu", ac(), cuda=False)
        add(P, "device_a2c+vanilla", ac(vnat(), device_a2c=True))
        add(P, "fc_phi_body+actor_body", ac(net("acfc2", lambda: rl.CategoricalActorCriticNet(
            None, 4, phi_body=rl.FCBody(16), actor_body=rl.FCBody(512)))))
        add(P, "actor_body+noisy_config", ac(acnat(actor_fc=True), noisy_linear=True))
        add(P, "actions+normalizer", ac(acnat(32), state_normalizer=rl.MeanStdNormalizer()))
        add(P, "adam_weight_decay+cpu", ac(opt=lambda n: adam(n, weight_decay=1e-4)), cuda=False)
    P = "ppo_graph_unsupported"
    add(P, "not_shared", ac(shared_repr=False))
    add(P, "short_minibatch", ac(mini_batch_size=300))
    add(P, "one_row", ac(rollout_length=1, num_workers=1, mini_batch_size=1))
    add(P, "no_cuda_graph+not_shared", ac(cuda_graph=False, shared_repr=False))
    add(P, "not_shared+short_minibatch", ac(shared_repr=False, mini_batch_size=300))
    add(P, "short_minibatch+fp32", ac(mini_batch_size=300), dtype=torch.float32)

    # ---- dqn_graph_unsupported(config, agent)
    space = lambda shape=(4, 84, 84), dtype=np.uint8: types.SimpleNamespace(
        observation_space=types.SimpleNamespace(shape=shape, dtype=dtype))

    class Hooked(rl.DQNAgent):
        def reduce_loss(self, loss):
            return loss.pow(2).mean()

    class OtherReplay:
        pass

    def dg(cls=rl.DQNAgent, network=None, opt=None, replay=None, env=None, **kw):
        n = network or vnat()
        c = _config(rl, dict(cuda_graph=True, state_normalizer=rl.ImageNormalizer(), async_actor=True), kw)
        c._eval_env = env or space()
        return lambda: (c, _agent(cls, c, n, (opt or rms)(n), replay=replay or _wrapper(rl)))

    cnat = lambda: net("cnat", lambda: rl.CategoricalNet(4, 51, rl.NatureConvBody()))
    qnat = lambda: net("qnat", lambda: rl.QuantileNet(4, 20, rl.NatureConvBody()))
    P = "dqn_graph_unsupported"
    add(P, "accepted", dg())
    add(P, "accepted_dueling", dg(network=net("dnat", None)))
    add(P, "accepted_prioritized", dg(replay=_wrapper(rl, rl.PrioritizedReplay)))
    add(P, "accepted_c51", dg(rl.CategoricalDQNAgent, cnat()))
    add(P, "accepted_qr", dg(rl.QuantileRegressionDQNAgent, qnat()))
    add(P, "no_cuda_graph", dg(cuda_graph=False))
    for flag in ("device_dqn", "device_c51", "device_qr", "device_rainbow"):
        add(P, flag, dg(**{flag: True}))
    add(P, "not_a_wrapper", dg(replay=types.SimpleNamespace(async_=True)))
    add(P, "sync_wrapper", dg(replay=_wrapper(rl, async_=False)))
    add(P, "replay_class", dg(replay=_wrapper(rl, OtherReplay)))
    add(P, "qr_prioritized", dg(rl.QuantileRegressionDQNAgent, qnat(), replay=_wrapper(rl, rl.PrioritizedReplay)))
    add(P, "rainbow_net", dg(network=net("rnat", lambda: rl.RainbowNet(4, 51, rl.NatureConvBody(), noisy_linear=False))))
    add(P, "noisy_config", dg(noisy_linear=True))
    add(P, "dqn_categorical_net", dg(network=cnat()))
    add(P, "c51_vanilla_net", dg(rl.CategoricalDQNAgent, vnat()))
    add(P, "fc_body", dg(network=net("vfc", None)))
    add(P, "noisy_body", dg(network=vnat(noisy_linear=True)))
    add(P, "fp32", dg(), dtype=torch.float32)
    add(P, "library", dg(), backend="library")
    add(P, "fused_bwd_off", dg(), fused_bwd=False)
    add(P, "normalizer", dg(state_normalizer=rl.MeanStdNormalizer()))
    add(P, "channels", dg(network=vnat(in_channels=1)))
    add(P, "history_length", dg(replay=_wrapper(rl, history_length=1)))
    add(P, "float_frames", dg(env=space(dtype=np.float32)))
    add(P, "frame_shape", dg(env=space(shape=(84, 84))))
    add(P, "no_eval_env", dg(env=types.SimpleNamespace()))
    add(P, "workers", dg(num_workers=2))
    add(P, "sgd", dg(opt=sgd))
    add(P, "hooks", dg(Hooked))
    add(P, "primed", dg(replay=_wrapper(rl, primed=True)))
    add(P, "cpu", dg(), cuda=False)
    add(P, "device_dqn+sync_wrapper", dg(replay=_wrapper(rl, async_=False), device_dqn=True))
    add(P, "qr_prioritized+noisy_config", dg(rl.QuantileRegressionDQNAgent, qnat(), replay=_wrapper(rl, rl.PrioritizedReplay),
                                             noisy_linear=True))
    add(P, "normalizer+float_frames", dg(env=space(dtype=np.float32), state_normalizer=rl.MeanStdNormalizer()))
    add(P, "workers+sgd", dg(opt=sgd, num_workers=2))
    add(P, "hooks+primed", dg(Hooked, replay=_wrapper(rl, primed=True)))
    add(P, "primed+cpu", dg(replay=_wrapper(rl, primed=True)), cuda=False)

    # ---- q_actor_unsupported(config, network, states, async_ok): the decision only
    def qa(network=None, states=uint8, async_ok=False, **kw):
        n = network or vnat()
        c = _config(rl, dict(cuda_graph=True, state_normalizer=rl.ImageNormalizer(), async_actor=False), kw)
        return lambda: (c, n, states, async_ok)

    P = "q_actor_unsupported"
    add(P, "accepted", qa())
    add(P, "accepted_async_ordered", qa(async_actor=True, async_ok=True))
    add(P, "async_unordered", qa(async_actor=True))
    add(P, "no_cuda_graph", qa(cuda_graph=False))
    add(P, "noisy_config", qa(noisy_linear=True))
    add(P, "fc_body", qa(net("vfc", None)))
    add(P, "no_body", qa(acnat()))
    add(P, "noisy_body", qa(vnat(noisy_linear=True)))
    add(P, "channels", qa(vnat(in_channels=1)))
    add(P, "fp32", qa(), dtype=torch.float32)
    add(P, "library", qa(), backend="library")
    add(P, "fused_bwd_off", qa(), fused_bwd=False)
    add(P, "normalizer", qa(state_normalizer=rl.MeanStdNormalizer()))
    add(P, "float_frames", qa(states=[np.zeros((4, 84, 84), np.float32)]))
    add(P, "cpu", qa(), cuda=False)

    # ---- a2c_unsupported(network, optimizer, config)
    def fc(D=8, hidden=(64, 64), gate=torch.tanh, noisy=False):
        return rl.FCBody(D, hidden, gate=gate, noisy_linear=noisy)

    cat = lambda A=4, **k: net(("cat", A, tuple(k.items())), lambda: rl.CategoricalActorCriticNet(
        None, A, phi_body=fc(**k)))
    gauss = lambda A=2, actor=None, critic=None, phi=None: net(("gauss", A, actor, critic, phi), lambda: (
        rl.GaussianActorCriticNet(None, A, phi_body=None if phi is None else fc(**dict(phi)),
                                  actor_body=fc(**dict(actor or ())), critic_body=fc(**dict(critic or ())))))

    def a2(network=None, opt=None, **kw):
        n = network or cat()
        c = _config(rl, dict(num_workers=16, rollout_length=5), kw)
        return lambda: (n, (opt or rms)(n), c)

    P = "a2c_unsupported"
    add(P, "accepted_categorical", a2())
    add(P, "accepted_gaussian", a2(gauss()))
    add(P, "accepted_relu", a2(cat(gate=F.relu)))
    add(P, "categorical_dummy_phi", a2(net("cat_dummy", lambda: rl.CategoricalActorCriticNet(8, 4))))
    add(P, "categorical_three_layers", a2(cat(hidden=(64, 64, 64))))
    add(P, "categorical_noisy", a2(cat(noisy=True)))
    add(P, "categorical_actor_body", a2(net("cat_actor", lambda: rl.CategoricalActorCriticNet(
        None, 4, phi_body=fc(), actor_body=fc(64)))))
    add(P, "gaussian_fc_phi", a2(gauss(phi=(("hidden", (8, 8)),))))
    add(P, "gaussian_three_layers", a2(gauss(actor=(("hidden", (64, 64, 64)),))))
    add(P, "other_network", a2(net("vfc8", lambda: rl.VanillaNet(4, fc()))))
    add(P, "widths", a2(gauss(critic=(("hidden", (32, 32)),))))
    add(P, "gates", a2(gauss(critic=(("gate", F.relu),))))
    add(P, "gate", a2(cat(gate=torch.sigmoid)))
    add(P, "cpu", a2(), cuda=False)
    add(P, "state_dim", a2(cat(D=300)))
    add(P, "hidden1", a2(cat(hidden=(129, 64))))
    add(P, "hidden2", a2(cat(hidden=(64, 129))))
    add(P, "actions", a2(cat(33)))
    add(P, "adam", a2(opt=adam))
    add(P, "image_normalizer", a2(state_normalizer=rl.ImageNormalizer()))
    add(P, "smem", a2(), smem=300 * 1024)
    add(P, "smem_zero", a2(), smem=0)
    add(P, "gate+cpu", a2(cat(gate=torch.sigmoid)), cuda=False)
    add(P, "cpu+state_dim", a2(cat(D=300)), cuda=False)
    add(P, "actions+adam", a2(cat(33), opt=adam))
    add(P, "adam+normalizer", a2(opt=adam, state_normalizer=rl.MeanStdNormalizer()))
    add(P, "normalizer+smem", a2(state_normalizer=rl.MeanStdNormalizer()), smem=300 * 1024)

    # ---- nstep_dqn_unsupported(network, optimizer, config)
    van = lambda A=4, **k: net(("van", A, tuple(k.items())), lambda: rl.VanillaNet(A, fc(**k)))

    def ns(network=None, opt=None, **kw):
        n = network or van()
        c = _config(rl, dict(num_workers=16, rollout_length=5), kw)
        return lambda: (n, (opt or rms)(n), c)

    P = "nstep_dqn_unsupported"
    add(P, "accepted", ns())
    add(P, "accepted_relu", ns(van(gate=F.relu)))
    add(P, "dueling", ns(net("duel", lambda: rl.DuelingNet(4, fc()))))
    add(P, "dummy_body", ns(net("vdummy", lambda: rl.VanillaNet(4, rl.DummyBody(8)))))
    add(P, "noisy", ns(van(noisy=True)))
    add(P, "three_layers", ns(van(hidden=(64, 64, 64))))
    add(P, "gate", ns(van(gate=torch.sigmoid)))
    add(P, "cpu", ns(), cuda=False)
    add(P, "state_dim", ns(van(D=300)))
    add(P, "one_action", ns(van(1)))
    add(P, "actions", ns(van(33)))
    add(P, "adam", ns(opt=adam))
    add(P, "image_normalizer", ns(state_normalizer=rl.ImageNormalizer()))
    add(P, "smem", ns(), smem=300 * 1024)
    add(P, "noisy+three_layers", ns(van(noisy=True, hidden=(64, 64, 64))))
    add(P, "three_layers+gate", ns(van(hidden=(64, 64, 64), gate=torch.sigmoid)))
    add(P, "gate+cpu", ns(van(gate=torch.sigmoid)), cuda=False)
    add(P, "actions+adam", ns(van(33), opt=adam))
    add(P, "normalizer+smem", ns(state_normalizer=rl.MeanStdNormalizer()), smem=300 * 1024)

    # ---- dqn_unsupported(agent)
    class OwnLoss(rl.DQNAgent):
        def reduce_loss(self, loss):
            return loss.pow(2).mean()

    def dq(cls=rl.DQNAgent, network=None, opt=None, flat=True, **kw):
        n = network or van()
        c = _config(rl, dict(async_actor=False, history_length=1, batch_size=32), kw)
        return lambda: (_agent(cls, c, n, (opt or rms)(n), flat),)

    cfc = lambda K=51, **k: net(("cfc", K, tuple(k.items())), lambda: rl.CategoricalNet(4, K, fc(**k)))
    P = "dqn_unsupported"
    add(P, "accepted", dq())
    add(P, "accepted_dueling", dq(network=net("duel", None)))
    add(P, "accepted_double_q", dq(double_q=True))
    add(P, "categorical_net", dq(network=cfc()))
    add(P, "hooks", dq(OwnLoss))
    add(P, "nature_body", dq(network=vnat()))
    add(P, "dummy_body", dq(network=net("vdummy", None)))
    add(P, "noisy_body", dq(network=van(noisy=True)))
    add(P, "noisy_config", dq(noisy_linear=True))
    add(P, "three_layers", dq(network=van(hidden=(64, 64, 64))))
    add(P, "gate", dq(network=van(gate=torch.sigmoid)))
    add(P, "cpu", dq(), cuda=False)
    add(P, "state_dim", dq(network=van(D=300)))
    add(P, "one_action", dq(network=van(1)))
    add(P, "adam", dq(opt=adam))
    add(P, "no_flat", dq(flat=False))
    add(P, "image_normalizer", dq(state_normalizer=rl.ImageNormalizer()))
    add(P, "async_actor", dq(async_actor=True))
    add(P, "history_length", dq(history_length=4))
    add(P, "smem", dq(), smem=300 * 1024)
    add(P, "categorical_net+hooks", dq(OwnLoss, network=cfc()))
    add(P, "hooks+nature_body", dq(OwnLoss, network=vnat()))
    add(P, "nature_body+noisy_config", dq(network=vnat(), noisy_linear=True))
    add(P, "gate+cpu", dq(network=van(gate=torch.sigmoid)), cuda=False)
    add(P, "cpu+state_dim", dq(network=van(D=300)), cuda=False)
    add(P, "normalizer+async_actor", dq(state_normalizer=rl.MeanStdNormalizer(), async_actor=True))
    add(P, "async_actor+history_length", dq(async_actor=True, history_length=4))
    add(P, "history_length+smem", dq(history_length=4), smem=300 * 1024)

    # ---- dist_dqn_unsupported(agent)
    class OwnKL(rl.CategoricalDQNAgent):
        def reduce_loss(self, loss):
            return loss.sum()

    class OwnQuantile(rl.QuantileRegressionDQNAgent):
        def reduce_loss(self, loss):
            return loss.sum()

    qfc = lambda K=20, **k: net(("qfc", K, tuple(k.items())), lambda: rl.QuantileNet(4, K, fc(**k)))
    rfc = lambda noisy=False, **k: net(("rfc", noisy, tuple(k.items())), lambda: rl.RainbowNet(
        4, 51, fc(noisy=noisy, **k), noisy_linear=noisy))

    def dd(cls=rl.CategoricalDQNAgent, network=None, opt=None, flat=True, replay=None, **kw):
        n = network or (cfc() if cls is not rl.QuantileRegressionDQNAgent and cls is not OwnQuantile else qfc())
        c = _config(rl, dict(async_actor=True, batch_size=32), kw)
        return lambda: (_agent(cls, c, n, (opt or rms)(n), flat, replay or _wrapper(rl, history_length=1)),)

    QR = rl.QuantileRegressionDQNAgent
    P = "dist_dqn_unsupported"
    add(P, "accepted_c51", dd())
    add(P, "accepted_qr", dd(QR))
    add(P, "accepted_c51_prioritized", dd(replay=_wrapper(rl, rl.PrioritizedReplay)))
    add(P, "accepted_history_length_1", dd(history_length=1))
    add(P, "accepted_plain_replay", dd(QR, replay=types.SimpleNamespace()))
    add(P, "rainbow_net", dd(network=rfc()))
    add(P, "c51_quantile_net", dd(network=qfc()))
    add(P, "qr_categorical_net", dd(QR, cfc()))
    add(P, "hooks_c51", dd(OwnKL))
    add(P, "hooks_qr", dd(OwnQuantile))
    add(P, "nature_body", dd(network=cnat()))
    add(P, "noisy_body", dd(network=cfc(noisy=True)))
    add(P, "three_layers", dd(network=cfc(hidden=(64, 64, 64))))
    add(P, "gate", dd(network=cfc(gate=torch.sigmoid)))
    add(P, "cpu", dd(), cuda=False)
    add(P, "atoms", dd(network=cfc(K=300)))
    add(P, "quantiles", dd(QR, qfc(K=1)))
    add(P, "state_dim", dd(network=cfc(D=300)))
    add(P, "adam", dd(opt=adam))
    add(P, "no_flat", dd(flat=False))
    add(P, "image_normalizer", dd(state_normalizer=rl.ImageNormalizer()))
    add(P, "history_length", dd(history_length=4))
    add(P, "qr_prioritized", dd(QR, replay=_wrapper(rl, rl.PrioritizedReplay)))
    add(P, "smem", dd(), smem=300 * 1024)
    add(P, "rainbow_net+hooks", dd(OwnKL, rfc()))
    add(P, "hooks+noisy_body", dd(OwnKL, cfc(noisy=True)))
    add(P, "cpu+atoms", dd(network=cfc(K=300)), cuda=False)
    add(P, "history_length+qr_prioritized", dd(QR, replay=_wrapper(rl, rl.PrioritizedReplay), history_length=4))
    add(P, "qr_prioritized+smem", dd(QR, replay=_wrapper(rl, rl.PrioritizedReplay)), smem=300 * 1024)

    # ---- rainbow_unsupported(agent)
    def rb(cls=rl.CategoricalDQNAgent, network=None, opt=None, flat=True, noisy=True, **kw):
        n = network or rfc(noisy)
        c = _config(rl, dict(async_actor=True, batch_size=32, noisy_linear=noisy), kw)
        return lambda: (_agent(cls, c, n, (opt or rms)(n), flat),)

    P = "rainbow_unsupported"
    add(P, "accepted_noisy", rb())
    add(P, "accepted_linear", rb(noisy=False))
    add(P, "dqn_agent", rb(rl.DQNAgent))
    add(P, "categorical_net", rb(network=cfc()))
    add(P, "hooks", rb(OwnKL))
    add(P, "nature_body", rb(network=net("rnat", None), noisy=False))
    add(P, "dummy_body", rb(network=net("rdummy", lambda: rl.RainbowNet(4, 51, rl.DummyBody(8), noisy_linear=False))))
    add(P, "three_layers", rb(network=rfc(True, hidden=(64, 64, 64))))
    add(P, "mixed_noise", rb(noisy_linear=False))
    add(P, "gate", rb(network=rfc(True, gate=torch.sigmoid)))
    add(P, "cpu", rb(), cuda=False)
    add(P, "atoms", rb(network=net("r300", lambda: rl.RainbowNet(4, 300, fc(noisy=True), noisy_linear=True))))
    add(P, "one_action", rb(network=net("r1", lambda: rl.RainbowNet(1, 51, fc(noisy=True), noisy_linear=True))))
    add(P, "adam", rb(opt=adam))
    add(P, "no_flat", rb(flat=False))
    add(P, "image_normalizer", rb(state_normalizer=rl.ImageNormalizer()))
    add(P, "history_length", rb(history_length=4))
    add(P, "smem", rb(), smem=300 * 1024)
    add(P, "dqn_agent+categorical_net", rb(rl.DQNAgent, cfc()))
    add(P, "three_layers+mixed_noise", rb(network=rfc(True, hidden=(64, 64, 64)), noisy_linear=False))
    add(P, "mixed_noise+gate", rb(network=rfc(True, gate=torch.sigmoid), noisy_linear=False))
    add(P, "gate+cpu", rb(network=rfc(True, gate=torch.sigmoid)), cuda=False)
    add(P, "history_length+smem", rb(history_length=4), smem=300 * 1024)
    return rows


def evaluate(rl, predicates, fake_cuda):
    """{"predicate/label": what the predicate returned} over ``cases``; ``fake_cuda(flag)``: a context in which the networks
    are (``True``) or are not on a CUDA device."""
    out = {}
    for pred, label, cuda, smem, change, make in cases(rl):
        args = make()
        with _settings(rl, smem, **change), fake_cuda(cuda):
            out[pred + "/" + label] = predicates[pred](*args)
    return out


@pytest.fixture
def rl():
    import deeprl_b200 as rl
    rl.select_device(-1)
    return rl


def test_every_predicate_returns_its_pinned_reason(rl, monkeypatch):
    from deeprl_b200.component import coverage

    @contextlib.contextmanager
    def fake_cuda(flag):
        with monkeypatch.context() as m:
            m.setattr(coverage, "on_cuda", lambda network: flag)
            yield

    predicates = {name: getattr(coverage, name) for name in {k.split("/")[0] for k in EXPECTED}}
    predicates["q_actor_unsupported"] = lambda *a: coverage.q_actor_unsupported(*a) is None
    got = evaluate(rl, predicates, fake_cuda)
    assert sorted(got) == sorted(EXPECTED)
    for key, want in EXPECTED.items():
        assert got[key] == want, (key, got[key], want)


def test_every_predicate_has_an_accepted_row_and_a_cpu_row():
    """Every predicate has an accepted row and a row that fails only the device check, which is the reason it reports."""
    cuda = "the network is not on a CUDA device (select_device(0))"
    for pred in {k.split("/")[0] for k in EXPECTED}:
        accepted = [k for k in EXPECTED if k.startswith(pred + "/accepted")]
        assert accepted and all(EXPECTED[k] in (None, True) for k in accepted), pred
        if pred != "q_actor_unsupported":
            assert EXPECTED[pred + "/cpu"] == cuda, pred


EXPECTED = {
    'nstep_q_graph_unsupported/accepted': None,
    'nstep_q_graph_unsupported/no_cuda_graph': 'config.cuda_graph is not set',
    'nstep_q_graph_unsupported/device_nstep_dqn': 'config.device_nstep_dqn is set; it runs the agent on the device itself',
    'nstep_q_graph_unsupported/dueling': 'the network is a DuelingNet; the captured update implements VanillaNet',
    'nstep_q_graph_unsupported/fc_body': 'the body is a FCBody; the captured update implements NatureConvBody',
    'nstep_q_graph_unsupported/noisy_body': 'the network has NoisyLinear layers; the captured update implements nn.Linear',
    'nstep_q_graph_unsupported/noisy_config': 'the network has NoisyLinear layers; the captured update implements nn.Linear',
    'nstep_q_graph_unsupported/channels':
        'the NatureConvBody takes 1 channels; the captured update reads stacks of 4 frames',
    'nstep_q_graph_unsupported/fp32':
        ("the compute dtype is torch.float32 with the 'tcgen05' dense backend; the captured update runs bf16 on the wgmma "
         'kernels (tcgen05)'),
    'nstep_q_graph_unsupported/library':
        ("the compute dtype is torch.bfloat16 with the 'library' dense backend; the captured update runs bf16 on the wgmma"
         ' kernels (tcgen05)'),
    'nstep_q_graph_unsupported/fused_bwd_off':
        'the fused backward epilogues are switched off; the captured update needs the fused update tail',
    'nstep_q_graph_unsupported/conv_slab_off':
        'the fused backward epilogues are switched off; the captured update needs the fused update tail',
    'nstep_q_graph_unsupported/actions': '32 actions; the narrow head and loss kernels take fewer than 32',
    'nstep_q_graph_unsupported/normalizer':
        'the state normalizer is MeanStdNormalizer; the captured update folds a RescaleNormalizer into conv1',
    'nstep_q_graph_unsupported/float_frames': 'the envs do not return uint8 4 x 84 x 84 frame stacks',
    'nstep_q_graph_unsupported/frame_shape': 'the envs do not return uint8 4 x 84 x 84 frame stacks',
    'nstep_q_graph_unsupported/sgd':
        ('the optimizer is SGD; the fused update tail implements RMSprop (centered or not) and Adam without momentum, '
         'weight decay or amsgrad'),
    'nstep_q_graph_unsupported/rmsprop_momentum':
        ('the optimizer is RMSprop; the fused update tail implements RMSprop (centered or not) and Adam without momentum, '
         'weight decay or amsgrad'),
    'nstep_q_graph_unsupported/adam_amsgrad':
        ('the optimizer is Adam; the fused update tail implements RMSprop (centered or not) and Adam without momentum, '
         'weight decay or amsgrad'),
    'nstep_q_graph_unsupported/cpu': 'the network is not on a CUDA device (select_device(0))',
    'nstep_q_graph_unsupported/no_cuda_graph+device_flag': 'config.cuda_graph is not set',
    'nstep_q_graph_unsupported/fc_body+noisy_config': 'the body is a FCBody; the captured update implements NatureConvBody',
    'nstep_q_graph_unsupported/fp32+cpu':
        ("the compute dtype is torch.float32 with the 'tcgen05' dense backend; the captured update runs bf16 on the wgmma "
         'kernels (tcgen05)'),
    'nstep_q_graph_unsupported/normalizer+float_frames':
        'the state normalizer is MeanStdNormalizer; the captured update folds a RescaleNormalizer into conv1',
    'nstep_q_graph_unsupported/sgd+cpu':
        ('the optimizer is SGD; the fused update tail implements RMSprop (centered or not) and Adam without momentum, '
         'weight decay or amsgrad'),
    'a2c_graph_unsupported/accepted': None,
    'a2c_graph_unsupported/no_cuda_graph': 'config.cuda_graph is not set',
    'a2c_graph_unsupported/device_a2c': 'config.device_a2c is set; it runs the agent on the device itself',
    'a2c_graph_unsupported/vanilla': 'the network is a VanillaNet; the captured update implements CategoricalActorCriticNet',
    'a2c_graph_unsupported/fc_phi_body': 'the phi_body is a FCBody; the captured update implements NatureConvBody',
    'a2c_graph_unsupported/actor_body':
        'the actor / critic bodies are FCBody / DummyBody; the captured update implements DummyBody for both',
    'a2c_graph_unsupported/noisy_body': 'the network has NoisyLinear layers; the captured update implements nn.Linear',
    'a2c_graph_unsupported/noisy_config': 'the network has NoisyLinear layers; the captured update implements nn.Linear',
    'a2c_graph_unsupported/channels': 'the NatureConvBody takes 1 channels; the captured update reads stacks of 4 frames',
    'a2c_graph_unsupported/fp32':
        ("the compute dtype is torch.float32 with the 'tcgen05' dense backend; the captured update runs bf16 on the wgmma "
         'kernels (tcgen05)'),
    'a2c_graph_unsupported/library':
        ("the compute dtype is torch.bfloat16 with the 'library' dense backend; the captured update runs bf16 on the wgmma"
         ' kernels (tcgen05)'),
    'a2c_graph_unsupported/fused_bwd_off':
        'the fused backward epilogues are switched off; the captured update needs the fused update tail',
    'a2c_graph_unsupported/actions': '32 actions; the actor-critic head and loss kernels take fewer than 32',
    'a2c_graph_unsupported/normalizer':
        'the state normalizer is MeanStdNormalizer; the captured update folds a RescaleNormalizer into conv1',
    'a2c_graph_unsupported/float_frames': 'the envs do not return uint8 4 x 84 x 84 frame stacks',
    'a2c_graph_unsupported/sgd':
        ('the optimizer is SGD; the fused update tail implements RMSprop (centered or not) and Adam without momentum, '
         'weight decay or amsgrad'),
    'a2c_graph_unsupported/adam_weight_decay':
        ('the optimizer is Adam; the fused update tail implements RMSprop (centered or not) and Adam without momentum, '
         'weight decay or amsgrad'),
    'a2c_graph_unsupported/cpu': 'the network is not on a CUDA device (select_device(0))',
    'a2c_graph_unsupported/device_a2c+vanilla': 'config.device_a2c is set; it runs the agent on the device itself',
    'a2c_graph_unsupported/fc_phi_body+actor_body':
        'the phi_body is a FCBody; the captured update implements NatureConvBody',
    'a2c_graph_unsupported/actor_body+noisy_config':
        'the actor / critic bodies are FCBody / DummyBody; the captured update implements DummyBody for both',
    'a2c_graph_unsupported/actions+normalizer': '32 actions; the actor-critic head and loss kernels take fewer than 32',
    'a2c_graph_unsupported/adam_weight_decay+cpu':
        ('the optimizer is Adam; the fused update tail implements RMSprop (centered or not) and Adam without momentum, '
         'weight decay or amsgrad'),
    'ppo_graph_unsupported/accepted': None,
    'ppo_graph_unsupported/no_cuda_graph': 'config.cuda_graph is not set',
    'ppo_graph_unsupported/device_a2c': 'config.device_a2c is set; it runs the agent on the device itself',
    'ppo_graph_unsupported/vanilla': 'the network is a VanillaNet; the captured update implements CategoricalActorCriticNet',
    'ppo_graph_unsupported/fc_phi_body': 'the phi_body is a FCBody; the captured update implements NatureConvBody',
    'ppo_graph_unsupported/actor_body':
        'the actor / critic bodies are FCBody / DummyBody; the captured update implements DummyBody for both',
    'ppo_graph_unsupported/noisy_body': 'the network has NoisyLinear layers; the captured update implements nn.Linear',
    'ppo_graph_unsupported/noisy_config': 'the network has NoisyLinear layers; the captured update implements nn.Linear',
    'ppo_graph_unsupported/channels': 'the NatureConvBody takes 1 channels; the captured update reads stacks of 4 frames',
    'ppo_graph_unsupported/fp32':
        ("the compute dtype is torch.float32 with the 'tcgen05' dense backend; the captured update runs bf16 on the wgmma "
         'kernels (tcgen05)'),
    'ppo_graph_unsupported/library':
        ("the compute dtype is torch.bfloat16 with the 'library' dense backend; the captured update runs bf16 on the wgmma"
         ' kernels (tcgen05)'),
    'ppo_graph_unsupported/fused_bwd_off':
        'the fused backward epilogues are switched off; the captured update needs the fused update tail',
    'ppo_graph_unsupported/actions': '32 actions; the actor-critic head and loss kernels take fewer than 32',
    'ppo_graph_unsupported/normalizer':
        'the state normalizer is MeanStdNormalizer; the captured update folds a RescaleNormalizer into conv1',
    'ppo_graph_unsupported/float_frames': 'the envs do not return uint8 4 x 84 x 84 frame stacks',
    'ppo_graph_unsupported/sgd':
        ('the optimizer is SGD; the fused update tail implements RMSprop (centered or not) and Adam without momentum, '
         'weight decay or amsgrad'),
    'ppo_graph_unsupported/adam_weight_decay':
        ('the optimizer is Adam; the fused update tail implements RMSprop (centered or not) and Adam without momentum, '
         'weight decay or amsgrad'),
    'ppo_graph_unsupported/cpu': 'the network is not on a CUDA device (select_device(0))',
    'ppo_graph_unsupported/device_a2c+vanilla': 'config.device_a2c is set; it runs the agent on the device itself',
    'ppo_graph_unsupported/fc_phi_body+actor_body':
        'the phi_body is a FCBody; the captured update implements NatureConvBody',
    'ppo_graph_unsupported/actor_body+noisy_config':
        'the actor / critic bodies are FCBody / DummyBody; the captured update implements DummyBody for both',
    'ppo_graph_unsupported/actions+normalizer': '32 actions; the actor-critic head and loss kernels take fewer than 32',
    'ppo_graph_unsupported/adam_weight_decay+cpu':
        ('the optimizer is Adam; the fused update tail implements RMSprop (centered or not) and Adam without momentum, '
         'weight decay or amsgrad'),
    'ppo_graph_unsupported/not_shared':
        'config.shared_repr is not set; the captured update implements one optimizer over the shared network',
    'ppo_graph_unsupported/short_minibatch':
        ("the rollout's 1024 rows are not a multiple of mini_batch_size 300; random_sample would yield a short last "
         'minibatch'),
    'ppo_graph_unsupported/one_row':
        "the rollout's 1 rows are not a multiple of mini_batch_size 1; random_sample would yield a short last minibatch",
    'ppo_graph_unsupported/no_cuda_graph+not_shared': 'config.cuda_graph is not set',
    'ppo_graph_unsupported/not_shared+short_minibatch':
        'config.shared_repr is not set; the captured update implements one optimizer over the shared network',
    'ppo_graph_unsupported/short_minibatch+fp32':
        ("the rollout's 1024 rows are not a multiple of mini_batch_size 300; random_sample would yield a short last "
         'minibatch'),
    'dqn_graph_unsupported/accepted': None,
    'dqn_graph_unsupported/accepted_dueling': None,
    'dqn_graph_unsupported/accepted_prioritized': None,
    'dqn_graph_unsupported/accepted_c51': None,
    'dqn_graph_unsupported/accepted_qr': None,
    'dqn_graph_unsupported/no_cuda_graph': 'config.cuda_graph is not set',
    'dqn_graph_unsupported/device_dqn': 'config.device_dqn is set; it runs the agent on the device itself',
    'dqn_graph_unsupported/device_c51': 'config.device_c51 is set; it runs the agent on the device itself',
    'dqn_graph_unsupported/device_qr': 'config.device_qr is set; it runs the agent on the device itself',
    'dqn_graph_unsupported/device_rainbow': 'config.device_rainbow is set; it runs the agent on the device itself',
    'dqn_graph_unsupported/not_a_wrapper':
        ('the replay is not ReplayWrapper(..., async_=True); the captured update with async replay implements its double '
         'buffer'),
    'dqn_graph_unsupported/sync_wrapper':
        ('the replay is not ReplayWrapper(..., async_=True); the captured update with async replay implements its double '
         'buffer'),
    'dqn_graph_unsupported/replay_class':
        'the replay is a OtherReplay; the captured update implements UniformReplay and PrioritizedReplay',
    'dqn_graph_unsupported/qr_prioritized':
        'QR-DQN with prioritized replay is undefined in the reference (its loss is per target quantile)',
    'dqn_graph_unsupported/rainbow_net':
        'the network is a RainbowNet or has NoisyLinear layers; the captured update implements nn.Linear heads',
    'dqn_graph_unsupported/noisy_config':
        'the network is a RainbowNet or has NoisyLinear layers; the captured update implements nn.Linear heads',
    'dqn_graph_unsupported/dqn_categorical_net':
        'the network is a CategoricalNet; the captured update implements VanillaNet / DuelingNet for DQNAgent',
    'dqn_graph_unsupported/c51_vanilla_net':
        'the network is a VanillaNet; the captured update implements CategoricalNet for CategoricalDQNAgent',
    'dqn_graph_unsupported/fc_body': 'the body is a FCBody; the captured update implements NatureConvBody',
    'dqn_graph_unsupported/noisy_body': 'the network has NoisyLinear layers; the captured update implements nn.Linear',
    'dqn_graph_unsupported/fp32':
        ("the compute dtype is torch.float32 with the 'tcgen05' dense backend; the captured update runs bf16 on the wgmma "
         'kernels (tcgen05)'),
    'dqn_graph_unsupported/library':
        ("the compute dtype is torch.bfloat16 with the 'library' dense backend; the captured update runs bf16 on the wgmma"
         ' kernels (tcgen05)'),
    'dqn_graph_unsupported/fused_bwd_off':
        'the fused backward epilogues are switched off; the captured update needs the fused update tail',
    'dqn_graph_unsupported/normalizer':
        'the state normalizer is MeanStdNormalizer; the captured update folds a RescaleNormalizer into conv1',
    'dqn_graph_unsupported/channels':
        ('the frames are uint8 (4, 84, 84) with history_length 4 into 1 channels; the captured update reads 84 x 84 uint8 '
         'frames with a history of 4'),
    'dqn_graph_unsupported/history_length':
        ('the frames are uint8 (4, 84, 84) with history_length 1 into 4 channels; the captured update reads 84 x 84 uint8 '
         'frames with a history of 4'),
    'dqn_graph_unsupported/float_frames':
        ('the frames are float32 (4, 84, 84) with history_length 4 into 4 channels; the captured update reads 84 x 84 '
         'uint8 frames with a history of 4'),
    'dqn_graph_unsupported/frame_shape':
        ('the frames are uint8 (84, 84) with history_length 4 into 4 channels; the captured update reads 84 x 84 uint8 '
         'frames with a history of 4'),
    'dqn_graph_unsupported/no_eval_env':
        ('the frames are float64 unknown with history_length 4 into 4 channels; the captured update reads 84 x 84 uint8 '
         'frames with a history of 4'),
    'dqn_graph_unsupported/workers':
        "2 envs per actor step; the staged feeds follow the reference's one-transition feed() calls",
    'dqn_graph_unsupported/sgd':
        ('the optimizer is SGD; the fused update tail implements RMSprop (centered or not) and Adam without momentum, '
         'weight decay or amsgrad'),
    'dqn_graph_unsupported/hooks': 'Hooked overrides compute_loss / reduce_loss; the captured update runs the stock loss',
    'dqn_graph_unsupported/primed':
        'the replay wrapper has already handed out an eager batch; its pending batch is not handed to the learner',
    'dqn_graph_unsupported/cpu': 'the network is not on a CUDA device (select_device(0))',
    'dqn_graph_unsupported/device_dqn+sync_wrapper': 'config.device_dqn is set; it runs the agent on the device itself',
    'dqn_graph_unsupported/qr_prioritized+noisy_config':
        'QR-DQN with prioritized replay is undefined in the reference (its loss is per target quantile)',
    'dqn_graph_unsupported/normalizer+float_frames':
        'the state normalizer is MeanStdNormalizer; the captured update folds a RescaleNormalizer into conv1',
    'dqn_graph_unsupported/workers+sgd':
        "2 envs per actor step; the staged feeds follow the reference's one-transition feed() calls",
    'dqn_graph_unsupported/hooks+primed':
        'Hooked overrides compute_loss / reduce_loss; the captured update runs the stock loss',
    'dqn_graph_unsupported/primed+cpu':
        'the replay wrapper has already handed out an eager batch; its pending batch is not handed to the learner',
    'q_actor_unsupported/accepted': True,
    'q_actor_unsupported/accepted_async_ordered': True,
    'q_actor_unsupported/async_unordered': False,
    'q_actor_unsupported/no_cuda_graph': False,
    'q_actor_unsupported/noisy_config': False,
    'q_actor_unsupported/fc_body': False,
    'q_actor_unsupported/no_body': False,
    'q_actor_unsupported/noisy_body': False,
    'q_actor_unsupported/channels': False,
    'q_actor_unsupported/fp32': False,
    'q_actor_unsupported/library': False,
    'q_actor_unsupported/fused_bwd_off': True,
    'q_actor_unsupported/normalizer': False,
    'q_actor_unsupported/float_frames': False,
    'q_actor_unsupported/cpu': False,
    'a2c_unsupported/accepted_categorical': None,
    'a2c_unsupported/accepted_gaussian': None,
    'a2c_unsupported/accepted_relu': None,
    'a2c_unsupported/categorical_dummy_phi':
        ('a CategoricalActorCriticNet needs a two-layer FCBody phi_body and DummyBody actor / critic bodies (got DummyBody'
         ' / DummyBody / DummyBody)'),
    'a2c_unsupported/categorical_three_layers':
        ('a CategoricalActorCriticNet needs a two-layer FCBody phi_body and DummyBody actor / critic bodies (got FCBody / '
         'DummyBody / DummyBody)'),
    'a2c_unsupported/categorical_noisy':
        ('a CategoricalActorCriticNet needs a two-layer FCBody phi_body and DummyBody actor / critic bodies (got FCBody / '
         'DummyBody / DummyBody)'),
    'a2c_unsupported/categorical_actor_body':
        ('a CategoricalActorCriticNet needs a two-layer FCBody phi_body and DummyBody actor / critic bodies (got FCBody / '
         'FCBody / DummyBody)'),
    'a2c_unsupported/gaussian_fc_phi':
        ('a GaussianActorCriticNet needs a DummyBody phi_body and two-layer FCBody actor / critic bodies (got FCBody / '
         'FCBody / FCBody)'),
    'a2c_unsupported/gaussian_three_layers':
        ('a GaussianActorCriticNet needs a DummyBody phi_body and two-layer FCBody actor / critic bodies (got DummyBody / '
         'FCBody / FCBody)'),
    'a2c_unsupported/other_network':
        'the network is a VanillaNet, not a CategoricalActorCriticNet or GaussianActorCriticNet',
    'a2c_unsupported/widths': 'the actor and critic bodies must have the same widths and gate',
    'a2c_unsupported/gates': 'the actor and critic bodies must have the same widths and gate',
    'a2c_unsupported/gate': 'the FCBody gate must be torch.tanh or F.relu',
    'a2c_unsupported/cpu': 'the network is not on a CUDA device (select_device(0))',
    'a2c_unsupported/state_dim':
        "sizes beyond the kernels' limits: state_dim 300 <= 256, hidden 64 / 64 <= 128, actions 4 <= 32",
    'a2c_unsupported/hidden1':
        "sizes beyond the kernels' limits: state_dim 8 <= 256, hidden 129 / 64 <= 128, actions 4 <= 32",
    'a2c_unsupported/hidden2':
        "sizes beyond the kernels' limits: state_dim 8 <= 256, hidden 64 / 129 <= 128, actions 4 <= 32",
    'a2c_unsupported/actions':
        "sizes beyond the kernels' limits: state_dim 8 <= 256, hidden 64 / 64 <= 128, actions 33 <= 32",
    'a2c_unsupported/adam': 'the optimizer is Adam; the device update implements RMSprop',
    'a2c_unsupported/image_normalizer':
        'the state normalizer is ImageNormalizer; the device actor applies RescaleNormalizer',
    'a2c_unsupported/smem':
        'a rollout of 6 x 16 rows needs 307200 bytes of shared memory, more than one SM has (b2rl_a2c_smem_bytes)',
    'a2c_unsupported/smem_zero':
        'a rollout of 6 x 16 rows needs 0 bytes of shared memory, more than one SM has (b2rl_a2c_smem_bytes)',
    'a2c_unsupported/gate+cpu': 'the FCBody gate must be torch.tanh or F.relu',
    'a2c_unsupported/cpu+state_dim': 'the network is not on a CUDA device (select_device(0))',
    'a2c_unsupported/actions+adam':
        "sizes beyond the kernels' limits: state_dim 8 <= 256, hidden 64 / 64 <= 128, actions 33 <= 32",
    'a2c_unsupported/adam+normalizer': 'the optimizer is Adam; the device update implements RMSprop',
    'a2c_unsupported/normalizer+smem':
        'the state normalizer is MeanStdNormalizer; the device actor applies RescaleNormalizer',
    'nstep_dqn_unsupported/accepted': None,
    'nstep_dqn_unsupported/accepted_relu': None,
    'nstep_dqn_unsupported/dueling': 'the network is a DuelingNet, not a VanillaNet',
    'nstep_dqn_unsupported/dummy_body': 'a VanillaNet needs an FCBody body (got DummyBody)',
    'nstep_dqn_unsupported/noisy': 'the FCBody has NoisyLinear layers; the device kernels implement nn.Linear',
    'nstep_dqn_unsupported/three_layers': 'the device kernels implement a two-layer FCBody (got 3 layers)',
    'nstep_dqn_unsupported/gate': 'the FCBody gate must be torch.tanh or F.relu',
    'nstep_dqn_unsupported/cpu': 'the network is not on a CUDA device (select_device(0))',
    'nstep_dqn_unsupported/state_dim':
        "sizes beyond the kernels' limits: state_dim 300 <= 256, hidden 64 / 64 <= 128, 2 <= actions 4 <= 32",
    'nstep_dqn_unsupported/one_action':
        "sizes beyond the kernels' limits: state_dim 8 <= 256, hidden 64 / 64 <= 128, 2 <= actions 1 <= 32",
    'nstep_dqn_unsupported/actions':
        "sizes beyond the kernels' limits: state_dim 8 <= 256, hidden 64 / 64 <= 128, 2 <= actions 33 <= 32",
    'nstep_dqn_unsupported/adam': 'the optimizer is Adam; the device update implements RMSprop',
    'nstep_dqn_unsupported/image_normalizer':
        'the state normalizer is ImageNormalizer; the device actor applies RescaleNormalizer',
    'nstep_dqn_unsupported/smem':
        'a rollout of 6 x 16 rows needs 307200 bytes of shared memory, more than one SM has (b2rl_nstep_dqn_smem_bytes)',
    'nstep_dqn_unsupported/noisy+three_layers': 'the FCBody has NoisyLinear layers; the device kernels implement nn.Linear',
    'nstep_dqn_unsupported/three_layers+gate': 'the device kernels implement a two-layer FCBody (got 3 layers)',
    'nstep_dqn_unsupported/gate+cpu': 'the FCBody gate must be torch.tanh or F.relu',
    'nstep_dqn_unsupported/actions+adam':
        "sizes beyond the kernels' limits: state_dim 8 <= 256, hidden 64 / 64 <= 128, 2 <= actions 33 <= 32",
    'nstep_dqn_unsupported/normalizer+smem':
        'the state normalizer is MeanStdNormalizer; the device actor applies RescaleNormalizer',
    'dqn_unsupported/accepted': None,
    'dqn_unsupported/accepted_dueling': None,
    'dqn_unsupported/accepted_double_q': None,
    'dqn_unsupported/categorical_net':
        ('the network is a CategoricalNet; the device kernels implement VanillaNet and DuelingNet (C51, QR and Rainbow '
         'heads are not covered)'),
    'dqn_unsupported/hooks': "OwnLoss overrides compute_loss / reduce_loss; the device update implements DQNAgent's",
    'dqn_unsupported/nature_body': 'the body is a NatureConvBody; the device kernels implement a two-layer FCBody',
    'dqn_unsupported/dummy_body': 'the network needs an FCBody body (got DummyBody)',
    'dqn_unsupported/noisy_body': 'the network has NoisyLinear layers; the device kernels implement nn.Linear',
    'dqn_unsupported/noisy_config': 'the network has NoisyLinear layers; the device kernels implement nn.Linear',
    'dqn_unsupported/three_layers': 'the device kernels implement a two-layer FCBody (got 3 layers)',
    'dqn_unsupported/gate': 'the FCBody gate must be torch.tanh or F.relu',
    'dqn_unsupported/cpu': 'the network is not on a CUDA device (select_device(0))',
    'dqn_unsupported/state_dim':
        "sizes beyond the kernels' limits: state_dim 300 <= 256, hidden 64 / 64 <= 128, 2 <= actions 4 <= 32",
    'dqn_unsupported/one_action':
        "sizes beyond the kernels' limits: state_dim 8 <= 256, hidden 64 / 64 <= 128, 2 <= actions 1 <= 32",
    'dqn_unsupported/adam': 'the optimizer is Adam; the device update implements RMSprop',
    'dqn_unsupported/no_flat': 'the optimizer is RMSprop; the device update implements RMSprop',
    'dqn_unsupported/image_normalizer':
        'the state normalizer is ImageNormalizer; the device actor applies RescaleNormalizer',
    'dqn_unsupported/async_actor': "async_actor is set; the device actor runs in the agent's thread (async_actor=False)",
    'dqn_unsupported/history_length': 'history_length is 4; the device kernels read single 1-D states, not frame stacks',
    'dqn_unsupported/smem':
        'a batch of 32 needs 307200 bytes of shared memory, more than one SM has (b2rl_dqn_replay_smem_bytes)',
    'dqn_unsupported/categorical_net+hooks':
        ('the network is a CategoricalNet; the device kernels implement VanillaNet and DuelingNet (C51, QR and Rainbow '
         'heads are not covered)'),
    'dqn_unsupported/hooks+nature_body':
        "OwnLoss overrides compute_loss / reduce_loss; the device update implements DQNAgent's",
    'dqn_unsupported/nature_body+noisy_config':
        'the body is a NatureConvBody; the device kernels implement a two-layer FCBody',
    'dqn_unsupported/gate+cpu': 'the FCBody gate must be torch.tanh or F.relu',
    'dqn_unsupported/cpu+state_dim': 'the network is not on a CUDA device (select_device(0))',
    'dqn_unsupported/normalizer+async_actor':
        'the state normalizer is MeanStdNormalizer; the device actor applies RescaleNormalizer',
    'dqn_unsupported/async_actor+history_length':
        "async_actor is set; the device actor runs in the agent's thread (async_actor=False)",
    'dqn_unsupported/history_length+smem':
        'history_length is 4; the device kernels read single 1-D states, not frame stacks',
    'dist_dqn_unsupported/accepted_c51': None,
    'dist_dqn_unsupported/accepted_qr': None,
    'dist_dqn_unsupported/accepted_c51_prioritized': None,
    'dist_dqn_unsupported/accepted_history_length_1': None,
    'dist_dqn_unsupported/accepted_plain_replay': None,
    'dist_dqn_unsupported/rainbow_net':
        'the network is a RainbowNet; the device kernels implement CategoricalNet (RainbowNet / NoisyLinear is not covered)',
    'dist_dqn_unsupported/c51_quantile_net': 'the network is a QuantileNet; the device kernels implement CategoricalNet',
    'dist_dqn_unsupported/qr_categorical_net': 'the network is a CategoricalNet; the device kernels implement QuantileNet',
    'dist_dqn_unsupported/hooks_c51':
        "OwnKL overrides compute_loss / reduce_loss; the device update implements CategoricalDQNAgent's",
    'dist_dqn_unsupported/hooks_qr':
        "OwnQuantile overrides compute_loss / reduce_loss; the device update implements QuantileRegressionDQNAgent's",
    'dist_dqn_unsupported/nature_body': 'the body is a NatureConvBody; the device kernels implement a two-layer FCBody',
    'dist_dqn_unsupported/noisy_body': 'the network has NoisyLinear layers; the device kernels implement nn.Linear',
    'dist_dqn_unsupported/three_layers': 'the device kernels implement a two-layer FCBody (got 3 layers)',
    'dist_dqn_unsupported/gate': 'the FCBody gate must be torch.tanh or F.relu',
    'dist_dqn_unsupported/cpu': 'the network is not on a CUDA device (select_device(0))',
    'dist_dqn_unsupported/atoms':
        ("sizes beyond the kernels' limits: state_dim 8 <= 256, hidden 64 / 64 <= 128, 2 <= actions 4 <= 32, 2 <= atoms "
         '300 <= 256'),
    'dist_dqn_unsupported/quantiles':
        ("sizes beyond the kernels' limits: state_dim 8 <= 256, hidden 64 / 64 <= 128, 2 <= actions 4 <= 32, 2 <= "
         'quantiles 1 <= 256'),
    'dist_dqn_unsupported/state_dim':
        ("sizes beyond the kernels' limits: state_dim 300 <= 256, hidden 64 / 64 <= 128, 2 <= actions 4 <= 32, 2 <= atoms "
         '51 <= 256'),
    'dist_dqn_unsupported/adam': 'the optimizer is Adam; the device update implements RMSprop',
    'dist_dqn_unsupported/no_flat': 'the optimizer is RMSprop; the device update implements RMSprop',
    'dist_dqn_unsupported/image_normalizer':
        'the state normalizer is ImageNormalizer; the device actor applies RescaleNormalizer',
    'dist_dqn_unsupported/history_length':
        'history_length is 4; the device kernels read single 1-D states, not frame stacks',
    'dist_dqn_unsupported/qr_prioritized':
        ('QR-DQN with prioritized replay is undefined in the reference: its loss is per target quantile, not per sample '
         '(QuantileRegressionDQN_agent.py:74)'),
    'dist_dqn_unsupported/smem':
        'a batch of 32 needs 307200 bytes of shared memory, more than one SM has (b2rl_dist_dqn_smem_bytes)',
    'dist_dqn_unsupported/rainbow_net+hooks':
        'the network is a RainbowNet; the device kernels implement CategoricalNet (RainbowNet / NoisyLinear is not covered)',
    'dist_dqn_unsupported/hooks+noisy_body':
        "OwnKL overrides compute_loss / reduce_loss; the device update implements CategoricalDQNAgent's",
    'dist_dqn_unsupported/cpu+atoms': 'the network is not on a CUDA device (select_device(0))',
    'dist_dqn_unsupported/history_length+qr_prioritized':
        'history_length is 4; the device kernels read single 1-D states, not frame stacks',
    'dist_dqn_unsupported/qr_prioritized+smem':
        ('QR-DQN with prioritized replay is undefined in the reference: its loss is per target quantile, not per sample '
         '(QuantileRegressionDQN_agent.py:74)'),
    'rainbow_unsupported/accepted_noisy': None,
    'rainbow_unsupported/accepted_linear': None,
    'rainbow_unsupported/dqn_agent': 'the agent is a DQNAgent; Rainbow is a CategoricalDQNAgent on a RainbowNet',
    'rainbow_unsupported/categorical_net': 'the network is a CategoricalNet; the device kernels implement RainbowNet',
    'rainbow_unsupported/hooks':
        "OwnKL overrides compute_loss / reduce_loss; the device update implements CategoricalDQNAgent's",
    'rainbow_unsupported/nature_body': 'the body is a NatureConvBody; the device kernels implement a two-layer FCBody',
    'rainbow_unsupported/dummy_body': 'the network needs an FCBody body (got DummyBody)',
    'rainbow_unsupported/three_layers': 'the device kernels implement a two-layer FCBody (got 3 layers)',
    'rainbow_unsupported/mixed_noise':
        ('the body, the head and config.noisy_linear disagree: the device kernels implement all four layers NoisyLinear or'
         ' all four nn.Linear, not a mix'),
    'rainbow_unsupported/gate': 'the FCBody gate must be torch.tanh or F.relu',
    'rainbow_unsupported/cpu': 'the network is not on a CUDA device (select_device(0))',
    'rainbow_unsupported/atoms':
        ("sizes beyond the kernels' limits: state_dim 8 <= 256, hidden 64 / 64 <= 128, 2 <= actions 4 <= 32, 2 <= atoms "
         '300 <= 256'),
    'rainbow_unsupported/one_action':
        ("sizes beyond the kernels' limits: state_dim 8 <= 256, hidden 64 / 64 <= 128, 2 <= actions 1 <= 32, 2 <= atoms 51"
         ' <= 256'),
    'rainbow_unsupported/adam': 'the optimizer is Adam; the device update implements RMSprop',
    'rainbow_unsupported/no_flat': 'the optimizer is RMSprop; the device update implements RMSprop',
    'rainbow_unsupported/image_normalizer':
        'the state normalizer is ImageNormalizer; the device actor applies RescaleNormalizer',
    'rainbow_unsupported/history_length': 'history_length is 4; the device kernels read single 1-D states, not frame stacks',
    'rainbow_unsupported/smem':
        'a batch of 32 needs 307200 bytes of shared memory, more than one SM has (b2rl_rainbow_smem_bytes)',
    'rainbow_unsupported/dqn_agent+categorical_net':
        'the agent is a DQNAgent; Rainbow is a CategoricalDQNAgent on a RainbowNet',
    'rainbow_unsupported/three_layers+mixed_noise': 'the device kernels implement a two-layer FCBody (got 3 layers)',
    'rainbow_unsupported/mixed_noise+gate':
        ('the body, the head and config.noisy_linear disagree: the device kernels implement all four layers NoisyLinear or'
         ' all four nn.Linear, not a mix'),
    'rainbow_unsupported/gate+cpu': 'the FCBody gate must be torch.tanh or F.relu',
    'rainbow_unsupported/history_length+smem':
        'history_length is 4; the device kernels read single 1-D states, not frame stacks',
}
