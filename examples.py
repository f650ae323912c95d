"""Launchers with the reference's names, hyper-parameters and wiring (reference ``examples.py:11-617``), re-issued
for this package: ``from deeprl_b200 import *`` instead of ``from deep_rl import *`` and ``ReplayWrapper(..., async_)``
(the reference spells the argument ``async``, a reserved word since Python 3.7 -- examples.py:116,149,180,214 there
do not parse on Python 3.12).  In scope: DQN, QR-DQN, C51, Rainbow, A2C, PPO (SURVEY.md section 2.1 #24).

Every launcher is ``name(**kwargs)`` with ``game=...`` like the reference's; hyper-parameters live in one table per
launcher so they can be diffed against the reference line by line.  Games available offline: ``CartPole-v0``,
``SyntheticAtari-v0`` (84x84x4 uint8 frames), ``SyntheticCheetah-v0`` (17-dim observations); anything else is handed
to gym if it is installed.
"""
from deeprl_b200 import *  # noqa: F401,F403


def _config(kwargs, **defaults):
    generate_tag(kwargs)
    kwargs.setdefault("log_level", 0)
    for k, v in defaults.items():
        kwargs.setdefault(k, v)
    config = Config()
    config.merge(kwargs)
    config.task_fn = lambda: Task(config.game)
    config.eval_env = config.task_fn()
    return config


def _replay(config, cls, async_, **kw):
    kw.setdefault("batch_size", config.batch_size)
    config.replay_fn = lambda: ReplayWrapper(cls, kw, async_)


def _per_schedule(config):
    config.replay_eps, config.replay_alpha = 0.01, 0.5
    config.replay_beta = LinearSchedule(0.4, 1.0, config.max_steps)


_ATARI = dict(state_normalizer=ImageNormalizer, reward_normalizer=SignNormalizer, discount=0.99, sgd_update_frequency=4,
              batch_size=32)


def _apply(config, table):
    for k, v in table.items():
        setattr(config, k, v() if k.endswith("_normalizer") else v)


# ------------------------------------------------------------------------------------------------ DQN (examples.py:11-97)
def dqn_feature(**kwargs):
    config = _config(kwargs, n_step=1, replay_cls=UniformReplay, async_replay=True)
    config.optimizer_fn = lambda params: torch.optim.RMSprop(params, 0.001)
    config.network_fn = lambda: VanillaNet(config.action_dim, FCBody(config.state_dim))
    _apply(config, dict(history_length=1, batch_size=10, discount=0.99, max_steps=1e5, target_network_update_freq=200,
                        exploration_steps=1000, double_q=False, sgd_update_frequency=4, gradient_clip=5,
                        eval_interval=int(5e3), async_actor=False))
    _replay(config, config.replay_cls, config.async_replay, memory_size=int(1e4), n_step=config.n_step,
            discount=config.discount, history_length=config.history_length)
    _per_schedule(config)
    config.random_action_prob = LinearSchedule(1.0, 0.1, 1e4)
    run_steps(DQNAgent(config))


def dqn_pixel(**kwargs):
    config = _config(kwargs, n_step=1, replay_cls=UniformReplay, async_replay=True)
    config.optimizer_fn = lambda params: torch.optim.RMSprop(params, lr=0.00025, alpha=0.95, eps=0.01, centered=True)
    config.network_fn = lambda: VanillaNet(config.action_dim, NatureConvBody(in_channels=config.history_length))
    _apply(config, dict(_ATARI, history_length=4, max_steps=int(2e7), target_network_update_freq=10000,
                        exploration_steps=50000, gradient_clip=5, double_q=False, async_actor=True))
    _replay(config, config.replay_cls, config.async_replay, memory_size=int(1e6), n_step=config.n_step,
            discount=config.discount, history_length=config.history_length)
    _per_schedule(config)
    config.random_action_prob = LinearSchedule(1.0, 0.01, 1e6)
    run_steps(DQNAgent(config))


# ------------------------------------------------------------------------------------------------ QR-DQN (examples.py:101-160)
def quantile_regression_dqn_feature(**kwargs):
    config = _config(kwargs)
    config.optimizer_fn = lambda params: torch.optim.RMSprop(params, 0.001)
    config.network_fn = lambda: QuantileNet(config.action_dim, config.num_quantiles, FCBody(config.state_dim))
    _apply(config, dict(batch_size=10, discount=0.99, target_network_update_freq=200, exploration_steps=100,
                        num_quantiles=20, gradient_clip=5, sgd_update_frequency=4, eval_interval=int(5e3), max_steps=1e5))
    _replay(config, UniformReplay, True, memory_size=int(1e4))
    config.random_action_prob = LinearSchedule(1.0, 0.1, 1e4)
    run_steps(QuantileRegressionDQNAgent(config))


def quantile_regression_dqn_pixel(**kwargs):
    config = _config(kwargs)
    config.optimizer_fn = lambda params: torch.optim.Adam(params, lr=0.00005, eps=0.01 / 32)
    config.network_fn = lambda: QuantileNet(config.action_dim, config.num_quantiles, NatureConvBody())
    _apply(config, dict(_ATARI, target_network_update_freq=10000, exploration_steps=50000, gradient_clip=5,
                        num_quantiles=200, max_steps=int(2e7)))
    _replay(config, UniformReplay, True, memory_size=int(1e6), history_length=4)
    config.random_action_prob = LinearSchedule(1.0, 0.01, 1e6)
    run_steps(QuantileRegressionDQNAgent(config))


# ------------------------------------------------------------------------------------------------ C51 (examples.py:164-227)
def categorical_dqn_feature(**kwargs):
    config = _config(kwargs)
    config.optimizer_fn = lambda params: torch.optim.RMSprop(params, 0.001)
    config.network_fn = lambda: CategoricalNet(config.action_dim, config.categorical_n_atoms, FCBody(config.state_dim))
    _apply(config, dict(batch_size=10, discount=0.99, target_network_update_freq=200, exploration_steps=100,
                        categorical_v_max=100, categorical_v_min=-100, categorical_n_atoms=50, gradient_clip=5,
                        sgd_update_frequency=4, eval_interval=int(5e3), max_steps=1e5))
    _replay(config, UniformReplay, True, memory_size=int(1e4))
    config.random_action_prob = LinearSchedule(1.0, 0.1, 1e4)
    run_steps(CategoricalDQNAgent(config))


def categorical_dqn_pixel(**kwargs):
    config = _config(kwargs)
    config.optimizer_fn = lambda params: torch.optim.Adam(params, lr=0.00025, eps=0.01 / 32)
    config.network_fn = lambda: CategoricalNet(config.action_dim, config.categorical_n_atoms, NatureConvBody())
    _apply(config, dict(_ATARI, target_network_update_freq=10000, exploration_steps=50000, categorical_v_max=10,
                        categorical_v_min=-10, categorical_n_atoms=51, gradient_clip=0.5, max_steps=int(2e7)))
    _replay(config, UniformReplay, True, memory_size=int(1e6), history_length=4)
    config.random_action_prob = LinearSchedule(1.0, 0.01, 1e6)
    run_steps(CategoricalDQNAgent(config))


# ------------------------------------------------------------------------------------------------ Rainbow (examples.py:231-336)
def rainbow_feature(**kwargs):
    config = _config(kwargs, n_step=3, replay_cls=PrioritizedReplay, async_replay=True)
    config.max_steps = 1e5
    config.optimizer_fn = lambda params: torch.optim.RMSprop(params, 0.001)
    config.noisy_linear = True
    config.network_fn = lambda: RainbowNet(config.action_dim, config.categorical_n_atoms,
                                           FCBody(config.state_dim, noisy_linear=config.noisy_linear),
                                           noisy_linear=config.noisy_linear)
    _apply(config, dict(categorical_v_max=100, categorical_v_min=-100, categorical_n_atoms=50, discount=0.99, batch_size=32,
                        target_network_update_freq=200, exploration_steps=1000, double_q=True, sgd_update_frequency=4,
                        eval_interval=int(5e3), async_actor=True, gradient_clip=10))
    _replay(config, config.replay_cls, config.async_replay, memory_size=int(1e4), n_step=config.n_step,
            discount=config.discount, history_length=1)
    _per_schedule(config)
    config.random_action_prob = LinearSchedule(1.0, 0.1, 1e4)
    run_steps(CategoricalDQNAgent(config))


def rainbow_pixel(**kwargs):
    config = _config(kwargs, n_step=1, replay_cls=PrioritizedReplay, async_replay=True, noisy_linear=True)
    config.max_steps = int(2e7)
    Config.NOISY_LAYER_STD = 0.5
    config.optimizer_fn = lambda params: torch.optim.Adam(params, lr=0.000625, eps=1.5e-4)
    config.network_fn = lambda: RainbowNet(config.action_dim, config.categorical_n_atoms,
                                           NatureConvBody(noisy_linear=config.noisy_linear), noisy_linear=config.noisy_linear)
    _apply(config, dict(_ATARI, categorical_v_max=10, categorical_v_min=-10, categorical_n_atoms=51, history_length=4,
                        target_network_update_freq=2000, exploration_steps=20000, double_q=True, async_actor=True,
                        gradient_clip=10))
    _replay(config, config.replay_cls, config.async_replay, memory_size=int(1e6), n_step=config.n_step,
            discount=config.discount, history_length=config.history_length)
    _per_schedule(config)
    config.random_action_prob = LinearSchedule(1, 0.01, 25e4)
    run_steps(CategoricalDQNAgent(config))


# ------------------------------------------------------------------------------------------------ A2C (examples.py:340-404)
def a2c_feature(**kwargs):
    config = _config(kwargs)
    config.num_workers = kwargs.get("num_workers", 5)
    config.task_fn = lambda: Task(config.game, num_envs=config.num_workers)
    config.eval_env = Task(config.game)
    config.optimizer_fn = lambda params: torch.optim.RMSprop(params, 0.001)
    config.network_fn = lambda: CategoricalActorCriticNet(config.state_dim, config.action_dim,
                                                          FCBody(config.state_dim, gate=torch.tanh))
    _apply(config, dict(discount=0.99, use_gae=True, gae_tau=0.95, entropy_weight=0.01, rollout_length=5, gradient_clip=0.5))
    run_steps(A2CAgent(config))


def a2c_pixel(**kwargs):
    config = _config(kwargs)
    config.num_workers = kwargs.get("num_workers", 16)
    config.task_fn = lambda: Task(config.game, num_envs=config.num_workers)
    config.eval_env = Task(config.game)
    config.optimizer_fn = lambda params: torch.optim.RMSprop(params, lr=1e-4, alpha=0.99, eps=1e-5)
    config.network_fn = lambda: CategoricalActorCriticNet(config.state_dim, config.action_dim, NatureConvBody())
    _apply(config, dict(state_normalizer=ImageNormalizer, reward_normalizer=SignNormalizer, discount=0.99, use_gae=True,
                        gae_tau=1.0, entropy_weight=0.01, rollout_length=5, gradient_clip=5, max_steps=int(2e7)))
    run_steps(A2CAgent(config))


def a2c_continuous(**kwargs):
    """examples.py:384-404: A2C with a Gaussian policy over FC bodies (16 workers, rollout 5, RMSprop 7e-4)."""
    config = _config(kwargs)
    config.num_workers = kwargs.get("num_workers", 16)
    config.task_fn = lambda: Task(config.game, num_envs=config.num_workers)
    config.eval_env = Task(config.game)
    config.optimizer_fn = lambda params: torch.optim.RMSprop(params, lr=0.0007)
    config.network_fn = lambda: GaussianActorCriticNet(config.state_dim, config.action_dim, actor_body=FCBody(config.state_dim),
                                                       critic_body=FCBody(config.state_dim))
    _apply(config, dict(discount=0.99, use_gae=True, gae_tau=1.0, entropy_weight=0.01, rollout_length=5, gradient_clip=5,
                        max_steps=int(2e7)))
    run_steps(A2CAgent(config))


# ------------------------------------------------------------------------------------------------ n-step DQN (examples.py:408-446)
def n_step_dqn_feature(**kwargs):
    config = _config(kwargs)
    config.num_workers = kwargs.get("num_workers", 5)
    config.task_fn = lambda: Task(config.game, num_envs=config.num_workers)
    config.eval_env = Task(config.game)
    config.optimizer_fn = lambda params: torch.optim.RMSprop(params, 0.001)
    config.network_fn = lambda: VanillaNet(config.action_dim, FCBody(config.state_dim))
    config.random_action_prob = LinearSchedule(1.0, 0.1, 1e4)
    _apply(config, dict(discount=0.99, target_network_update_freq=200, rollout_length=5, gradient_clip=5))
    run_steps(NStepDQNAgent(config))


def n_step_dqn_pixel(**kwargs):
    config = _config(kwargs)
    config.num_workers = kwargs.get("num_workers", 16)
    config.task_fn = lambda: Task(config.game, num_envs=config.num_workers)
    config.eval_env = Task(config.game)
    config.optimizer_fn = lambda params: torch.optim.RMSprop(params, lr=1e-4, alpha=0.99, eps=1e-5)
    config.network_fn = lambda: VanillaNet(config.action_dim, NatureConvBody())
    config.random_action_prob = LinearSchedule(1.0, 0.05, 1e6)
    _apply(config, dict(state_normalizer=ImageNormalizer, reward_normalizer=SignNormalizer, discount=0.99,
                        target_network_update_freq=10000, rollout_length=5, gradient_clip=5, max_steps=int(2e7)))
    run_steps(NStepDQNAgent(config))


# ------------------------------------------------------------------------------------------------ PPO (examples.py:496-550)
def ppo_continuous(**kwargs):
    config = _config(kwargs)
    config.num_workers = kwargs.get("num_workers", 1)
    config.task_fn = lambda: Task(config.game, num_envs=config.num_workers)
    config.eval_env = Task(config.game)
    config.network_fn = lambda: GaussianActorCriticNet(
        config.state_dim, config.action_dim, actor_body=FCBody(config.state_dim, gate=torch.tanh),
        critic_body=FCBody(config.state_dim, gate=torch.tanh))
    config.actor_opt_fn = lambda params: torch.optim.Adam(params, 3e-4)
    config.critic_opt_fn = lambda params: torch.optim.Adam(params, 1e-3)
    _apply(config, dict(discount=0.99, use_gae=True, gae_tau=0.95, gradient_clip=0.5, rollout_length=2048,
                        optimization_epochs=10, mini_batch_size=64, ppo_ratio_clip=0.2, log_interval=2048, max_steps=3e6,
                        target_kl=0.01, state_normalizer=MeanStdNormalizer))
    run_steps(PPOAgent(config))


def ppo_pixel(**kwargs):
    config = _config(kwargs)
    config.num_workers = kwargs.get("num_workers", 8)
    config.task_fn = lambda: Task(config.game, num_envs=config.num_workers)
    config.eval_env = Task(config.game)
    config.optimizer_fn = lambda params: torch.optim.Adam(params, lr=2.5e-4)
    config.network_fn = lambda: CategoricalActorCriticNet(config.state_dim, config.action_dim, NatureConvBody())
    _apply(config, dict(state_normalizer=ImageNormalizer, reward_normalizer=SignNormalizer, discount=0.99, use_gae=True,
                        gae_tau=0.95, entropy_weight=0.01, gradient_clip=0.5, rollout_length=128, optimization_epochs=4,
                        mini_batch_size=128 * config.num_workers // 4, ppo_ratio_clip=0.1,
                        log_interval=128 * config.num_workers, max_steps=int(2e7), shared_repr=True))
    run_steps(PPOAgent(config))


if __name__ == "__main__":
    mkdir("log")
    mkdir("tf_log")
    set_one_thread()
    random_seed()
    select_device(-1)                      # select_device(0) for the H100 path (required by the DQN family: HBM replay)
    a2c_feature(game="CartPole-v0", max_steps=int(2e4))
