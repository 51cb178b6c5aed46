"""b200rl — H100-native (sm_90a) vectorised RL inner loop behind ReinforcementLearning.jl's
run(policy, env, stop, hook) surface.  Python host mirror of the Julia glue
(julia/B200RL.jl): thin ctypes calls into libb200rl.so; no compute happens in Python and
there is no CPU fallback."""
from . import _lib
from ._lib import B200RLError, Context, load
from .core import (AbstractHook, AbstractPolicy, BatchStepsPerEpisode, ComposedHook, DeviceEpisodeLog, DeviceEpisodeStats, DoEveryNSteps, DoOnExit, EmptyHook, Experiment, ResetAfterNSteps, ResetIfEnvTerminated,
                   RandomPolicy, StopAfterNEpisodes, StopAfterNoImprovement, StopAfterNSeconds, StopAfterNSteps, StopIfAll, StopIfAny,
                   StopSignal, TimePerStep, TotalBatchRewardPerEpisode, run)
from .envs import B200VecEnv, cartpole_params, mountaincar_params, pendulum_params
from .explorers import EpsilonGreedyExplorer, EpsilonSpeedyExplorer, GreedyExplorer, GumbelSoftmaxExplorer, WeightedSoftmaxExplorer
from .learners import (ACT_RELU, ACT_TANH, KIND_CATEGORICAL, KIND_DUELING, KIND_GAUSSIAN, KIND_Q, Agent, DQNLearner, EvaluationPolicy, InsertSampleRatioController,
                       Network, OnPolicyAgent, QBasedPolicy, Trajectory, dqn_config, evaluate, onpolicy_config)
from . import checkpoint, core, explorers, learners, sharding
from .returns import discount_rewards, discount_rewards_reduced, generalized_advantage_estimation

__all__ = [n for n in dir() if not n.startswith("_")]
