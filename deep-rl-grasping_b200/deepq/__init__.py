"""Import-compatibility namespace for ``stable_baselines.deepq`` (sb_helper.py:12): ``deepq.DQN`` is the dueling double DQN
learner of the DQN branch of ``SBPolicy.learn`` (sb_helper.py:155-165), ``deepq.policies.MlpPolicy`` its policy."""
from . import policies  # noqa: F401
from ..dqn import DQN, DQNLearner  # noqa: F401
from .policies import MlpPolicy  # noqa: F401
