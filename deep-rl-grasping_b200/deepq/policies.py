class MlpPolicy:
    """stable-baselines' deepq MlpPolicy: the dueling MLP (layers [64, 64], ReLU) that ``deepq.DQN`` builds.  A marker: the
    network itself lives in csrc/dqn.cu."""
    # deepq.DQN accepts this class by identity; every other learner that reads ``unsupported`` (SAC) refuses it
    unsupported = "deepq.policies.MlpPolicy is the DQN policy: use it with b200grasp.deepq.DQN"
