"""[SB2] common/evaluation.py ``evaluate_policy`` as called from base_callbacks.py:83-87: run ``n_eval_episodes`` episodes
of ``model.predict`` on a single (vectorised) environment and return the mean/std reward or the per-episode lists."""
from __future__ import annotations

import numpy as np


def evaluate_policy(model, env, n_eval_episodes=10, deterministic=True, render=False, callback=None, reward_threshold=None,
                    return_episode_rewards=False):
    vec = hasattr(env, "num_envs")
    if vec:
        assert env.num_envs == 1, "You must pass only one environment when using this function"
    episode_rewards, episode_lengths = [], []
    obs = None
    # A model whose own VecNormalize statistics live on its learner (SAC(device_obs_norm=True)) takes RAW observations in
    # predict and normalises them on the device; an evaluation wrapper that normalises on the host hands over its raw copy.
    host_vn = None
    if getattr(model, "predict_takes_raw_obs", False):
        from .base_model import unwrap_vec_normalize
        host_vn = unwrap_vec_normalize(env)
        if host_vn is not None and (not host_vn.norm_obs or getattr(host_vn, "learner_owns_obs_rms", False)):
            host_vn = None
    for i in range(n_eval_episodes):
        if not vec or i == 0:            # a VecEnv resets itself at the end of an episode
            obs = env.reset()
        done, state = False, None
        ep_rew, ep_len = 0.0, 0
        while not done:
            action, state = model.predict(obs if host_vn is None else host_vn.get_original_obs(), state=state,
                                          deterministic=deterministic)
            obs, reward, done, _info = env.step(action)
            if vec:
                reward, done = float(np.asarray(reward).reshape(-1)[0]), bool(np.asarray(done).reshape(-1)[0])
            ep_rew += reward
            if callback is not None:
                callback(locals(), globals())
            ep_len += 1
            if render:
                env.render()
        episode_rewards.append(ep_rew)
        episode_lengths.append(ep_len)
    mean_reward, std_reward = float(np.mean(episode_rewards)), float(np.std(episode_rewards))
    if reward_threshold is not None:
        assert mean_reward > reward_threshold, "Mean reward below threshold: {:.2f} < {:.2f}".format(mean_reward, reward_threshold)
    if return_episode_rewards:
        return episode_rewards, episode_lengths
    return mean_reward, std_reward
