"""Callback protocol the learner drives ([SB2] common/callbacks.py as used by
/root/reference/manipulation_main/training/base_callbacks.py:16-245 and sb_helper.py:25-54):
init_callback(model) -> on_training_start(locals, globals) -> {on_rollout_start, on_step -> bool,
on_rollout_end}* -> on_training_end; attributes n_calls, num_timesteps, model, training_env,
locals, globals, parent."""
from __future__ import annotations

import os
import warnings
from typing import List, Optional

import numpy as np


class BaseCallback:
    def __init__(self, verbose: int = 0):
        self.model = None
        self.training_env = None
        self.n_calls = 0
        self.num_timesteps = 0
        self.verbose = verbose
        self.locals = None
        self.globals = None
        self.logger = None
        self.parent = None

    def init_callback(self, model) -> None:
        self.model = model
        self.training_env = model.get_env()
        self._init_callback()

    def _init_callback(self) -> None:
        pass

    def on_training_start(self, locals_, globals_) -> None:
        self.locals, self.globals = locals_, globals_
        self._on_training_start()

    def _on_training_start(self) -> None:
        pass

    def on_rollout_start(self) -> None:
        self._on_rollout_start()

    def _on_rollout_start(self) -> None:
        pass

    def _on_step(self) -> bool:
        return True

    def on_step(self) -> bool:
        self.n_calls += 1
        self.num_timesteps = self.model.num_timesteps
        return self._on_step()

    def on_rollout_end(self) -> None:
        self._on_rollout_end()

    def _on_rollout_end(self) -> None:
        pass

    def on_training_end(self) -> None:
        self._on_training_end()

    def _on_training_end(self) -> None:
        pass


class EventCallback(BaseCallback):
    def __init__(self, callback: Optional[BaseCallback] = None, verbose: int = 0):
        super().__init__(verbose)
        self.callback = callback
        if callback is not None:
            callback.parent = self

    def init_callback(self, model) -> None:
        super().init_callback(model)
        if self.callback is not None:
            self.callback.init_callback(model)

    def _on_training_start(self) -> None:
        if self.callback is not None:
            self.callback.on_training_start(self.locals, self.globals)

    def _on_event(self) -> bool:
        return self.callback.on_step() if self.callback is not None else True


class CallbackList(BaseCallback):
    def __init__(self, callbacks: List[BaseCallback]):
        super().__init__()
        self.callbacks = callbacks

    def _init_callback(self) -> None:
        for c in self.callbacks:
            c.init_callback(self.model)

    def _on_training_start(self) -> None:
        for c in self.callbacks:
            c.on_training_start(self.locals, self.globals)

    def _on_rollout_start(self) -> None:
        for c in self.callbacks:
            c.on_rollout_start()

    def _on_step(self) -> bool:
        ok = True
        for c in self.callbacks:
            ok = c.on_step() and ok
        return ok

    def _on_rollout_end(self) -> None:
        for c in self.callbacks:
            c.on_rollout_end()

    def _on_training_end(self) -> None:
        for c in self.callbacks:
            c.on_training_end()


class _FnCallback(BaseCallback):
    """Legacy ``callback(locals, globals) -> bool`` functions."""

    def __init__(self, fn):
        super().__init__()
        self.fn = fn

    def _on_step(self) -> bool:
        r = self.fn(self.locals, self.globals)
        return True if r is None else bool(r)


def as_callback(cb) -> BaseCallback:
    if cb is None:
        return BaseCallback()
    if isinstance(cb, (list, tuple)):
        return CallbackList([as_callback(c) for c in cb])
    if callable(cb) and not hasattr(cb, "on_step"):
        return _FnCallback(cb)
    return cb


class CheckpointCallback(BaseCallback):
    """[SB2] CheckpointCallback(save_freq, save_path, name_prefix) as constructed at sb_helper.py:81-82: every
    ``save_freq`` calls the model is saved to ``<save_path>/<name_prefix>_<num_timesteps>_steps``."""

    def __init__(self, save_freq: int, save_path: str, name_prefix: str = "rl_model", verbose: int = 0):
        super().__init__(verbose)
        self.save_freq, self.save_path, self.name_prefix = save_freq, save_path, name_prefix

    def _init_callback(self) -> None:
        if self.save_path is not None:
            os.makedirs(self.save_path, exist_ok=True)

    def _on_step(self) -> bool:
        if self.n_calls % self.save_freq == 0:
            path = os.path.join(self.save_path, "{}_{}_steps".format(self.name_prefix, self.num_timesteps))
            self.model.save(path)
            if self.verbose > 1:
                print("Saving model checkpoint to {}".format(path))
        return True


class TrainingStateCallback(BaseCallback):
    """Every ``save_freq`` calls, writes the model's whole training state (``save_training_state``: parameters, optimiser
    moments, replay, VecNormalize statistics, counters) to ``save_dir``.  Only the latest checkpoint is kept, because the
    replay makes each one large; a new one replaces the old only once it is complete."""

    def __init__(self, save_freq: int, save_dir: str, verbose: int = 0):
        super().__init__(verbose)
        self.save_freq, self.save_dir = int(save_freq), save_dir

    def _on_step(self) -> bool:
        if self.save_freq > 0 and self.n_calls % self.save_freq == 0:
            self.model.save_training_state(self.save_dir)
            if self.verbose > 1:
                print("Saving training state to {}".format(self.save_dir))
        return True


class EveryNTimesteps(EventCallback):
    """[SB2] trigger the child callback every ``n_steps`` environment timesteps."""

    def __init__(self, n_steps: int, callback: BaseCallback):
        super().__init__(callback)
        self.n_steps, self.last_time_trigger = n_steps, 0

    def _on_step(self) -> bool:
        if self.num_timesteps - self.last_time_trigger >= self.n_steps:
            self.last_time_trigger = self.num_timesteps
            return self._on_event()
        return True


class EvalCallback(EventCallback):
    """[SB2] common/callbacks.py EvalCallback (imported at train_stable_baselines.py:13; the reference's own copy in
    base_callbacks.py:16-117 derives from the same EventCallback and keeps working unchanged on top of this module):
    every ``eval_freq`` calls, sync the VecNormalize statistics into ``eval_env``, run ``n_eval_episodes`` episodes,
    append to ``<log_path>/evaluations.npz``, save ``best_model`` on a new best mean reward and fire the child callback."""

    def __init__(self, eval_env, callback_on_new_best: Optional[BaseCallback] = None, n_eval_episodes: int = 5, eval_freq: int = 10000,
                 log_path: Optional[str] = None, best_model_save_path: Optional[str] = None, deterministic: bool = True,
                 render: bool = False, verbose: int = 1):
        super().__init__(callback_on_new_best, verbose=verbose)
        from .vec_env import DummyVecEnv, VecEnv
        self.n_eval_episodes, self.eval_freq = n_eval_episodes, eval_freq
        self.best_mean_reward, self.last_mean_reward = -np.inf, -np.inf
        self.deterministic, self.render = deterministic, render
        if not isinstance(eval_env, VecEnv) and not hasattr(eval_env, "num_envs"):
            eval_env = DummyVecEnv([lambda: eval_env])
        assert eval_env.num_envs == 1, "You must pass only one environment for evaluation"
        self.eval_env = eval_env
        self.best_model_save_path = best_model_save_path
        self.log_path = os.path.join(log_path, "evaluations") if log_path is not None else None
        self.evaluations_results, self.evaluations_timesteps, self.evaluations_length = [], [], []

    def _init_callback(self) -> None:
        if type(self.training_env) is not type(self.eval_env):
            warnings.warn("Training and eval env are not of the same type {} != {}".format(self.training_env, self.eval_env))
        if self.best_model_save_path is not None:
            os.makedirs(self.best_model_save_path, exist_ok=True)
        if self.log_path is not None:
            os.makedirs(os.path.dirname(self.log_path), exist_ok=True)

    def _evaluate(self):
        from .evaluation import evaluate_policy
        from .vec_env import sync_envs_normalization
        sync_envs_normalization(self.training_env, self.eval_env)       # eval env sees the training statistics
        return evaluate_policy(self.model, self.eval_env, n_eval_episodes=self.n_eval_episodes, render=self.render,
                               deterministic=self.deterministic, return_episode_rewards=True)

    def _record(self, rewards, lengths) -> None:
        if self.log_path is None:
            return
        self.evaluations_timesteps.append(self.num_timesteps)
        self.evaluations_results.append(rewards)
        self.evaluations_length.append(lengths)
        np.savez(self.log_path, timesteps=self.evaluations_timesteps, results=self.evaluations_results, ep_lengths=self.evaluations_length)

    def _on_step(self) -> bool:
        due = self.eval_freq > 0 and self.n_calls % self.eval_freq == 0
        if not due:
            return True
        rewards, lengths = self._evaluate()
        self._record(rewards, lengths)
        self.last_mean_reward = float(np.mean(rewards))
        if self.verbose > 0:
            print("[eval] t={} reward {:.2f} +/- {:.2f}, length {:.1f} +/- {:.1f}".format(
                self.num_timesteps, self.last_mean_reward, float(np.std(rewards)), float(np.mean(lengths)), float(np.std(lengths))))
        if self.last_mean_reward < self.best_mean_reward:        # '>=' keeps a tie as the new best, like base_callbacks.py:104
            return True
        self.best_mean_reward = self.last_mean_reward
        if self.best_model_save_path is not None:
            self.model.save(os.path.join(self.best_model_save_path, "best_model"))
        if self.verbose > 0:
            print("[eval] new best mean reward {:.2f}".format(self.best_mean_reward))
        return self._on_event() if self.callback is not None else True
