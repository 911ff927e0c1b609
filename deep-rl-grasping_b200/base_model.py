"""``BaseModel`` -- what the SAC, BDQ, DQN, PPO2 and TRPO front ends share: the env plumbing, the device ownership of VecNormalize's
observation statistics, parameters, the stable-baselines zip and training-state directories (training_state.py).  Each
algorithm (PPO2 and TRPO through ``actor_critic.ActorCriticModel``) keeps its constructor, ``setup_model`` (and with it every parameter-initialisation rule), ``learn``, ``predict``,
``_data`` (the zip's hyper-parameters) and ``_host_state`` (host.json).
"""
from __future__ import annotations

import os
from collections import OrderedDict
from typing import Optional

import numpy as np

from . import _lib, sb_io, training_state
from .tensorboard import StepLog, TensorboardWriter
from .vec_env import DummyVecEnv, VecNormalize, unwrap_encode_depth


def unwrap_vec_normalize(env) -> Optional[VecNormalize]:
    e = env
    while e is not None:
        if isinstance(e, VecNormalize) or type(e).__name__ == "VecNormalize":
            return e
        e = getattr(e, "venv", None)
    return None


class BaseModel:
    _algo = ""                     # host.json's "algo"
    _policy = "MlpPolicy"          # what load_training_state passes as the constructor's policy
    device_obs_norm = False
    tensorboard_log = None
    #: per-gradient-step summaries of the replay learners: tag -> column of the learner's metrics ring (_lib.LOG_COLS)
    _step_tags = None
    learner = None
    env = None
    _vec_normalize_env = None

    def _replay_kwargs(self):
        """The learner's frame_capacity for BDQ / DQN's ``replay_frames`` (nothing without it: the default layout)."""
        f = getattr(self, "replay_frames", None)
        return {} if f is None else {"frame_capacity": f}

    # ------------------------------------------------------------------ TensorBoard (tensorboard.py)
    def _learn_logged(self, tb_log_name, reset_num_timesteps, run):
        """run(writer, step_log) inside stable-baselines' TensorboardWriter: writer is None without tensorboard_log and on
        ranks other than 0; step_log drains the learner's metrics ring (replay learners) and is drained once more on the
        way out, also when a callback stops the run or an exception ends it."""
        dp = getattr(self, "_dev", None) or getattr(self, "_dp", None) or {}
        path = self.tensorboard_log if int(dp.get("rank", 0)) == 0 else None
        with TensorboardWriter(path, tb_log_name, new_tb_log=reset_num_timesteps) as writer:
            steps = None
            if writer is not None and self._step_tags is not None:
                cols = _lib.LOG_COLS[self.learner._abi]
                steps = StepLog(self.learner, writer, list(self._step_tags), [cols.index(c) for c in self._step_tags.values()])
            try:
                return run(writer, steps)
            finally:
                if steps is not None:
                    steps.close()

    # ------------------------------------------------------------------ env plumbing
    def _set_env(self, env):
        if not hasattr(env, "num_envs"):
            env = DummyVecEnv([lambda: env])
        self.env, self.n_envs = env, int(env.num_envs)
        self.observation_space, self.action_space = env.observation_space, env.action_space
        self._vec_normalize_env = unwrap_vec_normalize(env)
        self._check_env()

    def _check_env(self):
        """Refuses an env this algorithm does not train on (called once the env is set)."""

    def get_env(self):
        return self.env

    def get_vec_normalize_env(self):
        return self._vec_normalize_env

    def close(self):
        """Releases the device learner.  Observation statistics it owned go back to the VecNormalize wrapper first."""
        if self.learner is not None:
            if self._owns_obs_rms():
                self._vec_normalize_env.take_obs_rms_back()
            ve = unwrap_encode_depth(self.env)
            if ve is not None and ve.encoder_owner is self.learner:
                ve.take_encoder_back()
            self.learner.close()
            self.learner = None

    # ------------------------------------------------------------------ VecNormalize's obs_rms on the device (device_obs_norm)
    def _owns_obs_rms(self) -> bool:
        vn = self._vec_normalize_env
        return vn is not None and self.learner is not None and getattr(vn, "obs_rms_owner", None) is self.learner

    @property
    def predict_takes_raw_obs(self) -> bool:
        """True while a learner owns the statistics of this model's VecNormalize: that wrapper returns raw observations and
        ``predict`` normalises them on the device (``evaluate_policy`` feeds an evaluation wrapper's raw copy accordingly)."""
        return bool(getattr(self._vec_normalize_env, "learner_owns_obs_rms", False))

    def _attach_device_norm(self):
        """device_obs_norm: the wrapper's obs_rms moves to this learner, unless another learner owns it already (a second
        model built on the same env, e.g. a parameter donor: it reads the owner's statistics and leaves them where they are)."""
        vn = self._vec_normalize_env
        if self.device_obs_norm and isinstance(vn, VecNormalize) and vn.norm_obs and not vn.learner_owns_obs_rms:
            vn.give_obs_rms_to(self.learner)

    # ------------------------------------------------------------------ the perception encoder on the device (VecEncodeDepth)
    def _attach_obs_encoder(self):
        """device_obs_norm on a stack with a VecEncodeDepth: the learner takes the encoder and the wrapper passes raw depth rows
        (one upload per frame, encoded on the device).  It stays in host mode while a host VecNormalize above it needs
        encoded rows, or while another learner has the encoder."""
        ve = unwrap_encode_depth(self.env)
        if ve is None or not self.device_obs_norm or ve.encoder_owner is not None:
            return
        if self._vec_normalize_env is not None and not self._owns_obs_rms():
            return
        self.learner.set_obs_encoder(ve.encoder, ve.tail)
        ve.give_encoder_to(self.learner)

    def _check_encoded(self, observation):
        """``predict`` takes encoded observations: a raw depth row of this model's VecEncodeDepth is refused."""
        ve = unwrap_encode_depth(self.env)
        if ve is not None and ve.raw_width != ve.observation_space.shape[0] and np.shape(observation)[-1:] == (ve.raw_width,):
            raise ValueError(f"predict takes encoded observations of {ve.observation_space.shape[0]} floats, got raw rows of "
                             f"{ve.raw_width}: wrap the env in a host-mode VecEncodeDepth (as the evaluation env is)")

    def _encoder_host(self):
        """host.json's record of the encoder a learner encodes with: its directory, weight digest and precision (None
        without one)."""
        ve = unwrap_encode_depth(self.env)
        if ve is None or ve.encoder_owner is not self.learner:
            return None
        return {"dir": getattr(ve.encoder, "model_dir", None), "digest": ve.encoder.weights_digest(),
                "precision": getattr(ve.encoder, "precision", "fp32")}

    @staticmethod
    def _check_encoder_digest(path, host, env):
        want = host.get("obs_encoder")
        if want is None:
            return
        ve = unwrap_encode_depth(env)
        if ve is None:
            raise ValueError(f"{path} was trained on the device encoder of {want['dir']}: wrap the env in a VecEncodeDepth")
        want_prec, got_prec = want.get("precision", "fp32"), getattr(ve.encoder, "precision", "fp32")   # older files: fp32
        if got_prec != want_prec:
            raise ValueError(f"{path} was trained through the {want_prec} encoder of {want['dir']}; the env's VecEncodeDepth "
                             f"encodes in {got_prec}")
        got = ve.encoder.weights_digest()
        if got != want["digest"]:
            raise ValueError(f"{path} was trained through encoder weights {want['digest'][:12]} ({want['dir']}); the env's "
                             f"VecEncodeDepth holds {got[:12]}")

    # ------------------------------------------------------------------ parameters / persistence
    def get_parameters(self):
        return OrderedDict((n + ":0", a) for n, a in self.learner.get_parameters().items())

    def load_parameters(self, load_path_or_dict, exact_match=True):
        params = load_path_or_dict
        if isinstance(params, str):
            _, params = sb_io.load_sb_zip(params)
        self.learner.load_parameters(params, exact_match=exact_match)

    def save(self, save_path, cloudpickle=False):
        """A stable-baselines zip: ``data`` (hyper-parameters), ``parameter_list`` and ``parameters`` in the learner's order."""
        d = os.path.dirname(save_path)
        if d:
            os.makedirs(d, exist_ok=True)
        sb_io.save_sb_zip(save_path, self._data(), self.learner.get_parameters())

    @staticmethod
    def _read_zip(load_path):
        """``load``'s (data, params) of ``load_path``, or of ``load_path + ".zip"`` when only that exists."""
        if not os.path.exists(load_path) and os.path.exists(load_path + ".zip"):
            load_path += ".zip"
        return sb_io.load_sb_zip(load_path)

    def _finish_load(self, env, observation_space, action_space, params):
        """``load``'s last steps: ``env``, or without one the spaces the zip implies; then the learner and the zip's
        parameters."""
        if env is not None:
            self._set_env(env)
        else:
            self.env, self.n_envs, self._vec_normalize_env = None, 1, None
            self.observation_space, self.action_space = observation_space, action_space
        self.setup_model()
        self.learner.load_parameters(params, exact_match=True)
        return self

    # ------------------------------------------------------------------ training state (training_state.py)
    def save_training_state(self, path):
        """Writes directory ``path``: model.zip, learner.state (parameters, Adam moments, counters and what the learner
        stores: the replay and its priority trees, a device obs_rms), vecnormalize.pkl and host.json.  The previous contents
        stay loadable until the new directory is complete."""
        return training_state.save_training_state(self, path)

    @classmethod
    def load_training_state(cls, path, env, **kwargs):
        """Rebuilds the model ``save_training_state`` wrote into ``path`` on ``env`` and restores the saved VecNormalize
        statistics into ``env``'s wrapper.  ``learn(n, reset_num_timesteps=False)`` then continues the run."""
        path = training_state.resolve(path)
        host = training_state.read_host(path)
        if host.get("algo") != cls._algo:
            raise ValueError(f"{path} holds a {host.get('algo')} training state")
        cls._check_encoder_digest(path, host, env)
        model = cls(cls._policy_from_host(host), env, **dict(host["init"], **kwargs))
        training_state.restore_vec_normalize(path, model.env)
        model._attach_device_norm()        # the restored statistics go back to the learner; learner.state carries the same ones
        model.load_parameters(os.path.join(path, training_state.MODEL_FILE))
        model.learner.load_state(os.path.join(path, training_state.STATE_FILE))
        model._restore_host_state(host)
        return model

    @classmethod
    def _policy_from_host(cls, host):
        return cls._policy

    def _restore_host_state(self, host):
        """The counters and generators of ``_host_state``, after the learner's state is back."""
        raise NotImplementedError
