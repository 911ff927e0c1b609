"""``DQN`` -- the dueling double DQN behind the ``sb.DQN`` call sites of the reference
(/root/reference/manipulation_main/training/sb_helper.py:155-165,183-199, train_stable_baselines.py:45-48,101-102), i.e.
stable-baselines 2.10.1 ``deepq`` with its defaults (dueling MLP policy [64, 64], double Q, Huber loss, per-variable gradient
clipping at 10, prioritised replay).  The learner runs on the GPU (csrc/dqn.cu); the algorithm is restated in
oracle/dqn_ref.py, which also lists what trained_models/DQN_4pads/DQN_simple_4pads.zip pins.  Import it as
``b200grasp.deepq.DQN`` (the stable-baselines path ``stable_baselines.deepq.DQN``).
"""
from __future__ import annotations

import ctypes as C
from collections import OrderedDict
from typing import Optional

import numpy as np

from . import _lib, training_state
from .base_model import BaseModel
from .callbacks import as_callback
from .tensorboard import EpisodeRewardLogger
from .learner import TransitionReplayLearner, _f32, _fp
from .vec_env import VecNormalize

_ONLINE, _TARGET = "deepq/model/", "deepq/target_q_func/model/"


class DQNLearner(TransitionReplayLearner):
    """numpy-facing wrapper of one ``b2g_dqn`` handle (maps 1:1 onto the C ABI)."""
    _abi = "dqn"

    def __init__(self, obs_dim=100, n_actions=12, layers=(64, 64), batch_size=32, buffer_size=50000, gamma=0.99, seed=0, device=0,
                 prioritized_replay=False, prioritized_replay_alpha=0.6, prioritized_replay_eps=1e-6, frame_capacity=None):
        """frame_capacity: the replay frame pool of BDQLearner (include/b200grasp.h: b2g_dqn_create2); None = two rows per slot."""
        self.lib = _lib.load()
        if len(layers) != 2:
            raise NotImplementedError(f"layers={list(layers)}: the DQN learner builds two hidden layers")
        cfg = _lib.DqnCfg(obs_dim, n_actions, int(layers[0]), int(layers[1]), batch_size, buffer_size, gamma, seed, device,
                          int(bool(prioritized_replay)), float(prioritized_replay_alpha), float(prioritized_replay_eps))
        self.prioritized_replay = bool(prioritized_replay)
        self.frame_capacity = None if frame_capacity is None else int(frame_capacity)
        self._create(cfg, self._replay_cfg(self.frame_capacity))
        self.obs_dim = self.obs_elems = obs_dim
        self.n_actions, self.batch_size = n_actions, batch_size
        self._act_width = 1
        self.obs_shape = (obs_dim,)          # shape of obs_rms_get's arrays (DQN sets the env's observation shape)

    def _has_grad(self, name):
        return name.startswith(_ONLINE)

    def set_eps(self, eps: float):
        """deepq/eps: the exploration epsilon the last action was taken with."""
        a = np.full(1, eps, np.float32)
        _lib.check(self.lib.b2g_dqn_set_param(self.h, b"deepq/eps", _fp(a), 1))

    def replay_add(self, obs, act, rew, next_obs, done):
        obs, next_obs = _f32(obs).reshape(-1, self.obs_dim), _f32(next_obs).reshape(-1, self.obs_dim)
        act, rew, done = _f32(np.reshape(act, -1)), _f32(np.reshape(rew, -1)), _f32(np.reshape(done, -1))
        n = rew.shape[0]
        assert obs.shape[0] == n and next_obs.shape[0] == n and act.size == n and done.size == n
        _lib.check(self.lib.b2g_dqn_replay_add(self.h, _fp(obs), _fp(act), _fp(rew), _fp(next_obs), _fp(done), n))

    def replay_size(self):
        return int(self.lib.b2g_dqn_replay_size(self.h))

    def step(self, n_steps=1, lr=5e-4):
        m = _lib.DqnMetrics()
        _lib.check(self.lib.b2g_dqn_step(self.h, n_steps, lr, C.byref(m)))
        return m.as_dict()

    def set_per_beta(self, beta: float):
        _lib.check(self.lib.b2g_dqn_set_per_beta(self.h, float(beta)))

    def last_per(self):
        """Slots, importance weights and new priorities (|td| + eps) of the last sampled step (weights and priorities with
        prioritised replay only)."""
        B = self.batch_size
        idx, w, p = np.empty(B, np.int32), np.empty(B, np.float32), np.empty(B, np.float32)
        _lib.check(self.lib.b2g_dqn_get_last_per(self.h, idx.ctypes.data_as(C.POINTER(C.c_int32)), _fp(w), _fp(p)))
        return idx, w, p

    def step_explicit(self, obs, act, rew, next_obs, done, weights=None, lr=5e-4, apply_update=True):
        B = self.batch_size
        td = np.empty(B, np.float32)
        w = _fp(_f32(weights)) if weights is not None else None
        m = _lib.DqnMetrics()
        _lib.check(self.lib.b2g_dqn_step_explicit(self.h, _fp(_f32(obs)), _fp(_f32(np.reshape(act, -1))), _fp(_f32(np.reshape(rew, -1))),
                                                   _fp(_f32(next_obs)), _fp(_f32(np.reshape(done, -1))), w, lr, int(apply_update),
                                                   C.byref(m), _fp(td)))
        out = m.as_dict()
        out["td"] = td
        return out

    def update_target(self):
        _lib.check(self.lib.b2g_dqn_update_target(self.h))

    def act(self, obs, with_q=False):
        """Greedy actions [n] of the online network on observations as the network sees them (a VecNormalize wrapper's
        output: nothing is normalised here), and with ``with_q`` the Q rows [n, n_actions]."""
        obs = _f32(obs).reshape(-1, self.obs_dim)
        n = obs.shape[0]
        out = np.empty(n, np.int32)
        q = np.empty((n, self.n_actions), np.float32) if with_q else None
        _lib.check(self.lib.b2g_dqn_act(self.h, _fp(obs), n, out.ctypes.data_as(C.POINTER(C.c_int32)), None if q is None else _fp(q)))
        return (out, q) if with_q else out

    def act_raw(self, obs, with_q=False):
        """``act`` on raw observations, normalised on the device with the learner's ``obs_rms`` (predict while the learner
        owns VecNormalize's statistics)."""
        obs = _f32(obs).reshape(-1, self.obs_dim)
        n = obs.shape[0]
        out = np.empty(n, np.int32)
        q = np.empty((n, self.n_actions), np.float32) if with_q else None
        _lib.check(self.lib.b2g_dqn_act_raw(self.h, _fp(obs), n, out.ctypes.data_as(C.POINTER(C.c_int32)), None if q is None else _fp(q)))
        return (out, q) if with_q else out

    # ---- the actor loop on one upload per frame (include/b200grasp.h: b2g_dqn_observe_*)
    def observe_act(self, obs, n=None, update_stats=True, eps=0.0, act=True):
        """``obs``: n raw observations to upload, merge into ``obs_rms`` (``update_stats``) and stage as the current
        observation of env i; ``None`` acts on the ones already staged.  Returns the [n] epsilon-greedy actions, or None
        with ``act=False``."""
        if obs is not None:
            obs = _f32(obs).reshape(-1, self.frame_elems)
            n = obs.shape[0]
            self.obs_rms_version += bool(update_stats)
        out = np.empty(int(n), np.int32) if act else None
        _lib.check(self.lib.b2g_dqn_observe_act(self.h, None if obs is None else _fp(obs), int(n), int(bool(update_stats)), float(eps),
                                                None if out is None else out.ctypes.data_as(C.POINTER(C.c_int32))))
        return out

    def observe_add(self, act, rew, next_obs, done, reset_obs=None, update_stats=True):
        """Transition i = (staged obs_i, act_i, rew_i, next_obs_i, done_i); ``reset_obs`` holds, for every finished env,
        the frame its auto-reset returned (the other rows are not read)."""
        act, next_obs = _f32(np.reshape(act, -1)), _f32(next_obs)
        rew, done = _f32(np.reshape(rew, -1)), _f32(np.reshape(done, -1))
        n = rew.shape[0]
        assert next_obs.size == n * self.frame_elems and act.size == n and done.size == n
        if reset_obs is not None:
            reset_obs = _f32(reset_obs)
            assert reset_obs.size == next_obs.size
        _lib.check(self.lib.b2g_dqn_observe_add(self.h, _fp(act), _fp(rew), _fp(next_obs), _fp(done),
                                                None if reset_obs is None else _fp(reset_obs), n, int(bool(update_stats))))
        self.obs_rms_version += bool(update_stats)



def _linear(t, span, p0, p1):
    """stable-baselines' LinearSchedule(span, initial_p=p0, final_p=p1).value(t)"""
    return p0 + min(float(t) / max(1, span), 1.0) * (p1 - p0)


def _check_policy_kwargs(policy_kwargs):
    kw = dict(policy_kwargs or {})
    unknown = set(kw) - {"layers", "dueling", "layer_norm", "act_fun"}
    if unknown:
        raise NotImplementedError(f"policy_kwargs {sorted(unknown)} are not built for DQN")
    if not kw.get("dueling", True):
        raise NotImplementedError("dueling=False: only the dueling DQN network is built")
    if kw.get("layer_norm", False):
        raise NotImplementedError("layer_norm=True: layer-normalised DQN policies are not built")
    if kw.get("act_fun") is not None and getattr(kw["act_fun"], "__name__", "") != "relu":
        raise NotImplementedError("act_fun: only ReLU is built")
    layers = list(kw.get("layers", [64, 64]))
    if len(layers) != 2:
        raise NotImplementedError(f"layers={layers}: the DQN learner builds exactly two hidden layers")
    return kw, [int(x) for x in layers]


class DQN(BaseModel):
    """stable-baselines 2.10 ``DQN(policy, env, ...)`` with its signature and defaults, plus ``device`` and ``seed``:
    ``learn / predict / save / load / get_parameters / load_parameters / get_env / get_vec_normalize_env`` and
    ``save_training_state / load_training_state``.  One environment (stable-baselines' DQN refuses a VecEnv of more)."""
    _algo = "DQN"

    def __init__(self, policy, env, gamma=0.99, learning_rate=5e-4, buffer_size=50000, exploration_fraction=0.1,
                 exploration_final_eps=0.02, exploration_initial_eps=1.0, train_freq=1, batch_size=32, double_q=True, learning_starts=1000,
                 target_network_update_freq=500, prioritized_replay=False, prioritized_replay_alpha=0.6, prioritized_replay_beta0=0.4,
                 prioritized_replay_beta_iters=None, prioritized_replay_eps=1e-6, param_noise=False, n_cpu_tf_sess=None, verbose=0,
                 tensorboard_log=None, _init_setup_model=True, policy_kwargs=None, full_tensorboard_log=False, seed=None, device=0,
                 replay_frames=None, device_obs_norm=False):
        if not double_q:
            raise NotImplementedError("double_q=False: only the double-Q target is built")
        if param_noise:
            raise NotImplementedError("param_noise=True: parameter-noise exploration is not built")
        if isinstance(policy, str):
            if policy != "MlpPolicy":
                raise NotImplementedError(f"policy '{policy}': only the MLP DQN policy is built")
        else:
            from .deepq.policies import MlpPolicy
            if policy is not MlpPolicy:
                raise NotImplementedError(f"policy {getattr(policy, '__name__', policy)}: only deepq.policies.MlpPolicy is built")
        self.policy_kwargs, self.layers = _check_policy_kwargs(policy_kwargs)
        self.gamma, self.learning_rate, self.buffer_size, self.batch_size = gamma, learning_rate, int(buffer_size), int(batch_size)
        self.exploration_fraction, self.exploration_final_eps = exploration_fraction, exploration_final_eps
        self.exploration_initial_eps = exploration_initial_eps
        self.train_freq, self.learning_starts, self.target_network_update_freq = int(train_freq), int(learning_starts), int(target_network_update_freq)
        self.prioritized_replay = bool(prioritized_replay)
        self.per_alpha, self.per_beta0, self.per_beta_iters, self.per_eps = prioritized_replay_alpha, prioritized_replay_beta0, \
            prioritized_replay_beta_iters, prioritized_replay_eps
        self.replay_frames = None if replay_frames is None else int(replay_frames)    # DQNLearner's frame_capacity
        # learn() feeds the actor, the statistics and the replay from one upload per frame (DQNLearner.observe_act / _add), a
        # VecNormalize with norm_obs hands its obs_rms to the device learner and a VecEncodeDepth its encoder
        self.device_obs_norm = bool(device_obs_norm)
        self.verbose, self.seed, self.device = verbose, seed, device
        self.tensorboard_log = tensorboard_log
        self.num_timesteps = 0
        self.n_target_updates = 0
        self._rng = np.random.default_rng(seed)            # epsilon-greedy draws of learn()
        self.predict_rng = np.random.default_rng(seed)     # softmax(Q) draws of predict(deterministic=False)
        self.learner: Optional[DQNLearner] = None
        if env is not None:
            self._set_env(env)
            if _init_setup_model:
                self.setup_model()

    def set_env(self, env):
        self._set_env(env)
        if self.learner is not None:
            self._attach_device_norm()
            self._attach_obs_encoder()

    def _check_env(self):
        if self.n_envs > 1:      # stable-baselines' own refusal (deepq/dqn.py: "...cannot be used with more than one env")
            raise ValueError("Error: DQN cannot be used with more than one environment (num_envs > 1)")

    def setup_model(self):
        if not hasattr(self.action_space, "n"):
            raise NotImplementedError(f"DQN needs a Discrete action space, got {self.action_space}")
        obs_dim = int(np.prod(self.observation_space.shape))
        self.learner = DQNLearner(obs_dim, int(self.action_space.n), tuple(self.layers), self.batch_size, self.buffer_size, self.gamma,
                                  int(self.seed or 0), self.device, prioritized_replay=self.prioritized_replay,
                                  prioritized_replay_alpha=self.per_alpha, prioritized_replay_eps=self.per_eps,
                                  **self._replay_kwargs())
        rng = np.random.default_rng(self.seed)
        p = OrderedDict()
        for n, shp in self.learner.param_shapes.items():
            if n == "deepq/eps":
                p[n] = np.float32(0.0)          # tf.constant_initializer(0) in deepq/build_graph.py build_act
            elif n.startswith(_TARGET):
                p[n] = p[n.replace(_TARGET, _ONLINE)].copy()
            elif len(shp) == 2:                 # tf.contrib.layers.fully_connected: Xavier uniform weights, zero biases
                lim = np.sqrt(6.0 / (shp[0] + shp[1]))
                p[n] = rng.uniform(-lim, lim, shp).astype(np.float32)
            else:
                p[n] = np.zeros(shp, np.float32)
        self.learner.load_parameters(p)
        self.learner.obs_shape = tuple(self.observation_space.shape)
        self._attach_device_norm()
        self._attach_obs_encoder()

    def _attach_device_norm(self):
        super()._attach_device_norm()
        if self._owns_obs_rms():
            self._sync_norm_stats()

    def _sync_norm_stats(self):
        """The wrapper's statistics for the gather of the sampled step; a learner that owns obs_rms takes the reward scalars
        and clips only (the observation statistics are its own)."""
        vn = self._vec_normalize_env
        if self._owns_obs_rms():
            self.learner.set_norm_stats(None, None, float(vn.ret_rms.var), vn.clip_obs, vn.clip_reward, vn.epsilon,
                                        norm_obs=vn.norm_obs, norm_reward=vn.norm_reward)
            return
        self.learner.set_norm_stats(vn.obs_rms.mean, vn.obs_rms.var, float(vn.ret_rms.var), vn.clip_obs, vn.clip_reward, vn.epsilon,
                                    norm_obs=vn.norm_obs, norm_reward=vn.norm_reward)

    _step_tags = {"loss": "loss", "mean_q": "mean_q", "mean_abs_td_error": "mean_abs_td", "grad_norm": "grad_norm"}

    def learn(self, total_timesteps, callback=None, log_interval=100, tb_log_name="DQN", reset_num_timesteps=True, replay_wrapper=None):
        """stable-baselines 2.10 DQN.learn: per environment step act epsilon-greedily, step, count, call back, store the raw
        transition, then (past learning_starts, every train_freq steps) one gradient step, and every
        target_network_update_freq environment steps the hard target copy.  With tensorboard_log every gradient step's
        losses are written from the device metrics ring (tensorboard.py)."""
        if replay_wrapper is not None:
            raise NotImplementedError("replay_wrapper: the replay lives on the device")
        return self._learn_logged(tb_log_name, reset_num_timesteps,
                                  lambda writer, steps: self._learn(total_timesteps, callback, reset_num_timesteps, writer, steps))

    def _learn(self, total_timesteps, callback, reset_num_timesteps, writer, steps):
        callback = as_callback(callback)
        callback.init_callback(self)
        callback.on_training_start({"self": self, "writer": writer}, globals())
        vn = self._vec_normalize_env
        lr = self.learning_rate if not callable(self.learning_rate) else self.learning_rate(1.0)
        # reset_num_timesteps=False continues a run: the schedules follow num_timesteps over a run that ends total_timesteps from
        # now, so an interrupted and resumed run takes the steps of an uninterrupted one
        t0 = 0 if reset_num_timesteps else self.num_timesteps
        if reset_num_timesteps:
            self.num_timesteps = 0
        horizon = t0 + total_timesteps
        eps_span = int(self.exploration_fraction * horizon)
        beta_span = self.per_beta_iters or horizon
        dev = self.device_obs_norm
        if dev and vn is not None:
            if not isinstance(vn, VecNormalize) or not vn.norm_obs:
                raise RuntimeError("device_obs_norm=True needs the env's VecNormalize to have norm_obs=True")
            if not self._owns_obs_rms():
                raise RuntimeError("learn: the env's VecNormalize statistics are owned by another model's learner (close that model, "
                                   "or build this one with device_obs_norm=True before it)")
        obs = self.env.reset()
        raw = vn.get_original_obs() if vn is not None else obs
        stats = dev and vn is not None
        if dev:      # the reset frames: uploaded once, merged (VecNormalize.reset's update), staged as the current observation
            self.learner.observe_act(np.asarray(raw, np.float32), update_stats=stats and vn.training, act=False)
        eps = self.exploration_initial_eps
        ep_log = EpisodeRewardLogger(1) if writer is not None else None
        for _ in range(total_timesteps):
            eps = _linear(self.num_timesteps, eps_span, self.exploration_initial_eps, self.exploration_final_eps)
            if dev:      # the staged frame, current statistics, epsilon-greedy on the device (Philox stream 3)
                action = int(self.learner.observe_act(None, n=1, eps=eps)[0])
            else:
                greedy = self.learner.act(np.asarray(obs, np.float32))     # the wrapper's output, as stable-baselines' act sees it
                action = int(self._rng.integers(0, self.learner.n_actions)) if self._rng.random() < eps else int(greedy[0])
            new_obs, rew, done, infos = self.env.step(np.array([action]))
            self.num_timesteps += 1
            if callback.on_step() is False:
                break
            new_raw = vn.get_original_obs() if vn is not None else new_obs
            rew_raw = vn.get_original_reward() if vn is not None else rew
            nxt = np.array(new_raw, np.float32, copy=True).reshape(1, -1)
            info = infos[0] if infos else {}
            if done[0] and isinstance(info, dict) and "terminal_observation" in info and vn is None:
                nxt[0] = np.asarray(info["terminal_observation"], np.float32).reshape(-1)
            if dev:      # next_obs crosses once; a finished env's reset frame is merged and staged
                self.learner.observe_add(np.float32(action), rew_raw, nxt, np.asarray(done, np.float32),
                                         reset_obs=np.asarray(new_raw, np.float32).reshape(1, -1) if done[0] else None,
                                         update_stats=stats and vn.training)       # step_wait's update; a callback may switch it
            else:
                self.learner.replay_add(np.asarray(raw, np.float32), np.float32(action), rew_raw, nxt, np.asarray(done, np.float32))
            obs, raw = new_obs, new_raw
            if ep_log is not None:
                ep_log(writer, rew_raw, done, self.num_timesteps)
            can_sample = self.learner.replay_size() >= self.batch_size
            if can_sample and self.num_timesteps > self.learning_starts and self.num_timesteps % self.train_freq == 0:
                if self.prioritized_replay:
                    self.learner.set_per_beta(_linear(self.num_timesteps, beta_span, self.per_beta0, 1.0))
                if vn is not None:       # the sample is normalised with the statistics of this moment
                    self._sync_norm_stats()
                self.learner.step(1, lr)
                if steps is not None:
                    steps.queued(1, self.num_timesteps)
            if can_sample and self.num_timesteps > self.learning_starts and self.num_timesteps % self.target_network_update_freq == 0:
                self.learner.update_target()
                self.n_target_updates += 1
        self.learner.set_eps(eps)
        callback.on_training_end()
        return self

    def predict(self, observation, state=None, mask=None, deterministic=True):
        """Greedy actions, or with ``deterministic=False`` a draw from softmax(Q) per row (the deepq policy's ``step``; the
        uniform comes from ``self.predict_rng``).  ``observation`` is what the env hands out: with a VecNormalize wrapper its
        normalised output, which the network takes as it is, or its raw output while this model's learner owns the
        statistics (``predict_takes_raw_obs``), which the learner normalises on the device."""
        self._check_encoded(observation)
        obs = np.asarray(observation, np.float32).reshape(-1, self.learner.obs_dim)
        act = self.learner.act_raw if self.predict_takes_raw_obs else self.learner.act
        idx, q = act(obs, with_q=True)
        if not deterministic:
            q = q.astype(np.float64)
            p = np.exp(q - q.max(1, keepdims=True))
            p /= p.sum(1, keepdims=True)
            idx = np.empty(len(q), np.int64)
            for i in range(len(q)):          # numpy's choice(n, p=p): inverse CDF of one uniform
                cdf = np.cumsum(p[i])
                cdf /= cdf[-1]
                idx[i] = int(np.searchsorted(cdf, self.predict_rng.random(), side="right"))
        idx = np.asarray(idx, np.int64)
        single = np.ndim(observation) == len(getattr(self.observation_space, "shape", (self.learner.obs_dim,)))
        return (int(idx[0]) if single else idx), None

    def _data(self):
        data = {"double_q": True, "param_noise": False, "learning_starts": self.learning_starts, "train_freq": self.train_freq,
                "prioritized_replay": self.prioritized_replay, "prioritized_replay_eps": self.per_eps, "batch_size": self.batch_size,
                "target_network_update_freq": self.target_network_update_freq, "prioritized_replay_alpha": self.per_alpha,
                "prioritized_replay_beta0": self.per_beta0, "prioritized_replay_beta_iters": self.per_beta_iters,
                "exploration_final_eps": self.exploration_final_eps, "exploration_fraction": self.exploration_fraction,
                "exploration_initial_eps": self.exploration_initial_eps, "learning_rate": self.learning_rate, "gamma": self.gamma,
                "verbose": self.verbose, "n_envs": 1, "seed": self.seed, "policy_kwargs": dict(self.policy_kwargs)}
        if callable(self.learning_rate):
            data["learning_rate"] = None
        return data

    @classmethod
    def load(cls, load_path, env=None, custom_objects=None, **kwargs):
        """Reads a stable-baselines DQN zip (the shipped DQN_simple_4pads.zip / best_model.zip unchanged): the number of actions
        and the widths come from the parameter shapes, the hyper-parameters from ``data``."""
        from .spaces import Box, Discrete
        data, params = cls._read_zip(load_path)
        w0 = params[_ONLINE + "action_value/fully_connected/weights"]
        w1 = params[_ONLINE + "action_value/fully_connected_1/weights"]
        w2 = params[_ONLINE + "action_value/fully_connected_2/weights"]
        kw = {k: data[k] for k in ("gamma", "learning_rate", "batch_size", "learning_starts", "train_freq", "target_network_update_freq",
                                   "exploration_fraction", "exploration_final_eps", "prioritized_replay", "prioritized_replay_alpha",
                                   "prioritized_replay_beta0", "prioritized_replay_beta_iters", "prioritized_replay_eps", "seed")
              if k in data and not isinstance(data[k], dict)}
        kw["policy_kwargs"] = dict(data.get("policy_kwargs") or {}, layers=[int(w0.shape[1]), int(w1.shape[1])])
        kw.update(kwargs)        # stable-baselines 2.10 does not save buffer_size: its default (50000) unless given here
        m = cls("MlpPolicy", None, _init_setup_model=False, **kw)
        return m._finish_load(env, Box(-np.inf, np.inf, (w0.shape[0],)), Discrete(w2.shape[1]), params)

    # ------------------------------------------------------------------ training state (training_state.py)
    def _host_state(self):
        if callable(self.learning_rate):
            raise NotImplementedError("save_training_state needs a constant learning_rate")
        init = dict(gamma=self.gamma, learning_rate=self.learning_rate, buffer_size=self.buffer_size,
                    exploration_fraction=self.exploration_fraction, exploration_final_eps=self.exploration_final_eps,
                    exploration_initial_eps=self.exploration_initial_eps, train_freq=self.train_freq, batch_size=self.batch_size,
                    learning_starts=self.learning_starts, target_network_update_freq=self.target_network_update_freq,
                    prioritized_replay=self.prioritized_replay, prioritized_replay_alpha=self.per_alpha,
                    prioritized_replay_beta0=self.per_beta0, prioritized_replay_beta_iters=self.per_beta_iters,
                    prioritized_replay_eps=self.per_eps, policy_kwargs=self.policy_kwargs, verbose=self.verbose, seed=self.seed,
                    device=self.device)
        if self.replay_frames is not None:
            init["replay_frames"] = self.replay_frames
        if self.device_obs_norm:
            init["device_obs_norm"] = True
        host = {"algo": "DQN", "init": init, "num_timesteps": int(self.num_timesteps), "n_target_updates": int(self.n_target_updates),
                "rng": training_state.rng_state(self._rng), "predict_rng": training_state.rng_state(self.predict_rng)}
        enc = self._encoder_host()
        if enc is not None:
            host["obs_encoder"] = enc
        return host

    def _restore_host_state(self, host):
        self.num_timesteps = int(host["num_timesteps"])
        self.n_target_updates = int(host.get("n_target_updates", 0))
        training_state.set_rng_state(self._rng, host["rng"])
        training_state.set_rng_state(self.predict_rng, host["predict_rng"])
