"""``BDQ`` -- branching dueling Q-network learner behind the ``sb.BDQ`` call sites of the reference
(/root/reference/manipulation_main/training/train_stable_baselines.py:103-104, sb_helper.py:202-226; hyper-parameters
config/gripper_grasp.yaml:104-118).  The reference's implementation is the author's stable-baselines fork ``bdq_sb``
(absent from the tree), so this follows the published algorithm with the variable names of the shipped zips; see
oracle/bdq_ref.py for every choice that is not pinned.  Prioritised replay (zip data ``prioritized_replay True, alpha .6,
beta0 .4``; config/simplified_object_picking.yaml:108-110) runs on device-resident sum / min segment trees; data
parallelism (BASELINE config 4) = one replay shard per rank + one NCCL all-reduce of the gradients per step.  Actions
are branch bin indices, mapped to linspace(-1, 1, n_bins).
"""
from __future__ import annotations

import ctypes as C
import os
from collections import OrderedDict
from typing import Optional

import numpy as np

from . import _lib, sb_io, training_state
from .callbacks import as_callback
from .learner import HandleLearner, _f32, _fp
from .vec_env import DummyVecEnv, VecNormalize


class BDQLearner(HandleLearner):
    """numpy-facing wrapper of one ``b2g_bdq`` handle (maps 1:1 onto the C ABI)."""
    _abi = "bdq"

    def __init__(self, obs_dim=100, n_branches=3, n_bins=8, layers=((64, 64), (32,), (32,)), batch_size=64, buffer_size=100000,
                 gamma=0.99, target_network_update_freq=1000, trunk_grad_rescale=True, seed=0, device=0, rank=0, nranks=1, nccl_id=None,
                 prioritized_replay=False, prioritized_replay_alpha=0.6, prioritized_replay_eps=1e-6):
        self.lib = _lib.load()
        if layers[1][0] != layers[2][0]:
            raise NotImplementedError("branch and state-value hidden widths must match (every shipped zip / config)")
        self._id_buf, idp, libp = None, None, None
        if nranks > 1:
            if nccl_id is None or len(nccl_id) != 128:
                raise ValueError("nranks > 1 needs the 128-byte nccl_id shared by all ranks")
            self._id_buf = C.create_string_buffer(bytes(nccl_id), 128)
            idp = C.cast(self._id_buf, C.c_void_p)
            lp = _lib.default_nccl_lib()
            libp = lp.encode() if lp else None
        cfg = _lib.BdqCfg(obs_dim, n_branches, n_bins, layers[0][0], layers[0][1], layers[1][0], batch_size, buffer_size, gamma,
                          target_network_update_freq, int(trunk_grad_rescale), seed, device, rank, nranks, idp, libp,
                          int(bool(prioritized_replay)), float(prioritized_replay_alpha), float(prioritized_replay_eps))
        self.prioritized_replay = bool(prioritized_replay)
        self._create(cfg)
        self.obs_dim, self.n_branches, self.n_bins, self.batch_size = obs_dim, n_branches, n_bins, batch_size
        self.obs_shape = (obs_dim,)          # shape of obs_rms_get's arrays (BDQ sets the env's observation shape)

    def _has_grad(self, name):
        return name.startswith("bdq/model/")

    def replay_add(self, obs, act_idx, rew, next_obs, done):
        obs, next_obs, act = _f32(obs), _f32(next_obs), _f32(act_idx)
        rew, done = _f32(np.reshape(rew, -1)), _f32(np.reshape(done, -1))
        _lib.check(self.lib.b2g_bdq_replay_add(self.h, _fp(obs), _fp(act), _fp(rew), _fp(next_obs), _fp(done), rew.shape[0]))

    def replay_size(self):
        return int(self.lib.b2g_bdq_replay_size(self.h))

    def load_state(self, path: str):
        """Restores a ``save_state`` file into this learner, which must have the same configuration (and own a device
        ``obs_rms`` exactly when the file carries one)."""
        super().load_state(path)
        self.obs_rms_version += 1

    def set_norm_stats(self, obs_mean=None, obs_var=None, ret_var=1.0, clip_obs=10.0, clip_reward=10.0, epsilon=1e-8,
                       norm_obs=True, norm_reward=True):
        """VecNormalize's statistics for the gather of the gradient step and act().  ``obs_mean = obs_var = None`` with
        ``norm_obs``: a learner that owns ``obs_rms`` keeps its device statistics and takes the scalars only."""
        dp = C.POINTER(C.c_double)
        mp = vp = None
        if norm_obs and obs_mean is not None:
            m = np.ascontiguousarray(obs_mean, np.float64).reshape(-1)
            v = np.ascontiguousarray(obs_var, np.float64).reshape(-1)
            assert m.size == self.obs_dim and v.size == self.obs_dim
            mp, vp = m.ctypes.data_as(dp), v.ctypes.data_as(dp)
        _lib.check(self.lib.b2g_bdq_set_norm_stats(self.h, mp, vp, float(ret_var), float(clip_obs), float(clip_reward),
                                                    float(epsilon), int(bool(norm_obs)), int(bool(norm_reward))))
        if mp is not None:
            self.obs_rms_version += 1

    # ---- device-resident obs_rms and the actor loop on one upload per frame (include/b200grasp.h: b2g_bdq_observe_*)
    #: bumped by every call that may change the device statistics (DeviceRunningMeanStd caches against it)
    obs_rms_version = 0

    def obs_rms_set(self, mean, var, count):
        """Creates (first call) or overwrites the device ``obs_rms``: float64 mean / var of the observation + count."""
        dp = C.POINTER(C.c_double)
        m = np.ascontiguousarray(mean, np.float64).reshape(-1)
        v = np.ascontiguousarray(var, np.float64).reshape(-1)
        assert m.size == self.obs_dim and v.size == self.obs_dim
        _lib.check(self.lib.b2g_bdq_obs_rms_set(self.h, m.ctypes.data_as(dp), v.ctypes.data_as(dp), float(count)))
        self.obs_rms_version += 1

    def obs_rms_get(self):
        """(mean, var, count) of the device ``obs_rms`` in ``obs_shape``; waits for the work enqueued on the handle."""
        dp = C.POINTER(C.c_double)
        m, v = np.empty(self.obs_shape, np.float64), np.empty(self.obs_shape, np.float64)
        cnt = C.c_double()
        _lib.check(self.lib.b2g_bdq_obs_rms_get(self.h, m.ctypes.data_as(dp), v.ctypes.data_as(dp), C.byref(cnt)))
        return m, v, float(cnt.value)

    def observe_act(self, obs, n=None, update_stats=True, eps=0.0, act=True):
        """``obs``: n raw observations to upload, merge into ``obs_rms`` (``update_stats``) and stage as the current
        observation of env i; ``None`` acts on the ones already staged.  Returns the [n, n_branches] epsilon-greedy bin
        indices, or None with ``act=False``."""
        if obs is not None:
            obs = _f32(obs).reshape(-1, self.obs_dim)
            n = obs.shape[0]
            self.obs_rms_version += bool(update_stats)
        out = np.empty((int(n), self.n_branches), np.int32) if act else None
        _lib.check(self.lib.b2g_bdq_observe_act(self.h, None if obs is None else _fp(obs), int(n), int(bool(update_stats)), float(eps),
                                                None if out is None else out.ctypes.data_as(C.POINTER(C.c_int32))))
        return out

    def observe_add(self, act_idx, rew, next_obs, done, reset_obs=None, update_stats=True):
        """Transition i = (staged obs_i, act_idx_i, rew_i, next_obs_i, done_i); ``reset_obs`` holds, for every finished env,
        the frame its auto-reset returned (the other rows are not read)."""
        act, next_obs = _f32(act_idx), _f32(next_obs)
        rew, done = _f32(np.reshape(rew, -1)), _f32(np.reshape(done, -1))
        n = rew.shape[0]
        assert next_obs.size == n * self.obs_dim and act.size == n * self.n_branches and done.size == n
        if reset_obs is not None:
            reset_obs = _f32(reset_obs)
            assert reset_obs.size == next_obs.size
        _lib.check(self.lib.b2g_bdq_observe_add(self.h, _fp(act), _fp(rew), _fp(next_obs), _fp(done),
                                                None if reset_obs is None else _fp(reset_obs), n, int(bool(update_stats))))
        self.obs_rms_version += bool(update_stats)

    def upload_bytes(self) -> dict:
        """Bytes copied host -> device so far: by ``observe_*`` / ``obs_rms_set``, and by ``act`` + ``replay_add`` +
        ``set_norm_stats``."""
        a, b = C.c_int64(), C.c_int64()
        _lib.check(self.lib.b2g_bdq_upload_bytes(self.h, C.byref(a), C.byref(b)))
        return {"observe": int(a.value), "other": int(b.value)}

    def step(self, n_steps=1, lr=1e-4):
        m = _lib.BdqMetrics()
        _lib.check(self.lib.b2g_bdq_step(self.h, n_steps, lr, C.byref(m)))
        return m.as_dict()

    def set_per_beta(self, beta: float):
        _lib.check(self.lib.b2g_bdq_set_per_beta(self.h, float(beta)))

    def last_per(self):
        """Slots, importance weights and new priorities (sum_d |TD_d| + eps) of the last sampled step.  The slots are valid
        with uniform replay too (the Philox draw of the step); weights and priorities only with prioritised replay."""
        B = self.batch_size
        idx, w, p = np.empty(B, np.int32), np.empty(B, np.float32), np.empty(B, np.float32)
        _lib.check(self.lib.b2g_bdq_get_last_per(self.h, idx.ctypes.data_as(C.POINTER(C.c_int32)), _fp(w), _fp(p)))
        return idx, w, p

    def step_explicit(self, obs, act_idx, rew, next_obs, done, weights=None, lr=1e-4, apply_update=True):
        B, D = self.batch_size, self.n_branches
        td = np.empty((B, D), np.float32)
        w = _fp(_f32(weights)) if weights is not None else None
        m = _lib.BdqMetrics()
        _lib.check(self.lib.b2g_bdq_step_explicit(self.h, _fp(_f32(obs)), _fp(_f32(act_idx)), _fp(_f32(np.reshape(rew, -1))),
                                                   _fp(_f32(next_obs)), _fp(_f32(np.reshape(done, -1))), w, lr, int(apply_update),
                                                   C.byref(m), _fp(td)))
        out = m.as_dict()
        out["td"] = td
        return out

    def act(self, obs):
        obs = _f32(obs).reshape(-1, self.obs_dim)
        out = np.empty((obs.shape[0], self.n_branches), np.int32)
        _lib.check(self.lib.b2g_bdq_act(self.h, _fp(obs), obs.shape[0], out.ctypes.data_as(C.POINTER(C.c_int32))))
        return out


class BDQ:
    """SB-shaped front end: ``BDQ(policy, env, policy_kwargs={'layers': [[64,64],[32],[32]]}, num_actions_pad=33, ...)``
    with ``learn / predict / save / load / get_parameters / load_parameters`` (sb_helper.py:202-226)."""

    def __init__(self, policy, env, gamma=0.99, learning_rate=1e-4, buffer_size=1000000, exploration_fraction=0.1,
                 exploration_final_eps=0.02, train_freq=1, batch_size=64, learning_starts=1000, target_network_update_freq=1000,
                 num_actions_pad=33, prioritized_replay=False, prioritized_replay_alpha=0.6, prioritized_replay_beta0=0.4,
                 prioritized_replay_beta_iters=None, prioritized_replay_eps=1e-6, epsilon_greedy=True, policy_kwargs=None, verbose=0,
                 tensorboard_log=None, seed=None, device=0, rank=0, nranks=1, nccl_id=None, _init_setup_model=True,
                 device_obs_norm=False, **_ignored):
        if device_obs_norm and nranks > 1:
            raise NotImplementedError("device_obs_norm=True keeps VecNormalize's obs_rms on one learner handle; with nranks > 1 every "
                                      "rank would own different statistics")
        # learn() stores raw transitions (stable-baselines' rule), feeds the actor, the statistics and the replay from one upload
        # per frame, and a VecNormalize with norm_obs hands its obs_rms to the device learner (BDQLearner.observe_act / _add)
        self.device_obs_norm = bool(device_obs_norm)
        self.prioritized_replay = bool(prioritized_replay)
        self.per_alpha, self.per_beta0, self.per_beta_iters, self.per_eps = prioritized_replay_alpha, prioritized_replay_beta0, \
            prioritized_replay_beta_iters, prioritized_replay_eps
        self._dp = dict(rank=rank, nranks=nranks, nccl_id=nccl_id)
        self.policy_kwargs = dict(policy_kwargs or {})
        self.layers = self.policy_kwargs.get("layers", [[64, 64], [32], [32]])
        self.gamma, self.learning_rate, self.buffer_size, self.batch_size = gamma, learning_rate, int(buffer_size), int(batch_size)
        self.exploration_fraction, self.exploration_final_eps = exploration_fraction, exploration_final_eps
        self.train_freq, self.learning_starts = train_freq, learning_starts
        self.target_network_update_freq, self.num_actions_pad = target_network_update_freq, int(num_actions_pad)
        self.verbose, self.seed, self.device = verbose, seed, device
        self.num_timesteps = 0
        self._rng = np.random.default_rng(seed)
        self.learner: Optional[BDQLearner] = None
        self.env = None
        self._vec_normalize_env = None
        if env is not None:
            self.env = env if hasattr(env, "num_envs") else DummyVecEnv([lambda: env])
            self.observation_space, self.action_space = self.env.observation_space, self.env.action_space
            self._vec_normalize_env = self.get_vec_normalize_env()
            if _init_setup_model:
                self.setup_model()

    def setup_model(self):
        obs_dim = int(np.prod(self.observation_space.shape))
        n_br = int(np.prod(self.action_space.shape))
        self.learner = BDQLearner(obs_dim, n_br, self.num_actions_pad, tuple(tuple(l) for l in self.layers), self.batch_size,
                                  self.buffer_size, self.gamma, self.target_network_update_freq, True, int(self.seed or 0), self.device,
                                  prioritized_replay=self.prioritized_replay, prioritized_replay_alpha=self.per_alpha,
                                  prioritized_replay_eps=self.per_eps, **self._dp)
        rng = np.random.default_rng(self.seed)
        p = OrderedDict()
        for n, shp in self.learner.param_shapes.items():
            if n == "bdq/eps":
                p[n] = np.float32(1.0)
            elif n.startswith("bdq/target_q_func/"):
                p[n] = p[n.replace("bdq/target_q_func/model", "bdq/model")].copy()
            elif len(shp) == 2:
                lim = np.sqrt(6.0 / (shp[0] + shp[1]))
                p[n] = rng.uniform(-lim, lim, shp).astype(np.float32)
            else:
                p[n] = np.zeros(shp, np.float32)
        self.learner.load_parameters(p)
        self.learner.obs_shape = tuple(self.observation_space.shape)
        self._bins = np.linspace(-1.0, 1.0, self.num_actions_pad).astype(np.float32)
        self._attach_device_norm()

    def close(self):
        """Releases the device learner.  Observation statistics it owned go back to the VecNormalize wrapper first."""
        if self.learner is not None:
            if self._owns_obs_rms():
                self._vec_normalize_env.take_obs_rms_back()
            self.learner.close()
            self.learner = None

    def _owns_obs_rms(self) -> bool:
        vn = self._vec_normalize_env
        return vn is not None and self.learner is not None and getattr(vn, "obs_rms_owner", None) is self.learner

    @property
    def predict_takes_raw_obs(self) -> bool:
        """True while a learner owns the statistics of this model's VecNormalize: that wrapper returns raw observations and
        ``predict`` normalises them on the device."""
        return bool(getattr(self._vec_normalize_env, "learner_owns_obs_rms", False))

    def _attach_device_norm(self):
        """device_obs_norm: the wrapper's obs_rms moves to this learner, unless another learner owns it already (a second
        model on the same env reads the owner's statistics and leaves them where they are)."""
        vn = self._vec_normalize_env
        if self.device_obs_norm and isinstance(vn, VecNormalize) and vn.norm_obs and not vn.learner_owns_obs_rms:
            vn.give_obs_rms_to(self.learner)
        if self._owns_obs_rms():
            self._sync_norm_stats()

    def _sync_norm_stats(self):
        """The owner's reward scalars and clips for the gather (the observation statistics are the learner's own)."""
        vn = self._vec_normalize_env
        self.learner.set_norm_stats(None, None, float(vn.ret_rms.var), vn.clip_obs, vn.clip_reward, vn.epsilon,
                                    norm_obs=vn.norm_obs, norm_reward=vn.norm_reward)

    def get_env(self):
        return self.env

    def _epsilon(self, t, total):
        frac = min(1.0, t / max(1.0, self.exploration_fraction * total))
        return 1.0 + frac * (self.exploration_final_eps - 1.0)

    def learn(self, total_timesteps, callback=None, log_interval=100, tb_log_name="BDQ", reset_num_timesteps=True):
        callback = as_callback(callback)
        callback.init_callback(self)
        callback.on_training_start({"self": self, "writer": None}, globals())
        dev = self.device_obs_norm
        vn = self._vec_normalize_env
        if dev:
            if not isinstance(vn, VecNormalize) or not vn.norm_obs:
                raise RuntimeError("device_obs_norm=True needs the env wrapped in a VecNormalize with norm_obs=True")
            if not self._owns_obs_rms():
                raise RuntimeError("learn: the env's VecNormalize statistics are owned by another model's learner (close that model, "
                                   "or build this one with device_obs_norm=True before it)")
        obs = self.env.reset()
        n_env, D = self.env.num_envs, self.learner.n_branches
        lr = self.learning_rate if not callable(self.learning_rate) else self.learning_rate(1.0)
        if dev:      # the reset frames: uploaded once, merged (VecNormalize.reset's update), staged as every env's current observation
            self.learner.observe_act(np.asarray(obs, np.float32), update_stats=vn.training, act=False)
        # reset_num_timesteps=False continues a run: epsilon and beta follow num_timesteps over the schedule of a run that ends
        # total_timesteps from now (the stable-baselines DQN rule)
        resume = not reset_num_timesteps
        horizon = self.num_timesteps + total_timesteps if resume else total_timesteps
        for t in range(0, total_timesteps, n_env):
            eps = self._epsilon(self.num_timesteps if resume else t, horizon)
            if dev:      # the staged frames, current statistics, epsilon-greedy on the device
                idx = self.learner.observe_act(None, n=n_env, eps=eps)
            else:
                idx = self.learner.act(np.asarray(obs, np.float32))
                explore = self._rng.random((n_env, D)) < eps                   # independent epsilon-greedy per branch
                idx = np.where(explore, self._rng.integers(0, self.num_actions_pad, (n_env, D)), idx)
            new_obs, rew, done, infos = self.env.step(self._bins[idx])
            self.num_timesteps += n_env
            if callback.on_step() is False:
                break
            nxt = np.array(new_obs, np.float32, copy=True)
            for i, info in enumerate(infos):
                if done[i] and isinstance(info, dict) and "terminal_observation" in info:
                    nxt[i] = np.asarray(info["terminal_observation"], np.float32).reshape(nxt[i].shape)
            if dev:      # raw transitions; next_obs crosses once, a finished env's reset frame is merged and staged
                self.learner.observe_add(idx.astype(np.float32), vn.get_original_reward(), nxt, np.asarray(done, np.float32),
                                         reset_obs=np.asarray(new_obs, np.float32) if np.any(done) else None,
                                         update_stats=vn.training)       # step_wait's update; a callback may switch it
            else:
                self.learner.replay_add(np.asarray(obs, np.float32), idx.astype(np.float32), rew, nxt, np.asarray(done, np.float32))
            obs = new_obs
            if self.num_timesteps > self.learning_starts and self.num_timesteps % self.train_freq == 0 and \
                    self.learner.replay_size() >= self.batch_size:
                if self.prioritized_replay:          # [SB2] LinearSchedule(beta_iters, initial_p=beta0, final_p=1.0)
                    iters = self.per_beta_iters or horizon
                    self.learner.set_per_beta(self.per_beta0 + min(1.0, self.num_timesteps / iters) * (1.0 - self.per_beta0))
                if dev:      # the sample is normalised with the statistics of this moment: obs_rms on the device, ret_rms here
                    self._sync_norm_stats()
                self.learner.step(1, lr)
        callback.on_training_end()
        return self

    def predict(self, observation, state=None, mask=None, deterministic=True):
        obs = np.asarray(observation, np.float32).reshape(-1, self.learner.obs_dim)
        idx = self.learner.act(obs)
        act = self._bins[idx]
        return (act[0] if np.ndim(observation) == 1 else act), None

    def get_parameters(self):
        return OrderedDict((n + ":0", a) for n, a in self.learner.get_parameters().items())

    def load_parameters(self, params, exact_match=True):
        if isinstance(params, str):
            _, params = sb_io.load_sb_zip(params)
        self.learner.load_parameters(params, exact_match=exact_match)

    def save(self, save_path, cloudpickle=False):
        d = os.path.dirname(save_path)
        if d:
            os.makedirs(d, exist_ok=True)
        data = {"gamma": self.gamma, "learning_rate": float(self.learning_rate), "batch_size": self.batch_size, "buffer_size": self.buffer_size,
                "exploration_fraction": self.exploration_fraction, "exploration_final_eps": self.exploration_final_eps,
                "train_freq": self.train_freq, "learning_starts": self.learning_starts, "num_actions_pad": self.num_actions_pad,
                "target_network_update_freq": self.target_network_update_freq, "prioritized_replay": self.prioritized_replay,
                "prioritized_replay_alpha": self.per_alpha, "prioritized_replay_beta0": self.per_beta0, "double_q": True,
                "epsilon_greedy": True, "policy_kwargs": {"layers": self.layers}}
        sb_io.save_sb_zip(save_path, data, self.learner.get_parameters())

    def get_vec_normalize_env(self):
        from .sac_model import unwrap_vec_normalize
        return unwrap_vec_normalize(self.env)

    # ------------------------------------------------------------------ training state (training_state.py)
    def _host_state(self):
        if callable(self.learning_rate):
            raise NotImplementedError("save_training_state needs a constant learning_rate")
        init = dict(gamma=self.gamma, learning_rate=self.learning_rate, buffer_size=self.buffer_size,
                    exploration_fraction=self.exploration_fraction, exploration_final_eps=self.exploration_final_eps,
                    train_freq=self.train_freq, batch_size=self.batch_size, learning_starts=self.learning_starts,
                    target_network_update_freq=self.target_network_update_freq, num_actions_pad=self.num_actions_pad,
                    prioritized_replay=self.prioritized_replay, prioritized_replay_alpha=self.per_alpha,
                    prioritized_replay_beta0=self.per_beta0, prioritized_replay_beta_iters=self.per_beta_iters,
                    prioritized_replay_eps=self.per_eps, policy_kwargs=self.policy_kwargs, verbose=self.verbose, seed=self.seed,
                    device=self.device)
        if self.device_obs_norm:
            init["device_obs_norm"] = True
        return {"algo": "BDQ", "init": init, "num_timesteps": int(self.num_timesteps), "rng": training_state.rng_state(self._rng)}

    def save_training_state(self, path):
        """Writes directory ``path``: model.zip, learner.state (parameters, Adam moments, counters, the replay and its
        priority trees), vecnormalize.pkl and host.json.  The previous contents stay loadable until the new one is complete."""
        return training_state.save_training_state(self, path)

    @classmethod
    def load_training_state(cls, path, env, **kwargs):
        """Rebuilds the model ``save_training_state`` wrote into ``path`` on ``env``; ``learn(n, reset_num_timesteps=False)``
        then continues with epsilon and beta taken from ``num_timesteps``."""
        path = training_state.resolve(path)
        host = training_state.read_host(path)
        if host.get("algo") != "BDQ":
            raise ValueError(f"{path} holds a {host.get('algo')} training state")
        model = cls("MlpActPolicy", env, **dict(host["init"], **kwargs))
        training_state.restore_vec_normalize(path, model.env)
        model._attach_device_norm()        # the restored statistics go back to the learner; learner.state carries the same ones
        model.load_parameters(os.path.join(path, training_state.MODEL_FILE))
        model.learner.load_state(os.path.join(path, training_state.STATE_FILE))
        model.num_timesteps = int(host["num_timesteps"])
        training_state.set_rng_state(model._rng, host["rng"])
        return model

    @classmethod
    def load(cls, load_path, env=None, **kwargs):
        from .spaces import Box
        if not os.path.exists(load_path) and os.path.exists(load_path + ".zip"):
            load_path += ".zip"
        data, params = sb_io.load_sb_zip(load_path)
        w0 = params["bdq/model/common_net/fully_connected/weights"]
        w1 = params["bdq/model/common_net/fully_connected_1/weights"]
        wb = params["bdq/model/action_value/fully_connected/weights"]
        wo = params["bdq/model/action_value/fully_connected_1/weights"]
        n_br = sum(1 for n in params if n.startswith("bdq/model/action_value/") and n.endswith("/weights")) // 2

        class _Spaces:
            num_envs = 1
            observation_space = Box(-np.inf, np.inf, (w0.shape[0],))
            action_space = Box(-1.0, 1.0, (n_br,))
        e = env if env is not None else _Spaces()
        kw = dict(gamma=data.get("gamma", 0.99), batch_size=data.get("batch_size", 64), num_actions_pad=wo.shape[1],
                  policy_kwargs={"layers": [[w0.shape[1], w1.shape[1]], [wb.shape[1]], [wb.shape[1]]]},
                  buffer_size=min(int(data.get("buffer_size", 1000)), 1000) if env is None else data.get("buffer_size", 100000))
        kw.update(kwargs)
        m = cls("MlpActPolicy", None, _init_setup_model=False, **kw)
        m.env = e if env is not None else None
        m._vec_normalize_env = m.get_vec_normalize_env() if env is not None else None
        m.observation_space, m.action_space = e.observation_space, e.action_space
        m.setup_model()
        m.learner.load_parameters(params, exact_match=True)
        return m
