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
from collections import OrderedDict
from typing import Optional

import numpy as np

from . import _lib, training_state
from .base_model import BaseModel
from .callbacks import as_callback
from .tensorboard import EpisodeRewardLogger
from .learner import TransitionReplayLearner, _f32, _fp, nccl_config
from .vec_env import VecNormalize


class BDQLearner(TransitionReplayLearner):
    """numpy-facing wrapper of one ``b2g_bdq`` handle (maps 1:1 onto the C ABI)."""
    _abi = "bdq"

    def __init__(self, obs_dim=100, n_branches=3, n_bins=8, layers=((64, 64), (32,), (32,)), batch_size=64, buffer_size=100000,
                 gamma=0.99, target_network_update_freq=1000, trunk_grad_rescale=True, seed=0, device=0, rank=0, nranks=1, nccl_id=None,
                 prioritized_replay=False, prioritized_replay_alpha=0.6, prioritized_replay_eps=1e-6, frame_capacity=None):
        """frame_capacity: the replay holds that many observation frames and a slot refers to its obs / next_obs frames
        (include/b200grasp.h: b2g_bdq_create2); None = two fp32 rows per slot."""
        self.lib = _lib.load()
        if layers[1][0] != layers[2][0]:
            raise NotImplementedError("branch and state-value hidden widths must match (every shipped zip / config)")
        self._id_buf, idp, libp = nccl_config(nranks, nccl_id)
        cfg = _lib.BdqCfg(obs_dim, n_branches, n_bins, layers[0][0], layers[0][1], layers[1][0], batch_size, buffer_size, gamma,
                          target_network_update_freq, int(trunk_grad_rescale), seed, device, rank, nranks, idp, libp,
                          int(bool(prioritized_replay)), float(prioritized_replay_alpha), float(prioritized_replay_eps))
        self.prioritized_replay = bool(prioritized_replay)
        self.frame_capacity = None if frame_capacity is None else int(frame_capacity)
        self._create(cfg, self._replay_cfg(self.frame_capacity))
        self.obs_dim = self.obs_elems = obs_dim
        self.n_branches, self.n_bins, self.batch_size = n_branches, n_bins, batch_size
        self._act_width = n_branches
        self.obs_shape = (obs_dim,)          # shape of obs_rms_get's arrays (BDQ sets the env's observation shape)

    def _has_grad(self, name):
        return name.startswith("bdq/model/")

    def replay_add(self, obs, act_idx, rew, next_obs, done):
        obs, next_obs, act = _f32(obs), _f32(next_obs), _f32(act_idx)
        rew, done = _f32(np.reshape(rew, -1)), _f32(np.reshape(done, -1))
        _lib.check(self.lib.b2g_bdq_replay_add(self.h, _fp(obs), _fp(act), _fp(rew), _fp(next_obs), _fp(done), rew.shape[0]))

    def replay_size(self):
        return int(self.lib.b2g_bdq_replay_size(self.h))

    # ---- the actor loop on one upload per frame (include/b200grasp.h: b2g_bdq_observe_*)
    def observe_act(self, obs, n=None, update_stats=True, eps=0.0, act=True):
        """``obs``: n raw observations to upload, merge into ``obs_rms`` (``update_stats``) and stage as the current
        observation of env i; ``None`` acts on the ones already staged.  Returns the [n, n_branches] epsilon-greedy bin
        indices, or None with ``act=False``."""
        if obs is not None:
            obs = _f32(obs).reshape(-1, self.frame_elems)
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
        assert next_obs.size == n * self.frame_elems and act.size == n * self.n_branches and done.size == n
        if reset_obs is not None:
            reset_obs = _f32(reset_obs)
            assert reset_obs.size == next_obs.size
        _lib.check(self.lib.b2g_bdq_observe_add(self.h, _fp(act), _fp(rew), _fp(next_obs), _fp(done),
                                                None if reset_obs is None else _fp(reset_obs), n, int(bool(update_stats))))
        self.obs_rms_version += bool(update_stats)

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


class BDQ(BaseModel):
    """SB-shaped front end: ``BDQ(policy, env, policy_kwargs={'layers': [[64,64],[32],[32]]}, num_actions_pad=33, ...)``
    with ``learn / predict / save / load / get_parameters / load_parameters`` (sb_helper.py:202-226)."""
    _algo, _policy = "BDQ", "MlpActPolicy"

    def __init__(self, policy, env, gamma=0.99, learning_rate=1e-4, buffer_size=1000000, exploration_fraction=0.1,
                 exploration_final_eps=0.02, train_freq=1, batch_size=64, learning_starts=1000, target_network_update_freq=1000,
                 num_actions_pad=33, prioritized_replay=False, prioritized_replay_alpha=0.6, prioritized_replay_beta0=0.4,
                 prioritized_replay_beta_iters=None, prioritized_replay_eps=1e-6, epsilon_greedy=True, policy_kwargs=None, verbose=0,
                 tensorboard_log=None, seed=None, device=0, rank=0, nranks=1, nccl_id=None, _init_setup_model=True,
                 device_obs_norm=False, replay_frames=None, **_ignored):
        if replay_frames is not None and nranks > 1:
            raise NotImplementedError("replay_frames with nranks > 1: the frame pool is built for one learner handle")
        if device_obs_norm and nranks > 1:
            raise NotImplementedError("device_obs_norm=True keeps VecNormalize's obs_rms on one learner handle; with nranks > 1 every "
                                      "rank would own different statistics")
        # learn() stores raw transitions (stable-baselines' rule), feeds the actor, the statistics and the replay from one upload
        # per frame, and a VecNormalize with norm_obs hands its obs_rms to the device learner (BDQLearner.observe_act / _add)
        self.device_obs_norm = bool(device_obs_norm)
        # replay storage: F observation frames, slot s referring to its obs / next_obs frames (BDQLearner: frame_capacity);
        # None = two fp32 rows per slot
        self.replay_frames = None if replay_frames is None else int(replay_frames)
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
        self.tensorboard_log = tensorboard_log
        self.num_timesteps = 0
        self._rng = np.random.default_rng(seed)
        self.learner: Optional[BDQLearner] = None
        if env is not None:
            self._set_env(env)
            if _init_setup_model:
                self.setup_model()

    def setup_model(self):
        obs_dim = int(np.prod(self.observation_space.shape))
        n_br = int(np.prod(self.action_space.shape))
        self.learner = BDQLearner(obs_dim, n_br, self.num_actions_pad, tuple(tuple(l) for l in self.layers), self.batch_size,
                                  self.buffer_size, self.gamma, self.target_network_update_freq, True, int(self.seed or 0), self.device,
                                  prioritized_replay=self.prioritized_replay, prioritized_replay_alpha=self.per_alpha,
                                  prioritized_replay_eps=self.per_eps, **self._dp, **self._replay_kwargs())
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
        self._attach_obs_encoder()

    def _attach_device_norm(self):
        super()._attach_device_norm()
        if self._owns_obs_rms():
            self._sync_norm_stats()

    def _sync_norm_stats(self):
        """The owner's reward scalars and clips for the gather (the observation statistics are the learner's own)."""
        vn = self._vec_normalize_env
        self.learner.set_norm_stats(None, None, float(vn.ret_rms.var), vn.clip_obs, vn.clip_reward, vn.epsilon,
                                    norm_obs=vn.norm_obs, norm_reward=vn.norm_reward)

    def _epsilon(self, t, total):
        frac = min(1.0, t / max(1.0, self.exploration_fraction * total))
        return 1.0 + frac * (self.exploration_final_eps - 1.0)

    _step_tags = {"loss": "loss", "mean_q": "mean_q", "grad_norm": "grad_norm", "learning_rate": "learning_rate"}

    def learn(self, total_timesteps, callback=None, log_interval=100, tb_log_name="BDQ", reset_num_timesteps=True):
        """With tensorboard_log every gradient step's losses are written from the device metrics ring (tensorboard.py)."""
        return self._learn_logged(tb_log_name, reset_num_timesteps,
                                  lambda writer, steps: self._learn(total_timesteps, callback, reset_num_timesteps, writer, steps))

    def _learn(self, total_timesteps, callback, reset_num_timesteps, writer, steps):
        callback = as_callback(callback)
        callback.init_callback(self)
        callback.on_training_start({"self": self, "writer": writer}, globals())
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
        ep_log = EpisodeRewardLogger(n_env) if writer is not None else None
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
            if ep_log is not None:
                ep_log(writer, vn.get_original_reward() if vn is not None else rew, done, self.num_timesteps)
            if self.num_timesteps > self.learning_starts and self.num_timesteps % self.train_freq == 0 and \
                    self.learner.replay_size() >= self.batch_size:
                if self.prioritized_replay:          # [SB2] LinearSchedule(beta_iters, initial_p=beta0, final_p=1.0)
                    iters = self.per_beta_iters or horizon
                    self.learner.set_per_beta(self.per_beta0 + min(1.0, self.num_timesteps / iters) * (1.0 - self.per_beta0))
                if dev:      # the sample is normalised with the statistics of this moment: obs_rms on the device, ret_rms here
                    self._sync_norm_stats()
                self.learner.step(1, lr)
                if steps is not None:
                    steps.queued(1, self.num_timesteps)
        callback.on_training_end()
        return self

    def predict(self, observation, state=None, mask=None, deterministic=True):
        self._check_encoded(observation)
        obs = np.asarray(observation, np.float32).reshape(-1, self.learner.obs_dim)
        idx = self.learner.act(obs)
        act = self._bins[idx]
        return (act[0] if np.ndim(observation) == 1 else act), None

    def _data(self):
        return {"gamma": self.gamma, "learning_rate": float(self.learning_rate), "batch_size": self.batch_size, "buffer_size": self.buffer_size,
                "exploration_fraction": self.exploration_fraction, "exploration_final_eps": self.exploration_final_eps,
                "train_freq": self.train_freq, "learning_starts": self.learning_starts, "num_actions_pad": self.num_actions_pad,
                "target_network_update_freq": self.target_network_update_freq, "prioritized_replay": self.prioritized_replay,
                "prioritized_replay_alpha": self.per_alpha, "prioritized_replay_beta0": self.per_beta0, "double_q": True,
                "epsilon_greedy": True, "policy_kwargs": {"layers": self.layers}}

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
        if self.replay_frames is not None:
            init["replay_frames"] = self.replay_frames
        host = {"algo": "BDQ", "init": init, "num_timesteps": int(self.num_timesteps), "rng": training_state.rng_state(self._rng)}
        enc = self._encoder_host()
        if enc is not None:
            host["obs_encoder"] = enc
        return host

    def _restore_host_state(self, host):
        self.num_timesteps = int(host["num_timesteps"])
        training_state.set_rng_state(self._rng, host["rng"])

    @classmethod
    def load(cls, load_path, env=None, **kwargs):
        from .spaces import Box
        data, params = cls._read_zip(load_path)
        w0 = params["bdq/model/common_net/fully_connected/weights"]
        w1 = params["bdq/model/common_net/fully_connected_1/weights"]
        wb = params["bdq/model/action_value/fully_connected/weights"]
        wo = params["bdq/model/action_value/fully_connected_1/weights"]
        n_br = sum(1 for n in params if n.startswith("bdq/model/action_value/") and n.endswith("/weights")) // 2
        kw = dict(gamma=data.get("gamma", 0.99), batch_size=data.get("batch_size", 64), num_actions_pad=wo.shape[1],
                  policy_kwargs={"layers": [[w0.shape[1], w1.shape[1]], [wb.shape[1]], [wb.shape[1]]]},
                  buffer_size=min(int(data.get("buffer_size", 1000)), 1000) if env is None else data.get("buffer_size", 100000))
        kw.update(kwargs)
        m = cls("MlpActPolicy", None, _init_setup_model=False, **kw)
        return m._finish_load(env, Box(-np.inf, np.inf, (w0.shape[0],)), Box(-1.0, 1.0, (n_br,)), params)
