"""``SAC`` -- the stable-baselines model object the reference constructs and drives
(/root/reference/manipulation_main/training/sb_helper.py:104-128,175,186-198,241-247;
train_stable_baselines.py:95-106; utils.py:71; base_callbacks.py:84-111,145-146), re-hosted on the
H100 learner.  Same constructor keywords, ``learn / predict / save / load / get_parameters /
load_parameters / get_env / get_vec_normalize_env``, same callback protocol, same zip format.

What runs where: env stepping (PyBullet) and this loop stay on host cores; replay storage,
minibatch sampling, VecNormalize-at-sample-time, the whole gradient step and the target update
run on the GPU behind the C ABI (include/b200grasp.h).  There is no CPU fallback.
"""
from __future__ import annotations

import time
from collections import OrderedDict, deque
from typing import Optional

import numpy as np

from . import _lib, sb_io, training_state
from .base_model import BaseModel, unwrap_vec_normalize  # noqa: F401  (unwrap_vec_normalize: also imported from here)
from .callbacks import as_callback
from .tensorboard import EpisodeRewardLogger
from .learner import Learner


class CnnPolicy:      # sentinels standing in for stable_baselines.sac.policies.{CnnPolicy,MlpPolicy}
    pass


class MlpPolicy:
    pass


_PRECISIONS = {"fp32": _lib.B2G_PREC_FP32_SIMT, "bf16x3": _lib.B2G_PREC_BF16X3, "bf16": _lib.B2G_PREC_BF16}
HEAD_WIDTHS = (64, 128, 192, 256)      # SAC.layers [H, H] the device learner builds (b2g_sac_cfg.hidden)


def head_width(layers) -> int:
    """policy_kwargs['layers'] -> the head width H; anything but two equal widths from HEAD_WIDTHS raises."""
    layers = [int(x) for x in layers]
    if len(layers) != 2 or layers[0] != layers[1] or layers[0] not in HEAD_WIDTHS:
        raise NotImplementedError(f"SAC.layers must be [H, H] with H in {list(HEAD_WIDTHS)} (got {layers})")
    return layers[0]


def extractor_of(cnn_extractor) -> str:
    """policy_kwargs['cnn_extractor'] -> the learner's extractor: stable-baselines' plain ``nature_cnn`` (the sentinel
    ``b200grasp.common.policies.nature_cnn``, or the string "nature_cnn" a training state stores); any other value means
    ``create_augmented_nature_cnn(1)``."""
    from .common.policies import nature_cnn
    return "nature_cnn" if cnn_extractor is nature_cnn or cnn_extractor == "nature_cnn" else "augmented"


def zip_extractor(params):
    """The CNN extractor a parameter dict was written by (conv1's variable name), or None for an MLP policy."""
    names = {n[:-2] if n.endswith(":0") else n for n in params}
    if "model/pi/c1/w" in names:
        return "nature_cnn"
    return "augmented" if "model/pi/cnn1/w" in names else None


def _constfn(v):
    return v if callable(v) else (lambda _frac: float(v))


class SAC(BaseModel):
    _algo = "SAC"

    def __init__(self, policy, env, gamma=0.99, learning_rate=3e-4, buffer_size=50000, learning_starts=100, train_freq=1,
                 batch_size=64, tau=0.005, ent_coef="auto", target_update_interval=1, gradient_steps=1,
                 target_entropy="auto", action_noise=None, random_exploration=0.0, verbose=0, tensorboard_log=None,
                 _init_setup_model=True, policy_kwargs=None, full_tensorboard_log=False, seed=None, n_cpu_tf_sess=None,
                 precision="bf16x3", device=0, rank=0, nranks=1, nccl_id=None, replay_frames=None, replay_u8_planes=(),
                 device_obs_norm=False):
        if device_obs_norm and nranks > 1:
            raise NotImplementedError("device_obs_norm=True keeps VecNormalize's obs_rms on one learner handle; with nranks > 1 every "
                                      "rank would own different statistics")
        if ent_coef != "auto":
            raise NotImplementedError("only ent_coef='auto' (every shipped zip; SURVEY.md section 8c) is built")
        if target_update_interval != 1:
            raise NotImplementedError("target_update_interval must be 1 (every shipped zip)")
        if action_noise is not None:
            raise NotImplementedError("action_noise is not used by the reference (zip: action_noise None)")
        if getattr(policy, "unsupported", None):
            raise NotImplementedError(policy.unsupported)
        self.policy = policy
        self.policy_kwargs = dict(policy_kwargs or {})
        self.hidden = head_width(self.policy_kwargs.get("layers", [64, 64]))
        if self.policy_kwargs.get("layer_norm", False):
            raise NotImplementedError("layer_norm=True is not used by the reference (sb_helper.py:95)")
        self.gamma, self.tau = float(gamma), float(tau)
        self.learning_rate = learning_rate
        self.buffer_size, self.batch_size = int(buffer_size), int(batch_size)
        self.learning_starts, self.train_freq, self.gradient_steps = int(learning_starts), int(train_freq), int(gradient_steps)
        self.random_exploration = float(random_exploration)
        self.verbose, self.tensorboard_log, self.seed = verbose, tensorboard_log, seed
        self.ent_coef, self.target_entropy = ent_coef, target_entropy
        self.precision = precision
        # replay storage (Learner: frame_capacity, u8_planes); None / () = two fp32 frames per replay slot
        self.replay_frames = None if replay_frames is None else int(replay_frames)
        self.replay_u8_planes = tuple(int(c) for c in replay_u8_planes)
        # learn() feeds the actor, the statistics and the replay from one upload per frame, and a VecNormalize with norm_obs
        # hands its obs_rms to the device learner (Learner.observe_act / observe_add)
        self.device_obs_norm = bool(device_obs_norm)
        self._dev = dict(device=device, rank=rank, nranks=nranks, nccl_id=nccl_id)
        self._layout_from_zip = False
        self.extractor = extractor_of(self.policy_kwargs.get("cnn_extractor"))
        self.num_timesteps, self.n_updates = 0, 0
        self.episode_rewards = [0.0]
        self.ep_info_buf = deque(maxlen=100)
        self.learner: Optional[Learner] = None
        self._rng = np.random.default_rng(seed)
        if env is not None:
            self.set_env(env)
            if _init_setup_model:
                self.setup_model()

    # ------------------------------------------------------------------ env plumbing
    def set_env(self, env):
        self._set_env(env)
        if self.learner is not None:
            self._attach_device_norm()
            self._attach_obs_encoder()
            self._sync_norm_stats()

    def setup_model(self):
        obs_shape = tuple(self.observation_space.shape)
        n_act = int(np.prod(self.action_space.shape))
        if len(obs_shape) == 3 and "cnn_extractor" not in self.policy_kwargs and not self._layout_from_zip:
            # sb_helper.py:93-95: CnnPolicy with policy_kwargs={} means stable-baselines' plain nature_cnn over ALL planes and
            # no direct feature -- a different network (and different zip variables) from augmented_nature_cnn.  The
            # extractor is asked for by name instead of by omission.  (SAC.load knows the layout from the zip itself.)
            raise NotImplementedError("CnnPolicy without policy_kwargs['cnn_extractor'] selects stable-baselines' plain nature_cnn "
                                      "(simplified + depth branch, sb_helper.py:93-95); pass cnn_extractor=nature_cnn "
                                      "(b200grasp.common.policies) for that network, or "
                                      "cnn_extractor=create_augmented_nature_cnn(1) as sb_helper.py:88-91 does")
        tgt = -float(n_act) if self.target_entropy == "auto" else float(self.target_entropy)
        self.learner = Learner(obs_shape, n_act=n_act, hidden=self.hidden, batch_size=self.batch_size, buffer_size=self.buffer_size,
                               gamma=self.gamma, tau=self.tau, target_entropy=tgt, seed=int(self.seed or 0),
                               precision=_PRECISIONS[self.precision], frame_capacity=self.replay_frames,
                               u8_planes=self.replay_u8_planes, **self._net_kwargs(obs_shape), **self._dev)
        self._init_parameters()
        self._attach_device_norm()
        self._attach_obs_encoder()
        self._sync_norm_stats()

    def _net_kwargs(self, obs_shape):
        """Learner's extractor argument: only the plain nature_cnn departs from the default."""
        return {"extractor": "nature_cnn"} if len(obs_shape) == 3 and self.extractor == "nature_cnn" else {}

    def _init_parameters(self):
        """[SB2] ortho_init(sqrt 2) for conv/linear, Glorot-uniform for tf.layers.dense, zero biases,
        log_ent_coef = 0, target = copy of values_fn."""
        rng = np.random.default_rng(self.seed)
        p = OrderedDict()
        for name, shape in self.learner.param_shapes.items():
            if name.startswith("target/"):
                p[name] = p["model/" + name[len("target/"):]].copy()
            elif name.endswith("/w"):
                flat = (int(np.prod(shape[:-1])), shape[-1])
                u, _, v = np.linalg.svd(rng.standard_normal(flat), full_matrices=False)
                q = u if u.shape == flat else v
                p[name] = (np.sqrt(2.0) * q.reshape(shape)).astype(np.float32)
            elif name.endswith("/kernel"):
                lim = np.sqrt(6.0 / (shape[0] + shape[1]))
                p[name] = rng.uniform(-lim, lim, size=shape).astype(np.float32)
            else:
                p[name] = np.zeros(shape, np.float32)
        self.learner.load_parameters(p)

    def load_parameters(self, load_path_or_dict, exact_match=True):
        """A donor of the other CNN extractor is refused before any variable is written (its head fc0 kernels differ in
        shape, so even exact_match=False would leave the learner half loaded)."""
        params = load_path_or_dict
        if isinstance(params, str):
            _, params = sb_io.load_sb_zip(params)
        theirs = zip_extractor(params)
        if len(self.observation_space.shape) == 3 and theirs is not None and theirs != self.extractor:
            raise ValueError(f"the parameters belong to the {theirs} extractor; this model's CNN policy is {self.extractor}")
        super().load_parameters(params, exact_match=exact_match)

    def _sync_norm_stats(self):
        vn = self._vec_normalize_env
        if vn is None:
            self.learner.set_norm_stats(norm_obs=False, norm_reward=False)
        elif self._owns_obs_rms():            # the scalars only: the statistics are this learner's own
            self.learner.set_norm_stats(None, None, float(vn.ret_rms.var), vn.clip_obs, vn.clip_reward, vn.epsilon,
                                        norm_obs=vn.norm_obs, norm_reward=vn.norm_reward)
        else:
            self.learner.set_norm_stats(vn.obs_rms.mean, vn.obs_rms.var, float(vn.ret_rms.var), vn.clip_obs, vn.clip_reward,
                                        vn.epsilon, norm_obs=vn.norm_obs, norm_reward=vn.norm_reward)

    # ------------------------------------------------------------------ action scaling ([SB2] common/math_util.py)
    def _scale_action(self, a):
        low, high = self.action_space.low, self.action_space.high
        return 2.0 * ((a - low) / (high - low)) - 1.0

    def _unscale_action(self, a):
        low, high = self.action_space.low, self.action_space.high
        return low + 0.5 * (a + 1.0) * (high - low)

    # ------------------------------------------------------------------ learn
    _step_tags = {t: t for t in ("policy_loss", "qf1_loss", "qf2_loss", "value_loss", "entropy", "ent_coef_loss", "ent_coef",
                                 "learning_rate")}

    def learn(self, total_timesteps, callback=None, log_interval=4, tb_log_name="SAC", reset_num_timesteps=True,
              replay_wrapper=None):
        """[SB2] SAC.learn: one env step then (every train_freq steps) gradient_steps minibatch updates.  With tensorboard_log
        every gradient step's losses are written from the device metrics ring (tensorboard.py)."""
        return self._learn_logged(tb_log_name, reset_num_timesteps,
                                  lambda writer, steps: self._learn(total_timesteps, callback, log_interval, reset_num_timesteps,
                                                                    writer, steps))

    def _learn(self, total_timesteps, callback, log_interval, reset_num_timesteps, writer, steps):
        if reset_num_timesteps:
            self.num_timesteps = 0
        callback = as_callback(callback)
        callback.init_callback(self)
        lr_fn = _constfn(self.learning_rate)
        vn = self._vec_normalize_env
        n_env = self.n_envs
        obs = self.env.reset()
        obs_ = vn.get_original_obs() if vn is not None else obs          # un-normalised copy stored in the replay
        dev = self.device_obs_norm
        owned = dev and self._owns_obs_rms()
        if getattr(vn, "learner_owns_obs_rms", False) and not owned:
            raise RuntimeError("learn: the env's VecNormalize statistics are owned by another model's learner (close that model, "
                               "or build this one with device_obs_norm=True before it)")
        if dev:      # the reset frames: uploaded once, merged (VecNormalize.reset's update), staged as every env's current observation
            self.learner.observe_act(np.asarray(obs_, np.float32), update_stats=owned and vn.training, act=False)
        ep_rew = np.zeros(n_env)
        infos_values = {}
        t_start = time.time()
        ep_log = EpisodeRewardLogger(n_env) if writer is not None else None
        self._locals = {"self": self, "writer": writer, "total_timesteps": total_timesteps}
        callback.on_training_start(self._locals, globals())
        callback.on_rollout_start()
        step = 0
        while step < total_timesteps:
            if self.num_timesteps < self.learning_starts or self._rng.random() < self.random_exploration:
                unscaled = np.stack([np.asarray(self.action_space.sample()) for _ in range(n_env)])
                action = self._scale_action(unscaled)
            elif dev:
                action = self.learner.observe_act(None, n=n_env, deterministic=False)      # the staged frames, current statistics
                unscaled = self._unscale_action(action)
            else:
                src = obs_ if vn is not None else obs        # the device normalises raw obs with the same statistics
                if vn is not None:
                    self._sync_norm_stats()                  # act on the wrapper's CURRENT statistics, like SB does
                action = self.learner.act(np.asarray(src, np.float32), deterministic=False)
                unscaled = self._unscale_action(action)
            new_obs, reward, done, infos = self.env.step(unscaled)
            self.num_timesteps += n_env
            step += n_env
            if callback.on_step() is False:
                break
            new_obs_ = vn.get_original_obs() if vn is not None else new_obs
            reward_ = vn.get_original_reward() if vn is not None else reward
            # DummyVecEnv auto-resets: the transition's next_obs is the terminal observation
            nxt = np.array(new_obs_, np.float32, copy=True)
            for i, info in enumerate(infos):
                if done[i] and isinstance(info, dict) and "terminal_observation" in info:
                    nxt[i] = info["terminal_observation"]
            if dev:      # next_obs crosses once; a finished env's reset frame is merged and staged, its terminal frame stored
                self.learner.observe_add(np.asarray(action, np.float32), np.asarray(reward_, np.float32), nxt, np.asarray(done, np.float32),
                                         reset_obs=np.asarray(new_obs_, np.float32) if np.any(done) else None,
                                         update_stats=owned and vn.training)      # step_wait's update; a callback may switch it
            else:
                self.learner.replay_add(np.asarray(obs_, np.float32), np.asarray(action, np.float32), np.asarray(reward_, np.float32),
                                        nxt, np.asarray(done, np.float32))
            obs, obs_ = new_obs, new_obs_
            ep_rew += np.asarray(reward_, np.float64).reshape(-1)
            if ep_log is not None:
                ep_log(writer, reward_, done, self.num_timesteps)
            for i in range(n_env):
                if done[i]:
                    self.episode_rewards.append(float(ep_rew[i]))
                    self.ep_info_buf.append({"r": float(ep_rew[i])})
                    ep_rew[i] = 0.0
            if (self.num_timesteps // n_env) % self.train_freq == 0:
                callback.on_rollout_end()
                if self.learner.replay_size() >= self.batch_size and self.num_timesteps >= self.learning_starts:
                    if vn is not None:
                        self._sync_norm_stats()              # statistics current at sample time ([SB2] ReplayBuffer.sample(env=))
                    frac = 1.0 - step / total_timesteps
                    lr = float(lr_fn(frac))
                    # enqueue only: the gradient step runs on the device while the host goes on to the next env.step(); the losses
                    # (SB's infos_values, used for logging alone) are read back when something is actually logged
                    self.learner.step_async(self.gradient_steps, lr)
                    self.n_updates += self.gradient_steps
                    self._last_lr = lr
                    if steps is not None:
                        steps.queued(self.gradient_steps, self.num_timesteps)
                callback.on_rollout_start()
            if self.verbose >= 1 and done.any() and log_interval and len(self.episode_rewards) % log_interval == 0:
                fps = int(step / max(1e-9, time.time() - t_start))
                if steps is not None:
                    steps.drain()
                if self.n_updates:
                    infos_values = self.learner.step(0, getattr(self, "_last_lr", 3e-4))       # 0 steps: just fetch the latest losses
                print({"episodes": len(self.episode_rewards), "mean 100 episode reward": round(float(np.mean(self.episode_rewards[-101:-1] or [0])), 1),
                       "n_updates": self.n_updates, "fps": fps, "total timesteps": self.num_timesteps,
                       **{k: infos_values.get(k) for k in ("policy_loss", "qf1_loss", "qf2_loss", "value_loss", "entropy", "ent_coef")}})
        callback.on_training_end()
        return self

    # ------------------------------------------------------------------ predict ([SB2] SAC.predict)
    def predict(self, observation, state=None, mask=None, deterministic=True):
        observation = np.asarray(observation, np.float32)
        self._check_encoded(observation)
        single = observation.shape == tuple(self.observation_space.shape)
        obs = observation.reshape((-1,) + tuple(self.observation_space.shape))
        vn = self._vec_normalize_env
        if vn is not None and vn.norm_obs:
            # ``predict`` receives observations ALREADY normalised by the VecNormalize wrapper (utils.py:71 feeds
            # task.reset()/step() outputs); the device normalises raw ones, so undo the wrapper's transform.  A wrapper whose
            # obs_rms a learner owns returns RAW observations: nothing to undo.  (Observations an evaluation wrapper
            # normalised belong to the model built on that wrapper, or are passed through its ``get_original_obs``.)
            if not self.predict_takes_raw_obs:
                obs = obs * np.sqrt(vn.obs_rms.var + vn.epsilon) + vn.obs_rms.mean
            self._sync_norm_stats()
        act = self.learner.act(obs.astype(np.float32), deterministic=deterministic)
        act = self._unscale_action(act.reshape((-1,) + tuple(self.action_space.shape)))
        return (act[0] if single else act), None

    # ------------------------------------------------------------------ persistence
    def _data(self):
        return {
            "gamma": self.gamma, "learning_rate": self.learning_rate if not callable(self.learning_rate) else float(self.learning_rate(1.0)),
            "buffer_size": self.buffer_size, "learning_starts": self.learning_starts, "train_freq": self.train_freq,
            "batch_size": self.batch_size, "tau": self.tau, "ent_coef": self.ent_coef,
            "target_entropy": self.target_entropy if isinstance(self.target_entropy, str) else float(self.target_entropy),
            "verbose": self.verbose, "n_envs": getattr(self, "n_envs", 1), "seed": self.seed, "action_noise": None,
            "random_exploration": self.random_exploration, "_vectorize_action": True, "n_cpu_tf_sess": None,
            "policy": "CnnPolicy" if len(self.observation_space.shape) == 3 else "MlpPolicy",
            "policy_kwargs": {k: v for k, v in self.policy_kwargs.items() if k != "cnn_extractor"},
            "observation_space": {"shape": list(self.observation_space.shape), "low": float(np.min(self.observation_space.low)),
                                  "high": float(np.max(self.observation_space.high))},
            "action_space": {"shape": list(self.action_space.shape), "low": [float(x) for x in np.ravel(self.action_space.low)],
                             "high": [float(x) for x in np.ravel(self.action_space.high)]},
            "b200grasp": {"precision": self.precision, "n_updates": self.n_updates, "replay_frames": self.replay_frames,
                          "replay_u8_planes": list(self.replay_u8_planes), "device_obs_norm": self.device_obs_norm},
        }

    # ------------------------------------------------------------------ training state (training_state.py)
    def _host_state(self):
        kw = self.policy_kwargs.get("cnn_extractor")
        policy_kwargs = dict(self.policy_kwargs)
        if kw is not None and not isinstance(kw, str):         # the extractor by name (the learner builds these two)
            policy_kwargs["cnn_extractor"] = "nature_cnn" if self.extractor == "nature_cnn" else "augmented_nature_cnn"
        if callable(self.learning_rate):
            raise NotImplementedError("save_training_state needs a constant learning_rate")
        init = dict(gamma=self.gamma, learning_rate=self.learning_rate, buffer_size=self.buffer_size, learning_starts=self.learning_starts,
                    train_freq=self.train_freq, batch_size=self.batch_size, tau=self.tau, ent_coef=self.ent_coef,
                    gradient_steps=self.gradient_steps, target_entropy=self.target_entropy, random_exploration=self.random_exploration,
                    verbose=self.verbose, seed=self.seed, policy_kwargs=policy_kwargs, precision=self.precision,
                    replay_frames=self.replay_frames, replay_u8_planes=list(self.replay_u8_planes))
        if self.device_obs_norm:
            init["device_obs_norm"] = True
        host = {"algo": "SAC", "policy": "CnnPolicy" if len(self.observation_space.shape) == 3 else "MlpPolicy", "init": init,
                "num_timesteps": int(self.num_timesteps), "n_updates": int(self.n_updates),
                "episode_rewards": [float(r) for r in self.episode_rewards], "ep_info_buf": list(self.ep_info_buf),
                "rng": training_state.rng_state(self._rng)}
        enc = self._encoder_host()
        if enc is not None:
            host["obs_encoder"] = enc
        return host

    @classmethod
    def _policy_from_host(cls, host):
        return {"CnnPolicy": CnnPolicy, "MlpPolicy": MlpPolicy}[host["policy"]]

    def _restore_host_state(self, host):
        self._sync_norm_stats()
        self.num_timesteps, self.n_updates = int(host["num_timesteps"]), int(host["n_updates"])
        self.episode_rewards = [float(r) for r in host["episode_rewards"]]
        self.ep_info_buf = deque(host["ep_info_buf"], maxlen=100)
        training_state.set_rng_state(self._rng, host["rng"])

    @classmethod
    def load(cls, load_path, env=None, custom_objects=None, **kwargs):
        """Reads zips written by this class or by stable-baselines 2.10 (e.g.
        trained_models/SAC_depth_1mbuffer/best_model/best_model.zip)."""
        from .spaces import Box
        data, params = cls._read_zip(load_path)
        extractor = zip_extractor(params)
        if extractor == "nature_cnn":         # nature_cnn's conv1 reads every plane
            obs_space = Box(0.0, 255.0, (64, 64, params["model/pi/c1/w"].shape[2]))
        elif extractor == "augmented":
            obs_space = Box(0.0, 255.0, (64, 64, params["model/pi/cnn1/w"].shape[2] + 1))
        else:
            obs_space = Box(-np.inf, np.inf, (params["model/pi/fc0/kernel"].shape[0],))
        kw = {}
        for k in ("gamma", "buffer_size", "learning_starts", "train_freq", "batch_size", "tau"):
            if isinstance(data.get(k), (int, float)):
                kw[k] = data[k]
        if isinstance(data.get("learning_rate"), (int, float)):
            kw["learning_rate"] = data["learning_rate"]
        # The zip's buffer_size (1e6 in every shipped model) is the TRAINING ring: 2 * 1e6 * (H*W*Ci + 4) * 4 B = 32.8 GB for
        # depth, 131 GB for RGB-D.  A loaded model is used for inference or as a parameter donor (sb_helper.py:113-115 builds
        # a second model just to call get_parameters), so it gets a small ring unless the caller asks for one explicitly.
        kw["buffer_size"] = min(int(kw.get("buffer_size", 1000)), 1000)
        if (data.get("b200grasp") or {}).get("device_obs_norm"):
            kw["device_obs_norm"] = True
        kw.update(kwargs)
        # the head widths are the zip's own: the actor's fc0 / fc1 kernels give [H1, H2], and SAC's constructor refuses any
        # layers the learner cannot build (unequal widths included) with the message that names the supported ones
        # (nature_cnn's actor names its second layer fc1_1: learner.py, INTEGRATION.md)
        fc1 = "model/pi/fc1_1/kernel" if extractor == "nature_cnn" else "model/pi/fc1/kernel"
        layers = [int(params["model/pi/fc0/kernel"].shape[1]), int(params[fc1].shape[1])]
        if "model/pi/fc2/kernel" in params:
            layers.append(int(params["model/pi/fc2/kernel"].shape[1]))
        pkw = {"layers": layers}
        if extractor == "nature_cnn":
            pkw["cnn_extractor"] = "nature_cnn"
        model = cls(policy=data.get("policy", "CnnPolicy"), env=None, _init_setup_model=False, policy_kwargs=pkw, **kw)
        model._layout_from_zip = True
        return model._finish_load(env, obs_space, Box(-1.0, 1.0, (params["model/pi/dense/kernel"].shape[1],)), params)
