"""What the PPO2 (ppo2.py) and TRPO (trpo_mpi.py) front ends share: ``common.policies.MlpPolicy``'s checks and initialisation,
the wrapper base of their handles (csrc/actor_critic.cuh) and ``ActorCriticModel``: ``predict``, the Box check, the rollout
loop of ``learn``, ``load`` and the numpy generator of the training state.  Each algorithm keeps its own ``learn`` outer loop,
hyper-parameters and ``_data``.
"""
from __future__ import annotations

import ctypes as C
from collections import OrderedDict

import numpy as np

from . import _lib
from .base_model import BaseModel, unwrap_vec_normalize
from .callbacks import as_callback
from .learner import HandleLearner, _f32, _fp
from .tensorboard import EpisodeRewardLogger, Summary
from .vec_env import VecNormalize


def check_policy(policy, algo):
    from .common.policies import MlpPolicy
    if isinstance(policy, str):
        if policy != "MlpPolicy":
            raise NotImplementedError(f"policy '{policy}': only common.policies.MlpPolicy is built for {algo}")
    elif policy is not MlpPolicy:
        raise NotImplementedError(f"policy {getattr(policy, '__name__', policy)}: only common.policies.MlpPolicy is built for {algo} "
                                  "(CNN, recurrent and layer-norm policies are not)")


def check_policy_kwargs(policy_kwargs, algo):
    """-> (policy_kwargs as a dict, [h0, h1])"""
    kw = dict(policy_kwargs or {})
    unknown = set(kw) - {"layers", "net_arch", "act_fun", "feature_extraction", "layer_norm"}
    if unknown:
        raise NotImplementedError(f"policy_kwargs {sorted(unknown)} are not built for {algo}")
    if kw.get("feature_extraction", "mlp") != "mlp":
        raise NotImplementedError(f"feature_extraction: only the MLP extractor is built for {algo}")
    if kw.get("layer_norm", False):
        raise NotImplementedError("layer_norm=True: layer-normalised policies are not built")
    act = kw.get("act_fun")
    if act is not None and getattr(act, "__name__", str(act)) != "tanh":
        raise NotImplementedError(f"act_fun: only tanh is built for {algo}")
    layers = [int(x) for x in kw.get("layers", None) or [64, 64]]
    if "net_arch" in kw and kw["net_arch"] is not None:
        na = list(kw["net_arch"])
        if len(na) != 1 or not isinstance(na[0], dict):
            raise NotImplementedError(f"net_arch={na}: shared layers are not built; give net_arch=[dict(pi=[h0, h1], vf=[h0, h1])]")
        pi, vf = [int(x) for x in na[0].get("pi", [])], [int(x) for x in na[0].get("vf", [])]
        if pi != vf:
            raise NotImplementedError(f"net_arch pi={pi} vf={vf}: the towers must have the same widths")
        layers = pi
    if len(layers) != 2:
        raise NotImplementedError(f"layers={layers}: the {algo} learner builds exactly two hidden layers")
    return kw, layers


def init_params(obs_dim, n_actions, layers, seed, rng=None, scope="model/"):
    """common/tf_layers.py ortho_init in the variables' creation order: the orthogonal factor of an SVD of a standard normal
    matrix, scaled sqrt(2) for the hidden layers, 1 for vf, 0.01 for pi and q; zero biases and logstd.  The normal draws come
    from ``rng``, by default a generator seeded with ``seed``; the names carry ``scope``."""
    rng = np.random.default_rng(seed) if rng is None else rng
    h0, h1 = layers
    p = OrderedDict()
    for name, shape in (("pi_fc0/w", (obs_dim, h0)), ("pi_fc0/b", (h0,)), ("vf_fc0/w", (obs_dim, h0)), ("vf_fc0/b", (h0,)),
                        ("pi_fc1/w", (h0, h1)), ("pi_fc1/b", (h1,)), ("vf_fc1/w", (h0, h1)), ("vf_fc1/b", (h1,)), ("vf/w", (h1, 1)),
                        ("vf/b", (1,)), ("pi/w", (h1, n_actions)), ("pi/b", (n_actions,)), ("pi/logstd", (1, n_actions)),
                        ("q/w", (h1, n_actions)), ("q/b", (n_actions,))):
        if name == "pi/logstd" or len(shape) == 1:
            p[scope + name] = np.zeros(shape, np.float32)
            continue
        scale = 1.0 if name == "vf/w" else (0.01 if name in ("pi/w", "q/w") else np.sqrt(2.0))
        u, _, v = np.linalg.svd(rng.normal(0.0, 1.0, shape), full_matrices=False)
        w = u if u.shape == shape else v
        p[scope + name] = (scale * w.reshape(shape)).astype(np.float32)
    return p


class ActorCriticLearner(HandleLearner):
    """What the ``b2g_ppo`` and ``b2g_trpo`` wrappers share, the device ``obs_rms`` and its observe path included
    (include/b200grasp.h: b2g_ppo_observe_act)."""
    n_envs = 1

    @property
    def obs_elems(self) -> int:
        return self.obs_dim

    @property
    def obs_shape(self):
        """shape of obs_rms_get's arrays (the model sets the env's observation shape)"""
        return getattr(self, "_obs_shape", None) or (self.obs_dim,)

    @obs_shape.setter
    def obs_shape(self, shape):
        self._obs_shape = tuple(int(s) for s in shape)

    def set_norm_stats(self, clip_obs=10.0, epsilon=1e-8, norm_obs=True):
        """VecNormalize's clip_obs, epsilon and norm_obs for the rows observe_act and act(raw=True) normalise."""
        _lib.check(self._fn("set_norm_stats")(self.h, float(clip_obs), float(epsilon), int(bool(norm_obs))))

    def observe_act(self, obs, update_stats=True, act=True):
        """``obs``: the n_envs raw frames to upload once, merge into ``obs_rms`` (``update_stats``) and normalise into the
        current rollout row (row t, or t + 1 once row t's action is drawn); ``None`` acts on the row already staged.
        Returns the unclipped actions [n_envs, n_actions] of rollout step t, or None with ``act=False``."""
        if obs is not None:
            obs = _f32(obs).reshape(self.n_envs, self.frame_elems)
            self.obs_rms_version += bool(update_stats)
        out = np.empty((self.n_envs, self.n_actions), np.float32) if act else None
        _lib.check(self._fn("observe_act")(self.h, None if obs is None else _fp(obs), self.n_envs, int(bool(update_stats)),
                                            None if out is None else _fp(out)))
        return out

    def rollout_reset(self):
        _lib.check(self._fn("rollout_reset")(self.h))

    def steps(self):
        """(Adam step, noise-stream step, rollout rows filled); TRPO's Adam is the value function's"""
        a, b, t = C.c_int64(), C.c_int64(), C.c_int32()
        _lib.check(self._fn("get_step")(self.h, C.byref(a), C.byref(b), C.byref(t)))
        return a.value, b.value, t.value


class ActorCriticModel(BaseModel):
    """The PPO2 and TRPO front ends' common part.  A subclass sets ``_scope`` (the zip's scope of the live network),
    ``_branch`` (the reference's name of it), ``_zip_hyper`` (the hyper-parameters ``load`` reads) and ``_update_tags``."""
    _scope = ""
    _branch = ""
    _zip_hyper = ()
    _update_tags = {}
    _boundary = None                # (num_timesteps, numpy global state) after the last completed update
    last_metrics = None

    def _check_env(self):
        if not hasattr(self.action_space, "low"):
            raise NotImplementedError(f"{self._algo} here needs a Box action space, got {self.action_space} (the reference's "
                                      f"{self._branch} branch is continuous)")

    def predict(self, observation, state=None, mask=None, deterministic=False):
        """The Gaussian mean (deterministic) or a sample of stream 1, clipped to the action space.  While a learner owns the
        statistics of this model's VecNormalize (``predict_takes_raw_obs``) the observation is raw and is normalised as the
        wrapper would: on the device when this model's learner owns them, else by the wrapper's ``normalize_obs``."""
        self._check_encoded(observation)
        obs = np.asarray(observation, np.float32)
        single = obs.ndim == len(self.observation_space.shape)
        obs = obs.reshape(-1, self.learner.obs_dim)
        if self.predict_takes_raw_obs and self._owns_obs_rms():
            self._sync_norm_stats()
            a = self.learner.act(obs, deterministic=deterministic, raw=True)[0]
        else:
            if self.predict_takes_raw_obs:
                obs = np.asarray(self._vec_normalize_env.normalize_obs(obs), np.float32)
            a = self.learner.act(obs, deterministic=deterministic)[0]
        a = np.clip(a, self.action_space.low.reshape(-1), self.action_space.high.reshape(-1))
        a = a.reshape((-1,) + tuple(self.action_space.shape))
        return (a[0] if single else a), None

    # ------------------------------------------------------------------ VecNormalize's obs_rms on the device (device_obs_norm)
    @staticmethod
    def _normalises_obs(env) -> bool:
        vn = unwrap_vec_normalize(env) if env is not None else None
        return isinstance(vn, VecNormalize) and bool(vn.norm_obs)

    def _refuse_device_obs_norm_without_wrapper(self, env):
        """device_obs_norm=True moves VecNormalize's obs_rms to the learner, which then stores each frame as the wrapper
        would have returned it: refused, before any device work, for an env (or no env) without a VecNormalize that
        normalises observations -- there are no statistics to take over."""
        if self.device_obs_norm and not self._normalises_obs(env):
            raise NotImplementedError(f"device_obs_norm=True: {self._algo} takes over the observation statistics of the env's "
                                      "VecNormalize; pass an env wrapped in VecNormalize(norm_obs=True)")

    def _attach_device(self):
        """setup_model's last step: with device_obs_norm the wrapper's obs_rms and a VecEncodeDepth's encoder move to the
        learner (base_model.py)."""
        if self.device_obs_norm:
            self.learner.obs_shape = tuple(self.observation_space.shape)
        self._attach_device_norm()
        self._attach_obs_encoder()

    def _attach_device_norm(self):
        super()._attach_device_norm()
        if self._owns_obs_rms():
            self._sync_norm_stats()

    def _sync_norm_stats(self):
        """The owner's clip_obs, epsilon and norm_obs (the statistics are the learner's own)."""
        vn = self._vec_normalize_env
        self.learner.set_norm_stats(vn.clip_obs, vn.epsilon, vn.norm_obs)

    def _check_device_norm(self):
        """learn's refusals of the wrapper, before any device work."""
        vn = self._vec_normalize_env
        if getattr(vn, "learner_owns_obs_rms", False) and not self._owns_obs_rms():
            raise RuntimeError("learn: the env's VecNormalize statistics are owned by another model's learner (close that model, "
                               "or build this one with device_obs_norm=True before it)")
        if self.device_obs_norm and not (isinstance(vn, VecNormalize) and vn.norm_obs):
            raise RuntimeError("device_obs_norm=True needs the env wrapped in a VecNormalize with norm_obs=True")

    # ------------------------------------------------------------------ learn
    def _learn_start(self, callback, reset_num_timesteps, writer, globals_):
        """learn's first steps (globals_: the algorithm module's, for the callback) -> (callback, episode-reward logger or
        None, the first observations [n_envs, obs_dim]).  With device_obs_norm the reset frames are observed: uploaded once,
        merged (VecNormalize.reset's update) and normalised into rollout row 0."""
        self._check_device_norm()
        callback = as_callback(callback)
        callback.init_callback(self)
        if reset_num_timesteps:
            self.num_timesteps = 0
        callback.on_training_start({"self": self, "writer": writer}, globals_)
        ep_log = EpisodeRewardLogger(self.n_envs) if writer is not None else None
        obs = np.asarray(self.env.reset(), np.float32).reshape(self.n_envs, -1)
        self.learner.rollout_reset()
        if self.device_obs_norm:
            self._sync_norm_stats()
            self.learner.observe_act(obs, update_stats=self._vec_normalize_env.training, act=False)
        self.last_metrics = None
        return callback, ep_log, obs

    def _rollout(self, obs, n_steps, callback, writer, ep_log):
        """n_steps steps of every env into the learner's rollout (clipped actions to the env, num_timesteps += n_envs);
        callback.on_step() False stops it and empties the rollout -> (the last observations, stopped).  With device_obs_norm
        the wrapper returns raw frames: each is observed right after env.step (merged while the wrapper is training, as
        step_wait merges, and normalised into the next rollout row), so a callback sees the statistics the host path shows it."""
        L = self.learner
        dev = self.device_obs_norm
        low, high = self.action_space.low.reshape(-1), self.action_space.high.reshape(-1)
        callback.on_rollout_start()
        stopped = False
        for _ in range(n_steps):
            actions = L.observe_act(None) if dev else L.rollout_act(obs)
            clipped = np.clip(actions, low, high)
            new_obs, rew, done, infos = self.env.step(clipped.reshape((self.n_envs,) + tuple(self.action_space.shape)))
            self.num_timesteps += self.n_envs
            if dev:
                L.observe_act(np.asarray(new_obs, np.float32), update_stats=self._vec_normalize_env.training, act=False)
            if callback.on_step() is False:
                stopped = True
                break
            for info in infos or []:
                ep = info.get("episode") if isinstance(info, dict) else None
                if ep is not None:
                    self.ep_info_buf.append(ep)
            L.rollout_reward(np.asarray(rew, np.float32), np.asarray(done, np.float32))
            if ep_log is not None:
                ep_log(writer, rew, done, self.num_timesteps)
            obs = np.asarray(new_obs, np.float32).reshape(self.n_envs, -1)
        callback.on_rollout_end()
        if stopped:
            L.rollout_reset()
        return obs, stopped

    def _update_done(self, metrics, writer, extra=()):
        """After an update: its metrics, the training-state boundary and the update's summary (``_update_tags`` and the
        (tag, value) pairs of ``extra``)."""
        self.last_metrics = metrics
        self._boundary = (self.num_timesteps, np.random.get_state())
        if writer is not None:
            vals = [Summary.Value(t, metrics[k]) for t, k in self._update_tags.items()] + [Summary.Value(t, v) for t, v in extra]
            writer.add_summary(Summary(vals), self.num_timesteps)

    # ------------------------------------------------------------------ zip
    def _space_data(self):
        d = {"verbose": self.verbose, "n_envs": self.n_envs, "seed": self.seed, "policy_kwargs": dict(self.policy_kwargs),
             "observation_shape": list(self.observation_space.shape), "action_shape": list(self.action_space.shape),
             "action_low": np.asarray(self.action_space.low).reshape(-1).tolist(),
             "action_high": np.asarray(self.action_space.high).reshape(-1).tolist()}
        if self.device_obs_norm:
            d["device_obs_norm"] = True
        return d

    @classmethod
    def load(cls, load_path, env=None, custom_objects=None, **kwargs):
        """Reads a zip: widths and sizes from the parameter shapes under ``_scope``, hyper-parameters from ``data``."""
        from .spaces import Box
        data, params = cls._read_zip(load_path)
        w0, w1, wpi = (params[cls._scope + n] for n in ("pi_fc0/w", "pi_fc1/w", "pi/w"))
        kw = {k: data[k] for k in cls._zip_hyper if k in data and data[k] is not None}
        kw["policy_kwargs"] = dict(data.get("policy_kwargs") or {}, layers=[int(w0.shape[1]), int(w1.shape[1])])
        # a zip trained with device_obs_norm keeps it on an env whose VecNormalize normalises observations (the statistics
        # move to the learner again); without one it is a plain model, as the zip's parameters are
        dev = bool(kwargs.pop("device_obs_norm", bool(data.get("device_obs_norm")) and cls._normalises_obs(env)))
        kw.update(kwargs)
        m = cls("MlpPolicy", None, _init_setup_model=False, **kw)
        m.device_obs_norm = dev
        m._refuse_device_obs_norm_without_wrapper(env)
        if env is None:
            m._check_without_env()
        A = int(wpi.shape[1])
        return m._finish_load(env, Box(-np.inf, np.inf, tuple(data.get("observation_shape") or (w0.shape[0],))),
                              Box(np.asarray(data.get("action_low", [-1.0] * A), np.float32),
                                  np.asarray(data.get("action_high", [1.0] * A), np.float32), tuple(data.get("action_shape") or (A,))),
                              params)

    def _check_without_env(self):
        """``load`` without an env: what ``_check_env`` would refuse of the zip's configuration on one env."""

    # ------------------------------------------------------------------ training state (training_state.py)
    def _host_state(self):
        init = self._host_init()
        if self.device_obs_norm:
            init["device_obs_norm"] = True
        num, np_state = self._boundary if self._boundary is not None else (self.num_timesteps, np.random.get_state())
        host = {"algo": self._algo, "init": init, "num_timesteps": int(num),
                "np_random": [np_state[0], np.asarray(np_state[1]).tolist(), int(np_state[2]), int(np_state[3]), float(np_state[4])]}
        enc = self._encoder_host()
        if enc is not None:
            host["obs_encoder"] = enc
        return host

    def _restore_host_state(self, host):
        self.num_timesteps = int(host["num_timesteps"])
        s = host["np_random"]
        np.random.set_state((s[0], np.asarray(s[1], np.uint32), s[2], s[3], s[4]))
        self._boundary = (self.num_timesteps, np.random.get_state())
