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
from .base_model import BaseModel
from .callbacks import as_callback
from .learner import HandleLearner
from .tensorboard import EpisodeRewardLogger, Summary


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
    """What the ``b2g_ppo`` and ``b2g_trpo`` wrappers share."""

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
        """The Gaussian mean (deterministic) or a sample of stream 1, clipped to the action space."""
        obs = np.asarray(observation, np.float32)
        single = obs.ndim == len(self.observation_space.shape)
        a = self.learner.act(obs.reshape(-1, self.learner.obs_dim), deterministic=deterministic)[0]
        a = np.clip(a, self.action_space.low.reshape(-1), self.action_space.high.reshape(-1))
        a = a.reshape((-1,) + tuple(self.action_space.shape))
        return (a[0] if single else a), None

    # ------------------------------------------------------------------ learn
    def _learn_start(self, callback, reset_num_timesteps, writer, globals_):
        """learn's first steps (globals_: the algorithm module's, for the callback) -> (callback, episode-reward logger or
        None, the first observations [n_envs, obs_dim])"""
        callback = as_callback(callback)
        callback.init_callback(self)
        if reset_num_timesteps:
            self.num_timesteps = 0
        callback.on_training_start({"self": self, "writer": writer}, globals_)
        ep_log = EpisodeRewardLogger(self.n_envs) if writer is not None else None
        obs = np.asarray(self.env.reset(), np.float32).reshape(self.n_envs, -1)
        self.learner.rollout_reset()
        self.last_metrics = None
        return callback, ep_log, obs

    def _rollout(self, obs, n_steps, callback, writer, ep_log):
        """n_steps steps of every env into the learner's rollout (clipped actions to the env, num_timesteps += n_envs);
        callback.on_step() False stops it and empties the rollout -> (the last observations, stopped)"""
        L = self.learner
        low, high = self.action_space.low.reshape(-1), self.action_space.high.reshape(-1)
        callback.on_rollout_start()
        stopped = False
        for _ in range(n_steps):
            actions = L.rollout_act(obs)
            clipped = np.clip(actions, low, high)
            new_obs, rew, done, infos = self.env.step(clipped.reshape((self.n_envs,) + tuple(self.action_space.shape)))
            self.num_timesteps += self.n_envs
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
        return {"verbose": self.verbose, "n_envs": self.n_envs, "seed": self.seed, "policy_kwargs": dict(self.policy_kwargs),
                "observation_shape": list(self.observation_space.shape), "action_shape": list(self.action_space.shape),
                "action_low": np.asarray(self.action_space.low).reshape(-1).tolist(),
                "action_high": np.asarray(self.action_space.high).reshape(-1).tolist()}

    @classmethod
    def load(cls, load_path, env=None, custom_objects=None, **kwargs):
        """Reads a zip: widths and sizes from the parameter shapes under ``_scope``, hyper-parameters from ``data``."""
        from .spaces import Box
        data, params = cls._read_zip(load_path)
        w0, w1, wpi = (params[cls._scope + n] for n in ("pi_fc0/w", "pi_fc1/w", "pi/w"))
        kw = {k: data[k] for k in cls._zip_hyper if k in data and data[k] is not None}
        kw["policy_kwargs"] = dict(data.get("policy_kwargs") or {}, layers=[int(w0.shape[1]), int(w1.shape[1])])
        kw.update(kwargs)
        m = cls("MlpPolicy", None, _init_setup_model=False, **kw)
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
        num, np_state = self._boundary if self._boundary is not None else (self.num_timesteps, np.random.get_state())
        return {"algo": self._algo, "init": init, "num_timesteps": int(num),
                "np_random": [np_state[0], np.asarray(np_state[1]).tolist(), int(np_state[2]), int(np_state[3]), float(np_state[4])]}

    def _restore_host_state(self, host):
        self.num_timesteps = int(host["num_timesteps"])
        s = host["np_random"]
        np.random.set_state((s[0], np.asarray(s[1], np.uint32), s[2], s[3], s[4]))
        self._boundary = (self.num_timesteps, np.random.get_state())
