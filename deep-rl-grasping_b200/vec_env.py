"""Minimal VecEnv / VecNormalize with the surface the reference harness touches
(sb_helper.py:75,101-103,118-119; train_stable_baselines.py:52-54,88-91; utils.py:71-76;
base_callbacks.py:140-149).  Restates [SB2] common/vec_env/{dummy_vec_env,vec_normalize}.py and
common/running_mean_std.py so that a reference user can switch imports without gym's VecEnv
machinery.  Statistics are float64 numpy, exactly what the learner consumes at sample time.
"""
from __future__ import annotations

import pickle
import sys
import types
from typing import Optional,  Callable, List, Sequence

import numpy as np


class RunningMeanStd:
    """[SB2] common/running_mean_std.py (parallel-variance update, count starts at epsilon)."""

    def __init__(self, epsilon: float = 1e-4, shape=()):
        self.mean = np.zeros(shape, np.float64)
        self.var = np.ones(shape, np.float64)
        self.count = epsilon

    def update(self, arr: np.ndarray) -> None:
        arr = np.asarray(arr, np.float64)
        self.update_from_moments(arr.mean(axis=0), arr.var(axis=0), arr.shape[0])

    def update_from_moments(self, batch_mean, batch_var, batch_count: int) -> None:
        delta = batch_mean - self.mean
        tot = self.count + batch_count
        new_mean = self.mean + delta * batch_count / tot
        m_a = self.var * self.count
        m_b = batch_var * batch_count
        m_2 = m_a + m_b + np.square(delta) * self.count * batch_count / tot
        self.mean, self.var, self.count = new_mean, m_2 / tot, tot


class DeviceRunningMeanStd:
    """The ``obs_rms`` of a VecNormalize whose statistics live on the device learner (``SAC(device_obs_norm=True)``).
    ``owner`` provides ``obs_rms_get() -> (mean, var, count)``, ``obs_rms_set(mean, var, count)`` and a counter
    ``obs_rms_version`` that moves whenever the device statistics may have changed.  ``mean`` / ``var`` / ``count`` fetch on
    access (cached until the version moves) and assignment writes through, so everything that reads or copies a
    RunningMeanStd keeps working: pickling and ``copy.deepcopy`` give a plain RunningMeanStd holding the current numbers."""

    def __init__(self, owner):
        self.__dict__["_owner"] = owner
        self.__dict__["_cache"] = None

    def _fetch(self):
        ver = self._owner.obs_rms_version
        if self._cache is None or self._cache[0] != ver:
            self.__dict__["_cache"] = (ver,) + tuple(self._owner.obs_rms_get())
        return self._cache[1:]

    mean = property(lambda self: self._fetch()[0])
    var = property(lambda self: self._fetch()[1])
    count = property(lambda self: self._fetch()[2])

    def __setattr__(self, name, value):
        if name not in ("mean", "var", "count"):
            raise AttributeError(name)
        cur = dict(zip(("mean", "var", "count"), self._fetch()))
        cur[name] = value
        self._owner.obs_rms_set(cur["mean"], cur["var"], cur["count"])
        self.__dict__["_cache"] = None

    def update(self, arr) -> None:
        raise RuntimeError("the device learner merges observations into these statistics (Learner.observe_act / observe_add)")

    def snapshot(self) -> RunningMeanStd:
        r = RunningMeanStd.__new__(RunningMeanStd)
        m, v, c = self._fetch()
        r.mean, r.var, r.count = np.array(m, np.float64), np.array(v, np.float64), float(c)
        return r

    def __deepcopy__(self, memo):
        return self.snapshot()

    def __reduce__(self):
        return (_rebuild_rms, tuple(self.snapshot().__dict__.items()))


def _rebuild_rms(*items):
    r = RunningMeanStd.__new__(RunningMeanStd)
    r.__dict__.update(items)
    return r


class VecEnv:
    """Marker base class (``isinstance(env, VecEnv)`` in base_callbacks.py:50 and [SB2] evaluate_policy)."""
    num_envs = 1


class DummyVecEnv(VecEnv):
    """Sequential vectorised env: ``DummyVecEnv([lambda: env, ...])`` (train_stable_baselines.py:54)."""

    def __init__(self, env_fns: Sequence[Callable]):
        self.envs = [fn() for fn in env_fns]
        self.num_envs = len(self.envs)
        e = self.envs[0]
        self.observation_space, self.action_space = e.observation_space, e.action_space
        self.buf_infos: List[dict] = [{} for _ in self.envs]
        self._actions = None

    def reset(self):
        return np.stack([np.asarray(e.reset()) for e in self.envs])

    def step_async(self, actions):
        self._actions = actions

    def step_wait(self):
        obs, rews, dones = [], [], []
        for i, (e, a) in enumerate(zip(self.envs, self._actions)):
            o, r, d, info = e.step(a)
            if d:
                info = dict(info)
                info["terminal_observation"] = o
                o = e.reset()
            obs.append(np.asarray(o)); rews.append(r); dones.append(d)
            self.buf_infos[i] = info
        return np.stack(obs), np.asarray(rews, np.float32), np.asarray(dones), list(self.buf_infos)

    def step(self, actions):
        self.step_async(actions)
        return self.step_wait()

    def close(self):
        for e in self.envs:
            if hasattr(e, "close"):
                e.close()

    def get_attr(self, name, indices=None):
        return [getattr(e, name) for e in self.envs]

    def env_method(self, name, *a, **k):
        return [getattr(e, name)(*a, **k) for e in self.envs]


def _subproc_worker(remote, parent_remote, fn_bytes):
    """One environment per process ([SB2] common/vec_env/subproc_vec_env.py protocol: step / reset / close / get_spaces /
    get_attr / env_method); auto-reset on done with the terminal observation in ``info``."""
    import pickle
    parent_remote.close()
    env = pickle.loads(fn_bytes)()
    try:
        while True:
            cmd, data = remote.recv()
            if cmd == "step":
                o, r, d, info = env.step(data)
                if d:
                    info = dict(info)
                    info["terminal_observation"] = np.asarray(o)
                    o = env.reset()
                remote.send((np.asarray(o), r, d, info))
            elif cmd == "reset":
                remote.send(np.asarray(env.reset()))
            elif cmd == "get_spaces":
                remote.send((env.observation_space, env.action_space))
            elif cmd == "get_attr":
                remote.send(getattr(env, data))
            elif cmd == "env_method":
                remote.send(getattr(env, data[0])(*data[1], **data[2]))
            elif cmd == "close":
                if hasattr(env, "close"):
                    env.close()
                remote.close()
                break
            else:
                raise NotImplementedError(cmd)
    except (EOFError, KeyboardInterrupt):
        pass


class SubprocVecEnv(VecEnv):
    """Vectorised environments in worker processes: the host-side actor loop that feeds the GPU-resident replay buffer
    (BASELINE config 5: 128 PyBullet envs on host cores; the reference imports it at sb_helper.py:19).  ``step_async``
    sends every action first, ``step_wait`` collects, so the environments advance in parallel on the host cores while
    the previous batch of transitions is already on its way to the device."""

    def __init__(self, env_fns: Sequence[Callable], start_method: Optional[str] = None):
        import multiprocessing as mp
        import cloudpickle
        ctx = mp.get_context(start_method or ("forkserver" if "forkserver" in mp.get_all_start_methods() else "spawn"))
        self.num_envs = len(env_fns)
        self.remotes, self.work_remotes = zip(*[ctx.Pipe() for _ in env_fns])
        self.procs = []
        for wr, r, fn in zip(self.work_remotes, self.remotes, env_fns):
            p = ctx.Process(target=_subproc_worker, args=(wr, r, cloudpickle.dumps(fn)), daemon=True)
            p.start()
            self.procs.append(p)
            wr.close()
        self.remotes[0].send(("get_spaces", None))
        self.observation_space, self.action_space = self.remotes[0].recv()
        self.buf_infos: List[dict] = [{} for _ in env_fns]
        self.waiting = self.closed = False

    def step_async(self, actions):
        for r, a in zip(self.remotes, actions):
            r.send(("step", a))
        self.waiting = True

    def step_wait(self):
        res = [r.recv() for r in self.remotes]
        self.waiting = False
        obs, rews, dones, infos = zip(*res)
        self.buf_infos = list(infos)
        return np.stack(obs), np.asarray(rews, np.float32), np.asarray(dones), list(infos)

    def step(self, actions):
        self.step_async(actions)
        return self.step_wait()

    def reset(self):
        for r in self.remotes:
            r.send(("reset", None))
        return np.stack([r.recv() for r in self.remotes])

    def get_attr(self, name, indices=None):
        idx = range(self.num_envs) if indices is None else indices
        for i in idx:
            self.remotes[i].send(("get_attr", name))
        return [self.remotes[i].recv() for i in idx]

    def env_method(self, name, *a, **k):
        for r in self.remotes:
            r.send(("env_method", (name, a, k)))
        return [r.recv() for r in self.remotes]

    @property
    def envs(self):
        raise AttributeError("SubprocVecEnv has no in-process envs; use get_attr / env_method")

    def close(self):
        if self.closed:
            return
        if self.waiting:
            for r in self.remotes:
                r.recv()
        for r in self.remotes:
            r.send(("close", None))
        for p in self.procs:
            p.join(timeout=5)
        self.closed = True


class VecEncodeDepth(VecEnv):
    """Owns the perception encoder of the encoded-depth configuration for a stack of envs whose sensor defers the encoding
    (``encoders.DeferredEncodedDepthImgSensor``): each raw observation is ``[H*W*C depth | tail]``, ``tail`` floats of actuator
    state or time feature (default: whatever follows the pixels).  ``observation_space`` is what the reference env reports,
    ``Box(-1, 1, (encoding_dim,))`` followed by the raw space's last ``tail`` bounds, so a VecNormalize on top keeps the
    shipped ``obs_rms`` layout.

    Host mode (the default): every ``reset`` / ``step`` makes one ``encoder.encode`` call for the frames of all envs and the
    terminal observations of the finished ones, and returns encoded rows.  Pass-raw mode: a SAC or BDQ learner built with
    ``device_obs_norm=True`` took the encoder (``give_encoder_to``) and encodes on its device, so ``reset`` / ``step`` and the
    terminal observations hand the raw rows through; ``take_encoder_back`` returns to host mode."""

    def __init__(self, venv, encoder, tail=None):
        from .spaces import Box
        self.venv, self.encoder = venv, encoder
        self.num_envs = venv.num_envs
        self.input_shape = tuple(int(d) for d in encoder.input_shape)
        self.pixels = int(np.prod(self.input_shape))
        self.raw_observation_space = raw = venv.observation_space
        self.raw_width = int(np.prod(raw.shape))
        self.tail = self.raw_width - self.pixels if tail is None else int(tail)
        if self.tail < 0 or self.pixels + self.tail != self.raw_width:
            raise ValueError(f"VecEncodeDepth: raw observations of {self.raw_width} floats are not {self.pixels} pixels "
                             f"{self.input_shape} + {self.tail} tail floats")
        dim = int(encoder.encoding_dim)
        low = np.concatenate([np.full(dim, -1.0), np.ravel(raw.low)[self.pixels:]])
        high = np.concatenate([np.full(dim, 1.0), np.ravel(raw.high)[self.pixels:]])
        self.observation_space = Box(low, high, (dim + self.tail,), np.float32)
        self.action_space = venv.action_space
        self._owner = None

    # ---- the encoder handed to a device learner (SAC / BDQ with device_obs_norm)
    @property
    def pass_raw(self) -> bool:
        return self._owner is not None

    @property
    def encoder_owner(self):
        return self._owner

    def give_encoder_to(self, owner) -> None:
        """From here on ``owner`` (a learner with the encoder attached) encodes: observations go through raw."""
        if self._owner is not None and self._owner is not owner:
            raise RuntimeError("this VecEncodeDepth's encoder is already attached to another learner")
        self._owner = owner

    def take_encoder_back(self) -> None:
        """Host mode again (the owner is about to go away)."""
        self._owner = None

    def encode(self, rows) -> np.ndarray:
        """Raw rows [n, H*W*C + tail] -> encoded rows [n, encoding_dim + tail] (one ``encoder.encode`` call)."""
        rows = np.asarray(rows, np.float32).reshape(-1, self.raw_width)
        enc = np.asarray(self.encoder.encode(rows[:, :self.pixels].reshape((-1,) + self.input_shape)), np.float32)
        return np.concatenate([enc, rows[:, self.pixels:]], axis=1)

    # ---- VecEnv surface
    @property
    def envs(self):
        return self.venv.envs

    @property
    def buf_infos(self):
        return self.venv.buf_infos

    def reset(self):
        obs = self.venv.reset()
        return obs if self.pass_raw else self.encode(obs)

    def step_async(self, actions):
        self.venv.step_async(actions)

    def step_wait(self):
        obs, rews, dones, infos = self.venv.step_wait()
        if self.pass_raw:
            return obs, rews, dones, infos
        # the reference env encodes the terminal frame too: it joins the same call
        term = [i for i, info in enumerate(infos) if dones[i] and isinstance(info, dict) and "terminal_observation" in info]
        n = self.num_envs
        rows = np.concatenate([np.asarray(obs, np.float32).reshape(n, -1)] +
                              [np.asarray(infos[i]["terminal_observation"], np.float32).reshape(1, -1) for i in term])
        enc = self.encode(rows)
        infos = list(infos)
        for k, i in enumerate(term):
            infos[i] = dict(infos[i], terminal_observation=enc[n + k])
        return enc[:n], rews, dones, infos

    def step(self, actions):
        self.step_async(actions)
        return self.step_wait()

    def close(self):
        self.venv.close()

    def get_attr(self, name, indices=None):
        return self.venv.get_attr(name, indices)

    def env_method(self, name, *a, **k):
        return self.venv.env_method(name, *a, **k)


def unwrap_encode_depth(env) -> Optional[VecEncodeDepth]:
    e = env
    while e is not None:
        if isinstance(e, VecEncodeDepth):
            return e
        e = getattr(e, "venv", None)
    return None


class VecNormalize(VecEnv):
    """[SB2] VecNormalize(venv, training=True, norm_obs=True, norm_reward=True, clip_obs=10.,
    clip_reward=10., gamma=0.99, epsilon=1e-8)."""

    def __init__(self, venv, training=True, norm_obs=True, norm_reward=True, clip_obs=10.0, clip_reward=10.0, gamma=0.99,
                 epsilon=1e-8):
        self.venv = venv
        self.num_envs = venv.num_envs
        self.observation_space, self.action_space = venv.observation_space, venv.action_space
        self.obs_rms = RunningMeanStd(shape=self.observation_space.shape)
        self.ret_rms = RunningMeanStd(shape=())
        self.clip_obs, self.clip_reward = clip_obs, clip_reward
        self.ret = np.zeros(self.num_envs)
        self.gamma, self.epsilon = gamma, epsilon
        self.training, self.norm_obs, self.norm_reward = training, norm_obs, norm_reward
        self.old_obs, self.old_rews = np.array([]), np.array([])

    # ---- statistics owned by the device learner (SAC(device_obs_norm=True))
    @property
    def learner_owns_obs_rms(self) -> bool:
        return isinstance(self.obs_rms, DeviceRunningMeanStd)

    def give_obs_rms_to(self, owner) -> None:
        """Hands the current ``obs_rms`` to ``owner`` (a Learner): from here on ``reset`` / ``step_wait`` return the RAW
        observation and leave the update and the normalisation of observations to the device; the reward side is unchanged.
        ``normalize_obs`` called explicitly still works, from the fetched statistics.  A wrapper has one owner at a time:
        another one must wait for ``take_obs_rms_back``."""
        if self.learner_owns_obs_rms:
            if self.obs_rms_owner is owner:
                return
            raise RuntimeError("this VecNormalize's obs_rms is already owned by another learner")
        owner.obs_rms_set(self.obs_rms.mean, self.obs_rms.var, self.obs_rms.count)
        self.obs_rms = DeviceRunningMeanStd(owner)

    @property
    def obs_rms_owner(self):
        return self.obs_rms._owner if self.learner_owns_obs_rms else None

    def take_obs_rms_back(self) -> None:
        """The statistics return to the host as a plain RunningMeanStd holding the owner's current numbers (the owner is
        about to go away): the wrapper updates and normalises again itself."""
        if self.learner_owns_obs_rms:
            self.obs_rms = self.obs_rms.snapshot()

    # ---- VecEnv surface
    @property
    def envs(self):
        return self.venv.envs

    @property
    def buf_infos(self):
        return self.venv.buf_infos

    def step_async(self, actions):
        self.venv.step_async(actions)

    def step_wait(self):
        obs, rews, news, infos = self.venv.step_wait()
        self.ret = self.ret * self.gamma + rews
        self.old_obs, self.old_rews = obs, rews
        owned = self.learner_owns_obs_rms
        if self.training:
            if not owned:
                self.obs_rms.update(obs)
            self.ret_rms.update(self.ret)
        if not owned:
            obs = self.normalize_obs(obs)
        rews = self.normalize_reward(rews)
        self.ret[news] = 0
        return obs, rews, news, infos

    def step(self, actions):
        self.step_async(actions)
        return self.step_wait()

    def reset(self):
        obs = self.venv.reset()
        self.old_obs = obs
        self.ret = np.zeros(self.num_envs)
        if self.learner_owns_obs_rms:
            return obs
        if self.training:
            self.obs_rms.update(obs)
        return self.normalize_obs(obs)

    def close(self):
        self.venv.close()

    def get_attr(self, name, indices=None):
        return self.venv.get_attr(name, indices)

    # ---- normalisation (float64 like numpy in SB2; the learner applies the same formula on the device)
    def normalize_obs(self, obs):
        if self.norm_obs:
            obs = np.clip((obs - self.obs_rms.mean) / np.sqrt(self.obs_rms.var + self.epsilon), -self.clip_obs, self.clip_obs)
        return obs

    def normalize_reward(self, reward):
        if self.norm_reward:
            reward = np.clip(reward / np.sqrt(self.ret_rms.var + self.epsilon), -self.clip_reward, self.clip_reward)
        return reward

    def get_original_obs(self):
        return self.old_obs.copy()

    def get_original_reward(self):
        return self.old_rews.copy()

    # ---- persistence (vecnormalize.pkl; sb_helper.py:246-247, train_stable_baselines.py:88-91)
    def __getstate__(self):
        st = self.__dict__.copy()
        for k in ("venv", "num_envs", "ret"):
            st.pop(k, None)
        if self.learner_owns_obs_rms:
            st["obs_rms"] = self.obs_rms.snapshot()
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)
        self.venv = None

    def set_venv(self, venv):
        self.venv = venv
        self.num_envs = venv.num_envs
        self.ret = np.zeros(self.num_envs)

    def save(self, path: str, sb_compatible: bool = True):
        """Pickle.  With ``sb_compatible`` the pickle names stable_baselines' own classes so that the
        reference's ``VecNormalize.load`` (train_stable_baselines.py:91) can read it back."""
        if not sb_compatible:
            with open(path, "wb") as f:
                pickle.dump(self, f)
            return
        # The pickle must NAME stable_baselines' classes.  Stand-in classes carrying those module / class names are
        # registered in sys.modules only for the duration of the dump; whatever was there before (a real stable_baselines
        # install included) is put back in `finally`, also when the dump raises.
        vn_mod, rm_mod = "stable_baselines.common.vec_env.vec_normalize", "stable_baselines.common.running_mean_std"
        vn_cls = type("VecNormalize", (), {"__module__": vn_mod})
        rm_cls = type("RunningMeanStd", (), {"__module__": rm_mod})
        created, missing = [], object()
        saved = {}
        try:
            for name in ("stable_baselines", "stable_baselines.common", "stable_baselines.common.vec_env", vn_mod, rm_mod):
                if name not in sys.modules:
                    sys.modules[name] = types.ModuleType(name)
                    created.append(name)
            for mod, attr, cls in ((vn_mod, "VecNormalize", vn_cls), (rm_mod, "RunningMeanStd", rm_cls)):
                saved[(mod, attr)] = getattr(sys.modules[mod], attr, missing)
                setattr(sys.modules[mod], attr, cls)
            obj = vn_cls.__new__(vn_cls)
            st = self.__getstate__()
            for k in ("obs_rms", "ret_rms"):
                r = rm_cls.__new__(rm_cls)
                r.__dict__.update(st[k].__dict__)
                st[k] = r
            for k in ("observation_space", "action_space"):      # our Box is not importable on the reference side
                st.pop(k, None)
            obj.__dict__.update(st)
            with open(path, "wb") as f:
                pickle.dump(obj, f)
        finally:
            for (mod, attr), old in saved.items():
                if mod in sys.modules and mod not in created:
                    if old is missing:
                        try:
                            delattr(sys.modules[mod], attr)
                        except AttributeError:
                            pass
                    else:
                        setattr(sys.modules[mod], attr, old)
            for name in created:
                sys.modules.pop(name, None)

    @staticmethod
    def load(path: str, venv):
        """Reads either our pickle or one written by stable-baselines (trained_models/*/vecnormalize.pkl)."""
        from .sb_io import load_vecnormalize
        d = load_vecnormalize(path)
        vn = VecNormalize(venv, training=True, norm_obs=d["norm_obs"], norm_reward=d["norm_reward"], clip_obs=d["clip_obs"],
                          clip_reward=d["clip_reward"], gamma=d["gamma"], epsilon=d["epsilon"])
        vn.obs_rms.mean, vn.obs_rms.var, vn.obs_rms.count = d["obs_mean"], d["obs_var"], d["obs_count"]
        vn.ret_rms.mean, vn.ret_rms.var, vn.ret_rms.count = np.float64(d["ret_mean"]), np.float64(d["ret_var"]), d["ret_count"]
        return vn


def sync_envs_normalization(env, eval_env) -> None:
    """[SB2] common/vec_env/__init__.py: copy the running statistics of every VecNormalize layer of ``env`` into the
    matching layer of ``eval_env`` (base_callbacks.py:81 before each evaluation)."""
    import copy
    e, ev = env, eval_env
    while e is not None and ev is not None:
        if isinstance(e, VecNormalize) and isinstance(ev, VecNormalize):
            ev.obs_rms = copy.deepcopy(e.obs_rms)
            ev.ret_rms = copy.deepcopy(e.ret_rms)
        e, ev = getattr(e, "venv", None), getattr(ev, "venv", None)
