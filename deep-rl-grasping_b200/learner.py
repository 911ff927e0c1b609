"""Thin numpy-facing wrappers of the device-resident learners' handles.

``HandleLearner`` is what the wrappers of the ``b2g_sac``, ``b2g_bdq``, ``b2g_dqn``, ``b2g_ppo`` and ``b2g_trpo`` handles share.
``Learner`` wraps one ``b2g_sac`` handle and is what ``SAC`` (sac_model.py, the stable-baselines-shaped front end) drives;
tests and bench.py also use it directly because it maps 1:1 onto the C ABI entry points.
"""
from __future__ import annotations

import ctypes as C
import os
from collections import OrderedDict
from typing import Optional, Sequence

import numpy as np

from . import _lib


def _fp(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _f32(a) -> np.ndarray:
    a = np.asarray(a, dtype=np.float32)          # (ascontiguousarray would promote 0-d to 1-d)
    return a if a.flags.c_contiguous else a.copy()


def nccl_config(nranks: int, nccl_id: Optional[bytes]):
    """(id buffer, id pointer, NCCL library path) for a handle's configuration; all None with one rank.  The buffer must
    outlive the create call that reads the pointer."""
    if nranks <= 1:
        return None, None, None
    if nccl_id is None or len(nccl_id) != 128:
        raise ValueError("nranks > 1 needs the 128-byte nccl_id shared by all ranks")
    buf = C.create_string_buffer(bytes(nccl_id), 128)
    lib_path = _lib.default_nccl_lib()
    return buf, C.cast(buf, C.c_void_p), lib_path.encode() if lib_path else None


class HandleLearner:
    """What the numpy-facing wrappers of the learner handles share: the handle's lifetime, its named parameters
    (``param_*``, ``get_param``, ``set_param``, ``get_grad``), its training-state files and, for the learners that take
    VecNormalize's statistics, ``set_norm_stats``, the device ``obs_rms`` and the upload counters.  A subclass sets
    ``_abi`` and ``_has_grad`` and calls ``_create`` with its configuration, or fills ``_info`` itself.  Entry point
    ``name`` is ``b2g_<abi>_<name>`` unless ``_names`` maps it to another symbol."""
    _abi = ""
    _names = {}
    log_capacity = 0

    #: bumped by every call that may change the device statistics (DeviceRunningMeanStd caches against it)
    obs_rms_version = 0
    #: floats of a raw row observe_* take while an observation encoder is attached (set_obs_encoder), else None
    raw_obs_elems = None

    def _has_grad(self, name: str) -> bool:
        raise NotImplementedError

    def metrics_log(self, capacity: int):
        """Per-step metrics ring of ``capacity`` rows on the device (0 turns it off); SAC, BDQ and DQN handles only."""
        _lib.check(self._fn("metrics_log")(self.h, int(capacity)))
        self.log_capacity = int(capacity)

    def metrics_drain(self, max_rows: Optional[int] = None):
        """Rows the steps appended since the last drain: ``(first_step, rows [n, K] float32, lost)``; row i is the metrics of
        optimiser step ``first_step + i`` (columns ``_lib.LOG_COLS[abi]``) and ``lost`` counts rows overwritten before this
        drain."""
        K = len(_lib.LOG_COLS[self._abi])
        cap = self.log_capacity if max_rows is None else int(max_rows)
        rows = np.empty((max(cap, 1), K), np.float32)
        first, n, lost = C.c_int64(), C.c_int(), C.c_int64()
        _lib.check(self._fn("metrics_drain")(self.h, _fp(rows.reshape(-1)), cap, C.byref(first), C.byref(n), C.byref(lost)))
        return int(first.value), rows[:n.value].copy(), int(lost.value)

    def _fn(self, name: str):
        return getattr(self.lib, self._names.get(name) or f"b2g_{self._abi}_{name}")

    def _create(self, cfg, replay=None):
        """``replay``: an ``_lib.ReplayCfg`` for the ``create2`` call (BDQ / DQN replay frames); None = ``create``."""
        self.h = C.c_void_p()
        if replay is None:
            _lib.check(self._fn("create")(C.byref(cfg), C.byref(self.h)))
        else:
            _lib.check(self._fn("create2")(C.byref(cfg), C.byref(replay), C.byref(self.h)))
        self._info = OrderedDict()
        buf = C.create_string_buffer(256)
        rows, cols, nd = C.c_int64(), C.c_int64(), C.c_int32()
        for i in range(self._fn("param_count")(self.h)):
            _lib.check(self._fn("param_info")(self.h, i, buf, 256, C.byref(rows), C.byref(cols), C.byref(nd)))
            self._info[buf.value.decode()] = () if nd.value == 0 else ((rows.value, cols.value) if nd.value == 2 else (cols.value,))

    def close(self):
        if getattr(self, "h", None) is not None and self.h:
            self._fn("destroy")(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def param_shapes(self):
        return self._info

    def get_parameters(self):
        out = OrderedDict()
        for n, shp in self._info.items():
            a = np.empty(shp, np.float32)
            _lib.check(self._fn("get_param")(self.h, n.encode(), _fp(a.reshape(-1)), a.size))
            out[n] = a
        return out

    def load_parameters(self, params, exact_match=True):
        seen = set()
        for n, a in params.items():
            key = n[:-2] if n.endswith(":0") else n
            if key not in self._info:
                if exact_match:
                    raise ValueError(f"unknown variable {n}")
                continue
            a = _f32(a)
            if tuple(a.shape) != self._info[key]:
                raise ValueError(f"shape mismatch for {n}: {a.shape} vs {self._info[key]}")
            _lib.check(self._fn("set_param")(self.h, key.encode(), _fp(a.reshape(-1)), a.size))
            seen.add(key)
        if exact_match and seen != set(self._info):
            raise ValueError(f"missing variables: {sorted(set(self._info) - seen)}")

    def get_gradients(self):
        """The last step's gradients of the trained variables, after the learner's gradient clip."""
        out = OrderedDict()
        for n, shp in self._info.items():
            if self._has_grad(n):
                a = np.empty(shp, np.float32)
                _lib.check(self._fn("get_grad")(self.h, n.encode(), _fp(a.reshape(-1)), a.size))
                out[n] = a
        return out

    def save_state(self, path: str):
        """Parameters, Adam moments, counters and, for the replay learners, the live replay rows and the prioritised-replay
        trees -> ``path`` (waits for enqueued steps)."""
        _lib.check(self._fn("state_save")(self.h, os.fsencode(path)))

    def load_state(self, path: str):
        """Restores a ``save_state`` file into this learner, which must have the same configuration (SAC's precision aside)
        and own a device ``obs_rms`` exactly when the file carries one.  Other normalisation statistics are not part of the
        file: set them again with ``set_norm_stats``."""
        _lib.check(self._fn("state_load")(self.h, os.fsencode(path)))
        self.obs_rms_version += 1

    # ---- VecNormalize's statistics (``obs_elems`` floats per observation)
    def set_norm_stats(self, obs_mean=None, obs_var=None, ret_var=1.0, clip_obs=10.0, clip_reward=10.0, epsilon=1e-8,
                       norm_obs=True, norm_reward=True):
        """The statistics of the gradient step's gather (and of act() where the learner normalises).  ``obs_mean = obs_var
        = None`` with ``norm_obs``: a learner that owns ``obs_rms`` keeps its device statistics and takes the scalars only."""
        dp = C.POINTER(C.c_double)
        mp = vp = None
        if norm_obs and obs_mean is not None:
            m = np.ascontiguousarray(obs_mean, np.float64).reshape(-1)
            v = np.ascontiguousarray(obs_var, np.float64).reshape(-1)
            assert m.size == self.obs_elems and v.size == self.obs_elems
            mp, vp = m.ctypes.data_as(dp), v.ctypes.data_as(dp)
        _lib.check(self._fn("set_norm_stats")(self.h, mp, vp, float(ret_var), float(clip_obs), float(clip_reward), float(epsilon),
                                               int(bool(norm_obs)), int(bool(norm_reward))))
        if mp is not None:
            self.obs_rms_version += 1

    def obs_rms_set(self, mean, var, count):
        """Creates (first call) or overwrites the device ``obs_rms``: float64 mean / var of the observation + count."""
        dp = C.POINTER(C.c_double)
        m = np.ascontiguousarray(mean, np.float64).reshape(-1)
        v = np.ascontiguousarray(var, np.float64).reshape(-1)
        assert m.size == self.obs_elems and v.size == self.obs_elems
        _lib.check(self._fn("obs_rms_set")(self.h, m.ctypes.data_as(dp), v.ctypes.data_as(dp), float(count)))
        self.obs_rms_version += 1

    def obs_rms_get(self):
        """(mean, var, count) of the device ``obs_rms`` in ``obs_shape``; waits for the work enqueued on the handle."""
        dp = C.POINTER(C.c_double)
        m, v = np.empty(self.obs_shape, np.float64), np.empty(self.obs_shape, np.float64)
        cnt = C.c_double()
        _lib.check(self._fn("obs_rms_get")(self.h, m.ctypes.data_as(dp), v.ctypes.data_as(dp), C.byref(cnt)))
        return m, v, float(cnt.value)

    # ---- an observation encoder on the observe path (SAC's MLP policy and BDQ; include/b200grasp.h: b2g_*_set_obs_encoder)
    def set_obs_encoder(self, encoder, tail: int = 0):
        """``encoder`` (an ``encoders.SimpleAutoEncoder`` with weights): its geometry and weights are copied into this learner,
        and from then on ``observe_act`` / ``observe_add`` take raw rows ``[H*W*C depth | tail]`` and encode them on the
        device into the ``[encoding_dim | tail]`` rows everything else works on.  ``None`` detaches.  Either way the staged
        observations are cleared."""
        if encoder is None:
            _lib.check(self._fn("set_obs_encoder")(self.h, None, 0))
            self.raw_obs_elems = None
            return
        _lib.check(self._fn("set_obs_encoder")(self.h, encoder._handle, int(tail)))
        self.raw_obs_elems = int(np.prod(encoder.input_shape)) + int(tail)

    @property
    def frame_elems(self) -> int:
        """Floats per frame of observe_act / observe_add."""
        return self.raw_obs_elems or self.obs_elems

    def upload_bytes(self) -> dict:
        """Bytes copied host -> device so far: by ``observe_*`` / ``obs_rms_set``, and by ``act`` + ``replay_add`` +
        ``set_norm_stats``."""
        a, b = C.c_int64(), C.c_int64()
        _lib.check(self._fn("upload_bytes")(self.h, C.byref(a), C.byref(b)))
        return {"observe": int(a.value), "other": int(b.value)}

    def replay_info(self) -> dict:
        """SAC, BDQ and DQN handles: capacity, size, frame_capacity and live_frames (0 without frames), bytes (device memory
        of the replay: rows or frames and frame indices, actions, rewards, dones), evicted_early."""
        keys = ("capacity", "size", "frame_capacity", "live_frames", "bytes", "evicted_early")
        vals = [C.c_int64() for _ in keys]
        _lib.check(self._fn("replay_info")(self.h, *[C.byref(v) for v in vals]))
        return {k: int(v.value) for k, v in zip(keys, vals)}


class TransitionReplayLearner(HandleLearner):
    """The transition replay the BDQ and DQN handles share (include/b200grasp.h: b2g_bdq_create2, b2g_*_replay_info)."""

    @staticmethod
    def _replay_cfg(frame_capacity: Optional[int]):
        """``frame_capacity``: keep obs / next_obs in a pool of that many frames (at least buffer_size + 1); None = two rows
        per slot."""
        return None if frame_capacity is None else _lib.ReplayCfg(int(frame_capacity), 0)

    def replay_get(self, slot: int) -> dict:
        """The stored transition of a live slot: obs, act, rew, next_obs, done, and frames = its (obs, next_obs) frame ids
        (-1 without frames)."""
        o, nx = np.empty(self.obs_dim, np.float32), np.empty(self.obs_dim, np.float32)
        a = np.empty(self._act_width, np.float32)
        r, d = np.empty(1, np.float32), np.empty(1, np.float32)
        fr = np.empty(2, np.int32)
        _lib.check(self._fn("replay_get")(self.h, int(slot), _fp(o), _fp(a), _fp(r), _fp(nx), _fp(d), fr.ctypes.data_as(C.POINTER(C.c_int32))))
        return {"obs": o, "act": a, "rew": float(r[0]), "next_obs": nx, "done": float(d[0]), "frames": (int(fr[0]), int(fr[1]))}


def transition_replay_bytes(buffer_size: int, obs_dim: int, act_width: int, frame_capacity: Optional[int] = None) -> int:
    """Device bytes of the BDQ / DQN replay of that shape without allocating it (``act_width``: n_branches, 1 for DQN;
    ``frame_capacity`` None = two rows per slot); the prioritised-replay trees are not counted."""
    return int(_lib.load().b2g_transition_replay_bytes(int(buffer_size), int(obs_dim), int(act_width), int(frame_capacity or 0)))


class Learner(HandleLearner):
    _abi = "sac"
    _names = {n: "b2g_" + n for n in ("get_param", "set_param", "get_grad", "set_norm_stats", "obs_rms_set", "obs_rms_get",
                                      "upload_bytes", "replay_info")}

    def __init__(self, obs_shape: Sequence[int], n_act: int = 5, hidden: int = 64, batch_size: int = 64,
                 buffer_size: int = 100000, gamma: float = 0.99, tau: float = 0.005,
                 target_entropy: Optional[float] = None, seed: int = 0, precision: int = _lib.B2G_PREC_FP32_SIMT,
                 device: int = 0, rank: int = 0, nranks: int = 1, nccl_id: Optional[bytes] = None,
                 frame_capacity: Optional[int] = None, u8_planes: Sequence[int] = (), extractor: str = "augmented"):
        """frame_capacity / u8_planes: replay storage (include/b200grasp.h, b2g_replay_cfg).  None and () keep two fp32
        frames per replay slot; a smaller frame budget shares each obs with the previous row's next_obs when they are
        equal, and u8_planes lists image channels stored as one byte per pixel (values must be integers in [0, 255]).
        extractor: the CNN policy's feature extractor, "augmented" (create_augmented_nature_cnn(1): the last plane is the
        actuator feature) or "nature_cnn" (stable-baselines' plain nature_cnn over every plane; b2g_sac_net_cfg)."""
        if extractor not in _lib.EXTRACTORS:
            raise ValueError(f"extractor must be one of {sorted(_lib.EXTRACTORS)} (got {extractor!r})")
        self.extractor = extractor
        self.lib = _lib.load()
        self.obs_shape = tuple(int(s) for s in obs_shape)
        self.n_act, self.batch_size = int(n_act), int(batch_size)
        cfg = _lib.SacCfg()
        if len(self.obs_shape) == 3:
            cfg.obs_h, cfg.obs_w, cfg.obs_c = self.obs_shape
            cfg.obs_dim = 0
        elif len(self.obs_shape) == 1:
            cfg.obs_h = cfg.obs_w = cfg.obs_c = 0
            cfg.obs_dim = self.obs_shape[0]
        else:
            raise ValueError(f"unsupported observation shape {obs_shape}")
        cfg.n_act, cfg.hidden, cfg.batch, cfg.buffer_capacity = n_act, hidden, batch_size, buffer_size
        cfg.gamma, cfg.tau = gamma, tau
        cfg.target_entropy = float(-n_act if target_entropy is None else target_entropy)
        cfg.seed, cfg.precision, cfg.device, cfg.rank, cfg.nranks = seed, precision, device, rank, nranks
        self._id_buf, cfg.nccl_id, cfg.nccl_lib = nccl_config(nranks, nccl_id)
        self.h = C.c_void_p()
        self.frame_capacity = None if frame_capacity is None else int(frame_capacity)
        self.u8_planes = tuple(int(c) for c in u8_planes)
        rcfg = None
        if self.frame_capacity is not None or self.u8_planes:
            if any(not 0 <= c < 32 for c in self.u8_planes):
                raise ValueError(f"u8_planes must be channel indices (got {self.u8_planes})")
            rcfg = _lib.ReplayCfg(2 * int(buffer_size) if self.frame_capacity is None else self.frame_capacity,
                                  sum(1 << c for c in set(self.u8_planes)))
        ncfg = _lib.SacNetCfg(_lib.EXTRACTORS[extractor])
        _lib.check(self.lib.b2g_sac_create3(C.byref(cfg), None if rcfg is None else C.byref(rcfg), C.byref(ncfg), C.byref(self.h)))
        self.obs_elems = int(np.prod(self.obs_shape))
        self._info = OrderedDict()
        name, numel, ndim = C.c_char_p(), C.c_int64(), C.c_int32()
        shape = (C.c_int64 * 4)()
        for i in range(self.lib.b2g_param_count(self.h)):
            _lib.check(self.lib.b2g_param_info(self.h, i, C.byref(name), C.byref(numel), C.byref(ndim), shape))
            self._info[name.value.decode()] = tuple(int(shape[k]) for k in range(ndim.value))

    # ---- peer-memory data parallelism (include/b200grasp.h: b2g_sac_dp_export / b2g_sac_dp_connect)
    DP_EXPORT_BYTES = 192

    def dp_export(self) -> bytes:
        buf = C.create_string_buffer(self.DP_EXPORT_BYTES)
        _lib.check(self.lib.b2g_sac_dp_export(self.h, C.cast(buf, C.c_void_p)))
        return buf.raw

    def dp_connect(self, exports: "list[bytes]"):
        """exports: the dp_export() blob of every rank, in rank order.  From here on the optimiser launch of each step reduces
        the gradients, updates this rank's slice and writes the new parameters into every replica through NVLink peer memory."""
        blob = b"".join(exports)
        if len(blob) != self.DP_EXPORT_BYTES * len(exports):
            raise ValueError("every export blob must be DP_EXPORT_BYTES long")
        buf = C.create_string_buffer(blob, len(blob))
        _lib.check(self.lib.b2g_sac_dp_connect(self.h, C.cast(buf, C.c_void_p), len(exports)))

    def dp_connect_torch(self):
        """dp_export + all_gather over the initialised torch.distributed process group + dp_connect."""
        import torch.distributed as dist
        blobs = [None] * dist.get_world_size()
        dist.all_gather_object(blobs, self.dp_export())
        self.dp_connect(blobs)
        dist.barrier()

    @staticmethod
    def nccl_unique_id() -> bytes:
        lib = _lib.load()
        buf = C.create_string_buffer(128)
        p = _lib.default_nccl_lib()
        _lib.check(lib.b2g_nccl_unique_id(C.cast(buf, C.c_void_p), p.encode() if p else None))
        return buf.raw

    def _has_grad(self, name):
        return not name.startswith("target/")

    def get_adam(self, name: str):
        shp = self._info[name]
        m, v = np.empty(shp, np.float32), np.empty(shp, np.float32)
        _lib.check(self.lib.b2g_get_adam(self.h, name.encode(), _fp(m.reshape(-1)), _fp(v.reshape(-1)), m.size))
        return m, v

    def reset_optimizer(self):
        _lib.check(self.lib.b2g_reset_optimizer(self.h))

    # ---- replay
    def replay_add(self, obs, act, rew, next_obs, done):
        obs, next_obs, act = _f32(obs), _f32(next_obs), _f32(act)
        rew, done = _f32(np.reshape(rew, -1)), _f32(np.reshape(done, -1))
        n = rew.shape[0]
        assert obs.size == n * self.obs_elems and next_obs.size == obs.size and act.size == n * self.n_act
        _lib.check(self.lib.b2g_replay_add(self.h, _fp(obs), _fp(act), _fp(rew), _fp(next_obs), _fp(done), n))

    def replay_size(self) -> int:
        return int(self.lib.b2g_replay_size(self.h))

    def replay_get(self, slot: int) -> dict:
        """One stored (raw) transition, like ``ReplayBuffer.storage[slot]``."""
        obs, nxt = np.empty(self.obs_shape, np.float32), np.empty(self.obs_shape, np.float32)
        act, rew, done = np.empty(self.n_act, np.float32), np.empty(1, np.float32), np.empty(1, np.float32)
        _lib.check(self.lib.b2g_replay_get(self.h, int(slot), _fp(obs.reshape(-1)), _fp(act), _fp(rew), _fp(nxt.reshape(-1)), _fp(done)))
        return dict(obs=obs, act=act, rew=float(rew[0]), next_obs=nxt, done=float(done[0]))

    def last_batch(self) -> dict:
        """Replay slots, policy noise and per-sample outputs of the LAST gradient step (graph path included)."""
        B = self.batch_size
        idx = np.empty(B, np.int32)
        eps, ps, pi = np.empty((B, self.n_act), np.float32), np.empty((7, B), np.float32), np.empty((B, self.n_act), np.float32)
        _lib.check(self.lib.b2g_get_last_batch(self.h, idx.ctypes.data_as(C.POINTER(C.c_int32)), _fp(eps.reshape(-1)),
                                               _fp(ps.reshape(-1)), _fp(pi.reshape(-1))))
        out = dict(indices=idx, eps=eps, pi=pi)
        for i, k in enumerate(("q1", "q2", "v", "logp", "v_targ", "q1_pi", "q2_pi")):
            out[k] = ps[i].copy()
        return out

    # ---- the actor loop on one upload per frame (include/b200grasp.h: b2g_sac_observe_*)
    def observe_act(self, obs, n=None, update_stats=True, deterministic=False, act=True):
        """``obs``: n raw observations to upload, merge into ``obs_rms`` (``update_stats``) and stage as the current
        observation of env i; ``None`` acts on the ones already staged.  Returns the n actions, or None with ``act=False``."""
        if obs is not None:
            obs = _f32(obs).reshape(-1, self.frame_elems)
            n = obs.shape[0]
            self.obs_rms_version += bool(update_stats)
        out = np.empty((int(n), self.n_act), np.float32) if act else None
        _lib.check(self.lib.b2g_sac_observe_act(self.h, None if obs is None else _fp(obs), int(n), int(bool(update_stats)),
                                                int(deterministic), None if out is None else _fp(out)))
        return out

    def observe_add(self, act, rew, next_obs, done, reset_obs=None, update_stats=True):
        """Transition i = (staged obs_i, act_i, rew_i, next_obs_i, done_i); ``reset_obs`` holds, for every finished env,
        the frame its auto-reset returned (the other rows are not read)."""
        act, next_obs = _f32(act), _f32(next_obs)
        rew, done = _f32(np.reshape(rew, -1)), _f32(np.reshape(done, -1))
        n = rew.shape[0]
        assert next_obs.size == n * self.frame_elems and act.size == n * self.n_act and done.size == n
        if reset_obs is not None:
            reset_obs = _f32(reset_obs)
            assert reset_obs.size == next_obs.size
        _lib.check(self.lib.b2g_sac_observe_add(self.h, _fp(act), _fp(rew), _fp(next_obs), _fp(done),
                                                None if reset_obs is None else _fp(reset_obs), n, int(bool(update_stats))))
        self.obs_rms_version += bool(update_stats)

    # ---- hot path
    def step(self, n_steps: int = 1, lr: float = 3e-4) -> dict:
        m = _lib.SacMetrics()
        _lib.check(self.lib.b2g_sac_step(self.h, n_steps, lr, C.byref(m)))
        return m.as_dict()

    def step_async(self, n_steps: int = 1, lr: float = 3e-4):
        _lib.check(self.lib.b2g_sac_step_async(self.h, n_steps, lr))

    def sync(self):
        _lib.check(self.lib.b2g_sync(self.h))

    def step_explicit(self, obs, act, rew, next_obs, done, eps, lr: float = 3e-4, apply_update: bool = True):
        B = self.batch_size
        obs, next_obs, act, eps = _f32(obs), _f32(next_obs), _f32(act), _f32(eps)
        rew, done = _f32(np.reshape(rew, -1)), _f32(np.reshape(done, -1))
        assert obs.size == B * self.obs_elems and act.size == B * self.n_act and eps.size == B * self.n_act and rew.size == B
        ps = np.empty((7, B), np.float32)
        pi = np.empty((B, self.n_act), np.float32)
        m = _lib.SacMetrics()
        _lib.check(self.lib.b2g_sac_step_explicit(self.h, _fp(obs), _fp(act), _fp(rew), _fp(next_obs), _fp(done), _fp(eps),
                                                   lr, int(apply_update), C.byref(m), _fp(ps), _fp(pi)))
        out = m.as_dict()
        for i, k in enumerate(("q1", "q2", "v", "logp", "v_targ", "q1_pi", "q2_pi")):
            out[k] = ps[i].copy()
        out["pi"] = pi
        return out

    def step_host_pipelined(self, obs, act, rew, next_obs, done, eps, lr: float = 3e-4):
        """Enqueue one step on a HOST batch (arrays must stay alive until the next call / flush; pinned float32
        arrays overlap the copy with the previous step).  Returns the previous step's losses, or None."""
        B = self.batch_size
        arrs = [_f32(obs), _f32(act), _f32(np.reshape(rew, -1)), _f32(next_obs), _f32(np.reshape(done, -1)), _f32(eps)]
        assert arrs[0].size == B * self.obs_elems and arrs[1].size == B * self.n_act and arrs[2].size == B
        self._pipe_keep = (getattr(self, "_pipe_keep", ()) + (arrs,))[-2:]   # host buffers stay alive while copies fly
        m, have = _lib.SacMetrics(), C.c_int(0)
        _lib.check(self.lib.b2g_sac_step_host_pipelined(self.h, *[_fp(a) for a in arrs], lr, C.byref(m), C.byref(have)))
        return m.as_dict() if have.value else None

    def pipeline_flush(self) -> dict:
        m = _lib.SacMetrics()
        _lib.check(self.lib.b2g_sac_pipeline_flush(self.h, C.byref(m)))
        return m.as_dict()

    def act(self, obs, deterministic: bool = True) -> np.ndarray:
        obs = _f32(obs).reshape(-1, self.obs_elems)
        out = np.empty((obs.shape[0], self.n_act), np.float32)
        _lib.check(self.lib.b2g_sac_act(self.h, _fp(obs), obs.shape[0], int(deterministic), _fp(out)))
        return out

    def launches_per_step(self) -> int:
        return int(self.lib.b2g_launches_per_step(self.h))

    def last_step_ms(self) -> float:
        return float(self.lib.b2g_last_step_ms(self.h))

    def profile_step(self, lr: float = 3e-4) -> "OrderedDict[str, float]":
        cap = 64
        names = (C.c_char_p * cap)()
        ms = (C.c_float * cap)()
        n = _lib.check(self.lib.b2g_profile_step(self.h, lr, names, ms, cap))
        return OrderedDict((names[i].decode(), float(ms[i])) for i in range(n))
