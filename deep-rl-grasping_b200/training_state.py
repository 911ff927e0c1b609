"""Training-state directories: everything a stopped SAC / BDQ / DQN / PPO2 / TRPO run needs to continue where it stopped.

``<dir>/`` holds
  model.zip          the stable-baselines zip of ``model.save`` (parameters only, loadable on its own)
  learner.state      the device learner's file (include/b200grasp.h, b2g_sac_state_save / b2g_bdq_state_save): parameters,
                     Adam moments, counters and the whole replay
  vecnormalize.pkl   the VecNormalize statistics, when the model's env has a VecNormalize wrapper
  host.json          the host side: num_timesteps, episode bookkeeping, the numpy generator state and the constructor keywords

A directory is written as ``<dir>.tmp`` and swapped in only once every file is complete, so a writer that dies half way leaves
the previous checkpoint loadable.  The environment's own state is not saved: a resumed run starts a fresh episode.
"""
from __future__ import annotations

import json
import os
import shutil

FORMAT = 1
STATE_FILE, MODEL_FILE, VECNORM_FILE, HOST_FILE = "learner.state", "model.zip", "vecnormalize.pkl", "host.json"


def _json_default(o):
    import numpy as np
    if isinstance(o, np.integer):
        return int(o)
    if isinstance(o, np.floating):
        return float(o)
    if isinstance(o, np.ndarray):
        return o.tolist()
    raise TypeError(f"not JSON serialisable: {type(o).__name__}")


def save_training_state(model, path: str) -> str:
    """Writes ``model``'s training state to directory ``path`` (replaced atomically).  ``model`` provides ``save(path)``,
    ``learner.save_state(path)``, ``get_vec_normalize_env()`` and ``_host_state() -> dict``."""
    path = os.path.normpath(path)
    tmp, old = path + ".tmp", path + ".old"
    if os.path.exists(tmp):
        shutil.rmtree(tmp)
    os.makedirs(tmp)
    try:
        model.save(os.path.join(tmp, MODEL_FILE))
        model.learner.save_state(os.path.join(tmp, STATE_FILE))
        vn = model.get_vec_normalize_env()
        if vn is not None:
            vn.save(os.path.join(tmp, VECNORM_FILE))
        host = dict(model._host_state(), format=FORMAT)
        with open(os.path.join(tmp, HOST_FILE), "w") as f:
            json.dump(host, f, default=_json_default)
    except BaseException:
        shutil.rmtree(tmp, ignore_errors=True)
        raise
    # swap: between the two renames only <path>.old exists, and resolve() finds it there
    if os.path.exists(path):
        if os.path.exists(old):
            shutil.rmtree(old)
        os.rename(path, old)
        os.rename(tmp, path)
        shutil.rmtree(old)
    else:
        os.rename(tmp, path)
    return path


def resolve(path: str) -> str:
    """The checkpoint directory to read: ``path``, or ``<path>.old`` when a writer stopped between the two renames."""
    path = os.path.normpath(path)
    if os.path.isfile(os.path.join(path, HOST_FILE)):
        return path
    if os.path.isfile(os.path.join(path + ".old", HOST_FILE)):
        return path + ".old"
    raise FileNotFoundError(f"no training state in {path}")


def read_host(path: str) -> dict:
    with open(os.path.join(path, HOST_FILE)) as f:
        host = json.load(f)
    if host.get("format") != FORMAT:
        raise ValueError(f"{path}: unsupported training-state format {host.get('format')}")
    return host


def restore_vec_normalize(path: str, env) -> None:
    """Copies the saved VecNormalize statistics into ``env``'s own VecNormalize wrapper (when both exist)."""
    from .base_model import unwrap_vec_normalize
    from .vec_env import VecNormalize
    vn = unwrap_vec_normalize(env) if env is not None else None
    f = os.path.join(path, VECNORM_FILE)
    if vn is None or not os.path.exists(f):
        return
    saved = VecNormalize.load(f, vn.venv)
    vn.obs_rms, vn.ret_rms = saved.obs_rms, saved.ret_rms
    vn.clip_obs, vn.clip_reward, vn.gamma, vn.epsilon = saved.clip_obs, saved.clip_reward, saved.gamma, saved.epsilon
    vn.norm_obs, vn.norm_reward = saved.norm_obs, saved.norm_reward


def rng_state(rng) -> dict:
    return rng.bit_generator.state


def set_rng_state(rng, state: dict) -> None:
    rng.bit_generator.state = state
