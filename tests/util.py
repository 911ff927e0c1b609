"""Shared helpers for the parity tests: seeded batches from the committed fixtures."""
import os

import numpy as np

import b200grasp
from b200grasp import synth
from oracle import sac_ref as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_case(key):
    """key in {'sac_depth', 'sac_encoder'} -> (cfg, trained params, vecnormalize stats)."""
    vn = dict(np.load(os.path.join(GOLD, f"vecnorm_{key}.npz")))
    cfg = R.SACConfig(obs_shape=tuple(vn["obs_mean"].shape))
    raw = dict(np.load(os.path.join(GOLD, f"{key}_params.npz")))
    params = {n: raw[n] for n, _ in R.param_specs(cfg)}
    return cfg, params, vn


def _switch(vn, key):
    return bool(vn[key]) if key in vn else True


def normalize(tr, vn, idx=slice(None)):
    """What the learner feeds the step for the raw transitions ``tr[idx]`` under the VecNormalize statistics ``vn``: its own
    clip_obs, clip_reward and epsilon, and each of norm_obs / norm_reward (absent = on) switching its half off."""
    clip_o, clip_r, e = float(vn["clip_obs"]), float(vn["clip_reward"]), float(vn["epsilon"])

    def obs(o):
        if not _switch(vn, "norm_obs"):
            return np.asarray(o, np.float32)
        return R.normalize_obs(o, vn["obs_mean"], vn["obs_var"], clip=clip_o, eps=e)

    rew = tr["rew"][idx]
    if _switch(vn, "norm_reward"):
        rew = R.normalize_reward(rew, float(vn["ret_var"]), clip=clip_r, eps=e)
    return dict(obs=obs(tr["obs"][idx]), next_obs=obs(tr["next_obs"][idx]), act=tr["act"][idx],
                rew=np.asarray(rew, np.float32), done=tr["done"][idx])


def make_batch(vn, B, seed=synth.DATA_SEED, n_act=5):
    raw = synth.make_transitions(B, vn["obs_mean"], vn["obs_var"], seed=seed, n_act=n_act)
    return raw, normalize(raw, vn), synth.make_eps(B, n_act=n_act, seed=seed + 1)


def make_learner(cfg, vn, B, params=None, buffer_size=1024, precision=0, **kw):
    L = b200grasp.Learner(cfg.obs_shape, n_act=cfg.n_act, batch_size=B, buffer_size=buffer_size, gamma=cfg.gamma,
                          tau=cfg.tau, target_entropy=cfg.target_entropy, precision=precision, **kw)
    L.set_norm_stats(vn["obs_mean"], vn["obs_var"], float(vn["ret_var"]), float(vn["clip_obs"]), float(vn["clip_reward"]),
                     float(vn["epsilon"]), norm_obs=_switch(vn, "norm_obs"), norm_reward=_switch(vn, "norm_reward"))
    if params is not None:
        L.load_parameters(params)
    return L


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))
