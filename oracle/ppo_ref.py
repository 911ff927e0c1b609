"""float64 restatement of the stable-baselines 2.10.1 PPO2 update with ``common.policies.MlpPolicy``.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  The reference builds PPO through ``sb.PPO2(MlpPolicy, env, verbose=2,
gamma=..., learning_rate=config['PPO']['learning_rate'])`` (/root/reference/manipulation_main/training/sb_helper.py:137-154)
and runs ``algorithm: ppo`` zips through ``sb.PPO2.load`` (train_stable_baselines.py:99-100).  The stable-baselines source is
not in the reference tree and no PPO zip is shipped, so nothing in the reference pins the algorithm, the variable names or the
defaults below: they are restated from stable-baselines 2.10.1 (ppo2/ppo2.py, common/policies.py, common/distributions.py).

  policy   FeedForwardPolicy, net_arch=[dict(pi=[h0, h1], vf=[h0, h1])], tanh; obs cast to float32 and flattened (no /255)
           pi: tanh(tanh(x W_pi0 + b) W_pi1 + b) W_pi + b = mean;  vf: ... W_vf + b = value;  pi/logstd [1, A] (zeros);
           q (vf latent -> A) exists and is never trained
  init     orthogonal: sqrt(2) hidden layers, 1 vf, 0.01 pi and q; zero biases
  neglogp  0.5 sum((a - mean) / std)^2 + 0.5 log(2 pi) A + sum logstd;  entropy = sum(logstd + 0.5 log(2 pi e))
  GAE      delta = r + gamma V' (1 - d') - V,  adv = delta + gamma lam (1 - d') adv',  returns = adv + V
  loss     adv normalised over the minibatch (population std, + 1e-8);  ratio = exp(old_nlp - nlp)
           pg = mean max(-adv ratio, -adv clip(ratio, 1 +- c));  vf = 0.5 mean max((v - R)^2, (v_clip - R)^2),
           v_clip = old_v + clip(v - old_v, +- c_vf) (no clip when c_vf < 0);  loss = pg - ent_coef entropy + vf_coef vf
  step     tf.clip_by_global_norm(max_grad_norm), then TF1 Adam (b1 .9, b2 .999, epsilon 1e-5)
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict

import numpy as np
import torch

ADAM_B1, ADAM_B2, ADAM_EPS = 0.9, 0.999, 1e-5
HALF_LOG_2PI = 0.5 * np.log(2.0 * np.pi)
HALF_LOG_2PIE = 0.5 * np.log(2.0 * np.pi * np.e)
SCOPE = "model/"
TRAINED = ("pi_fc0/w", "pi_fc0/b", "vf_fc0/w", "vf_fc0/b", "pi_fc1/w", "pi_fc1/b", "vf_fc1/w", "vf_fc1/b", "vf/w", "vf/b", "pi/w",
           "pi/b", "pi/logstd")


def param_specs(obs_dim: int, n_actions: int, layers=(64, 64)):
    """(name, shape) in creation order under model/ (the order of the zip's parameter_list)."""
    h0, h1 = layers
    return [("model/pi_fc0/w", (obs_dim, h0)), ("model/pi_fc0/b", (h0,)), ("model/vf_fc0/w", (obs_dim, h0)), ("model/vf_fc0/b", (h0,)),
            ("model/pi_fc1/w", (h0, h1)), ("model/pi_fc1/b", (h1,)), ("model/vf_fc1/w", (h0, h1)), ("model/vf_fc1/b", (h1,)),
            ("model/vf/w", (h1, 1)), ("model/vf/b", (1,)), ("model/pi/w", (h1, n_actions)), ("model/pi/b", (n_actions,)),
            ("model/pi/logstd", (1, n_actions)), ("model/q/w", (h1, n_actions)), ("model/q/b", (n_actions,))]


def ortho(shape, scale, rng):
    """common/tf_layers.py ortho_init: the orthogonal factor of an SVD of a standard normal matrix, times scale."""
    a = rng.normal(0.0, 1.0, shape)
    u, _, v = np.linalg.svd(a, full_matrices=False)
    w = u if u.shape == tuple(shape) else v
    return (scale * w.reshape(shape)).astype(np.float32)


def init_params(obs_dim, n_actions, layers=(64, 64), rng=None) -> "OrderedDict[str, np.ndarray]":
    rng = rng if rng is not None else np.random.default_rng(0)
    p = OrderedDict()
    for name, shape in param_specs(obs_dim, n_actions, layers):
        short = name[len(SCOPE):]
        if short == "pi/logstd" or len(shape) == 1:
            p[name] = np.zeros(shape, np.float32)
        else:
            scale = 1.0 if short == "vf/w" else (0.01 if short in ("pi/w", "q/w") else np.sqrt(2.0))
            p[name] = ortho(shape, scale, rng)
    return p


def _t(x):
    return torch.as_tensor(np.asarray(x), dtype=torch.float64)


def forward(params, obs):
    """-> mean [n, A], value [n] (float64 numpy)."""
    P = {k[len(SCOPE):] if k.startswith(SCOPE) else k: _t(v) for k, v in params.items()}
    with torch.no_grad():
        mean, v = _forward(P, _t(obs).reshape(len(obs), -1))
    return mean.numpy(), v.numpy()


def _forward(P, x):
    hp = torch.tanh(torch.tanh(x @ P["pi_fc0/w"] + P["pi_fc0/b"]) @ P["pi_fc1/w"] + P["pi_fc1/b"])
    hv = torch.tanh(torch.tanh(x @ P["vf_fc0/w"] + P["vf_fc0/b"]) @ P["vf_fc1/w"] + P["vf_fc1/b"])
    return hp @ P["pi/w"] + P["pi/b"], (hv @ P["vf/w"] + P["vf/b"])[:, 0]


def neglogp(mean, logstd, act):
    mean, act, logstd = np.asarray(mean, np.float64), np.asarray(act, np.float64), np.asarray(logstd, np.float64).reshape(-1)
    z = (act - mean) / np.exp(logstd)
    return 0.5 * (z * z).sum(-1) + HALF_LOG_2PI * act.shape[-1] + logstd.sum()


def entropy(logstd):
    logstd = np.asarray(logstd, np.float64).reshape(-1)
    return float((logstd + HALF_LOG_2PIE).sum())


def gae(rewards, values, dones, last_values, last_dones, gamma, lam):
    """ppo2.py Runner._run: rewards / values / dones [n_steps, n_envs] (dones[t] = episode-start flags of step t), last_values
    and last_dones [n_envs] -> advantages, returns [n_steps, n_envs] (float64)."""
    r, v, d = (np.asarray(x, np.float64) for x in (rewards, values, dones))
    T = r.shape[0]
    adv = np.zeros_like(r)
    last = 0.0
    for t in reversed(range(T)):
        if t == T - 1:
            nnt, nv = 1.0 - np.asarray(last_dones, np.float64), np.asarray(last_values, np.float64)
        else:
            nnt, nv = 1.0 - d[t + 1], v[t + 1]
        delta = r[t] + gamma * nv * nnt - v[t]
        adv[t] = last = delta + gamma * lam * nnt * last
    return adv, adv + v


def swap_and_flatten(a):
    """[n_steps, n_envs, ...] -> [n_envs * n_steps, ...] env-major (ppo2.py swap_and_flatten)."""
    a = np.asarray(a)
    s = a.shape
    return a.swapaxes(0, 1).reshape(s[0] * s[1], *s[2:])


def loss_and_grads(params, obs, returns, actions, values, old_nlp, cliprange, cliprange_vf=None, ent_coef=0.01, vf_coef=0.5):
    """ppo2.py _train_step's graph on one minibatch -> (loss, metrics dict, OrderedDict of float64 gradients of the trained
    variables).  cliprange_vf None uses cliprange; a negative value turns value clipping off."""
    names = [SCOPE + n for n in TRAINED]
    P = {k[len(SCOPE):]: _t(v).clone().requires_grad_(k in names) for k, v in params.items()}
    x = _t(obs).reshape(len(obs), -1)
    R, A, V0, NLP0 = _t(returns).reshape(-1), _t(actions).reshape(len(obs), -1), _t(values).reshape(-1), _t(old_nlp).reshape(-1)
    mean, v = _forward(P, x)
    logstd = P["pi/logstd"].reshape(-1)
    adv = R - V0
    adv = (adv - adv.mean()) / (adv.std(unbiased=False) + 1e-8)
    z = (A - mean) / torch.exp(logstd)
    nlp = 0.5 * (z * z).sum(-1) + HALF_LOG_2PI * A.shape[1] + logstd.sum()
    ent = (logstd + HALF_LOG_2PIE).sum()
    ratio = torch.exp(NLP0 - nlp)
    pg = torch.maximum(-adv * ratio, -adv * torch.clamp(ratio, 1.0 - cliprange, 1.0 + cliprange)).mean()
    cvf = cliprange if cliprange_vf is None else cliprange_vf
    vc = v if cvf < 0 else V0 + torch.clamp(v - V0, -cvf, cvf)
    vf = 0.5 * torch.maximum((v - R) ** 2, (vc - R) ** 2).mean()
    loss = pg - ent_coef * ent + vf_coef * vf
    loss.backward()
    with torch.no_grad():
        kl = 0.5 * ((nlp - NLP0) ** 2).mean()
        cf = ((ratio - 1.0).abs() > cliprange).double().mean()
    grads = OrderedDict((SCOPE + n, P[n].grad.numpy().copy()) for n in TRAINED)
    met = dict(policy_loss=pg.item(), value_loss=vf.item(), entropy=ent.item(), approxkl=kl.item(), clipfrac=cf.item())
    return loss.item(), met, grads


def clip_global(grads, max_norm):
    """tf.clip_by_global_norm -> (clipped grads, global norm)."""
    norm = float(np.sqrt(sum(float((g * g).sum()) for g in grads.values())))
    s = max_norm / max(norm, max_norm)
    return OrderedDict((k, g * s) for k, g in grads.items()), norm


class Adam:
    """TF1 AdamOptimizer(epsilon=1e-5) over the trained variables, float64."""

    def __init__(self):
        self.t, self.m, self.v = 0, {}, {}

    def step(self, params, grads, lr):
        self.t += 1
        lr_t = lr * np.sqrt(1.0 - ADAM_B2 ** self.t) / (1.0 - ADAM_B1 ** self.t)
        out = OrderedDict((k, np.asarray(a, np.float64).copy()) for k, a in params.items())
        for k, g in grads.items():
            m = self.m.get(k, np.zeros_like(g)) * ADAM_B1 + (1 - ADAM_B1) * g
            v = self.v.get(k, np.zeros_like(g)) * ADAM_B2 + (1 - ADAM_B2) * g * g
            self.m[k], self.v[k] = m, v
            out[k] = out[k] - lr_t * m / (np.sqrt(v) + ADAM_EPS)
        return out


def train_step(params, opt: Adam, obs, returns, actions, values, old_nlp, lr, cliprange, cliprange_vf=None, ent_coef=0.01,
               vf_coef=0.5, max_grad_norm=0.5):
    """One minibatch step -> (new params, metrics incl. grad_norm, clipped grads)."""
    _, met, g = loss_and_grads(params, obs, returns, actions, values, old_nlp, cliprange, cliprange_vf, ent_coef, vf_coef)
    gc, norm = clip_global(g, max_grad_norm)
    met["grad_norm"] = norm
    return opt.step(params, gc, lr), met, gc


def update(params, opt: Adam, obs, returns, actions, values, old_nlp, perms, nminibatches, lr, cliprange, cliprange_vf=None,
           ent_coef=0.01, vf_coef=0.5, max_grad_norm=0.5):
    """ppo2.py's update loop over flattened (env-major) rollout arrays: for each epoch's permutation, contiguous minibatches of
    n_batch // nminibatches rows -> (params, mean metrics)."""
    n_batch = len(returns)
    mb = n_batch // nminibatches
    mets = []
    for perm in perms:
        for s in range(0, n_batch, mb):
            i = np.asarray(perm[s:s + mb])
            params, met, _ = train_step(params, opt, obs[i], returns[i], actions[i], values[i], old_nlp[i], lr, cliprange, cliprange_vf,
                                        ent_coef, vf_coef, max_grad_norm)
            mets.append(met)
    return params, {k: float(np.mean([m[k] for m in mets])) for k in mets[0]}


def as_float64(params) -> Dict[str, np.ndarray]:
    return OrderedDict((k, np.asarray(v, np.float64)) for k, v in params.items())


__all__ = ["param_specs", "init_params", "forward", "neglogp", "entropy", "gae", "swap_and_flatten", "loss_and_grads", "clip_global",
           "Adam", "train_step", "update", "ortho"]
