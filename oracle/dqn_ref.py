"""PyTorch-CPU restatement of the stable-baselines 2.10.1 dueling double DQN step.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  The reference trains DQN through ``sb.DQN(DQNMlpPolicy, env, gamma,
batch_size, prioritized_replay)`` (/root/reference/manipulation_main/training/sb_helper.py:155-165) with stable-baselines
2.10.1 (setup.py:7), whose source is not in the tree.  This restates deepq/policies.py ``FeedForwardPolicy`` (dueling=True,
layers=[64, 64], ReLU, no layer norm), deepq/build_graph.py ``build_train`` (double_q=True, grad_norm_clipping=10 as dqn.py
passes it, tf_util.huber_loss) and the TF1 Adam that follows.

What trained_models/DQN_4pads/DQN_simple_4pads.zip pins:
  * the variable names and shapes (``all_specs``: deepq/eps, the online net, the target net, in the zip's order);
  * the ``data`` hyper-parameters (``ZIP_DATA``), among them gamma 1.0, batch 32, learning_rate 5e-4 and prioritized_replay;
  * the spaces: Discrete(12) actions, Box(-1, 1, (100,)) observations.
The network, loss, clipping and optimiser are the library's code paths for those values, restated here, not pinned by the zip.

  Q(s)  = V(s) + (A(s) - mean_n A(s))                   two towers obs -> h0 -> h1 -> {n, 1}, each with its own first layer
  a*    = argmax_n Q_online(s'),  y = r + gamma (1 - done) Q_target(s', a*)
  td    = Q(s, a) - y;  loss = mean_b w_b huber(td_b),  huber(x) = 0.5 x^2 (|x| < 1) else |x| - 0.5
  g     <- g * 10 / max(||g||_2, 10)  per variable (tf.clip_by_norm), then TF1 Adam (b1 .9, b2 .999, eps 1e-8)
  new priorities |td| + 1e-6
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass
from typing import Dict, Tuple

import numpy as np
import torch
import torch.nn.functional as F

ADAM_B1, ADAM_B2, ADAM_EPS = 0.9, 0.999, 1e-8
GRAD_CLIP = 10.0
PER_EPS = 1e-6
ONLINE, TARGET = "deepq/model", "deepq/target_q_func/model"

#: the zip's ``data`` hyper-parameters (stable-baselines 2.10 does not save buffer_size; its default is 50000)
ZIP_DATA = dict(double_q=True, param_noise=False, learning_starts=1000, train_freq=1, batch_size=32, target_network_update_freq=500,
                prioritized_replay=True, prioritized_replay_alpha=0.6, prioritized_replay_beta0=0.4, prioritized_replay_beta_iters=None,
                prioritized_replay_eps=1e-6, exploration_fraction=0.1, exploration_final_eps=0.02, learning_rate=5e-4, gamma=1.0,
                policy_kwargs={})


@dataclass
class DQNConfig:
    obs_dim: int = 100
    n_actions: int = 12
    layers: Tuple[int, int] = (64, 64)
    gamma: float = 1.0


def _fc(i: int) -> str:
    return "fully_connected" if i == 0 else f"fully_connected_{i}"


def param_specs(cfg: DQNConfig, scope: str = ONLINE):
    """(name, shape) of one network in the zip's order: per tower, per layer, weights then biases."""
    out = []
    for tower, n_out in (("action_value", cfg.n_actions), ("state_value", 1)):
        dims = [cfg.obs_dim, cfg.layers[0], cfg.layers[1], n_out]
        for k in range(3):
            out.append((f"{scope}/{tower}/{_fc(k)}/weights", (dims[k], dims[k + 1])))
            out.append((f"{scope}/{tower}/{_fc(k)}/biases", (dims[k + 1],)))
    return out


def all_specs(cfg: DQNConfig):
    return [("deepq/eps", ())] + param_specs(cfg, ONLINE) + param_specs(cfg, TARGET)


def init_params(cfg: DQNConfig, seed: int = 0) -> "OrderedDict[str, np.ndarray]":
    """Xavier-uniform weights and zero biases (tf.contrib.layers.fully_connected), target = online, deepq/eps 0."""
    rng = np.random.default_rng(seed)
    p = OrderedDict()
    p["deepq/eps"] = np.float32(0.0)
    for name, shape in param_specs(cfg, ONLINE):
        if name.endswith("weights"):
            lim = np.sqrt(6.0 / (shape[0] + shape[1]))
            p[name] = rng.uniform(-lim, lim, shape).astype(np.float32)
        else:
            p[name] = np.zeros(shape, np.float32)
    for name, _ in param_specs(cfg, ONLINE):
        p[name.replace(ONLINE, TARGET)] = p[name].copy()
    return p


def q_values(p: Dict[str, torch.Tensor], obs: torch.Tensor, scope: str = ONLINE) -> torch.Tensor:
    """Q [B, n] of the network under ``scope``."""
    outs = []
    for tower in ("action_value", "state_value"):
        h = obs
        for k in range(2):
            h = F.relu(h @ p[f"{scope}/{tower}/{_fc(k)}/weights"] + p[f"{scope}/{tower}/{_fc(k)}/biases"])
        outs.append(h @ p[f"{scope}/{tower}/{_fc(2)}/weights"] + p[f"{scope}/{tower}/{_fc(2)}/biases"])
    a, v = outs
    return v + (a - a.mean(1, keepdim=True))


def huber(x):
    return torch.where(x.abs() < 1.0, 0.5 * x * x, x.abs() - 0.5)


def clip_by_norm(g: np.ndarray, clip: float = GRAD_CLIP):
    """tf.clip_by_norm: g * clip / max(||g||_2, clip) -> (clipped, norm before)"""
    n = float(np.sqrt((np.asarray(g, np.float64) ** 2).sum()))
    return (g * clip / max(n, clip)).astype(g.dtype), n


def dqn_step(params: Dict[str, np.ndarray], opt, batch: Dict[str, np.ndarray], lr: float, cfg: DQNConfig, dtype=torch.float64,
             a_star=None):
    """One train step.  batch: obs [B,obs], act [B] (ints), rew [B], next_obs, done [B], weights [B] (IS weights; ones without
    prioritised replay).  ``opt`` = dict(m, v, t).  ``a_star`` [B] (optional) replaces the online net's argmax at s' -- for rows
    whose top two Q values fp32 cannot order.  -> (outputs, clipped grads, new params, new opt); outputs hold loss, td, q,
    mean_q, mean_abs_td, priorities, grads_pre (before the clip), norms (per tensor), grad_norm (global, before the clip) and
    n_clipped."""
    np_dt = np.float64 if dtype == torch.float64 else np.float32
    tp = {n: torch.tensor(np.asarray(a, np_dt), dtype=dtype, requires_grad=n.startswith(ONLINE + "/")) for n, a in params.items()}
    obs = torch.tensor(np.asarray(batch["obs"], np_dt), dtype=dtype)
    nxt = torch.tensor(np.asarray(batch["next_obs"], np_dt), dtype=dtype)
    act = torch.tensor(np.asarray(batch["act"], np.int64).reshape(-1))
    rew = torch.tensor(np.asarray(batch["rew"], np_dt), dtype=dtype)
    done = torch.tensor(np.asarray(batch["done"], np_dt), dtype=dtype)
    w = torch.tensor(np.asarray(batch.get("weights", np.ones(len(rew))), np_dt), dtype=dtype)
    q = q_values(tp, obs, ONLINE)
    q_sa = q.gather(1, act.unsqueeze(1)).squeeze(1)
    with torch.no_grad():
        if a_star is None:
            a_star = q_values(tp, nxt, ONLINE).argmax(1)                   # online net selects
        else:
            a_star = torch.tensor(np.asarray(a_star, np.int64))
        q_t = q_values(tp, nxt, TARGET).gather(1, a_star.unsqueeze(1)).squeeze(1)
        y = rew + cfg.gamma * (1 - done) * q_t
    td = q_sa - y
    loss = (w * huber(td)).mean()
    names = [n for n, _ in param_specs(cfg, ONLINE)]
    gl = torch.autograd.grad(loss, [tp[n] for n in names])
    pre = {n: g.detach().numpy().astype(np_dt) for n, g in zip(names, gl)}
    grads, norms = {}, {}
    for n in names:
        grads[n], norms[n] = clip_by_norm(pre[n])
    new_p = OrderedDict((n, np.asarray(a, np_dt).copy()) for n, a in params.items())
    t = opt["t"] + 1
    lr_t = np_dt(lr) * np.sqrt(np_dt(1) - np_dt(ADAM_B2) ** t) / (np_dt(1) - np_dt(ADAM_B1) ** t)
    new_opt = {"t": t, "m": {}, "v": {}}
    for n in names:
        m = (ADAM_B1 * opt["m"].get(n, 0.0) + (1 - ADAM_B1) * grads[n]).astype(np_dt)
        v = (ADAM_B2 * opt["v"].get(n, 0.0) + (1 - ADAM_B2) * grads[n] ** 2).astype(np_dt)
        new_opt["m"][n], new_opt["v"][n] = m, v
        new_p[n] = (new_p[n] - lr_t * m / (np.sqrt(v) + np_dt(ADAM_EPS))).astype(np_dt)
    tdn = td.detach().numpy()
    out = dict(loss=float(loss.detach()), td=tdn, q=q.detach().numpy(), q_sa=q_sa.detach().numpy(), y=y.numpy(), a_star=a_star.numpy(),
               mean_q=float(q_sa.detach().mean()), mean_abs_td=float(np.abs(tdn).mean()), priorities=np.abs(tdn) + PER_EPS,
               grads_pre=pre, norms=norms, grad_norm=float(np.sqrt(sum(v * v for v in norms.values()))),
               n_clipped=int(sum(v > GRAD_CLIP for v in norms.values())))
    return out, grads, new_p, new_opt


def hard_target_update(params):
    for n in list(params):
        if n.startswith(ONLINE + "/"):
            params[n.replace(ONLINE, TARGET)] = np.array(params[n], copy=True)
    return params


def greedy_action(params, obs):
    """argmax_n Q (float64) and the Q rows."""
    tp = {n: torch.tensor(np.asarray(a, np.float64)) for n, a in params.items()}
    q = q_values(tp, torch.tensor(np.asarray(obs, np.float64)), ONLINE).numpy()
    return q.argmax(1), q


def softmax_action(q_rows, uniforms):
    """deepq policy step(deterministic=False): per row, numpy's choice(n, p=softmax(Q)) on the given uniform (inverse CDF)."""
    q = np.asarray(q_rows, np.float64)
    p = np.exp(q - q.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    out = np.empty(len(q), np.int64)
    for i in range(len(q)):
        cdf = np.cumsum(p[i])
        cdf /= cdf[-1]
        out[i] = int(np.searchsorted(cdf, uniforms[i], side="right"))
    return out, p
