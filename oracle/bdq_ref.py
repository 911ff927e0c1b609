"""PyTorch-CPU restatement of the branching dueling Q-network (BDQ) minibatch step.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  PARITY UNPINNED: the reference's BDQ lives in the
author's stable-baselines fork ``bdq_sb``, declared at /root/reference/.gitmodules:1-3 and ABSENT from the
tree; call sites: manipulation_main/training/train_stable_baselines.py:103-104, sb_helper.py:202-226;
hyper-parameters: config/gripper_grasp.yaml:104-118, config/simplified_object_picking.yaml:108-122.
What follows restates the published algorithm (Tavakoli, Pardo, Kormushev: "Action Branching Architectures
for Deep Reinforcement Learning", AAAI-18; code acknowledged at README.md:135) with the variable names and
shapes of the shipped zips (trained_models/BDQ_8pads, BDQ_33pads_big; SURVEY.md Appendix C):

  trunk   : bdq/model/common_net/fully_connected{,_1}          ReLU FC x2
  branch d: bdq/model/action_value/fully_connected_{2d,2d+1}   ReLU FC -> n advantages A_d
  value   : bdq/model/state_value/fully_connected{,_1}         ReLU FC -> V
  Q_d = V + A_d - mean_n(A_d)                                   (dueling, local mean)
  double-Q: a*_d = argmax_n Q_d^online(s'),  y = r + gamma (1-done) mean_d Q_d^target(s', a*_d)
  loss    = mean_b w_b mean_d (Q_d(s, a_d) - y)^2 ;  trunk gradient rescaled by 1/(D+1) (paper, section 4)
  Adam (TF1 form), hard target copy every ``target_network_update_freq`` steps.
Every detail not visible in the zips/configs (loss reduction, the 1/(D+1) rescale, no gradient clipping) is a
choice documented here, not a pinned fact.  trained_models/BDQ_8pads/logs.full.csv (mean_loss, mean_td_errors per log
interval) was examined as a possible pin: its early rows have mean_loss ~ 0.002 * mean_td_errors**2, below the Jensen
bound td**2 / 9 of the paper's definitions, so the fork's logged quantities are not the ones restated here and the
log cannot arbitrate.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass
from typing import Dict, Tuple

import numpy as np
import torch
import torch.nn.functional as F

ADAM_B1, ADAM_B2, ADAM_EPS = 0.9, 0.999, 1e-8


@dataclass
class BDQConfig:
    obs_dim: int = 100
    n_branches: int = 3
    n_bins: int = 8
    trunk: Tuple[int, int] = (64, 64)
    branch_hidden: int = 32
    value_hidden: int = 32
    gamma: float = 0.99
    trunk_grad_rescale: bool = True


def _fc(i: int) -> str:
    return "fully_connected" if i == 0 else f"fully_connected_{i}"


def param_specs(cfg: BDQConfig, scope: str = "bdq/model"):
    specs = [(f"{scope}/action_value/{_fc(2 * d + k)}/{wb}", shp)
             for d in range(cfg.n_branches)
             for k, dims in enumerate(((cfg.trunk[1], cfg.branch_hidden), (cfg.branch_hidden, cfg.n_bins)))
             for wb, shp in (("biases", (dims[1],)), ("weights", dims))]
    specs += [(f"{scope}/common_net/{_fc(k)}/{wb}", shp)
              for k, dims in enumerate(((cfg.obs_dim, cfg.trunk[0]), (cfg.trunk[0], cfg.trunk[1])))
              for wb, shp in (("biases", (dims[1],)), ("weights", dims))]
    specs += [(f"{scope}/state_value/{_fc(k)}/{wb}", shp)
              for k, dims in enumerate(((cfg.trunk[1], cfg.value_hidden), (cfg.value_hidden, 1)))
              for wb, shp in (("biases", (dims[1],)), ("weights", dims))]
    return specs


def all_specs(cfg: BDQConfig):
    """zip order (sorted names as np.savez keeps them): bdq/eps, online net, target net."""
    return [("bdq/eps", ())] + param_specs(cfg, "bdq/model") + param_specs(cfg, "bdq/target_q_func/model")


def init_params(cfg: BDQConfig, seed: int = 0) -> "OrderedDict[str, np.ndarray]":
    rng = np.random.default_rng(seed)
    p = OrderedDict()
    p["bdq/eps"] = np.float32(1.0)
    for name, shape in param_specs(cfg, "bdq/model"):
        if name.endswith("weights"):     # tf.contrib.layers.fully_connected default: Xavier uniform, zero biases
            lim = np.sqrt(6.0 / (shape[0] + shape[1]))
            p[name] = rng.uniform(-lim, lim, shape).astype(np.float32)
        else:
            p[name] = np.zeros(shape, np.float32)
    for name, _ in param_specs(cfg, "bdq/model"):
        p[name.replace("bdq/model", "bdq/target_q_func/model")] = p[name].copy()
    return p


def q_values(p: Dict[str, torch.Tensor], obs: torch.Tensor, cfg: BDQConfig, scope: str, rescale: bool = False):
    """Returns Q [B, D, n]."""
    h = obs
    for k in range(2):
        h = F.relu(h @ p[f"{scope}/common_net/{_fc(k)}/weights"] + p[f"{scope}/common_net/{_fc(k)}/biases"])
    if rescale:        # forward identity, backward scale 1/(D+1) on the way into the trunk
        s = 1.0 / (cfg.n_branches + 1)
        h = h * s + (h * (1 - s)).detach()
    hv = F.relu(h @ p[f"{scope}/state_value/{_fc(0)}/weights"] + p[f"{scope}/state_value/{_fc(0)}/biases"])
    v = hv @ p[f"{scope}/state_value/{_fc(1)}/weights"] + p[f"{scope}/state_value/{_fc(1)}/biases"]
    qs = []
    for d in range(cfg.n_branches):
        hb = F.relu(h @ p[f"{scope}/action_value/{_fc(2 * d)}/weights"] + p[f"{scope}/action_value/{_fc(2 * d)}/biases"])
        a = hb @ p[f"{scope}/action_value/{_fc(2 * d + 1)}/weights"] + p[f"{scope}/action_value/{_fc(2 * d + 1)}/biases"]
        qs.append(v + a - a.mean(1, keepdim=True))
    return torch.stack(qs, 1)


def bdq_step(params: Dict[str, np.ndarray], opt, batch: Dict[str, np.ndarray], lr: float, cfg: BDQConfig, dtype=torch.float32,
             a_star=None):
    """One train step.  batch: obs [B,obs], act_idx [B,D] (ints), rew [B], next_obs, done [B], weights [B] (IS weights,
    ones without prioritised replay).  ``opt`` = dict(m, v, t).  ``a_star`` [B,D] (optional) replaces the online net's
    argmax at s' -- for rows whose top two advantages fp32 cannot order.  Returns (outputs, grads, new_params, new_opt)."""
    np_dt = np.float64 if dtype == torch.float64 else np.float32
    tp = {n: torch.tensor(np.asarray(a, np_dt), dtype=dtype, requires_grad=n.startswith("bdq/model/")) for n, a in params.items()}
    obs = torch.tensor(np.asarray(batch["obs"], np_dt), dtype=dtype)
    nxt = torch.tensor(np.asarray(batch["next_obs"], np_dt), dtype=dtype)
    act = torch.tensor(np.asarray(batch["act_idx"], np.int64))
    rew = torch.tensor(np.asarray(batch["rew"], np_dt), dtype=dtype)
    done = torch.tensor(np.asarray(batch["done"], np_dt), dtype=dtype)
    w = torch.tensor(np.asarray(batch.get("weights", np.ones(len(rew))), np_dt), dtype=dtype)
    q = q_values(tp, obs, cfg, "bdq/model", rescale=cfg.trunk_grad_rescale)
    q_sa = q.gather(2, act.unsqueeze(2)).squeeze(2)                       # [B, D]
    with torch.no_grad():
        if a_star is None:
            a_star = q_values(tp, nxt, cfg, "bdq/model").argmax(2)         # online net selects
        else:
            a_star = torch.tensor(np.asarray(a_star, np.int64))
        q_t = q_values(tp, nxt, cfg, "bdq/target_q_func/model").gather(2, a_star.unsqueeze(2)).squeeze(2)
        y = rew + cfg.gamma * (1 - done) * q_t.mean(1)
    td = q_sa - y.unsqueeze(1)
    loss = (w * (td ** 2).mean(1)).mean()
    names = [n for n in tp if n.startswith("bdq/model/")]
    gl = torch.autograd.grad(loss, [tp[n] for n in names])
    grads = {n: g.detach().numpy().astype(np_dt) for n, g in zip(names, gl)}
    new_p = OrderedDict((n, np.asarray(a, np_dt).copy()) for n, a in params.items())
    t = opt["t"] + 1
    lr_t = np_dt(lr) * np.sqrt(np_dt(1) - np_dt(ADAM_B2) ** t) / (np_dt(1) - np_dt(ADAM_B1) ** t)
    new_opt = {"t": t, "m": {}, "v": {}}
    for n in names:
        m = (ADAM_B1 * opt["m"].get(n, 0.0) + (1 - ADAM_B1) * grads[n]).astype(np_dt)
        v = (ADAM_B2 * opt["v"].get(n, 0.0) + (1 - ADAM_B2) * grads[n] ** 2).astype(np_dt)
        new_opt["m"][n], new_opt["v"][n] = m, v
        new_p[n] = (new_p[n] - lr_t * m / (np.sqrt(v) + np_dt(ADAM_EPS))).astype(np_dt)
    out = dict(loss=float(loss.detach()), q_sa=q_sa.detach().numpy(), y=y.numpy(), td=td.detach().numpy(), a_star=a_star.numpy(),
               priorities=td.detach().abs().sum(1).numpy(), mean_q=float(q_sa.detach().mean()),
               grad_norm=float(np.sqrt(sum(float((g.astype(np.float64) ** 2).sum()) for g in grads.values()))))
    return out, grads, new_p, new_opt


def hard_target_update(params):
    for n in list(params):
        if n.startswith("bdq/model/"):
            params[n.replace("bdq/model", "bdq/target_q_func/model")] = params[n].copy()
    return params


def greedy_action(params, obs, cfg: BDQConfig):
    tp = {n: torch.tensor(a, dtype=torch.float32) for n, a in params.items()}
    idx = q_values(tp, torch.tensor(obs, dtype=torch.float32), cfg, "bdq/model").argmax(2).numpy()
    return idx, np.linspace(-1.0, 1.0, cfg.n_bins)[idx]
