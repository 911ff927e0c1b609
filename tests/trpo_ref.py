"""float64 restatement of the stable-baselines 2.10.1 TRPO iteration with ``common.policies.MlpPolicy`` and one environment.

TEST INFRASTRUCTURE ONLY.  The reference builds TRPO through ``sb.TRPO(MlpPolicy, env, verbose=2, gamma=...,
timesteps_per_batch=config['TRPO']['max_iters'], vf_stepsize=config['TRPO']['step_size'])`` (sb_helper.py:129-136).  No TRPO
zip ships, so nothing in the reference pins numbers; the algorithm is restated from stable-baselines 2.10.1 (trpo_mpi/trpo_mpi.py,
trpo_mpi/utils.py add_vtarg_and_adv, common/cg.py, common/mpi_adam.py, common/distributions.py).  The network is PPO2's
(oracle/ppo_ref.py); parameters are dicts keyed by the names without a scope ("pi_fc0/w", ...).

  atarg      (adv - mean) / (std + 1e-8), population std
  losses     [optimgain, meankl, entbonus, surrgain, meanent] of theta against theta_old
  F v        d^2 meankl / d theta^2 . v over the rows [::5] (torch double backprop), + cg_damping v
  cg         common/cg.py: p = r = g, x = 0; cg_iters iterations; stop when r.r < 1e-10
  step       shs = 0.5 x.Fx, fullstep = x / sqrt(|shs| / max_kl); ten candidates 0.5^k, the first with finite losses, meankl <=
             1.5 max_kl and optimgain - optimgain_before >= 0
  value      vf_iters passes of 128-row minibatches (partial dropped), loss mean (V - R)^2, MpiAdam (eps 1e-8)
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np
import torch

from oracle import ppo_ref

POLICY = ("pi_fc0/w", "pi_fc0/b", "pi_fc1/w", "pi_fc1/b", "pi/w", "pi/b", "pi/logstd")
VALUE = ("vf_fc0/w", "vf_fc0/b", "vf_fc1/w", "vf_fc1/b", "vf/w", "vf/b")
HALF_LOG_2PI, HALF_LOG_2PIE = ppo_ref.HALF_LOG_2PI, ppo_ref.HALF_LOG_2PIE


def _t(x):
    return torch.as_tensor(np.asarray(x), dtype=torch.float64)


def tensors(params, requires=()):
    """{short name: float64 tensor} of a dict whose names may carry a scope."""
    out = {}
    for k, v in params.items():
        s = k.split("model/", 1)[-1]
        out[s] = _t(v).clone().requires_grad_(s in requires)
    return out


def mean_of(P, x):
    return ppo_ref._forward(P, x)[0]


def standardize(adv):
    a = np.asarray(adv, np.float64)
    return (a - a.mean()) / (a.std() + 1e-8)


def losses_t(P, Pold, x, act, atarg, entcoeff):
    """[optimgain, meankl, entbonus, surrgain, meanent] as torch scalars."""
    mu, mu_o = mean_of(P, x), mean_of(Pold, x)
    ls, ls_o = P["pi/logstd"].reshape(-1), Pold["pi/logstd"].reshape(-1)
    logp = -(0.5 * (((act - mu) / torch.exp(ls)) ** 2).sum(-1) + HALF_LOG_2PI * act.shape[1] + ls.sum())
    logp_o = -(0.5 * (((act - mu_o) / torch.exp(ls_o)) ** 2).sum(-1) + HALF_LOG_2PI * act.shape[1] + ls_o.sum())
    surr = (torch.exp(logp - logp_o) * atarg).mean()
    kl = (ls - ls_o + (torch.exp(2 * ls_o) + (mu_o - mu) ** 2) / (2 * torch.exp(2 * ls)) - 0.5).sum(-1).mean()
    ent = (ls + HALF_LOG_2PIE).sum()
    eb = entcoeff * ent
    return [surr + eb, kl, eb, surr, ent]


def flat(P, names=POLICY):
    return np.concatenate([P[n].detach().numpy().reshape(-1) for n in names])


def unflat(vec, P, names=POLICY):
    out, k = {}, 0
    for n in names:
        m = P[n].numel()
        out[n] = _t(vec[k:k + m]).reshape(P[n].shape)
        k += m
    return out


def losses(params, old, obs, act, atarg, entcoeff=0.0):
    P, Po = tensors(params), tensors(old)
    with torch.no_grad():
        return np.array([float(v) for v in losses_t(P, Po, _t(obs).reshape(len(obs), -1), _t(act).reshape(len(obs), -1), _t(atarg),
                                                      entcoeff)])


def grad_at_old(params, obs, act, atarg, entcoeff=0.0):
    """(losses at theta_old, flat g = d optimgain / d var_list at theta_old)."""
    P, Po = tensors(params, POLICY), tensors(params)
    L = losses_t(P, Po, _t(obs).reshape(len(obs), -1), _t(act).reshape(len(obs), -1), _t(atarg), entcoeff)
    g = torch.autograd.grad(L[0], [P[n] for n in POLICY])
    return np.array([float(v) for v in L]), np.concatenate([x.numpy().reshape(-1) for x in g])


def fvp(params, obs_f, v, damping):
    """F v by double backprop of meankl at theta = theta_old, over the rows obs_f (already [::5])."""
    P, Po = tensors(params, POLICY), tensors(params)
    x = _t(obs_f).reshape(len(obs_f), -1)
    kl = losses_t(P, Po, x, torch.zeros(len(obs_f), P["pi/b"].numel(), dtype=torch.float64), torch.zeros(len(obs_f), dtype=torch.float64),
                  0.0)[1]
    g = torch.autograd.grad(kl, [P[n] for n in POLICY], create_graph=True)
    gf = torch.cat([t.reshape(-1) for t in g])
    hv = torch.autograd.grad((gf * _t(v)).sum(), [P[n] for n in POLICY])
    return np.concatenate([t.numpy().reshape(-1) for t in hv]) + damping * np.asarray(v, np.float64)


def fvp_gauss_newton(params, obs_f, v, damping):
    """The same product as J^T diag(1 / (sigma^2 N_f)) J v for the mean, 2 v for logstd (forward-mode tangent + backward)."""
    P = tensors(params, POLICY)
    x = _t(obs_f).reshape(len(obs_f), -1)
    V = unflat(np.asarray(v, np.float64), P)
    sig2 = torch.exp(2 * P["pi/logstd"].detach().reshape(-1))
    with torch.no_grad():
        z0 = x @ P["pi_fc0/w"] + P["pi_fc0/b"]
        y0 = torch.tanh(z0)
        dy0 = (1 - y0 ** 2) * (x @ V["pi_fc0/w"] + V["pi_fc0/b"])
        y1 = torch.tanh(y0 @ P["pi_fc1/w"] + P["pi_fc1/b"])
        dy1 = (1 - y1 ** 2) * (dy0 @ P["pi_fc1/w"] + y0 @ V["pi_fc1/w"] + V["pi_fc1/b"])
        jv = dy1 @ P["pi/w"] + y1 @ V["pi/w"] + V["pi/b"]
        u = jv / (sig2 * len(obs_f))
    mu = mean_of(P, x)
    g = torch.autograd.grad((mu * u).sum(), [P[n] for n in POLICY[:-1]])
    out = np.concatenate([t.numpy().reshape(-1) for t in g] + [2.0 * V["pi/logstd"].numpy().reshape(-1)])
    return out + damping * np.asarray(v, np.float64)


def cg(f_Ax, b, cg_iters=10, residual_tol=1e-10):
    """common/cg.py -> (x, iterations run)."""
    p, r = b.copy(), b.copy()
    x = np.zeros_like(b)
    rdotr = r.dot(r)
    it = 0
    for _ in range(cg_iters):
        z = f_Ax(p)
        v = rdotr / p.dot(z)
        x += v * p
        r -= v * z
        newrdotr = r.dot(r)
        p = r + newrdotr / rdotr * p
        rdotr = newrdotr
        it += 1
        if rdotr < residual_tol:
            break
    return x, it


def line_search(loss_at, before_gain, max_kl, n=10):
    """loss_at(k) -> the five losses at theta_before + 0.5^k fullstep.  -> (k, losses) of the first acceptable k, (-1, None)."""
    for k in range(n):
        L = np.asarray(loss_at(k), np.float64)
        if not np.isfinite(L).all() or L[1] > 1.5 * max_kl or L[0] - before_gain < 0:
            continue
        return k, L
    return -1, None


def value_minibatches(n, batch_size=128):
    return [(s, s + batch_size) for s in range(0, n - batch_size + 1, batch_size)]


class MpiAdam:
    """common/mpi_adam.py on one process, float64."""

    def __init__(self):
        self.t, self.m, self.v = 0, {}, {}

    def update(self, params, grads, lr, b1=0.9, b2=0.999, eps=1e-8):
        self.t += 1
        a = lr * np.sqrt(1 - b2 ** self.t) / (1 - b1 ** self.t)
        out = OrderedDict((k, np.asarray(x, np.float64).copy()) for k, x in params.items())
        for k, g in grads.items():
            self.m[k] = b1 * self.m.get(k, 0.0) + (1 - b1) * g
            self.v[k] = b2 * self.v.get(k, 0.0) + (1 - b2) * g * g
            out[k] = out[k] - a * self.m[k] / (np.sqrt(self.v[k]) + eps)
        return out


def value_grad(params, obs, ret):
    """(loss mean (V - R)^2, {name: gradient}) of the vf tower on one minibatch."""
    P = tensors(params, VALUE)
    v = ppo_ref._forward(P, _t(obs).reshape(len(obs), -1))[1]
    loss = ((v - _t(ret)) ** 2).mean()
    g = torch.autograd.grad(loss, [P[n] for n in VALUE])
    return float(loss), {n: t.numpy() for n, t in zip(VALUE, g)}


def iteration(params, adam, obs, act, adv, tdlamret, perms, max_kl=0.01, cg_iters=10, cg_damping=1e-2, entcoeff=0.0, vf_stepsize=3e-4):
    """One policy step and value step on short-named float64 params -> (new params, record)."""
    params = OrderedDict((k, np.asarray(v, np.float64)) for k, v in params.items())
    atarg = standardize(adv)
    L0, g = grad_at_old(params, obs, act, atarg, entcoeff)
    rec = dict(losses_before=L0, g=g, accepted=-2, losses_after=L0, stepdir=None, fullstep=None, shs=0.0, expectedimprove=0.0,
               cg_iters=0)
    new = OrderedDict(params)
    if not np.allclose(g, 0):
        obs_f = np.asarray(obs)[::5]
        x, it = cg(lambda p: fvp(params, obs_f, p, cg_damping), g.copy(), cg_iters)
        assert np.isfinite(x).all()
        shs = 0.5 * x.dot(fvp(params, obs_f, x, cg_damping))
        fullstep = x / np.sqrt(abs(shs) / max_kl)
        th0 = flat(tensors(params))
        P0 = tensors(params)

        def at(k):
            cand = dict(params)
            cand.update({n: t.numpy() for n, t in unflat(th0 + 0.5 ** k * fullstep, P0).items()})
            return losses(cand, params, obs, act, atarg, entcoeff)
        rec["table"] = np.stack([at(k) for k in range(10)])     # the losses of every candidate 0.5^k
        k, La = line_search(at, L0[0], max_kl)
        rec.update(stepdir=x, fullstep=fullstep, shs=shs, expectedimprove=g.dot(fullstep), cg_iters=it, accepted=k)
        if k >= 0:
            rec["losses_after"] = La
            new.update({n: t.numpy() for n, t in unflat(th0 + 0.5 ** k * fullstep, P0).items()})
    vl = []
    for perm in perms:
        for s, e in value_minibatches(len(obs)):
            i = np.asarray(perm[s:e])
            loss, gr = value_grad(new, np.asarray(obs)[i], np.asarray(tdlamret)[i])
            vl.append(loss)
            new = adam.update(new, gr, vf_stepsize)
    rec["vf_loss"] = float(np.mean(vl)) if vl else 0.0
    return new, rec


__all__ = ["POLICY", "VALUE", "standardize", "losses", "grad_at_old", "fvp", "fvp_gauss_newton", "cg", "line_search",
           "value_minibatches", "MpiAdam", "value_grad", "iteration", "flat", "unflat", "tensors"]
