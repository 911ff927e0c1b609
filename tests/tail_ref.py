"""The SAC head tail (everything between fc0's contraction and its gradient: csrc/tail.cu's tail4_kernel and tailw_kernel<H>)
restated once, from SURVEY.md Appendix A and oracle/sac_ref_np.py, over an arithmetic backend:

  * `Bound` evaluates it in float64 and carries, beside every value, a first-order bound on how far an fp32 evaluation of the
    same formula can be from it (running error analysis, u = 2^-24): each fp32 add, multiply or FMA contributes u |result|
    (a*b + c is charged u |ab| + u |result|, so the bound holds with and without FMA); a sum of n terms in unknown order
    (warp shuffles, shared and global fp32 atomics) gamma_n sum|terms|; expf and tanhf 2 ulp, logf 1 ulp (CUDA's maximum
    errors; the build has no fast-math flag); IEEE division one rounding; input errors propagate through the derivative
    magnitudes, for exp, tanh, log and x / (x + eps) through the exact image of the input interval (these are monotone).
    Constants carry their fp32 representation error.  Callers hold |fp32 - value| <= SLACK * bound: the 1 % covers the
    second-order terms.
  * `Fp32` evaluates it in fp32 numpy, each contraction and batch sum in a chosen summation order, with or without FMA:
    the check that the bound bounds (tests/test_tail_ref_cpu.py).

The formulas are the tail's own: tanh of the replay action is never taken (the replay action enters Q as stored), the 1e-6
sits in t = (u - mu) / (std + 1e-6), in log(1 - pi^2 + 1e-6) and in the tanh seed's one_m / (one_m + 1e-6), and the policy
loss takes qf1 at pi alone.  qf1 and qf2 at pi reuse the replay action's fc0 output: z0(pi) = z0(a) + (pi - a) K0[action rows].

ReLU masks and the log_std clamp are discontinuities of the gradients.  Every mask is recorded; a caller that knows the side
the kernel took passes it in `masks`, and the bound is then the bound on that side.  `near[key]` marks inputs within their
bound of the kink (fp32 could take either side), `bad[key]` a given side that float64 says fp32 cannot take.
"""
import math

import numpy as np

U = 2.0 ** -24
SLACK = 1.01
EPS = 1e-6
LOG_STD_MAX, LOG_STD_MIN = 2.0, -20.0
LOG_2PI = math.log(2 * math.pi)
ENT_C = 0.5 * math.log(2 * math.pi * math.e)


def gamma(n):
    return n * U / (1 - n * U)


def _other_letter(subs):
    ins, out = subs.split("->")
    (k,) = {c for c in ins.replace(",", "") if c not in out}
    return k


# ================================================================================================ float64 + bound
class E:
    """A float64 value and a bound on |fp32 evaluation - value|."""
    __array_priority__ = 100

    def __init__(self, v, e=0.0):
        self.v = np.asarray(v, np.float64)
        self.e = np.broadcast_to(np.asarray(e, np.float64), self.v.shape).copy()

    @staticmethod
    def of(x):
        return x if isinstance(x, E) else E(x)

    @property
    def mag(self):
        """A bound on |fp32 value|."""
        return np.abs(self.v) + self.e

    def __add__(a, b):
        b = E.of(b)
        v = a.v + b.v
        return E(v, a.e + b.e + U * np.abs(v))

    __radd__ = __add__

    def __neg__(a):
        return E(-a.v, a.e)

    def __sub__(a, b):
        return a + (-E.of(b))

    def __rsub__(a, b):
        return E.of(b) + (-a)

    def __mul__(a, b):
        b = E.of(b)
        v = a.v * b.v
        return E(v, np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e + U * np.abs(v))

    __rmul__ = __mul__

    def __truediv__(a, b):
        b = E.of(b)
        d = np.abs(b.v) - b.e
        assert (d > 0).all(), "a divisor within its bound of 0"
        q = a.v / b.v
        return E(q, (a.e + np.abs(q) * b.e) / d + U * np.abs(q))

    def __getitem__(self, i):
        return E(self.v[i], self.e[i])


class Bound:
    """float64 values with running error bounds; `masks` holds the sides the fp32 evaluation took where they are known."""

    def __init__(self, masks=None):
        self.masks = dict(masks or {})
        self.side, self.near, self.bad = {}, {}, {}

    def lift(self, x):
        return E(np.asarray(x, np.float64))

    def const(self, c):
        return E(c, abs(float(np.float32(c)) - c))

    def _mono(self, f, x, ulps, lo=-np.inf):
        """f monotone: the image of [v - e, v + e] (clipped below at lo, a bound the fp32 input is known to keep), plus ulps."""
        v = f(x.v)
        a, b = f(np.maximum(x.v - x.e, lo)), f(x.v + x.e)
        m = np.maximum(np.abs(a - v), np.abs(b - v))
        return E(v, m + ulps * 2 * U * np.maximum(np.maximum(np.abs(a), np.abs(b)), np.abs(v)))

    def exp(self, x):
        return self._mono(np.exp, x, 2)

    def tanh(self, x):
        return self._mono(np.tanh, x, 2)

    def log(self, x, lo):
        return self._mono(np.log, x, 1, lo)

    def _side(self, key, z, cut=0.0):
        f64 = z.v > cut
        side = np.asarray(self.masks[key], bool) if key in self.masks else f64
        near = np.abs(z.v - cut) <= SLACK * z.e
        self.side[key], self.near[key] = side, near
        self.bad[key] = (side != f64) & ~near
        return side

    def relu(self, z, key):
        self._side(key, z)
        return E(np.maximum(z.v, 0.0), z.e)          # relu is 1-Lipschitz: the bound holds on either side

    def gate(self, key, x):
        m = self.side[key]
        return E(np.where(m, x.v, 0.0), np.where(m, x.e, 0.0))

    def clip_log_std(self, x, key):
        """clip(x, -20, 2) and the mask of x inside [-20, 2] (the log_std seed's gate)."""
        hi = self._side(key + "/max", -x, -LOG_STD_MAX)       # x < 2 ...
        lo = self._side(key + "/min", x, LOG_STD_MIN)         # ... and x > -20
        self.side[key] = hi & lo
        v = np.clip(x.v, LOG_STD_MIN, LOG_STD_MAX)
        out = (x.v - SLACK * x.e > LOG_STD_MAX) | (x.v + SLACK * x.e < LOG_STD_MIN)    # fp32 fminf / fmaxf return the bound
        return E(v, np.where(out, 0.0, x.e))

    def minimum(self, a, b):
        return E(np.minimum(a.v, b.v), np.maximum(a.e, b.e))

    def contract(self, subs, a, b, bias=None):
        """einsum(subs, a, b) (+ bias): one sum of n (+ 1) terms in unknown order."""
        a, b = E.of(a), E.of(b)
        k = _other_letter(subs)
        ins = subs.split("->")[0].split(",")
        n = (a.v.shape[ins[0].index(k)])
        v = np.einsum(subs, a.v, b.v)
        mag = np.einsum(subs, a.mag, b.mag)
        prop = np.einsum(subs, np.abs(a.v), b.e) + np.einsum(subs, a.e, np.abs(b.v)) + np.einsum(subs, a.e, b.e)
        if bias is not None:
            bias = E.of(bias)
            v, mag, prop, n = v + bias.v, mag + bias.mag, prop + bias.e, n + 1
        return E(v, gamma(n) * mag + prop)

    def total(self, x, axis=0):
        n = x.v.shape[axis]
        return E(x.v.sum(axis), gamma(n) * x.mag.sum(axis) + x.e.sum(axis))

    def shifted_diff(self, mu, eps, sd):
        """u = mu + eps sd, and u - mu as the fp32 evaluation forms it: mu's own error cancels in the difference, which is
        eps sd with the roundings of the product, of u and of the subtraction."""
        p = eps * sd
        u = mu + p
        d = E(u.v - mu.v, p.e + U * u.mag + U * np.abs(p.v) * (1 + U))
        return u, d

    def times_ratio(self, c, one_m, eps):
        """c one_m / (one_m + eps), one_m >= 0: x / (x + eps) is increasing in x and decreasing in eps; three roundings."""
        x0, x1 = np.maximum(one_m.v - one_m.e, 0.0), one_m.v + one_m.e
        e0, e1 = eps.v - eps.e, eps.v + eps.e
        r = one_m.v / (one_m.v + eps.v)
        m = np.maximum(np.abs(x0 / (x0 + e1) - r), np.abs(x1 / (x1 + e0) - r))
        return c * E(r, m + 3 * U * np.maximum(r, x1 / (x1 + e0)))


# ================================================================================================ fp32 evaluations
class Fp32:
    """fp32 numpy: every contraction and batch sum accumulated in `order` ('seq', 'rev', 'perm', 'tree'), the products fused
    into the accumulation (fma) or rounded first."""

    def __init__(self, order="seq", fma=True, seed=0):
        self.order, self.fma, self.rng = order, fma, np.random.default_rng(seed)
        self.side = {}

    lift = staticmethod(lambda x: np.asarray(x, np.float32))
    const = staticmethod(lambda c: np.float32(c))
    exp = staticmethod(np.exp)
    tanh = staticmethod(np.tanh)
    log = staticmethod(lambda x, lo: np.log(x))
    minimum = staticmethod(np.minimum)

    def relu(self, z, key):
        self.side[key] = z > 0
        return np.maximum(z, np.float32(0))

    def gate(self, key, x):
        return np.where(self.side[key], x, np.float32(0))

    def clip_log_std(self, x, key):
        self.side[key + "/max"], self.side[key + "/min"] = x <= LOG_STD_MAX, x >= LOG_STD_MIN
        self.side[key] = self.side[key + "/max"] & self.side[key + "/min"]
        return np.minimum(np.maximum(x, np.float32(LOG_STD_MIN)), np.float32(LOG_STD_MAX))

    def _acc(self, terms, init):
        """Sum float64 exact products terms[k] (k along axis 0) into the fp32 init."""
        n = terms.shape[0]
        if self.order == "tree":
            t = [np.float32(x) for x in terms] + ([np.asarray(init, np.float32)] if init is not None else [])
            while len(t) > 1:
                t = [np.float32(t[i] + t[i + 1]) if i + 1 < len(t) else t[i] for i in range(0, len(t), 2)]
            return np.asarray(t[0], np.float32)
        idx = {"seq": np.arange(n), "rev": np.arange(n)[::-1], "perm": self.rng.permutation(n)}[self.order]
        acc = np.zeros(terms.shape[1:], np.float32)
        if init is not None:
            acc = acc + np.asarray(init, np.float32)
        for k in idx:
            acc = np.float32(acc + terms[k]) if self.fma else np.float32(acc + np.float32(terms[k]))
        return acc

    def contract(self, subs, a, b, bias=None):
        k = _other_letter(subs)
        ins, out = subs.split("->")
        ka, kb = ins.split(",")
        terms = np.einsum(f"{ka},{kb}->{k}{out}", np.asarray(a, np.float64), np.asarray(b, np.float64))
        init = None if bias is None else np.broadcast_to(np.asarray(bias, np.float32), terms.shape[1:])
        return self._acc(terms, init)

    def total(self, x, axis=0):
        return self._acc(np.moveaxis(np.asarray(x, np.float64), axis, 0), None)

    def shifted_diff(self, mu, eps, sd):
        p64 = np.asarray(eps, np.float64) * np.asarray(sd, np.float64)
        u = np.float32(p64 + mu) if self.fma else np.float32(mu + np.float32(p64))
        return u, np.float32(u - mu)

    def times_ratio(self, c, one_m, eps):
        return np.float32(np.float32(c * one_m) / np.float32(one_m + eps))


# ================================================================================================ the tail
HEADS = ("pi", "vf", "qf1", "qf2")
PREFIX = {"pi": "model/pi", "vf": "model/values_fn/vf", "qf1": "model/values_fn/qf1", "qf2": "model/values_fn/qf2",
          "target": "target/values_fn/vf"}
OUT = {"vf": "vf", "qf1": "qf1", "qf2": "qf2", "target": "vf"}


def tail(X, z0, params, act, eps, rew, done, gamma_, target_entropy, feat_dim, pi_in=None):
    """X: Bound or Fp32.  z0[head] [B][H] for pi, vf, qf1, qf2, target: fc0 outputs without bias (qf at the replay action);
    params: the fp32 parameters by name; act, eps [B][A]; rew, done [B].  Returns a dict of every quantity the tail produces.

    pi_in: the fp32 pi the evaluation under test formed (the kernel stores it).  o["pi"] is then still held from the inputs,
    and everything downstream of pi (the log-prob's squashing term, Q at pi, the tanh seed) from pi_in: the Q-at-pi ReLU
    inputs and the actor's seeds keep bounds near fp32 round-off instead of inheriting pi's bound through K0."""
    P = {k: np.asarray(v, np.float64) for k, v in params.items()}
    B, A = np.shape(eps)
    L = X.lift
    invB = X.const(1.0 / B)
    log_alpha = L(P["model/log_ent_coef"])
    alpha = X.exp(log_alpha)
    EPSC = X.const(EPS)
    o = {}

    def fc(head, z):
        pre = PREFIX[head]
        a0 = X.relu(z + L(P[f"{pre}/fc0/bias"]), f"a0/{head}")
        a1 = X.relu(X.contract("bi,ij->bj", a0, L(P[f"{pre}/fc1/kernel"]), L(P[f"{pre}/fc1/bias"])), f"a1/{head}")
        return a0, a1

    def out1(head, a1):
        pre = PREFIX[head]
        return X.contract("bj,j->b", a1, L(P[f"{pre}/{OUT[head]}/kernel"][:, 0]), L(P[f"{pre}/{OUT[head]}/bias"][0]))

    # ---- actor: mu, log_std, the tanh-Gaussian sample and its log-prob
    a0 = {}
    a0["pi"], g = fc("pi", L(z0["pi"]))
    mu = X.contract("bj,ja->ba", g, L(P["model/pi/dense/kernel"]), L(P["model/pi/dense/bias"]))
    ls_raw = X.contract("bj,ja->ba", g, L(P["model/pi/dense_1/kernel"]), L(P["model/pi/dense_1/bias"]))
    ls = X.clip_log_std(ls_raw, "ls")
    sd = X.exp(ls)
    e = L(eps)
    u, u_mu = X.shifted_diff(mu, e, sd)
    tt = u_mu / (sd + EPSC)
    pi = o["pi"] = X.tanh(u)
    if pi_in is not None:
        pi = X.lift(pi_in)
    one_m = 1.0 - pi * pi
    logp = X.total(-0.5 * (tt * tt + 2.0 * ls + X.const(LOG_2PI)) - X.log(one_m + EPSC, float(np.float32(EPS))), axis=1)
    ent = X.total(ls + X.const(ENT_C), axis=1)
    # ---- critics at the replay action, the target vf at the next observation
    a1 = {"pi": g}
    q = {}
    for h in ("vf", "qf1", "qf2", "target"):
        a0[h], a1[h] = fc(h, L(z0[h]))
        q[h] = out1(h, a1[h])
    # ---- qf1, qf2 at pi: z0(pi) = z0(a) + (pi - a) K0[action rows]
    dlt = pi - L(act)
    qp, a0p, a1p = {}, {}, {}
    for h in ("qf1", "qf2"):
        pre = PREFIX[h]
        k0a = L(P[f"{pre}/fc0/kernel"][feat_dim:])
        zp = X.contract("ba,aj->bj", dlt, k0a, L(z0[h]))
        a0p[h] = X.relu(zp + L(P[f"{pre}/fc0/bias"]), f"a0p/{h}")
        a1p[h] = X.relu(X.contract("bi,ij->bj", a0p[h], L(P[f"{pre}/fc1/kernel"]), L(P[f"{pre}/fc1/bias"])), f"a1p/{h}")
        qp[h] = out1(h, a1p[h])
    # ---- value targets, losses and metrics
    v, v_targ, q1, q2 = q["vf"], q["target"], q["qf1"], q["qf2"]
    v_backup = X.minimum(qp["qf1"], qp["qf2"]) - alpha * logp
    ev = v - v_backup
    q_backup = L(rew) + (1.0 - L(done)) * X.const(gamma_) * v_targ
    e1, e2 = q1 - q_backup, q2 - q_backup
    te = X.const(target_entropy)
    o.update(q1=q1, q2=q2, v=v, logp=logp, v_targ=v_targ, q1_pi=qp["qf1"], q2_pi=qp["qf2"], ls_raw=ls_raw)
    o["policy_loss"] = X.total((alpha * logp - qp["qf1"]) * invB)
    o["ent_coef_loss"] = X.total(-log_alpha * (logp + te) * invB)
    o["entropy"] = X.total(ent * invB)
    o["mean_logp"] = X.total(logp * invB)
    o["value_loss"] = X.total(0.5 * ev * ev * invB)
    o["mean_v"] = X.total(v * invB)
    o["qf1_loss"] = X.total(0.5 * e1 * e1 * invB)
    o["qf2_loss"] = X.total(0.5 * e2 * e2 * invB)
    o["mean_q1"] = X.total(q1 * invB)
    o["mean_q2"] = X.total(q2 * invB)
    o["g/model/log_ent_coef"] = X.total(-(logp + te) * invB)
    # ---- the critics' backward seeds and output-layer gradients
    dz1 = {}
    for h, d in (("vf", ev * invB), ("qf1", e1 * invB), ("qf2", e2 * invB)):
        pre = PREFIX[h]
        o[f"g/{pre}/{h}/kernel"] = X.contract("bj,b->j", a1[h], d)
        o[f"g/{pre}/{h}/bias"] = X.total(d)
        dz1[h] = X.gate(f"a1/{h}", d[:, None] * L(P[f"{pre}/{h}/kernel"][:, 0])[None, :])
    # ---- d(-Q1(s, pi)) / d pi: back through qf1 at pi to its action rows (qf1's weights are constants here)
    pre = PREFIX["qf1"]
    dzp = X.gate("a1p/qf1", -invB * L(np.ones((B, 1))) * L(P[f"{pre}/qf1/kernel"][:, 0])[None, :])
    dz0p = X.gate("a0p/qf1", X.contract("bj,ij->bi", dzp, L(P[f"{pre}/fc1/kernel"])))
    dpi = X.contract("bj,aj->ba", dz0p, L(P[f"{pre}/fc0/kernel"][feat_dim:]))
    # ---- the actor's seeds: tanh squashing, the sample's std and the clamp
    du = X.times_ratio(alpha * invB * 2.0 * pi, one_m, EPSC) + dpi * one_m
    spe = sd + EPSC
    d = du * e * sd + alpha * invB * (-tt * e * sd * EPSC / (spe * spe) - 1.0)
    dls = X.gate("ls", d)
    o["g/model/pi/dense/kernel"] = X.contract("bj,ba->ja", g, du)
    o["g/model/pi/dense/bias"] = X.total(du)
    o["g/model/pi/dense_1/kernel"] = X.contract("bj,ba->ja", g, dls)
    o["g/model/pi/dense_1/bias"] = X.total(dls)
    seeds = _cat(X, du, dls)
    kk = L(np.concatenate([P["model/pi/dense/kernel"], P["model/pi/dense_1/kernel"]], 1))
    dz1["pi"] = X.gate("a1/pi", X.contract("ba,ja->bj", seeds, kk))
    # ---- fc0 pre-activation gradients
    dz0 = {h: X.gate(f"a0/{h}", X.contract("bj,ij->bi", dz1[h], L(P[f"{PREFIX[h]}/fc1/kernel"]))) for h in HEADS}
    for h in HEADS:
        o[f"a0/{h}"], o[f"dz1/{h}"], o[f"dz0/{h}"] = a0[h], dz1[h], dz0[h]
    o["a1/pi"] = g
    return o


def _cat(X, a, b):
    if isinstance(a, E):
        return E(np.concatenate([a.v, b.v], 1), np.concatenate([a.e, b.e], 1))
    return np.concatenate([a, b], 1)


PER_SAMPLE = ("q1", "q2", "v", "logp", "v_targ", "q1_pi", "q2_pi")
SUMS = ("policy_loss", "qf1_loss", "qf2_loss", "value_loss", "ent_coef_loss", "entropy", "mean_q1", "mean_q2", "mean_v",
        "mean_logp")
GRADS = ("model/pi/dense/kernel", "model/pi/dense/bias", "model/pi/dense_1/kernel", "model/pi/dense_1/bias",
         "model/values_fn/vf/vf/kernel", "model/values_fn/vf/vf/bias", "model/values_fn/qf1/qf1/kernel",
         "model/values_fn/qf1/qf1/bias", "model/values_fn/qf2/qf2/kernel", "model/values_fn/qf2/qf2/bias", "model/log_ent_coef")
# the gradient's masks no stored tensor shows (qf2 at pi enters the losses through min(q1_pi, q2_pi) only: no mask of its own)
UNREVEALED = ("ls/max", "ls/min", "a0p/qf1", "a1p/qf1")
