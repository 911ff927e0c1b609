"""The PPO2 and TRPO kernels (csrc/actor_critic.cu, csrc/ppo.cu, csrc/trpo.cu) restated kernel by kernel, from the inputs each
one read, over the arithmetic backends of tests/tail_ref.py:

  * `Bound` evaluates a formula in float64 and carries beside every value a first-order bound on how far an fp32 evaluation
    of it can be (u = 2^-24 per rounding; a sum of n terms in any order gamma_{n-1} sum|terms|, so the kernels' serial fmaf
    chains, fixed-order block sums and warp trees are all covered; expf / tanhf 2 ulp, logf / sincospif 1 ulp, sqrtf
    correctly rounded: the CUDA math guide's maximum errors without fast-math).  Scaling by a power of two is exact.
  * `Fp32` evaluates the same formula in fp32 numpy, sums in a chosen order: tests/test_ac_kernels_ref_cpu.py checks that the
    bound bounds it, and that an error a few bounds in size planted in one element fails.

Sums the kernels form in float64 (TRPO's head gradients, dot products, line-search partials) carry gamma64_n sum|terms| and
one fp32 rounding of the result.  Formulas that stable-baselines states are taken from oracle/ppo_ref.py (GAE, neglogp)
and oracle/philox_ref.py (the noise), in the kernels' own operation order where they differ only in that order.
"""
import math

import numpy as np

from oracle import philox_ref as PX
from tests import tail_ref as TR
from tests.tail_ref import E, U, SLACK

U64 = 2.0 ** -53
HALF_LOG_2PI = 0.91893853320467274
HALF_LOG_2PI_E = 1.4189385332046727
NORM_BLOCKS, NORM_THREADS = 128, 256
DOT_BLOCKS, LS_BLOCKS, LS_THREADS, NCAND, VF_BATCH = 128, 64, 256, 10, 128
SC = dict(RR=0, ALPHA=1, BETA=2, DONE=3, ZERO=4, BAD=5, ITERS=6, ACC=7, LM=8)
PM = dict(PG=0, VF=1, ENT=2, KL=3, CLIP=4, GN=5)
TM_BEFORE, TM_AFTER, TM_GG, TM_SHS, TM_EI, TM_VF = 0, 5, 10, 11, 12, 13
NOISE_ULPS = 0.5 * 2 + 1 + 2 + 1   # z = sqrtf(-2 logf u0) * sincospif: logf 1 ulp halved by the root, sqrtf, sincospif, the product


def gamma(n):
    n = max(int(n), 0)
    return n * U / (1 - n * U)


def gamma64(n):
    return n * U64 / (1 - n * U64)


def pow2(c):
    return c > 0 and math.frexp(c)[0] == 0.5


# ================================================================================================ backends
class Bound(TR.Bound):
    def sqrt(self, x):
        return self._mono(np.sqrt, x, 0.5, 0.0)

    def total(self, x, axis=0):
        n = x.v.shape[axis]
        return E(x.v.sum(axis), gamma(n - 1) * x.mag.sum(axis) + x.e.sum(axis))

    def scale(self, x, c):
        """x * c: exact for a power of two c, else one rounding and c's representation error"""
        if pow2(c):
            return E(x.v * c, x.e * c)
        return x * self.const(c)

    def cat(self, xs, axis):
        xs = [E.of(x) for x in xs]
        return E(np.concatenate([x.v for x in xs], axis), np.concatenate([x.e for x in xs], axis))

    def where(self, m, a, b):
        a, b = E.of(a), E.of(b)
        return E(np.where(m, a.v, b.v), np.where(m, a.e, b.e))

    def clip(self, x, lo, hi):
        lo, hi = E.of(lo), E.of(hi)
        return E(np.clip(x.v, lo.v, hi.v), np.maximum(x.e, np.maximum(lo.e, hi.e)))

    def maximum(self, a, b):
        return E(np.maximum(a.v, b.v), np.maximum(a.e, b.e))

    def square(self, x):
        return x * x

    def dsum(self, x, axis=0):
        """a float64 sum of fp32 values, rounded to fp32 once"""
        n = x.v.shape[axis]
        v = x.v.sum(axis)
        return E(v, gamma64(n) * x.mag.sum(axis) + x.e.sum(axis) + U * np.abs(v))


class Fp32(TR.Fp32):
    sqrt = staticmethod(np.sqrt)

    def scale(self, x, c):
        return (np.asarray(x, np.float32) * np.float32(c)).astype(np.float32)

    def cat(self, xs, axis):
        return np.concatenate([np.broadcast_to(np.asarray(x, np.float32), np.shape(xs[0])[:axis] + np.shape(x)[axis:])
                               if np.ndim(x) == np.ndim(xs[0]) else np.asarray(x, np.float32) for x in xs], axis)

    where = staticmethod(lambda m, a, b: np.where(m, a, b).astype(np.float32))
    clip = staticmethod(lambda x, lo, hi: np.minimum(np.maximum(x, np.float32(lo)), np.float32(hi)))
    maximum = staticmethod(np.maximum)
    square = staticmethod(lambda x: np.float32(x * x))

    def dsum(self, x, axis=0):
        return np.float32(np.asarray(x, np.float64).sum(axis))


def cst(X, c, c32, shape):
    """the constant c as the kernel holds it (fp32 value c32), broadcast to shape"""
    if isinstance(X, Bound):
        return E(np.full(shape, c), abs(float(c32) - c))
    return np.full(shape, np.float32(c32), np.float32)


# ================================================================================================ layout
def layout(D, A, H0, H1, copies=1):
    """actor_critic.cu ac_layout: arena offsets (each entry padded to 32 floats) -> dict, n_train, n_total"""
    off = 0
    o = {}

    def take(name, n):
        nonlocal off
        o[name] = off
        off += -(-n // 32) * 32

    take("W0", D * 2 * H0); take("b0", 2 * H0)
    for tw in range(2):
        take(f"W1_{tw}", H0 * H1); take(f"b1_{tw}", H1)
    take("Wvf", H1); take("bvf", 1); take("Wpi", H1 * A); take("bpi", A); take("ls", A)
    n_train = off
    take("Wq", H1 * A); take("bq", A)
    return o, n_train, off


def unpack(P, o, D, A, H0, H1):
    """the arena's blocks as float32 arrays: W0 [D, 2 H0] (pi | vf columns), b0 [2 H0], W1 [2][H0, H1], ..."""
    g = lambda k, n: P[o[k]:o[k] + n]
    return dict(W0=g("W0", D * 2 * H0).reshape(D, 2 * H0), b0=g("b0", 2 * H0),
                W1=[g(f"W1_{t}", H0 * H1).reshape(H0, H1) for t in range(2)], b1=[g(f"b1_{t}", H1) for t in range(2)],
                Wvf=g("Wvf", H1), bvf=g("bvf", 1), Wpi=g("Wpi", H1 * A).reshape(H1, A), bpi=g("bpi", A), ls=g("ls", A))


# ================================================================================================ shared kernels
def bias_tanh(X, Z, b):
    """ppo_bias_tanh_kernel: Y = tanhf(Z + b[col])"""
    return X.tanh(X.lift(Z) + X.lift(b))


def heads(X, Y1, net, H1):
    """ac_heads: mu = bpi + sum_k ypi[k] Wpi[k] and v = bvf + sum_k yvf[k] Wvf[k] (serial fmaf chains)"""
    ypi, yvf = Y1[:, :H1], Y1[:, H1:2 * H1]
    mu = X.contract("rk,kj->rj", X.lift(ypi), X.lift(net["Wpi"]), bias=X.lift(net["bpi"]))
    v = X.contract("rk,k->r", X.lift(yvf), X.lift(net["Wvf"]), bias=X.lift(net["bvf"][0]))
    return mu, v


def neglogp(X, z, ls):
    """A 0.5 log 2 pi + sum_k (0.5 z^2 + ls), the constant first (the kernels' order)"""
    R, A = np.shape(_val(z))
    t = X.scale(X.square(z), 0.5) + X.lift(ls)
    c = cst(X, HALF_LOG_2PI * A, np.float32(HALF_LOG_2PI) * np.float32(A), (R, 1))
    return X.total(X.cat([c, t], 1), axis=1)


def noise(key, step, rows, A):
    """stream-1 noise of one drawing call (oracle/philox_ref.py) and its fp32 bound"""
    z = PX.noise(key, step, rows * A).reshape(rows, A)
    return E(z, NOISE_ULPS * U * np.abs(z))


def act(X, Y1, net, H1, z):
    """ppo_act_kernel: act = mu + expf(ls) z, value, neglogp = sum(0.5 z^2 + ls) + A 0.5 log 2 pi"""
    mu, v = heads(X, Y1, net, H1)
    ls = X.lift(net["ls"])
    a = mu + X.exp(ls) * z
    return a, v, neglogp(X, z, net["ls"])


def gae(X, rew, val, done, lastv, gamma_, lam):
    """ppo_gae_kernel per env column: val [T + 1, E] (row T unused: lastv), done [T + 1, E] episode-start flags"""
    T = rew.shape[0]
    g, l = X.const(gamma_), X.const(lam)
    last = X.lift(np.zeros(rew.shape[1]))
    adv, ret = [None] * T, [None] * T
    for t in range(T - 1, -1, -1):
        nnt = X.lift(1.0 - done[t + 1])
        nv = X.lift(lastv if t == T - 1 else val[t + 1])
        delta = X.lift(rew[t]) + g * nv * nnt - X.lift(val[t])
        last = delta + g * l * nnt * last
        adv[t] = last
        ret[t] = last + X.lift(val[t])
    return adv, ret


# ================================================================================================ PPO2
def ppo_tail(X, Y1, net, H1, act_, oval, onlp, ret, clip, clipvf, ent_coef, vf_coef, side=None, vside=None, stored=None):
    """ppo_tail_kernel's per-row stage and its sums (rows already gathered through rowidx).  side [M]: the kernel's
    tf.maximum / clip_by_value gradient gate (None: float64's); vside [M]: the value loss took l2 with d outside the clip.
    stored: the kernel's fp32 sz, sv, snlp, sadv, which its later loops read back from global memory; the outputs o[...] of
    those names are still held from the inputs, and what follows is formed from the stored values (so that M = 1's
    adv - mean is exactly 0, as it is on the device)."""
    M, A = act_.shape
    mu, v = heads(X, Y1, net, H1)
    ls = X.lift(net["ls"])
    sig = X.exp(ls)
    z = (X.lift(act_) - mu) / sig
    nlp = neglogp(X, z, net["ls"])
    adv = X.lift(ret) - X.lift(oval)
    o = dict(sz=z, sv=v, snlp=nlp, sadv=adv)
    if stored is not None:
        z, v, nlp, adv = (X.lift(np.asarray(stored[k], np.float32).reshape(np.shape(_val(o[k])))) for k in ("sz", "sv", "snlp", "sadv"))
    invM = 1.0 / M
    mean = X.scale(X.total(adv), invM)
    d = adv - mean
    std = X.sqrt(X.scale(X.total(X.square(d)), invM))
    advn = d / (std + X.const(1e-8))
    ratio = X.exp(X.lift(onlp) - nlp)
    lo, hi = np.float32(1) - np.float32(clip), np.float32(1) + np.float32(clip)
    rc = X.clip(ratio, float(lo), float(hi))
    pg1, pg2 = -advn * ratio, -advn * rc
    o.update(advn=advn, ratio=ratio, pg1=pg1, pg2=pg2, lo=float(lo), hi=float(hi))
    if side is None:
        side = _val(pg1) >= _val(pg2)
        side = side | ((_val(ratio) >= lo) & (_val(ratio) <= hi))
    dratio = X.where(side, -advn, X.lift(np.zeros(M)))
    g_nlp = X.scale(-dratio * ratio, invM)
    R_, ov = X.lift(ret), X.lift(oval)
    dv = v - R_
    l1 = X.square(dv)
    if clipvf >= 0:
        dd = v - ov
        vc = ov + X.clip(dd, -float(np.float32(clipvf)), float(np.float32(clipvf)))
        l2 = X.square(vc - R_)
        if vside is None:
            vside = (_val(l2) > _val(l1)) & ((_val(dd) < -clipvf) | (_val(dd) > clipvf))
        o["vc"], o["dd"], o["l1"], o["l2"] = vc, dd, l1, l2
        l1 = X.maximum(l1, l2)
        if isinstance(X, Bound):
            # inside the clip l2 may win by a rounding: dv is then vc - R, the same float64 value as v - R but rounded
            # through vc = ov + d
            alt = vc - R_
            dv = E(dv.v, np.where(np.abs(dd.v) <= clipvf + dd.e, np.maximum(dv.e, alt.e), dv.e))
        dv = X.where(vside, X.lift(np.zeros(M)), dv)
    o["sdv"] = X.scale(X.const(vf_coef) * dv, invM)
    o["sdm"] = (-g_nlp)[:, None] * z / sig
    o["sdls"] = g_nlp[:, None] * (X.lift(np.ones((M, A))) - X.square(z))
    o["pg"] = X.scale(X.total(X.maximum(pg1, pg2)), invM)
    o["vf"] = X.scale(X.scale(X.total(l1), 0.5), invM)
    o["kl"] = X.scale(X.scale(X.total(X.square(nlp - X.lift(onlp))), 0.5), invM)
    o["ent"] = X.total(X.cat([cst(X, HALF_LOG_2PI_E * A, np.float32(HALF_LOG_2PI_E) * np.float32(A), (1,)), ls], 0))
    o["side"], o["vside"] = side, vside
    return o


def _val(x):
    return x.v if isinstance(x, E) else np.asarray(x, np.float64)


def ppo_dz1(X, Y1, net, H1, sdm, sdv):
    """the tail's head backward from its stored seeds: dZ1 pi = (sdm Wpi^T)(1 - y^2), dZ1 vf = sdv Wvf (1 - y^2)"""
    yp, yv = X.lift(Y1[:, :H1]), X.lift(Y1[:, H1:2 * H1])
    one = X.lift(np.ones_like(Y1[:, :H1]))
    dp = X.contract("rj,kj->rk", X.lift(sdm), X.lift(net["Wpi"])) * (one - X.square(yp))
    dvf = X.lift(sdv)[:, None] * X.lift(net["Wvf"])[None, :] * (one - X.square(yv))
    return dp, dvf


def ppo_head_grads(X, Y1, H1, sdm, sdls, sdv, ent_coef):
    """the tail's head and logstd gradients from its stored seeds (serial fp32 sums over the minibatch).  The bound is the
    fp32 accuracy of a serial M-term sum, gamma_{M-1} sum|terms|: at M = 16384 that is about 1e-3 of sum|y sdm|, more than
    one row's share, so a single dropped or wrong row of a large minibatch can sit inside it.  Rows are held one by one
    where they are per-row outputs (sdm, sdls, sdv, dZ1); the sums are held only to this accuracy."""
    yp, yv = X.lift(Y1[:, :H1]), X.lift(Y1[:, H1:2 * H1])
    gW = X.contract("rk,rj->kj", yp, X.lift(sdm))
    gb = X.total(X.lift(sdm))
    gWvf = X.contract("rk,r->k", yv, X.lift(sdv))
    gbvf = X.total(X.lift(sdv))
    gls = X.total(X.lift(sdls)) - X.const(ent_coef)
    return dict(Wpi=gW, bpi=gb, Wvf=gWvf, bvf=gbvf, ls=gls)


def norm_blocks(n_train):
    """ppo_norm_kernel's partial index of each arena element (float4 i4 of a grid-stride loop over 128 x 256 threads)"""
    i4 = np.arange(n_train // 4 * 4) // 4
    return (i4 % (NORM_BLOCKS * NORM_THREADS)) // NORM_THREADS


def norm_partials(G, rel=0.0):
    """ppo_norm_kernel: part[b] = sum of g^2 over block b's elements; rel: a relative uncertainty of the stored G"""
    blk = norm_blocks(G.size)
    g = np.asarray(G[:blk.size], np.float64)
    sq = g * g
    v = np.bincount(blk, sq, NORM_BLOCKS)
    n = np.bincount(blk, None, NORM_BLOCKS)
    e = np.array([gamma(k - 1) for k in n]) * v * (1 + 2 * rel) + v * (2 * rel + rel * rel)
    return E(v, e)


def adam_scale(part, max_norm):
    """ppo_adam_kernel's fp32 reduction of the 128 partials (lanes stride 32, then the xor tree): (norm, scale), bit for bit"""
    p = np.asarray(part, np.float32)
    lane = np.zeros(32, np.float32)
    for i in range(NORM_BLOCKS):
        lane[i % 32] = np.float32(lane[i % 32] + p[i])
    o = 16
    while o:
        lane = np.float32(lane + lane[np.arange(32) ^ o])
        o >>= 1
    norm = np.sqrt(lane[0], dtype=np.float32)
    mn = np.float32(max_norm)
    return norm, np.float32(mn / np.maximum(norm, mn))


def lr_t(lr, t, b1=0.9, b2=0.999):
    return np.float32(float(np.float32(lr)) * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t))


# the fp32 constants (b1, 1 - b1, b2, 1 - b2, eps) as each kernel holds them: ppo_adam_kernel forms 1.f - b1 in fp32,
# trpo_vadam_kernel writes the literals 0.1f and 0.001f
TF_ADAM = (np.float32(0.9), np.float32(1) - np.float32(0.9), np.float32(0.999), np.float32(1) - np.float32(0.999), np.float32(1e-5))
MPI_ADAM = (np.float32(0.9), np.float32(0.1), np.float32(0.999), np.float32(0.001), np.float32(1e-8))


def adam(X, p, m, v, g, lrt, b1, c1, b2, c2, eps):
    """TF1 / MpiAdam element update with the kernel's fp32 constants (b1, c1 = 1 - b1, b2, c2 = 1 - b2, eps):
    m = b1 m + c1 g, v = b2 v + c2 g^2, p -= lr_t m / (sqrtf(v) + eps)"""
    k = (lambda c: X.lift(np.float64(c))) if isinstance(X, Bound) else np.float32
    m2 = k(b1) * X.lift(m) + k(c1) * X.lift(g)
    v2 = k(b2) * X.lift(v) + k(c2) * X.square(X.lift(g))
    step = k(lrt) * m2 / (X.sqrt(v2) + k(eps))
    return m2, v2, X.lift(p) - step


# ================================================================================================ TRPO
def trpo_prep(X, Y1, net, H1, act_, adv, entcoeff):
    """trpo_prep_kernel: atarg from float64 mean / population std, mean and neglogp at theta_old, the seeds, the losses"""
    N, A = act_.shape
    a64 = np.asarray(adv, np.float64)
    mean = a64.sum() / N
    std = math.sqrt(((a64 - mean) ** 2).sum() / N)
    at64 = (a64 - mean) / (std + 1e-8)
    e_mean = gamma64(N + 1) * np.abs(a64).mean()
    e_std = gamma64(2 * N + 4) * std + e_mean
    atarg = E(at64, U * np.abs(at64) + (e_mean + np.abs(at64) * e_std) / (std + 1e-8) + 4 * U64 * np.abs(at64))
    mu, _ = heads(X, Y1, net, H1)
    ls = X.lift(net["ls"])
    sig = X.exp(ls)
    z = (X.lift(act_) - mu) / sig
    nlp = neglogp(X, z, net["ls"])
    return dict(atarg=atarg, mu_old=mu, nlp_old=nlp, z=z, sig=sig)


def trpo_seeds(X, atarg_f32, z, sig, N):
    """the seeds from the stored atarg: sdm = at z / sig / N, sdls = at (z^2 - 1) / N"""
    at = X.lift(atarg_f32)[:, None]
    sdm = at * z / sig
    sdls = at * (X.square(z) - X.lift(np.ones(np.shape(_val(z)))))
    return X.scale(sdm, 1.0 / N), X.scale(sdls, 1.0 / N)


def trpo_prep_losses(atarg, ls, entcoeff):
    """the losses at theta_old (met[0:5]) from the stored atarg, in float64: optimgain, meankl 0, entbonus, surrgain, entropy"""
    N = atarg.size
    surr = np.asarray(atarg, np.float64).sum() / N
    ent = HALF_LOG_2PI_E * ls.size + np.asarray(ls, np.float64).sum()
    eb = float(np.float32(entcoeff)) * ent
    v = np.array([surr + eb, 0.0, eb, surr, ent])
    mag = np.array([abs(surr) + abs(eb), 0, abs(eb), abs(surr), abs(ent)]) + np.abs(atarg).sum() / N
    return E(v, U * np.abs(v) + gamma64(N + ls.size + 4) * mag)


def head_bwd(X, seed, Wpi, Y1rows):
    """trpo_head_bwd_kernel: dZ1[r, k] = (sum_j seed[r, j] Wpi[k, j]) (1 - y[r, k]^2)"""
    one = X.lift(np.ones_like(Y1rows))
    return X.contract("rj,kj->rk", X.lift(seed), X.lift(Wpi)) * (one - X.square(X.lift(Y1rows)))


def head_grad(Y1rows, seed):
    """trpo_headgrad_kernel: float64 sums over rows, one fp32 rounding: gW [H1, A] = Y1^T seed, gb [A] = sum seed"""
    y, s = np.asarray(Y1rows, np.float64), np.asarray(seed, np.float64)
    M = y.shape[0]
    gW, gb = y.T @ s, s.sum(0)
    return (E(gW, U * np.abs(gW) + gamma64(M) * (np.abs(y).T @ np.abs(s))),
            E(gb, U * np.abs(gb) + gamma64(M) * np.abs(s).sum(0)))


def tangent(X, Tpre, vb, Yrows):
    """trpo_tangent_kernel: (1 - y^2)(T + vb)"""
    one = X.lift(np.ones_like(Yrows))
    return (one - X.square(X.lift(Yrows))) * (Tpre + X.lift(vb))


def fvp_head(X, T1, Y1rows, Wpi, Vpi, vbpi, ls, M):
    """trpo_fvp_head_kernel: u = (vbpi + sum_k T1 Wpi + Y1 Vpi) / (expf(2 ls) M), one serial chain of 2 H1 fmafs"""
    num = X.contract("rk,kj->rj", X.cat([X.lift(T1), X.lift(Y1rows)], 1), X.cat([X.lift(Wpi), X.lift(Vpi)], 0), bias=X.lift(vbpi))
    den = X.exp(X.scale(X.lift(ls), 2.0))
    den = X.scale(den, float(M)) if pow2(M) else den * X.lift(np.float64(np.float32(M)))
    return num / den


def ls_rows(Y1c, Wc, bc, lsc, act_, mu_old, nlp_old, atarg, ls_old):
    """trpo_ls_loss_kernel per row of one candidate: (surrogate ratio * atarg, KL) in float64 with their bounds"""
    X = Bound()
    mu = X.contract("rq,qj->rj", X.lift(Y1c), X.lift(Wc), bias=X.lift(bc))
    sig = X.exp(X.lift(lsc))
    z = (X.lift(act_) - mu) / sig
    nlp = neglogp(X, z, lsc)
    ratio = np.exp(np.asarray(nlp_old, np.float64) - nlp.v)
    at = np.asarray(atarg, np.float64)
    su = E(ratio * at, np.abs(ratio * at) * np.expm1(nlp.e) + 4 * U64 * np.abs(ratio * at))
    ls64, lo64 = np.asarray(lsc, np.float64), np.asarray(ls_old, np.float64)
    so, sn = np.exp(lo64), np.exp(ls64)
    dm = np.asarray(mu_old, np.float64) - mu.v
    t = ls64 - lo64 + (so * so + dm * dm) / (2 * sn * sn) - 0.5
    kl = E(t.sum(1), ((2 * np.abs(dm) * mu.e + mu.e ** 2) / (2 * sn * sn)).sum(1) + 16 * U64 * np.abs(t).sum(1) * (1 + ls64.size))
    return su, kl


def ls_partials(rows_val):
    """the 64 fixed-grid double partials of one candidate (grid-stride over 64 x 256 threads): rows -> blocks"""
    n = rows_val.v.size
    blk = (np.arange(n) % (LS_BLOCKS * LS_THREADS)) // LS_THREADS
    v = np.bincount(blk, rows_val.v, LS_BLOCKS)
    e = np.bincount(blk, rows_val.e, LS_BLOCKS) + gamma64(n) * np.bincount(blk, np.abs(rows_val.v), LS_BLOCKS)
    return E(v, e)


def ls_select(lspart, lsc, N, A, entcoeff, max_kl, before):
    """trpo_ls_select_kernel's decision from the stored partials, bit for bit: -> (k or -1, [K][5] losses as fp32)"""
    P = np.asarray(lspart, np.float64).reshape(NCAND, LS_BLOCKS, 2)
    out = []
    acc = -1
    for k in range(NCAND):
        su = kl = 0.0
        for b in range(LS_BLOCKS):
            su += P[k, b, 0]
            kl += P[k, b, 1]
        su /= N
        kl /= N
        ent = HALF_LOG_2PI_E * A
        for j in range(A):
            ent += float(lsc[k, j])
        ec = float(np.float32(entcoeff))
        l = np.array([su + ec * ent, kl, ec * ent, su, ent], np.float32)
        out.append(l)
        if acc < 0 and np.isfinite(l).all() and not l[1] > np.float32(1.5) * np.float32(max_kl) and not np.float32(l[0] - np.float32(before)) < 0:
            acc = k
    return acc, np.array(out)


def vf_tail(X, vY1, Wvf, bvf, ret_rows):
    """trpo_vf_tail_kernel: v (serial fmaf chain), e = v - R, dv = 2 e / 128, dZ1 = dv Wvf (1 - y^2), float64 head sums"""
    v = X.contract("rk,k->r", X.lift(vY1), X.lift(Wvf), bias=X.lift(bvf[0]))
    e = v - X.lift(ret_rows)
    dv = X.scale(X.scale(e, 2.0), 1.0 / VF_BATCH)
    one = X.lift(np.ones_like(vY1))
    dz1 = dv[:, None] * X.lift(Wvf)[None, :] * (one - X.square(X.lift(vY1)))
    return dict(v=v, e=e, dv=dv, dZ1=dz1)
