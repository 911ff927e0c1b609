"""The PPO2 and TRPO kernels held element by element to float64 of the inputs they read (tests/ac_kernels_ref.py).

The step-level tests (test_gpu_ppo.py, test_gpu_trpo.py) compare gradients and rollouts by relative norm or by
max|err| / max|ref|: one wrong action component, minibatch row, logstd entry, env column or [::5] Fisher row moves those by
less than their bars.  Here each case runs one explicit step, rollout, update or fvp call, reads the handle's device buffers
back (b2g_debug_ppo_tensor / b2g_debug_trpo_tensor) and checks:
  * bit for bit: the row maps of ppo_rows_kernel, trpo_rows_kernel and ac_iota_rows_kernel; trpo_cand_kernel and
    trpo_apply_kernel (p + 0.5^k f, entries with f == 0 untouched); trpo_vec_kernel op 3 (x / lm), and ops 0 and 1 of a
    one-iteration CG (x = alpha g); the logstd block of trpo_fvp_finish_kernel; the untouched q/* entries and the zero vf entries of
    the policy vectors (G, X, FS, Zv); ppo_adam_kernel's G <- G scale (scale reproduced from the stored partials) and the
    stream-1 step counter;
  * within a bound derived from the inputs (never a fitted constant), per element: ppo_bias_tanh_kernel; ppo_act_kernel's
    rollout mode and its predict mode, deterministic and stochastic; ppo_gae_kernel per env column; ppo_tail_kernel's
    sz sv snlp sadv, the normalised advantage, sdm sdls sdv, dZ1 of both towers, the head and logstd gradients and the five
    metrics; ppo_norm_kernel's partials; ppo_adam_kernel's m, v, p; trpo_prep_kernel (atarg, mu_old, nlp_old, seeds,
    losses); trpo_headgrad_kernel (the policy step's gradient and the Fisher product's head block); trpo_tangent_kernel (T0,
    T1); trpo_fvp_head_kernel (u); trpo_head_bwd_kernel over the [::5] rows; trpo_fvp_finish_kernel; trpo_dot_kernel through
    sc[RR]; trpo_ls_l0_kernel for all ten candidates; trpo_ls_loss_kernel's partials; trpo_vf_tail_kernel; trpo_vadam_kernel;
  * decisions, on the side the kernel revealed, which must be float64's unless its input lies within its bound of the
    threshold: the ratio clip / tf.maximum gate, the value clip, clipfrac, the global-norm clip, trpo_ls_select_kernel's
    first acceptable k (its fp32 KL compare reproduced bit for bit from the stored partials, and float64's choice held to it),
    CG_INIT's np.allclose(g, 0) zero test, CG's r.r < 1e-10 stop;
  * conjugate gradient iteration by iteration (b2g_debug_trpo_cg stops after k iterations and returns the state before the
    last): the Fisher product of that iteration's p, alpha, x and r (vec op 1), r.r, beta and p (vec op 2, which still runs
    under SC_DONE = 2), and after the stop that x, r and the scalars stay put; shs, lm and the expected improvement of the
    step; ppo_act_kernel's bootstrap mode through TRPO's value of the next batch's row 0; the four line-search outcomes of
    test_gpu_trpo.py's fixtures (accept at 0, after a KL rejection, after K and I, reject all); N = 127 runs no value step.

`pytest -s` prints each quantity's worst err/bar for every case.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from b200grasp import _lib
from b200grasp.ppo2 import PPO2Learner
from b200grasp.trpo_mpi import TRPOLearner
from oracle import philox_ref as PX
from oracle import ppo_ref as PR
from tests import ac_kernels_ref as K
from tests.ac_kernels_ref import Bound, E, SLACK, U
from tests.gg_tc_ref import Report

pytestmark = pytest.mark.gpu
INTS = {"rowidx", "rowoff", "perm", "act_rowoff", "vrowoff"}
MAX_GRAD_NORM, MAX_KL, CG_DAMPING = 0.5, 0.01, 1e-2


def read(L, kind, name):
    n, eb = C.c_int64(), C.c_int32()
    _lib.check(getattr(L.lib, f"b2g_debug_{kind}_tensor_info")(L.h, name.encode(), C.byref(n), C.byref(eb)))
    dt = {4: np.int32 if name in INTS else np.float32, 8: np.int64 if name == "counters" else np.float64}[eb.value]
    out = np.empty(n.value, dt)
    _lib.check(getattr(L.lib, f"b2g_debug_{kind}_tensor")(L.h, name.encode(), out.ctypes.data_as(C.c_void_p), out.nbytes))
    return out


def hold(rep, name, got, ref):
    rep.hold(name, np.asarray(got, np.float64).reshape(ref.v.shape), ref.v, SLACK * ref.e, 1.0)


def side_ok(rep, name, got, f64, near):
    """a decision the kernel revealed: float64's side unless the input is within its bound of the threshold"""
    bad = (np.asarray(got) != np.asarray(f64)) & ~np.asarray(near)
    rep.exact(f"{name} side", bad, np.zeros_like(bad))


# ================================================================================================ PPO2
@dataclasses.dataclass(frozen=True)
class PpoCase:
    name: str
    D: int
    A: int
    H: tuple
    M: int
    cvf: float = 0.2            # < 0: no value clipping
    clip: float = 0.2
    scale: float = 1.0          # observation scale: 0.01 keeps the global norm below max_grad_norm
    ent: float = 0.01
    clipped: object = None      # the global-norm clip side the case is built to take (None: either)


PPO_CASES = [
    PpoCase("d1_a1_w4_m1", 1, 1, (4, 4), 1),
    PpoCase("d7_a16_w256x4_m33", 7, 16, (256, 4), 33, cvf=0.05),
    PpoCase("d100_a3_w64_m31", 100, 3, (64, 64), 31, cvf=-1.0, clipped=True),
    PpoCase("d100_a3_w64_m32_small", 100, 3, (64, 64), 32, cvf=-1.0, scale=0.01, clipped=False),
    PpoCase("d100_a3_w8x256_m2", 100, 3, (8, 256), 2),
    PpoCase("d20480_a3_w64_m1023", 20480, 3, (64, 64), 1023, cvf=0.1),
    PpoCase("d100_a16_w256_m1025_small", 100, 16, (256, 256), 1025, cvf=-1.0, scale=0.01, ent=0.0),
    PpoCase("d7_a1_w4_m16384_clip0", 7, 1, (4, 4), 16384, clip=0.0),
]


def ppo_params(D, A, H, seed):
    p = PR.init_params(D, A, H, np.random.default_rng(seed))
    rng = np.random.default_rng(seed + 100)
    for k in p:
        if p[k].ndim == 1 or k.endswith("logstd"):
            p[k] = rng.uniform(-0.3, 0.3, p[k].shape).astype(np.float32)
    p["model/pi/w"] = (p["model/pi/w"] * 50).astype(np.float32)
    return p


def ppo_minibatch(p, M, D, A, seed, scale):
    rng = np.random.default_rng(seed)
    x = (rng.normal(0, 1, (M, D)) * scale / np.sqrt(D)).astype(np.float32)
    mean, v = PR.forward(p, x)
    std = np.exp(p["model/pi/logstd"].astype(np.float64).reshape(-1))
    act = (mean + std * rng.normal(0, 1, (M, A))).astype(np.float32)
    nlp = PR.neglogp(mean, p["model/pi/logstd"], act)
    return (x, (v + rng.uniform(-0.5, 0.5, M) + rng.normal(0, 1, M)).astype(np.float32), act,
            (v + rng.uniform(-0.5, 0.5, M)).astype(np.float32), (nlp + rng.uniform(-0.6, 0.6, M)).astype(np.float32))


def check_tail(rep, L, c, net, rows, act, oval, onlp, ret, clip, cvf, H1, vf_coef=0.5):
    """ppo_tail_kernel on the minibatch rows `rows` of the stored inputs"""
    M, A = len(rows), act.shape[1]
    T = {n: read(L, "ppo", n) for n in ("Y1", "sz", "sv", "snlp", "sadv", "sdm", "sdls", "sdv", "dZ1", "met", "G", "part", "hp")}
    Y1 = T["Y1"][:M * 2 * H1].reshape(M, 2 * H1)
    sdm, sdls, sdv = T["sdm"][:M * A].reshape(M, A), T["sdls"][:M * A].reshape(M, A), T["sdv"][:M]
    rep.exact("hp (lr, cliprange, cliprange_vf)", T["hp"][1:3], np.array([clip, cvf], np.float32))
    side = (sdm != 0).any(1) | (sdls != 0).any(1)
    vside = (sdv == 0) & (T["sv"][:M] != ret[rows]) if cvf >= 0 else None
    X = Bound()
    o = K.ppo_tail(X, Y1, net, H1, act[rows], oval[rows], onlp[rows], ret[rows], clip, cvf, c.ent, vf_coef, side=side, vside=vside,
                   stored={k: T[k][:M * (A if k == "sz" else 1)] for k in ("sz", "sv", "snlp", "sadv")})
    for k in ("sz", "sv", "snlp", "sadv", "sdm", "sdls", "sdv"):
        n = o[k].v.size
        hold(rep, f"tail {k}", T[k][:n], o[k])
    # the gate: float64's side unless ratio is within its bound of a clip edge or pg1 - pg2 of 0, or advn is 0
    r, adv = o["ratio"], o["advn"]
    g64 = (o["pg1"].v >= o["pg2"].v) | ((r.v >= o["lo"]) & (r.v <= o["hi"]))
    near = (np.abs(r.v - o["lo"]) <= SLACK * r.e) | (np.abs(r.v - o["hi"]) <= SLACK * r.e) | (np.abs(adv.v) <= SLACK * adv.e)
    near |= np.abs(o["pg1"].v - o["pg2"].v) <= SLACK * (o["pg1"].e + o["pg2"].e)
    side_ok(rep, "ratio clip / tf.maximum", side, g64, near)
    if cvf >= 0:
        dd, l1, l2 = o["dd"], o["l1"], o["l2"]
        v64 = (l2.v > l1.v) & ((dd.v < -cvf) | (dd.v > cvf))
        vnear = (np.abs(l2.v - l1.v) <= SLACK * (l1.e + l2.e)) | (np.abs(np.abs(dd.v) - cvf) <= SLACK * dd.e + U * cvf)
        vnear |= np.abs(o["sv"].v - ret[rows]) <= SLACK * o["sv"].e
        side_ok(rep, "value clip", vside, v64, vnear)
    met = T["met"]
    for k, key in (("pg", "PG"), ("vf", "VF"), ("ent", "ENT"), ("kl", "KL")):
        hold(rep, f"metric {k}", met[K.PM[key]:K.PM[key] + 1], E(o[k].v.reshape(1), o[k].e.reshape(1)))
    # clipfrac: the count of |ratio - 1| > clip, within the rows whose side fp32 could take either way
    dev = np.abs(r.v - 1.0)
    sure, maybe = dev - SLACK * r.e > clip, np.abs(dev - clip) <= SLACK * r.e + U
    lo_cf, hi_cf = sure.sum() / M, (sure | maybe).sum() / M
    cf = float(met[K.PM["CLIP"]])
    rep.exact("clipfrac within its undecided rows", np.array(lo_cf * (1 - 4 * U) <= cf <= hi_cf * (1 + 4 * U) + 0.0), np.array(True))
    # head backward and head gradients from the stored seeds
    dp, dvf = K.ppo_dz1(X, Y1, net, H1, sdm, sdv)
    dZ1 = T["dZ1"][:M * 2 * H1].reshape(M, 2 * H1)
    hold(rep, "dZ1 pi", dZ1[:, :H1], dp)
    hold(rep, "dZ1 vf", dZ1[:, H1:], dvf)
    # the stored gradient is g * scale (ppo_adam_kernel), scale reproduced bit for bit from the stored partials
    norm, sc = K.adam_scale(T["part"], MAX_GRAD_NORM)
    hold(rep, "grad norm metric", met[K.PM["GN"]:K.PM["GN"] + 1], E(np.array([float(norm)]), np.zeros(1)))
    gr = K.ppo_head_grads(X, Y1, H1, sdm, sdls, sdv, c.ent)
    o_, n_train, _ = K.layout(c.D, A, *c.H)
    G = T["G"]
    for k, blk in (("Wpi", "Wpi"), ("bpi", "bpi"), ("Wvf", "Wvf"), ("bvf", "bvf"), ("ls", "ls")):
        ref = gr[k] * X.lift(np.float64(sc)) if sc != 1 else gr[k]
        n = ref.v.size
        hold(rep, f"grad {k} (x scale)", G[o_[blk]:o_[blk] + n], ref)
    return T, norm, sc


def check_norm_adam(rep, L, c, T, norm, sc, P0, lr, n_train):
    """ppo_norm_kernel partials from the stored (scaled) G, the clip decision, ppo_adam_kernel's moments and parameters"""
    G = T["G"][:n_train]
    pre = G.astype(np.float64) / float(sc)
    part = K.norm_partials(pre, rel=0.0 if sc == 1 else 2 * U)
    hold(rep, "norm partials", T["part"], part)
    n64 = np.sqrt(part.v.sum())
    n_e = np.sqrt(part.v.sum() + part.e.sum() + K.gamma(128) * part.v.sum()) - n64
    clipped = sc != 1
    side_ok(rep, "global-norm clip", np.array(clipped), np.array(n64 > MAX_GRAD_NORM),
            np.array(abs(n64 - MAX_GRAD_NORM) <= SLACK * n_e + U * n64))
    if c.clipped is not None:
        rep.exact("global-norm clip taken as the case intends", np.array(clipped), np.array(c.clipped))
    Mo, Vo, P = (read(L, "ppo", n)[:n_train] for n in ("Mo", "Vo", "P"))
    cnt = read(L, "ppo", "counters")
    rep.exact("Adam step counter", cnt[0:1], np.array([1]))
    X = Bound()
    m2, v2, p2 = K.adam(X, P0[:n_train], np.zeros(n_train), np.zeros(n_train), G, K.lr_t(lr, 1), *K.TF_ADAM)
    hold(rep, "Adam m", Mo, m2)
    hold(rep, "Adam v", Vo, v2)
    hold(rep, "Adam p", P, p2)


@pytest.mark.parametrize("c", PPO_CASES, ids=lambda c: c.name)
def test_ppo_explicit_step_kernels(c):
    seed = c.D + 7 * c.A + c.M
    L = PPO2Learner(c.D, c.A, c.H, n_envs=1, n_steps=c.M, nminibatches=1, noptepochs=1, seed=seed, ent_coef=c.ent,
                    max_grad_norm=MAX_GRAD_NORM)
    rep = Report(f"PPO2 {c.name}")
    try:
        p = ppo_params(c.D, c.A, c.H, seed)
        L.load_parameters(p)
        x, ret, act, ov, onlp = ppo_minibatch(p, c.M, c.D, c.A, seed, c.scale)
        P0 = read(L, "ppo", "P")
        o_, n_train, n_total = K.layout(c.D, c.A, *c.H)
        net = K.unpack(P0, o_, c.D, c.A, *c.H)
        lr = 1e-3
        L.train_step_explicit(x, ret, act, ov, onlp, lr, c.clip, c.cvf, apply_update=True)
        H0, H1 = c.H
        Z0, Y0 = read(L, "ppo", "Z0"), read(L, "ppo", "Y0")
        n = c.M * 2 * H0
        hold(rep, "bias_tanh Y0", Y0[:n], K.bias_tanh(Bound(), Z0[:n].reshape(c.M, 2 * H0), net["b0"]))
        rows = np.arange(c.M)
        T, norm, sc = check_tail(rep, L, c, net, rows, act, ov, onlp, ret, c.clip, c.cvf, H1)
        check_norm_adam(rep, L, c, T, norm, sc, P0, lr, n_train)
        P = read(L, "ppo", "P")
        rep.exact("q/* untouched", P[n_train:n_total], P0[n_train:n_total])
    finally:
        L.close()
    rep.finish()


ROLLOUTS = [(1, 6, 3, (4, 4), 7), (3, 4, 16, (64, 64), 100), (1025, 2, 3, (8, 256), 1), (4096, 2, 16, (256, 4), 7)]


@pytest.mark.parametrize("E_,T_,A,H,D", ROLLOUTS, ids=lambda v: str(v))
def test_ppo_rollout_gae_update_kernels(E_, T_, A, H, D):
    """rollout rows (ac_iota_rows_kernel, ppo_act_kernel mode 0, stream-1 steps), GAE per env, ppo_rows_kernel, and the last
    minibatch's tail through its row map (lr 0 keeps the parameters the tail read); predict in both modes"""
    seed = 50 + E_ + A
    nmb = 2
    L = PPO2Learner(D, A, H, n_envs=E_, n_steps=T_, nminibatches=nmb, noptepochs=1, seed=seed, max_grad_norm=MAX_GRAD_NORM)
    rep = Report(f"PPO2 rollout E={E_} T={T_} A={A} H={H} D={D}")
    H0, H1 = H
    try:
        p = ppo_params(D, A, H, seed)
        L.load_parameters(p)
        P0 = read(L, "ppo", "P")
        o_, n_train, _ = K.layout(D, A, H0, H1)
        net = K.unpack(P0, o_, D, A, H0, H1)
        rng = np.random.default_rng(seed)
        obs = rng.normal(0, 1, (T_ + 1, E_, D)).astype(np.float32)
        rew = rng.normal(0, 1, (T_, E_)).astype(np.float32)
        done = (rng.random((T_, E_)) < 0.3).astype(np.float32)
        key = PX.act_seed(seed)
        X = Bound()
        XS = -(-D // 4) * 4
        for t in range(T_):
            step = int(read(L, "ppo", "counters")[1])
            a = L.rollout_act(obs[t])
            rep.exact("act_rowoff", read(L, "ppo", "act_rowoff"), ((t * E_ + np.arange(E_)) * XS).astype(np.int32))
            Y1 = read(L, "ppo", "Y1")[:E_ * 2 * H1].reshape(E_, 2 * H1)
            z = K.noise(key, step, E_, A)
            ra, rv, rn = K.act(X, Y1, net, H1, z)
            hold(rep, "act mode 0: actions", a, ra)
            ract = read(L, "ppo", "r_act").reshape(T_ + 1, E_, A)[t]
            rep.exact("act mode 0: stored row t", ract, a)
            hold(rep, "act mode 0: value", read(L, "ppo", "r_val").reshape(T_ + 1, E_)[t], rv)
            hold(rep, "act mode 0: neglogp", read(L, "ppo", "r_nlp").reshape(T_ + 1, E_)[t], rn)
            rep.exact("stream-1 step advanced once", read(L, "ppo", "counters")[1:2], np.array([step + 1]))
            L.rollout_reward(rew[t], done[t])
        perm = rng.permutation(T_ * E_)[None].astype(np.int32)
        L.update(obs[T_], perm, 0.0, 0.2, 0.2)
        r = {n: read(L, "ppo", n) for n in ("r_rew", "r_val", "r_done", "lastv", "r_adv", "r_ret", "rowidx", "rowoff", "r_act", "r_nlp")}
        val = r["r_val"].reshape(T_ + 1, E_)
        dn = r["r_done"].reshape(T_ + 1, E_)
        # the update copied row T's flags to row 0 after GAE read them: GAE saw row 0 as the rollout's first flags (zeros)
        dn_seen = dn.copy()
        dn_seen[0] = 0.0
        dn_seen[1:] = done
        adv, ret = K.gae(X, r["r_rew"].reshape(T_, E_), val, dn_seen, r["lastv"], 0.99, 0.95)
        for t in range(T_):
            hold(rep, "GAE adv (per env column)", r["r_adv"].reshape(T_, E_)[t], adv[t])
            hold(rep, "GAE ret (per env column)", r["r_ret"].reshape(T_, E_)[t], ret[t])
        f = perm[0]
        ridx = ((f % T_) * E_ + f // T_).astype(np.int32)
        rep.exact("ppo_rows rowidx", r["rowidx"], ridx)
        rep.exact("ppo_rows rowoff", r["rowoff"], (ridx * XS).astype(np.int32))
        # the last minibatch's tail through its row map
        M = T_ * E_ // nmb
        rows = ridx[(nmb - 1) * M:]
        c = PpoCase("rollout", D, A, H, M)
        act_all = r["r_act"].reshape(-1, A)
        check_tail(rep, L, c, net, rows, act_all, val.reshape(-1), r["r_nlp"], r["r_ret"], 0.2, 0.2, H1)
        rep.exact("lr 0 leaves P", read(L, "ppo", "P")[:n_train], P0[:n_train])
        # predict: deterministic (no draw), then stochastic (one draw)
        n = min(64, E_)
        xo = rng.normal(0, 1, (n, D)).astype(np.float32)
        for det in (True, False):
            step = int(read(L, "ppo", "counters")[1])
            a, v, nl = L.act(xo, deterministic=det)
            Y1 = read(L, "ppo", "Y1")[:n * 2 * H1].reshape(n, 2 * H1)
            z = K.noise(key, step, n, A) if not det else E(np.zeros((n, A)))
            ra, rv, rn = K.act(X, Y1, net, H1, z)
            hold(rep, f"predict det={det}: actions", a, ra)
            hold(rep, f"predict det={det}: value", v, rv)
            hold(rep, f"predict det={det}: neglogp", nl, rn)
            rep.exact(f"predict det={det}: stream-1 step", read(L, "ppo", "counters")[1:2], np.array([step + (0 if det else 1)]))
    finally:
        L.close()
    rep.finish()


# ================================================================================================ TRPO
@dataclasses.dataclass(frozen=True)
class TrpoCase:
    name: str
    D: int
    A: int
    H: tuple
    N: int
    ent: float = 0.0
    cg: int = 10
    vf_iters: int = 1
    seed: int = 0
    max_kl: float = MAX_KL
    ls: str = ""                # a line-search outcome fixture of tests/test_gpu_trpo.py (its shapes replace the case's)


TRPO_CASES = [
    TrpoCase("n1_d1_a1_w4", 1, 1, (4, 4), 1, cg=1, vf_iters=0),
    TrpoCase("n4_d7_a3_w256x4", 7, 3, (256, 4), 4, ent=0.01, cg=2, vf_iters=0),
    TrpoCase("n6_d100_a16_w4x256", 100, 16, (4, 256), 6, cg=1, vf_iters=0),
    TrpoCase("n127_d7_a3_w64_novalue", 7, 3, (64, 64), 127, vf_iters=2, seed=2),
    TrpoCase("n129_d7_a3_w64", 7, 3, (64, 64), 129, ent=0.01, vf_iters=1),
    TrpoCase("n1024_d100_a3_w256", 100, 3, (256, 256), 1024, cg=3, vf_iters=0, seed=3),
    TrpoCase("n16384_d20_a16_w8x256", 20, 16, (8, 256), 16384, cg=1, vf_iters=0, seed=4),
] + [TrpoCase(f"ls_{k}", 0, 0, (8, 8), 0, vf_iters=0, ls=k) for k in ("zero", "kl", "imp", "reject")]


def dot64(a, b):
    """a float64 dot product of fp32 vectors in any order: trpo_dot_kernel's fixed-grid partials and their sum"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    v = a @ b
    return E(np.array([v]), np.array([K.gamma64(a.size + K.DOT_BLOCKS) * (np.abs(a) @ np.abs(b))]))


def check_zero_test(rep, amax, G, sc):
    """trpo_dot_kernel's max partials (exact: a max of |g| over each block's grid-stride elements) and CG_INIT's
    np.allclose(g, 0) decision: every |g_i| <= 1e-8"""
    n = G.size
    blk = (np.arange(n) % (K.DOT_BLOCKS * 256)) // 256
    want = np.zeros(K.DOT_BLOCKS)
    np.maximum.at(want, blk, np.abs(G.astype(np.float64)))
    rep.exact("amax partials", amax, want)
    rep.exact("zero test (max |g| <= 1e-8)", np.array([sc[K.SC["ZERO"]]]), np.array([1.0 if want.max() <= 1e-8 else 0.0]))


def trpo_setup(c):
    """-> (learner, case with the fixture's shapes, obs, actions, advantages, returns)"""
    from b200grasp.trpo_mpi import init_params
    if c.ls:
        from tests.test_gpu_trpo import ls_fixture
        p, obs, act, adv, max_kl, _ = ls_fixture(c.ls)
        c = dataclasses.replace(c, D=obs.shape[1], A=act.shape[1], N=obs.shape[0], max_kl=max_kl)
        L = TRPOLearner(c.D, c.A, c.H, c.N, cg_iters=c.cg, vf_iters=0, seed=0, max_kl=c.max_kl, cg_damping=CG_DAMPING)
        L.load_parameters(p)
        return L, c, obs, act, adv, adv
    L = TRPOLearner(c.D, c.A, c.H, c.N, cg_iters=c.cg, vf_iters=c.vf_iters, entcoeff=c.ent, seed=c.seed, vf_stepsize=3e-4,
                    max_kl=c.max_kl, cg_damping=CG_DAMPING)
    p = init_params(c.D, c.A, c.H, c.seed)
    rng = np.random.default_rng(c.seed + 7)
    for s in ("pi/model/", "oldpi/model/"):
        p[s + "pi/logstd"] = rng.normal(0, 0.2, p[s + "pi/logstd"].shape).astype(np.float32)
        p[s + "pi/w"] = (p[s + "pi/w"] * 30).astype(np.float32)
        for k in ("pi_fc0/b", "pi_fc1/b", "vf_fc0/b", "vf_fc1/b", "pi/b", "vf/b"):
            p[s + k] = rng.normal(0, 0.1, p[s + k].shape).astype(np.float32)
    L.load_parameters(p)
    rng = np.random.default_rng(c.seed + 1)
    obs = (rng.uniform(0, 1, (c.N, c.D)) if c.D < 1000 else rng.normal(0, 1, (c.N, c.D)) / np.sqrt(c.D)).astype(np.float32)
    return L, c, obs, rng.normal(0, 1, (c.N, c.A)).astype(np.float32), rng.normal(0, 1, c.N).astype(np.float32), \
        rng.normal(0, 1, c.N).astype(np.float32)


def check_fvp(rep, L, c, net, Pv, o_):
    """the Fisher-vector product's kernels over the rows [::5], from what the last one left: Zv = F Pv at the parameters net"""
    D, A, (H0, H1), NF = c.D, c.A, c.H, (c.N + 4) // 5
    X = Bound()
    T = {n: read(L, "trpo", n) for n in ("Zv", "T0", "T1", "u", "dZ1", "Y0", "Y1", "r_obs")}
    Zv = T["Zv"]
    XS = -(-D // 4) * 4
    obs = T["r_obs"][:(c.N + 1) * XS].reshape(c.N + 1, XS)[:c.N:5, :D]
    Y0 = T["Y0"][:c.N * 2 * H0].reshape(c.N, 2 * H0)[::5, :H0]
    Y1 = T["Y1"][:c.N * 2 * H1].reshape(c.N, 2 * H1)[::5, :H1]
    vn = K.unpack(Pv, o_, D, A, H0, H1)
    # T0 = (1 - y0^2)(x V0 + vb0): the contraction's split-R atomics are a sum of D terms in unknown order
    t0 = X.contract("rd,dc->rc", X.lift(obs), X.lift(vn["W0"][:, :H0]))
    T0 = T["T0"][:NF * H0].reshape(NF, H0)
    hold(rep, "tangent T0", T0, K.tangent(X, t0, vn["b0"][:H0], Y0))
    t1 = X.contract("rk,kc->rc", X.cat([X.lift(T0), X.lift(Y0)], 1), X.cat([X.lift(net["W1"][0]), X.lift(vn["W1"][0])], 0))
    T1 = T["T1"][:NF * H1].reshape(NF, H1)
    hold(rep, "tangent T1", T1, K.tangent(X, t1, vn["b1"][0], Y1))
    u = T["u"][:NF * A].reshape(NF, A)
    hold(rep, "fvp_head u", u, K.fvp_head(X, T1, Y1, net["Wpi"], vn["Wpi"], vn["bpi"], net["ls"], NF))
    hold(rep, "head_bwd dZ1 over [::5]", T["dZ1"][:NF * H1].reshape(NF, H1), K.head_bwd(X, u, net["Wpi"], Y1))
    gW, gb = K.head_grad(Y1, u)
    d = np.float32(CG_DAMPING)
    for nm, g in (("Wpi", gW), ("bpi", gb)):
        n = g.v.size
        v = Pv[o_[nm]:o_[nm] + n].astype(np.float64)
        ref = E(g.v.reshape(-1) + float(d) * v, g.e.reshape(-1) + U * np.abs(float(d) * v) + U * (np.abs(g.v.reshape(-1)) + np.abs(float(d) * v)))
        hold(rep, f"fvp headgrad + finish {nm}", Zv[o_[nm]:o_[nm] + n], ref)
    v = Pv[o_["ls"]:o_["ls"] + A]
    rep.exact("fvp_finish logstd 2v + damping", Zv[o_["ls"]:o_["ls"] + A], np.float32(np.float32(0) + d * v) + np.float32(2) * v)


@pytest.mark.parametrize("c", TRPO_CASES, ids=lambda c: c.name)
def test_trpo_step_kernels(c):
    L, c, obs, act, adv, ret = trpo_setup(c)
    rep = Report(f"TRPO {c.name}")
    D, A, (H0, H1), N = c.D, c.A, c.H, c.N
    try:
        o_, n_train, n_total = K.layout(D, A, H0, H1)
        P0 = read(L, "trpo", "P")
        net = K.unpack(P0, o_, D, A, H0, H1)
        perms = np.stack([np.random.default_rng(c.seed + 9 + i).permutation(N) for i in range(c.vf_iters)]).astype(np.int32) \
            if c.vf_iters else np.zeros((0, N), np.int32)
        m, g, x, f = L.step_explicit(obs, act, adv, ret, perms)
        T = {n: read(L, "trpo", n) for n in ("atarg", "mu_old", "nlp_old", "sdm", "sdls", "met", "G", "X", "Rv", "FS", "sc", "cand",
                                             "P", "Y1", "Y0", "Z0", "dZls", "Y0c", "Y1c", "lspart", "Zv", "counters", "amax")}
        X = Bound()
        Y1 = T["Y1"][:N * 2 * H1].reshape(N, 2 * H1)
        pr = K.trpo_prep(X, Y1, net, H1, act, adv, c.ent)
        hold(rep, "prep atarg", T["atarg"], pr["atarg"])
        hold(rep, "prep mu_old", T["mu_old"], pr["mu_old"])
        hold(rep, "prep nlp_old", T["nlp_old"], pr["nlp_old"])
        sdm, sdls = K.trpo_seeds(X, T["atarg"], pr["z"], pr["sig"], N)
        hold(rep, "prep sdm", T["sdm"], sdm)
        hold(rep, "prep sdls", T["sdls"], sdls)
        met = T["met"]
        hold(rep, "prep losses", met[K.TM_BEFORE:K.TM_BEFORE + 5], K.trpo_prep_losses(T["atarg"], net["ls"], c.ent))
        # the policy gradient's head block (trpo_headgrad_kernel with the logstd seeds and entcoeff)
        gW, gb = K.head_grad(Y1[:, :H1], T["sdm"].reshape(N, A))
        gl = K.head_grad(np.ones((N, 1)), T["sdls"].reshape(N, A))[0]
        G = T["G"]
        hold(rep, "headgrad pi/w", G[o_["Wpi"]:o_["Wpi"] + H1 * A], E(gW.v.reshape(-1), gW.e.reshape(-1)))
        hold(rep, "headgrad pi/b", G[o_["bpi"]:o_["bpi"] + A], gb)
        ec = float(np.float32(c.ent))
        hold(rep, "headgrad logstd", G[o_["ls"]:o_["ls"] + A],
             E(gl.v.reshape(-1) + ec, gl.e.reshape(-1) + 2 * U * (np.abs(gl.v.reshape(-1)) + ec)))
        # vf entries of the policy vectors are 0; q/* untouched
        vf = np.zeros(n_train, bool)
        W0m = np.zeros((D, 2 * H0), bool)
        W0m[:, H0:] = True
        vf[o_["W0"]:o_["W0"] + D * 2 * H0] = W0m.reshape(-1)
        vf[o_["b0"] + H0:o_["b0"] + 2 * H0] = True
        for k, n in (("W1_1", H0 * H1), ("b1_1", H1), ("Wvf", H1), ("bvf", 1)):
            vf[o_[k]:o_[k] + n] = True
        for nm in ("G", "X", "FS", "Zv"):
            rep.exact(f"{nm} is 0 at the vf entries", T[nm][:n_train][vf], np.zeros(int(vf.sum()), np.float32))
        rep.exact("q/* untouched", T["P"][n_train:n_total], P0[n_train:n_total])
        sc = T["sc"]
        # CG: the zero test from the stored max partials, r.r of the stored residual, X = alpha g after one iteration, then
        # shs = 0.5 x.Fx (Zv = F x after the last Fisher product), lm = sqrt(|shs| / max_kl), the full step x / lm and
        # expectedimprove = g.fullstep, each from the stored vectors
        check_zero_test(rep, T["amax"], G[:n_train], sc)
        rr = T["Rv"][:n_train].astype(np.float64)
        hold(rep, "CG r.r", sc[K.SC["RR"]:K.SC["RR"] + 1], dot64(rr, rr))
        xs = T["X"][:n_train].astype(np.float64)
        if sc[K.SC["ZERO"]] == 0:
            shs = dot64(xs, T["Zv"][:n_train]) * 0.5
            hold(rep, "shs", met[K.TM_SHS:K.TM_SHS + 1], E(shs.v, shs.e + U * np.abs(shs.v)))
            lm = np.sqrt(np.abs(shs.v) / float(np.float32(c.max_kl)))
            hold(rep, "lm", sc[K.SC["LM"]:K.SC["LM"] + 1], E(lm, lm * (0.5 * shs.e / np.abs(shs.v) + 4 * K.U64)))
            ei = dot64(G[:n_train], T["FS"][:n_train])
            hold(rep, "expected improvement", met[K.TM_EI:K.TM_EI + 1], E(ei.v, ei.e + U * np.abs(ei.v)))
        else:
            rep.exact("zero gradient: no step", np.concatenate([T["FS"][:n_train], T["P"][:n_train] - P0[:n_train]]),
                      np.zeros(2 * n_train, np.float32))
            rep.exact("zero gradient: SC_ACC -2", sc[K.SC["ACC"]:K.SC["ACC"] + 1], np.array([-2.0]))
        if c.cg == 1 and sc[K.SC["ZERO"]] == 0:
            rep.exact("CG x = alpha g (one iteration)", T["X"][:n_train], np.float32(np.float32(sc[K.SC["ALPHA"]]) * G[:n_train]))
        if sc[K.SC["ZERO"]] == 0 and sc[K.SC["BAD"]] == 0:
            rep.exact("vec op 3: fullstep = x / lm", T["FS"][:n_train], (T["X"][:n_train].astype(np.float64) / sc[K.SC["LM"]]).astype(np.float32))
        # line search: the candidates bit for bit, layer 0 of all ten, the loss partials, the choice, the apply
        FS = T["FS"]
        Pold = T["P"][n_total:2 * n_total]
        rep.exact("oldpi copy = theta_old", Pold, P0[:n_total])
        cand = T["cand"]
        blocks = (("b0", H0), ("W1_0", H0 * H1), ("b1_0", H1), ("Wpi", H1 * A), ("bpi", A), ("ls", A))
        off = 0
        cb = {}
        for nm, n in blocks:
            want = np.stack([np.float32(Pold[o_[nm]:o_[nm] + n] + np.float32(2.0 ** -k) * FS[o_[nm]:o_[nm] + n]) for k in range(K.NCAND)])
            got = cand[off:off + K.NCAND * n].reshape(K.NCAND, n)
            rep.exact(f"cand {nm}", got, want)
            cb[nm] = got
            off += K.NCAND * n
        Z0 = T["Z0"][:N * 2 * H0].reshape(N, 2 * H0)[:, :H0]
        dZ = T["dZls"][:N * H0].reshape(N, H0)
        Y0c = T["Y0c"].reshape(K.NCAND, N, H0)
        Y1c = T["Y1c"].reshape(K.NCAND, N, H1)
        for k in range(K.NCAND):
            zk = X.lift(Z0) + X.scale(X.lift(dZ), 2.0 ** -k)
            hold(rep, "ls_l0 Y0c (all ten)", Y0c[k], X.tanh(zk + X.lift(cb["b0"][k])))
        parts = []
        for k in range(K.NCAND):
            su, kl = K.ls_rows(Y1c[k], cb["Wpi"][k].reshape(H1, A), cb["bpi"][k], cb["ls"][k], act, T["mu_old"].reshape(N, A),
                               T["nlp_old"], T["atarg"], net["ls"])
            ps, pk = K.ls_partials(su), K.ls_partials(kl)
            lp = T["lspart"].reshape(K.NCAND, K.LS_BLOCKS, 2)[k]
            hold(rep, "ls_loss surrogate partials", lp[:, 0], ps)
            hold(rep, "ls_loss KL partials", lp[:, 1], pk)
            parts.append((ps, pk))
        if sc[K.SC["ZERO"]] == 0 and sc[K.SC["BAD"]] == 0:
            acc, losses = K.ls_select(T["lspart"], cb["ls"], N, A, c.ent, c.max_kl, met[0])
            rep.exact("ls_select k (from the stored partials)", np.array([sc[K.SC["ACC"]]]), np.array([float(acc)]))
            if c.ls:                   # the fixture's outcome: accepted at k = 0, after a KL rejection, after K and I, or none
                from tests.test_gpu_trpo import ls_fixture
                rep.exact(f"line-search outcome {c.ls}", np.array([acc]), np.array([ls_fixture(c.ls)[5].find("A")]))
            if acc >= 0:
                rep.exact("losses after (the accepted k)", met[K.TM_AFTER:K.TM_AFTER + 5], losses[acc])
            # float64's choice: every k before the device's is rejected and the device's accepted, unless that compare is
            # within its bound (the KL compare in float64 against stable-baselines' 1.5 max_kl, the improvement against 0)
            for k in range(K.NCAND if acc < 0 else acc + 1):
                ps, pk = parts[k]
                klv, kle = pk.v.sum() / N, pk.e.sum() / N + 2 * U * abs(pk.v.sum() / N)
                ent = K.HALF_LOG_2PI_E * A + cb["ls"][k].astype(np.float64).sum()
                imp = ps.v.sum() / N + ec * ent - float(met[0])
                ime = ps.e.sum() / N + 4 * U * (abs(ps.v.sum() / N) + abs(ec * ent) + abs(float(met[0])))
                ok64 = klv <= 1.5 * c.max_kl and imp >= 0
                undecided = abs(klv - 1.5 * c.max_kl) <= SLACK * kle + 2 * U * c.max_kl or abs(imp) <= SLACK * ime
                side_ok(rep, "ls_select k (float64)", np.array(k == acc), np.array(ok64), np.array(undecided))
            want = Pold[:n_train].copy()
            if acc >= 0:
                nz = FS[:n_train] != 0
                want[nz] = np.float32(Pold[:n_train][nz] + np.float32(2.0 ** -acc) * FS[:n_train][nz])
            pol = ~vf
            rep.exact("apply (policy entries)", T["P"][:n_train][pol], want[pol])
        check_fvp(rep, L, c, net, read(L, "trpo", "Pv"), o_)
        if c.vf_iters and N >= K.VF_BATCH:
            check_value(rep, L, c, net, P0, T, perms, ret, o_, n_train, vf)
        else:                          # no full value minibatch (N < 128 drops the partial one): nothing of the value step runs
            rep.exact("no value step: Adam step, moments, vf entries", np.concatenate([
                T["counters"][0:1].astype(np.float32), read(L, "trpo", "Mo")[:n_train], read(L, "trpo", "Vo")[:n_train],
                T["P"][:n_train][vf] - P0[:n_train][vf]]), np.zeros(1 + 2 * n_train + int(vf.sum()), np.float32))
    finally:
        L.close()
    rep.finish()


def check_value(rep, L, c, net, P0, T, perms, ret, o_, n_train, vf):
    """one value minibatch (vf_iters 1, N / 128 = 1): trpo_rows_kernel, trpo_vf_tail_kernel from the stored vY1 and
    trpo_vadam_kernel from the stored Gv (only vf entries move, MpiAdam epsilon 1e-8)"""
    N, (H0, H1) = c.N, c.H
    XS = -(-c.D // 4) * 4
    rep.exact("trpo_rows vrowoff", read(L, "trpo", "vrowoff")[:N], (perms.reshape(-1) * XS).astype(np.int32))
    X = Bound()
    vY1 = read(L, "trpo", "vY1").reshape(K.VF_BATCH, H1)
    rows = perms.reshape(-1)[:K.VF_BATCH]
    o = K.vf_tail(X, vY1, net["Wvf"], net["bvf"], ret[rows])
    hold(rep, "vf_tail dZ1", read(L, "trpo", "vdZ1").reshape(K.VF_BATCH, H1), o["dZ1"])
    Gv = read(L, "trpo", "Gv")
    dv = o["dv"]
    gW = X.dsum(X.lift(vY1) * dv[:, None])
    hold(rep, "vf_tail gWvf", Gv[o_["Wvf"]:o_["Wvf"] + H1], gW)
    hold(rep, "vf_tail gbvf", Gv[o_["bvf"]:o_["bvf"] + 1], X.dsum(dv[:, None]))
    loss = X.dsum(X.square(o["e"]))
    hold(rep, "vf_tail loss", T["met"][K.TM_VF:K.TM_VF + 1], E(np.array([loss.v / K.VF_BATCH]), np.array([loss.e / K.VF_BATCH + U * loss.v / K.VF_BATCH])))
    rep.exact("value Adam step", T["counters"][0:1], np.array([1]))
    Mo, Vo = read(L, "trpo", "Mo")[:n_train], read(L, "trpo", "Vo")[:n_train]
    m2, v2, p2 = K.adam(X, P0[:n_train], np.zeros(n_train), np.zeros(n_train), Gv[:n_train], K.lr_t(3e-4, 1), *K.MPI_ADAM)
    hold(rep, "vadam m (vf entries)", Mo[vf], m2[vf])
    hold(rep, "vadam v (vf entries)", Vo[vf], v2[vf])
    hold(rep, "vadam p (vf entries)", T["P"][:n_train][vf], p2[vf])
    rep.exact("vadam leaves the policy moments", np.concatenate([Mo[~vf], Vo[~vf]]), np.zeros(2 * int((~vf).sum()), np.float32))


def test_matrix_covers_the_issue_shapes():
    widths = {c.H for c in PPO_CASES} | {c.H for c in TRPO_CASES} | {r[3] for r in ROLLOUTS}
    assert {(4, 4), (64, 64), (256, 256), (8, 256), (256, 4)} <= widths
    assert {1, 3, 16} <= {c.A for c in PPO_CASES} & {c.A for c in TRPO_CASES}
    assert {1, 7, 100, 20480} <= {c.D for c in PPO_CASES}
    assert {1, 2, 31, 33, 1023, 1025, 16384} <= {c.M for c in PPO_CASES}
    assert {-1.0, 0.2} <= {c.cvf for c in PPO_CASES} and 0.0 in {c.clip for c in PPO_CASES}
    assert {1, 3, 1025, 4096} <= {r[0] for r in ROLLOUTS}
    assert {1, 4, 6, 127, 129, 1024, 16384} <= {c.N for c in TRPO_CASES}
    assert {0.0, 0.01} <= {c.ent for c in TRPO_CASES}
    assert {"zero", "kl", "imp", "reject"} == {c.ls for c in TRPO_CASES if c.ls}
    assert {1, 2, 3} <= {k for c in CG_CASES for k in range(1, c.cg + 1)}
    assert {True, False} == {c.clipped for c in PPO_CASES if c.clipped is not None}


# ================================================================================================ TRPO: CG, iteration by iteration
CG_CASES = [
    # NF = 1 and A = 1: F = damping I + a rank-one block + 2 I on logstd has three eigenvalues, so r.r falls below 1e-10 at
    # iteration 3 (SC_DONE = 2) and iterations 4 to 6 run with it set (op 1 skipped, op 2 still run)
    TrpoCase("cg_n4_d1_a1_w4", 1, 1, (4, 4), 4, cg=6, vf_iters=0, seed=11),
    TrpoCase("cg_n64_d7_a3_w64", 7, 3, (64, 64), 64, cg=3, vf_iters=0, seed=12),
    TrpoCase("cg_n129_d100_a16_w8x256", 100, 16, (8, 256), 129, ent=0.01, cg=2, vf_iters=0, seed=13),
]


@pytest.mark.parametrize("c", CG_CASES, ids=lambda c: c.name)
def test_trpo_cg_iterations(c):
    """b2g_debug_trpo_cg runs the policy gradient and k CG iterations and hands back x, r, p and the scalars from before the
    last one: that iteration's Fisher product of p, alpha = r.r / p.z, x += alpha p, r -= alpha z, r.r, beta, the r.r < 1e-10
    stop and p = r + beta p are each held to float64 of what it read, for k = 1 .. cg_iters"""
    L, c, obs, act, adv, _ = trpo_setup(c)
    rep = Report(f"TRPO CG {c.name}")
    D, A, (H0, H1) = c.D, c.A, c.H
    o_, n, _ = K.layout(D, A, H0, H1)
    S = K.SC
    try:
        net = K.unpack(read(L, "trpo", "P"), o_, D, A, H0, H1)
        ran_done2 = False
        for k in range(1, c.cg + 1):
            prev = np.empty(3 * n + 2 * 16, np.float32)
            _lib.check(L.lib.b2g_debug_trpo_cg(L.h, obs.ctypes.data_as(C.POINTER(C.c_float)), act.ctypes.data_as(C.POINTER(C.c_float)),
                                               adv.ctypes.data_as(C.POINTER(C.c_float)), k, prev.ctypes.data_as(C.POINTER(C.c_float))))
            x0, r0, p0 = prev[:n], prev[n:2 * n], prev[2 * n:3 * n]
            s0 = prev[3 * n:].view(np.float64)
            T = {m: read(L, "trpo", m) for m in ("X", "Rv", "Pv", "Zv", "sc", "G", "amax")}
            sc, G = T["sc"], T["G"][:n]
            if k == 1:
                rep.exact("vec op 0: x = 0, r = p = g", np.concatenate([x0, r0, p0]), np.concatenate([np.zeros(n, np.float32), G, G]))
                check_zero_test(rep, T["amax"], G, sc)
                hold(rep, "CG_INIT g.g", s0[S["RR"]:S["RR"] + 1], dot64(G, G))
                assert sc[S["ZERO"]] == 0, "the case needs a non-zero gradient"
            check_fvp(rep, L, c, net, p0, o_)
            if s0[S["DONE"]] == 0:
                pz = dot64(p0, T["Zv"][:n])
                rr0 = s0[S["RR"]]
                al = rr0 / pz.v
                hold(rep, "alpha = r.r / p.z", sc[S["ALPHA"]:S["ALPHA"] + 1], E(al, np.abs(al) * (pz.e / np.abs(pz.v) + 2 * K.U64)))
                a32 = np.float64(np.float32(sc[S["ALPHA"]]))
                xr = a32 * p0.astype(np.float64) + x0
                rr_ = -a32 * T["Zv"][:n].astype(np.float64) + r0
                hold(rep, "vec op 1: x += alpha p", T["X"][:n], E(xr, U * np.abs(xr) + 2 * K.U64 * np.abs(a32 * p0)))
                hold(rep, "vec op 1: r -= alpha z", T["Rv"][:n], E(rr_, U * np.abs(rr_) + 2 * K.U64 * np.abs(a32 * T["Zv"][:n])))
                rr = dot64(T["Rv"][:n], T["Rv"][:n])
                hold(rep, "r.r", sc[S["RR"]:S["RR"] + 1], rr)
                b = rr.v / rr0
                hold(rep, "beta = r.r / r.r before", sc[S["BETA"]:S["BETA"] + 1], E(b, rr.e / rr0 + 2 * K.U64 * np.abs(b)))
                side_ok(rep, "r.r < 1e-10 stop (SC_DONE 2)", np.array(sc[S["DONE"]] == 2), np.array(rr.v[0] < 1e-10),
                        np.array(abs(rr.v[0] - 1e-10) <= SLACK * rr.e[0]))
                rep.exact("iteration count", sc[S["ITERS"]:S["ITERS"] + 1], s0[S["ITERS"]:S["ITERS"] + 1] + 1)
            else:                      # stopped before: op 1 and the scalars leave everything as it was
                rep.exact("after the stop: x, r unchanged", np.concatenate([T["X"][:n], T["Rv"][:n]]), np.concatenate([x0, r0]))
                rep.exact("after the stop: scalars unchanged", sc, s0)
            if sc[S["DONE"]] != 1:     # op 2 runs unless the zero test stopped CG (SC_DONE 2 included)
                pr = np.float64(np.float32(sc[S["BETA"]])) * p0.astype(np.float64) + T["Rv"][:n]
                hold(rep, "vec op 2: p = r + beta p", T["Pv"][:n], E(pr, U * np.abs(pr) + 2 * K.U64 * np.abs(pr)))
                ran_done2 |= s0[S["DONE"]] == 2
            else:
                rep.exact("zero test: p unchanged", T["Pv"][:n], p0)
        if c.name.startswith("cg_n4"):
            assert ran_done2, "no iteration ran with SC_DONE = 2"
    finally:
        L.close()
    rep.finish()


def test_trpo_bootstrap_value_after_update():
    """ppo_act_kernel's bootstrap mode (mode 1): after b2g_trpo_update, rollout row 0's value is the updated value tower's
    head over the boundary latents the last forward left in Y1 row 0"""
    c = TrpoCase("boot", 7, 3, (64, 64), 6, cg=2, vf_iters=0, seed=21)
    L, c, obs, act, adv, ret = trpo_setup(c)
    rep = Report("TRPO bootstrap value")
    D, A, (H0, H1) = c.D, c.A, c.H
    o_, n_train, _ = K.layout(D, A, H0, H1)
    try:
        rng = np.random.default_rng(3)
        for t in range(c.N):
            L.rollout_act(rng.normal(0, 1, D))
            L.rollout_reward(rng.normal(), float(t == 2))
        L.update(rng.normal(0, 1, D), np.zeros((0, c.N), np.int32))
        net = K.unpack(read(L, "trpo", "P"), o_, D, A, H0, H1)
        Y1 = read(L, "trpo", "Y1")[:2 * H1].reshape(1, 2 * H1)
        _, v = K.heads(Bound(), Y1, net, H1)
        hold(rep, "act mode 1: value into r_val[0]", read(L, "trpo", "r_val")[:1], v)
    finally:
        L.close()
    rep.finish()
