"""tests/ac_kernels_ref.py's bounds bound an fp32 evaluation and catch an error: every tier-2 quantity of
tests/test_gpu_ac_kernels.py is evaluated by the `Bound` backend and by the `Fp32` backend (fp32 numpy, sums in serial,
reversed, random and pairwise order, with and without fused products), and
  * the fp32 values lie within SLACK times the bound of float64;
  * an error of four bounds planted in one element (one row of a per-row output, one column of a gradient, one env column of
    GAE, one [::5] row of the Fisher product, one candidate's partial) is caught.
No GPU: this keeps the GPU test's bounds from going vacuous.
"""
import numpy as np
import pytest

from oracle import philox_ref as PX
from tests import ac_kernels_ref as K
from tests.ac_kernels_ref import E, SLACK

ORDERS = [("seq", True), ("rev", False), ("perm", True), ("tree", False)]


def within(got, ref):
    got = np.asarray(got, np.float64).reshape(ref.v.shape)
    return np.abs(got - ref.v) <= SLACK * ref.e


def plant_caught(got, ref, rng):
    """four bounds added to one element with a non-zero bound (the largest, and a random one) must fail the check"""
    g = np.asarray(got, np.float64).reshape(ref.v.shape).copy()
    flat = ref.e.reshape(-1)
    cand = np.flatnonzero(flat > 0)
    assert cand.size, "every bound is zero"
    for i in {int(np.argmax(flat)), int(rng.choice(cand))}:
        h = g.reshape(-1).copy()
        h[i] += 4 * flat[i] * (1 if rng.random() < 0.5 else -1)
        if within(h, ref).all():
            return False
    return True


def hold_all(outs32, outs64, rng):
    """each fp32 output within its bound, a planted error caught, and the bounds tight: the worst err/bar over the group
    exceeds 0.05 (a bound that were, say, 100 times too loose would leave every ratio below 0.01)"""
    worst = {}
    for k, ref in outs64.items():
        got = np.asarray(outs32[k], np.float64).reshape(ref.v.shape)
        if not ref.e.any():             # exact zeros (M = 1's seeds): nothing to plant against, equality instead
            assert (got == ref.v).all(), k
            continue
        ok = within(got, ref)
        assert ok.all(), (k, int((~ok).sum()), "of", ok.size)
        assert plant_caught(got, ref, rng), k
        worst[k] = float(np.max(np.abs(got - ref.v) / np.where(ref.e > 0, ref.e, np.inf)))
    print("worst err/bar " + ", ".join(f"{k} {v:.2f}" for k, v in sorted(worst.items(), key=lambda t: -t[1])))
    assert max(worst.values()) > 0.05, ("the bounds are not tight anywhere", worst)


def net_of(rng, D, A, H0, H1):
    o, n_train, n_total = K.layout(D, A, H0, H1)
    P = np.zeros(n_total, np.float32)
    P[:n_train] = rng.normal(0, 0.3, n_train)
    return K.unpack(P, o, D, A, H0, H1), P, o, n_train


def tanh32(rng, shape):
    return np.tanh(rng.normal(0, 1, shape)).astype(np.float32)


@pytest.mark.parametrize("order,fma", ORDERS)
@pytest.mark.parametrize("M,A,H1,cvf,clip", [(1, 1, 4, 0.2, 0.2), (31, 3, 64, -1.0, 0.2), (33, 16, 8, 0.05, 0.0)])
def test_ppo_tail(order, fma, M, A, H1, cvf, clip):
    rng = np.random.default_rng(M + A)
    net, *_ = net_of(rng, 3, A, 8, H1)
    Y1 = tanh32(rng, (M, 2 * H1))
    act = rng.normal(0, 1, (M, A)).astype(np.float32)
    ov, ret = rng.normal(0, 1, M).astype(np.float32), rng.normal(0, 1, M).astype(np.float32)
    onlp = (rng.normal(0, 1, M) + 3).astype(np.float32)
    f0 = K.ppo_tail(K.Fp32(order, fma, 1), Y1, net, H1, act, ov, onlp, ret, clip, cvf, 0.01, 0.5)
    st = {k: f0[k] for k in ("sz", "sv", "snlp", "sadv")}
    b = K.ppo_tail(K.Bound(), Y1, net, H1, act, ov, onlp, ret, clip, cvf, 0.01, 0.5, stored=st)
    f = K.ppo_tail(K.Fp32(order, fma, 1), Y1, net, H1, act, ov, onlp, ret, clip, cvf, 0.01, 0.5, side=b["side"], vside=b["vside"])
    if M == 1:
        assert f["advn"] == 0 and b["advn"].v == 0 and b["advn"].e == 0
    keys = ["sz", "sv", "snlp", "sadv", "sdm", "sdls", "sdv", "pg", "vf", "kl", "ent"] + (["advn"] if M > 1 else [])
    hold_all({k: f[k] for k in keys}, {k: b[k] for k in keys}, rng)
    sdm, sdls, sdv = (np.asarray(f[k], np.float32) for k in ("sdm", "sdls", "sdv"))
    dp, dv = K.ppo_dz1(K.Bound(), Y1, net, H1, sdm, sdv)
    dp32, dv32 = K.ppo_dz1(K.Fp32(order, fma, 2), Y1, net, H1, sdm, sdv)
    g = K.ppo_head_grads(K.Bound(), Y1, H1, sdm, sdls, sdv, 0.01)
    g32 = K.ppo_head_grads(K.Fp32(order, fma, 3), Y1, H1, sdm, sdls, sdv, 0.01)
    hold_all(dict(dp=dp32, dv=dv32, **g32), dict(dp=dp, dv=dv, **g), rng)


@pytest.mark.parametrize("order,fma", ORDERS)
@pytest.mark.parametrize("E_,A", [(1, 1), (3, 3), (37, 16)])
def test_act_and_gae(order, fma, E_, A):
    rng = np.random.default_rng(E_ * 10 + A)
    net, *_ = net_of(rng, 3, A, 8, 16)
    Y1 = tanh32(rng, (E_, 32))
    z = K.noise(PX.act_seed(5), 3, E_, A)
    # the device's fp32 noise formula with correctly rounded logf and sincospif
    r = PX._blocks(PX.act_seed(5), 3, (E_ * A + 3) // 4, PX.STREAM_NOISE).reshape(-1, 4)
    u = PX.u01(r)
    rr = np.sqrt(np.float32(-2) * np.float32(np.log(u[:, [0, 0, 2, 2]])))
    ang = np.pi * 2 * u[:, [1, 1, 3, 3]]
    sc = np.float32(np.where(np.arange(4) % 2 == 1, np.sin(ang), np.cos(ang)))
    z32 = (rr * sc).astype(np.float32).reshape(-1)[:E_ * A].reshape(E_, A)
    assert within(z32, z).all()
    X32 = K.Fp32(order, fma, 4)
    a, v, nl = K.act(K.Bound(), Y1, net, 16, z)
    a32, v32, nl32 = K.act(X32, Y1, net, 16, z32)
    T = 6
    rew = rng.normal(0, 1, (T, E_)).astype(np.float32)
    val = rng.normal(0, 1, (T + 1, E_)).astype(np.float32)
    done = (rng.random((T + 1, E_)) < 0.3).astype(np.float32)
    lastv = rng.normal(0, 1, E_).astype(np.float32)
    adv, ret = K.gae(K.Bound(), rew, val, done, lastv, 0.99, 0.95)
    adv32, ret32 = K.gae(X32, rew, val, done, lastv, 0.99, 0.95)
    outs64 = dict(a=a, v=v, nl=nl, adv=E(np.stack([x.v for x in adv]), np.stack([x.e for x in adv])),
                  ret=E(np.stack([x.v for x in ret]), np.stack([x.e for x in ret])))
    hold_all(dict(a=a32, v=v32, nl=nl32, adv=np.stack(adv32), ret=np.stack(ret32)), outs64, rng)


def test_norm_partials_and_adam():
    rng = np.random.default_rng(7)
    _, n_train, _ = K.layout(100, 3, 64, 64)
    G = (rng.normal(0, 1e-2, n_train)).astype(np.float32)
    part = K.norm_partials(G)
    blk = K.norm_blocks(n_train)
    p32 = np.zeros(K.NORM_BLOCKS, np.float32)
    for i in range(blk.size):            # the kernel's thread-serial then tree order is one order of many; serial is another
        p32[blk[i]] = np.float32(p32[blk[i]] + np.float32(G[i] * G[i]))
    P0 = rng.normal(0, 0.3, n_train).astype(np.float32)
    outs = {}
    for name, consts in (("tf", K.TF_ADAM), ("mpi", K.MPI_ADAM)):
        lrt = K.lr_t(1e-3, 1)
        m, v, p = K.adam(K.Bound(), P0, np.zeros(n_train), np.zeros(n_train), G, lrt, *consts)
        m32, v32, p32_ = K.adam(K.Fp32(), P0, np.zeros(n_train, np.float32), np.zeros(n_train, np.float32), G, lrt, *consts)
        outs[name] = ((m32, v32, p32_), (m, v, p))
    hold_all({"part": p32, **{f"{n}{i}": outs[n][0][i] for n in outs for i in range(3)}},
             {"part": part, **{f"{n}{i}": outs[n][1][i] for n in outs for i in range(3)}}, rng)
    norm, sc = K.adam_scale(p32, 0.5)
    assert sc == np.float32(0.5) / max(norm, np.float32(0.5))


@pytest.mark.parametrize("order,fma", ORDERS)
@pytest.mark.parametrize("N,A,H0,H1", [(1, 1, 4, 4), (6, 16, 4, 256), (129, 3, 64, 8)])
def test_trpo_prep_fvp_and_value(order, fma, N, A, H0, H1):
    rng = np.random.default_rng(N + A)
    net, P, o, n_train = net_of(rng, 5, A, H0, H1)
    Y1 = tanh32(rng, (N, 2 * H1))
    act = rng.normal(0, 1, (N, A)).astype(np.float32)
    adv = rng.normal(0, 1, N).astype(np.float32)
    X32 = K.Fp32(order, fma, 5)
    b = K.trpo_prep(K.Bound(), Y1, net, H1, act, adv, 0.01)
    f = K.trpo_prep(X32, Y1, net, H1, act, adv, 0.01)
    at32 = np.asarray(b["atarg"].v, np.float32)
    sdm, sdls = K.trpo_seeds(K.Bound(), at32, b["z"], b["sig"], N)
    sdm32, sdls32 = K.trpo_seeds(X32, at32, f["z"], f["sig"], N)
    NF = (N + 4) // 5
    T1, Y1r, Vpi = tanh32(rng, (NF, H1)), Y1[::5, :H1], rng.normal(0, 0.3, (H1, A)).astype(np.float32)
    vb = rng.normal(0, 0.3, A).astype(np.float32)
    u = K.fvp_head(K.Bound(), T1, Y1r, net["Wpi"], Vpi, vb, net["ls"], NF)
    u32 = K.fvp_head(X32, T1, Y1r, net["Wpi"], Vpi, vb, net["ls"], NF)
    uu = np.asarray(u32, np.float32)
    dz = K.head_bwd(K.Bound(), uu, net["Wpi"], Y1r)
    dz32 = K.head_bwd(X32, uu, net["Wpi"], Y1r)
    Tpre = K.Bound().lift(rng.normal(0, 1, (NF, H0)).astype(np.float32))
    Y0r, vb0 = tanh32(rng, (NF, H0)), rng.normal(0, 0.3, H0).astype(np.float32)
    tg, tg32 = K.tangent(K.Bound(), Tpre, vb0, Y0r), K.tangent(X32, np.float32(Tpre.v), vb0, Y0r)
    gW, gb = K.head_grad(Y1r, uu)
    gW32 = np.float32((Y1r.astype(np.float64).T @ uu.astype(np.float64)))
    vY1 = tanh32(rng, (K.VF_BATCH, H1))
    rr = rng.normal(0, 1, K.VF_BATCH).astype(np.float32)
    vt, vt32 = K.vf_tail(K.Bound(), vY1, net["Wvf"], net["bvf"], rr), K.vf_tail(X32, vY1, net["Wvf"], net["bvf"], rr)
    outs64 = dict(atarg=b["atarg"], mu=b["mu_old"], nlp=b["nlp_old"], sdm=sdm, sdls=sdls, u=u, dz=dz, gW=gW, vdz=vt["dZ1"], v=vt["v"])
    outs32 = dict(atarg=at32, mu=f["mu_old"], nlp=f["nlp_old"], sdm=sdm32, sdls=sdls32, u=u32, dz=dz32, gW=gW32, vdz=vt32["dZ1"],
                  v=vt32["v"])
    if N == 1:                          # std = 0: atarg and every seed is exactly 0, with a zero bound
        for k in ("atarg", "sdm", "sdls"):
            assert (np.asarray(outs32[k]) == 0).all() and (outs64[k].v == 0).all()
            del outs64[k], outs32[k]
    outs64["tangent"], outs32["tangent"] = tg, tg32
    hold_all(outs32, outs64, rng)


@pytest.mark.parametrize("N,A,H1", [(4, 1, 4), (300, 3, 16), (16500, 2, 4)])
def test_line_search_partials_and_select(N, A, H1):
    rng = np.random.default_rng(N)
    Y1 = tanh32(rng, (N, H1))
    W, b = rng.normal(0, 0.5, (H1, A)).astype(np.float32), rng.normal(0, 0.1, A).astype(np.float32)
    ls, ls_old = rng.normal(0, 0.1, A).astype(np.float32), rng.normal(0, 0.1, A).astype(np.float32)
    act = rng.normal(0, 1, (N, A)).astype(np.float32)
    mu_old = (Y1 @ W + b + rng.normal(0, 0.05, (N, A))).astype(np.float32)
    nlp_old = rng.normal(3, 0.1, N).astype(np.float32)
    at = rng.normal(0, 1, N).astype(np.float32)
    su, kl = K.ls_rows(Y1, W, b, ls, act, mu_old, nlp_old, at, ls_old)
    # the kernel's per-row evaluation: fp32 mean and neglogp, float64 ratio and KL
    X32 = K.Fp32("seq", True)
    mu = np.asarray(X32.contract("rq,qj->rj", Y1, W, bias=b), np.float64)
    z = np.float32((act - np.float32(mu)) / np.exp(ls))
    nlp = np.asarray(K.neglogp(X32, z, ls), np.float64)
    su32 = np.exp(nlp_old - nlp) * at
    dm = mu_old.astype(np.float64) - mu
    so, sn = np.exp(ls_old.astype(np.float64)), np.exp(ls.astype(np.float64))
    kl32 = (ls.astype(np.float64) - ls_old + (so * so + dm * dm) / (2 * sn * sn) - 0.5).sum(1)
    ps, pk = K.ls_partials(su), K.ls_partials(kl)
    blk = (np.arange(N) % (K.LS_BLOCKS * K.LS_THREADS)) // K.LS_THREADS
    hold_all(dict(su=su32, kl=kl32, ps=np.bincount(blk, su32, K.LS_BLOCKS), pk=np.bincount(blk, kl32, K.LS_BLOCKS)),
             dict(su=su, kl=kl, ps=ps, pk=pk), np.random.default_rng(1))
    # the select rule from partials: KL of candidate k over 1.5 max_kl rejects it, the first acceptable k wins
    part = np.zeros((K.NCAND, K.LS_BLOCKS, 2))
    part[:, 0, 0] = N * np.linspace(1.0, 0.1, K.NCAND)
    part[:, 0, 1] = N * 0.01 * np.array([3, 2, 1.6, 1.5, 1.4, 1, 1, 1, 1, 1])
    lsc = np.zeros((K.NCAND, A), np.float32)
    acc, _ = K.ls_select(part.reshape(-1), lsc, N, A, 0.0, 0.01, 0.0)
    assert acc == 3          # 0.015 is not > 1.5f * 0.01f in fp32
    acc, _ = K.ls_select(part.reshape(-1), lsc, N, A, 0.0, 0.01, 0.95)
    assert acc == -1         # no candidate improves on 0.95 ... until k = 0 gives 1.0 - 0.95 but its KL is rejected
