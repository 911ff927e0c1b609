"""tests/tail_ref.py without a GPU: its float64 side reproduces the float64 oracle (oracle/sac_ref_np.py), and its bound holds
for fp32 evaluations of the same formulas in several summation orders, with and without FMA, at random and edge inputs
(log_std past both clamps and just inside -20, where t = (u - mu) / (std + 1e-6) cancels; saturated actions, where
log(1 - pi^2 + 1e-6) and one_m / (one_m + 1e-6) cancel; done 0 and 1; rewards of both signs; log_ent_coef away from 0)."""
import numpy as np
import pytest

from oracle import sac_ref as R
from oracle import sac_ref_np as N
from tests import tail_ref as T

D = 24                    # MLP observation width of the cases here


def edge_params(cfg, seed, batch):
    """Fresh parameters, non-zero biases, log_ent_coef -0.7; dense_1 scaled so that raw log_std has mean -9 and spread 8 over
    the batch (past both clamps, and inside -20 with std << 1e-6); dense bias 3 on action 0 (with the wide noise of
    edge_batch, some actions saturate)."""
    p = R.init_params(cfg, seed=seed)
    rng = np.random.default_rng(seed)
    for k in [k for k in p if k.endswith("/bias")]:
        p[k] = (rng.standard_normal(p[k].shape) * 0.1).astype(np.float32)
    (_, ls), _ = N.mlp_fwd(batch["obs"].astype(np.float64), p, "model/pi", ("dense", "dense_1"), len(cfg.layers))
    p["model/pi/dense_1/kernel"] *= (8.0 / (ls - p["model/pi/dense_1/bias"]).std(0)).astype(np.float32)
    p["model/pi/dense_1/bias"][:] = np.float32(-9.0)
    p["model/pi/dense/bias"][0] = np.float32(3.0)
    p["model/log_ent_coef"] = np.array(-0.7, np.float32)
    for k in [k for k in p if k.startswith("target/")]:
        p[k] = (p[k] * np.float32(1.01)).astype(np.float32)
    return p


def edge_batch(cfg, B, seed):
    rng = np.random.default_rng(seed)
    A = cfg.n_act
    obs = (rng.standard_normal((B, D)) * 2).astype(np.float32)
    nxt = (rng.standard_normal((B, D)) * 2).astype(np.float32)
    act = rng.uniform(-1, 1, (B, A)).astype(np.float32)
    act[::5] = np.sign(act[::5])                                   # stored actions at +-1
    rew = (rng.standard_normal(B) * 3).astype(np.float32)
    done = (rng.random(B) < 0.4).astype(np.float32)
    eps = (rng.standard_normal((B, A)) * 2.5).astype(np.float32)
    return dict(obs=obs, next_obs=nxt, act=act, rew=rew, done=done), eps


def z0_of(p, batch, dtype):
    """The fc0 outputs (no bias) of the five heads, as the tail reads them."""
    f = lambda x: np.asarray(x, dtype)
    h, hn, a = f(batch["obs"]), f(batch["next_obs"]), f(batch["act"])
    ha = np.concatenate([h, a], 1)
    return {"pi": h @ f(p["model/pi/fc0/kernel"]), "vf": h @ f(p["model/values_fn/vf/fc0/kernel"]),
            "qf1": ha @ f(p["model/values_fn/qf1/fc0/kernel"]), "qf2": ha @ f(p["model/values_fn/qf2/fc0/kernel"]),
            "target": hn @ f(p["target/values_fn/vf/fc0/kernel"])}


def run(X, cfg, p, batch, eps, z0, pi_in=None):
    return T.tail(X, z0, p, batch["act"], eps, batch["rew"], batch["done"], cfg.gamma, cfg.target_entropy, cfg.feat_dim, pi_in)


# ------------------------------------------------------------------------------------------------ against the oracle
@pytest.mark.parametrize("H", [64, 256])
@pytest.mark.parametrize("A", [1, 8])
def test_float64_side_reproduces_the_oracle(H, A):
    cfg = R.SACConfig(obs_shape=(D,), n_act=A, layers=(H, H), target_entropy=-float(A))
    batch, eps = edge_batch(cfg, 96, seed=H * A)
    p = edge_params(cfg, H + A, batch)
    eps[0, 0] = 12.0                                          # u = mu + 12 std: saturated at any log_std above -1
    out, grads = N.sac_grads(p, batch, eps, cfg)
    X = T.Bound()
    o = run(X, cfg, p, batch, eps, z0_of(p, batch, np.float64))
    # the batch reaches every edge: log_std clamped at both bounds and inside, a saturated action, done 0 and 1, rewards +-
    assert (~X.side["ls/max"]).any() and (~X.side["ls/min"]).any() and X.side["ls"].any()
    assert (np.abs(out["pi"]) > 1 - 1e-7).any()
    assert {0.0, 1.0} <= set(batch["done"].tolist()) and (batch["rew"] > 0).any() and (batch["rew"] < 0).any()

    def same(name, got, want):
        got, want = np.asarray(got, np.float64).reshape(-1), np.asarray(want, np.float64).reshape(-1)
        scale = np.abs(want).max() + 1e-300
        assert np.abs(got - want).max() <= 1e-12 * scale, (name, np.abs(got - want).max() / scale)

    for k in T.PER_SAMPLE + ("pi",):
        same(k, o[k].v, out[k])
    for k in ("policy_loss", "qf1_loss", "qf2_loss", "value_loss", "ent_coef_loss"):
        same(k, o[k].v, out[k])
    same("entropy", o["entropy"].v, out["entropy"])
    for k in T.GRADS:
        same(k, o["g/" + k].v, grads[k])
    # dz1 and dz0 of the four heads, through the oracle's fc1 / fc0 gradients (linear in them)
    feats = {"pi": batch["obs"], "vf": batch["obs"], "qf1": np.concatenate([batch["obs"], batch["act"]], 1)}
    feats["qf2"] = feats["qf1"]
    for h in T.HEADS:
        pre = T.PREFIX[h]
        dz1, dz0, a0 = o[f"dz1/{h}"].v, o[f"dz0/{h}"].v, o[f"a0/{h}"].v
        same(f"{h} fc1/kernel", a0.T @ dz1, grads[f"{pre}/fc1/kernel"])
        same(f"{h} fc1/bias", dz1.sum(0), grads[f"{pre}/fc1/bias"])
        same(f"{h} fc0/bias", dz0.sum(0), grads[f"{pre}/fc0/bias"])
        same(f"{h} fc0/kernel", feats[h].astype(np.float64).T @ dz0, grads[f"{pre}/fc0/kernel"])


# ------------------------------------------------------------------------------------------------ the bound bounds
ORDERS = [("seq", True), ("rev", False), ("perm", True), ("perm", False), ("tree", False)]


def fp32_inputs(cfg, p, batch, eps):
    """What the tail reads: fp32 z0 (here a float64 product rounded once) and the fp32 parameters and batch."""
    return {k: v.astype(np.float32) for k, v in z0_of(p, batch, np.float64).items()}


@pytest.mark.parametrize("H,A,B,seed", [(64, 1, 768, 1), (64, 3, 768, 2), (64, 8, 512, 3), (128, 5, 256, 4), (256, 8, 160, 5)])
def test_bound_holds_for_fp32_evaluations(H, A, B, seed):
    cfg = R.SACConfig(obs_shape=(D,), n_act=A, layers=(H, H), target_entropy=-float(A))
    batch, eps = edge_batch(cfg, B, seed=100 + seed)
    p = edge_params(cfg, seed, batch)
    eps[1::7, -1] = np.float32(9.0)                               # saturated on some rows
    z0 = fp32_inputs(cfg, p, batch, eps)
    worst = {}
    saw_sat = False
    for i, (order, fma) in enumerate(ORDERS):
        F = T.Fp32(order, fma, seed=i)
        f = run(F, cfg, p, batch, eps, z0)
        X = T.Bound(masks=F.side)
        o = run(X, cfg, p, batch, eps, z0, pi_in=f["pi"] if i % 2 else None)       # the kernel's pi downstream, or not
        for key, bad in X.bad.items():
            assert not bad.any(), (order, fma, key, "an fp32 side the bound says fp32 cannot take")
        for key, ref in o.items():
            got = np.asarray(f[key], np.float64)
            err = np.abs(got - ref.v)
            bar = T.SLACK * ref.e
            ok = err <= bar
            assert ok.all(), (order, fma, key, float((err - bar).max()), np.argwhere(~ok)[:3])
            r = float(np.max(err / np.maximum(bar, 1e-300), initial=0.0))
            worst[key] = max(worst.get(key, 0.0), r)
        saw_sat |= bool((np.abs(f["pi"]) == 1).any())
    assert saw_sat, "no action saturated in fp32"
    assert X.side["ls"].any() and (~X.side["ls/max"]).any() and (~X.side["ls/min"]).any()
    # raw log_std inside the clamp but std << 1e-6 on some rows: there u - mu cancels in fp32 and t rests on the bound of u
    assert (X.side["ls"] & (o["ls_raw"].v < -14)).any()
    print(f"H={H} A={A} B={B}: worst err/bar " + ", ".join(f"{k} {v:.2f}" for k, v in sorted(worst.items(), key=lambda t: -t[1])[:8]))
    assert max(worst.values()) > 0.05, "the bound is not tight anywhere: the comparison is vacuous"
