"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on seeded batches.

Tolerance (BASELINE.json north_star): Q-values, losses and gradient norms within 1e-4 RELATIVE
fp32 of the reference learner on the same seeded replay batch.  Per-sample vectors are compared
as ||gpu - oracle||_2 / ||oracle||_2; scalars as |gpu - oracle| / |oracle|.
"""
import numpy as np
import pytest
import torch

from oracle import sac_ref as R
from tests.util import load_case, make_batch, make_learner, rel_err, GOLD

pytestmark = pytest.mark.gpu
TOL = 1e-4      # north_star tolerance
LR = 3e-4

SCALARS = ("policy_loss", "qf1_loss", "qf2_loss", "value_loss", "ent_coef_loss", "entropy",
           "grad_norm_pi", "grad_norm_values", "grad_ent")
VECTORS = ("q1", "q2", "v", "logp", "v_targ", "q1_pi", "q2_pi", "pi")


def _check_step(cfg, params, vn, B, tol=TOL, precision=0):
    """One explicit step on the GPU vs the oracle.

    The reference arithmetic is fp32 (TF1).  Errors are measured against the float64 oracle; the bar
    is ``tol`` (1e-4) unless fp32 arithmetic ITSELF cannot resolve the quantity that well, which the
    fp32 oracle reveals (e.g. logp = ... - log(1 - tanh(u)^2 + 1e-6) at saturated actions cancels
    catastrophically in fp32): then the bar is 3x the fp32 oracle's own distance from float64.
    """
    raw, norm, eps = make_batch(vn, B)
    L = make_learner(cfg, vn, B, params, precision=precision)
    out = L.step_explicit(raw["obs"], raw["act"], raw["rew"], raw["next_obs"], raw["done"], eps, lr=LR, apply_update=True)
    ref, grads, newp, newopt = R.sac_step(params, R.OptState.zeros(params), norm, eps, LR, cfg, torch.float32)
    ref64, grads64, newp64, _ = R.sac_step(params, R.OptState.zeros(params), norm, eps, LR, cfg, torch.float64)
    errs, bars = {}, {}
    for k in VECTORS:
        errs[k] = rel_err(out[k].reshape(-1), np.asarray(ref64[k]).reshape(-1))
        bars[k] = max(tol, 3 * rel_err(np.asarray(ref[k]).reshape(-1), np.asarray(ref64[k]).reshape(-1)))
    for k in SCALARS:
        errs[k] = abs(out[k] - float(ref64[k])) / (abs(float(ref64[k])) + 1e-30)
        bars[k] = max(tol, 3 * abs(float(ref[k]) - float(ref64[k])) / (abs(float(ref64[k])) + 1e-30))
    g = L.get_gradients()
    gerr = {n: rel_err(g[n], grads64[n]) for n in grads64}
    # per-tensor gradients, conditioning-aware: a tensor whose per-sample contributions cancel amplifies the unit
    # round-off of whatever arithmetic formed it, and the fp32 oracle's own distance from float64 measures that
    # amplification: <= max(1e-3, 3 x fp32-oracle error) for BOTH engines.  (Round 1 needed 1e-2 / 192x for the tensor
    # engine: its 2-plane BF16 forward and the truncating tensor-core accumulation cost two decimal digits; the 3-plane forward
    # with separate leading / correction accumulators is at fp32 level, tools/precision_emulation.py.)
    gtol = 10 * tol
    gbar = {n: max(gtol, 3.0 * rel_err(grads[n], grads64[n])) for n in grads64}
    worst_g = max(gerr, key=lambda n: gerr[n] / gbar[n])
    # post-update parameters (3x TF-Adam + Polyak), element-wise.  At t=1 an Adam step is
    # lr*g/(|g|+3.2e-7): entries with |g| <~ 1e-6 amplify fp32 noise in g to O(lr), so the
    # optimiser arithmetic is checked on the GPU's OWN gradients (whose parity is asserted above):
    # expected = oracle Adam formula applied to g_gpu in float64.
    p2 = L.get_parameters()
    worst_u = 0.0
    lr_t = LR * np.sqrt(1 - R.ADAM_B2) / (1 - R.ADAM_B1)
    exp_new = {}
    for n in params:
        if n.startswith("target/"):
            continue
        gg = g[n].astype(np.float64)
        m, v = (1 - R.ADAM_B1) * gg, (1 - R.ADAM_B2) * gg * gg
        exp_new[n] = params[n].astype(np.float64) - lr_t * m / (np.sqrt(v) + R.ADAM_EPS)
    for n in params:
        if n.startswith("target/"):
            src = "model/" + n[len("target/"):]
            ref_p = (1 - cfg.tau) * params[n].astype(np.float64) + cfg.tau * p2[src].astype(np.float64)
            bar = 2.5e-7 * np.abs(ref_p) + 1e-12
        else:
            ref_p = exp_new[n]
            bar = 1e-4 * LR + 2.5e-7 * np.abs(ref_p) + 1e-12
        d = np.abs(p2[n].astype(np.float64) - ref_p)
        worst_u = max(worst_u, float((d / bar).max()))
    # and against the oracle's own update where the gradient is well away from zero
    for n in ("model/values_fn/cnn_fc1/w", "model/pi/fc0/kernel", "model/log_ent_coef"):
        if n not in grads64:
            continue
        well = np.abs(grads64[n]) > 1e-4 * max(1e-30, float(np.abs(grads64[n]).max()))
        d = np.abs(p2[n].astype(np.float64) - newp64[n])[well]
        assert d.max() <= 2e-2 * LR + 1e-6 * np.abs(newp64[n]).max(), (n, d.max())
    print("errs", {k: f"{v:.2e}" for k, v in errs.items()})
    print("worst grad", worst_g, f"{gerr[worst_g]:.2e} (bar {gbar[worst_g]:.2e})", "worst update/bar", f"{worst_u:.3f}")
    print(f"B={B} precision={precision} worst err/bar: outputs {max(errs[k] / bars[k] for k in errs):.3f},",
          f"gradients {gerr[worst_g] / gbar[worst_g]:.3f}, update {worst_u:.3f}")
    L.close()
    bad = {k: (v, bars[k]) for k, v in errs.items() if not v <= bars[k]}
    assert not bad, f"outputs beyond tolerance: {bad}"
    assert gerr[worst_g] <= gbar[worst_g], f"gradient {worst_g} rel err {gerr[worst_g]} > {gbar[worst_g]}"
    assert worst_u <= 1.0, f"parameter update off by {worst_u} x tolerance"
    return errs


def test_depth_cnn_trained_weights_b32():
    cfg, params, vn = load_case("sac_depth")
    errs = _check_step(cfg, params, vn, 32)
    # committed regression vector (fp64 oracle, generated by tests/golden/make_fixtures.py)
    gold = np.load(f"{GOLD}/golden_step_sac_depth_b32.npz")
    raw, norm, eps = make_batch(vn, 32)
    L = make_learner(cfg, vn, 32, params)
    out = L.step_explicit(raw["obs"], raw["act"], raw["rew"], raw["next_obs"], raw["done"], eps, lr=LR, apply_update=False)
    for k in ("q1", "q2", "v", "logp"):
        assert rel_err(out[k], gold[k].reshape(-1)) <= TOL, k
    for k in ("policy_loss", "qf1_loss", "qf2_loss", "value_loss", "grad_norm_pi", "grad_norm_values"):
        assert abs(out[k] - float(gold[k])) <= TOL * abs(float(gold[k])), k
    L.close()


def test_depth_cnn_fresh_init_b256():
    cfg, _, vn = load_case("sac_depth")
    params = R.init_params(cfg, seed=3)
    _check_step(cfg, params, vn, 256)


@pytest.mark.parametrize("B", [32, 256])
def test_tcgen05_bf16x3_parity_mode(B):
    """Tensor-core engine (parity mode: BF16 plane split, fp32 accumulate): held to the SAME bars as the fp32 engine."""
    cfg, params, vn = load_case("sac_depth")
    _check_step(cfg, params, vn, B, precision=1)


def test_tcgen05_bf16x3_fresh_init_and_rgbd():
    cfg, _, vn = load_case("sac_depth")
    _check_step(cfg, R.init_params(cfg, seed=11), vn, 64, precision=1)
    vn5 = dict(np.load(f"{GOLD}/vecnorm_sac_rgbd.npz"))
    cfg5 = R.SACConfig(obs_shape=(64, 64, 5))
    _check_step(cfg5, R.init_params(cfg5, seed=5), vn5, 64, precision=1)


def test_tcgen05_bf16_fast_mode_tolerance():
    """Single-pass BF16 (fast mode) is NOT a parity mode: it is reported with its measured tolerance.
    Q-values/losses within 5e-3, gradient norms within 0.15 relative on the trained weights."""
    cfg, params, vn = load_case("sac_depth")
    B = 32
    raw, norm, eps = make_batch(vn, B)
    L = make_learner(cfg, vn, B, params, precision=2)
    out = L.step_explicit(raw["obs"], raw["act"], raw["rew"], raw["next_obs"], raw["done"], eps, lr=LR, apply_update=False)
    ref, _, _, _ = R.sac_step(params, R.OptState.zeros(params), norm, eps, LR, cfg, torch.float64)
    for k in ("q1", "q2", "v", "logp"):
        assert rel_err(out[k], np.asarray(ref[k]).reshape(-1)) <= 5e-3, k
    for k in ("grad_norm_pi", "grad_norm_values"):
        assert abs(out[k] - ref[k]) <= 0.15 * abs(ref[k]), k
    L.close()


def test_encoder_mlp_trained_weights_b64():
    cfg, params, vn = load_case("sac_encoder")
    _check_step(cfg, params, vn, 64)


def test_rgbd_cnn_fresh_init_b16():
    vn = dict(np.load(f"{GOLD}/vecnorm_sac_rgbd.npz"))
    cfg = R.SACConfig(obs_shape=(64, 64, 5))
    params = R.init_params(cfg, seed=5)
    _check_step(cfg, params, vn, 16)


def test_two_steps_optimizer_state():
    """Second step exercises non-zero Adam moments, t=2 bias correction and the moved target net."""
    cfg, params, vn = load_case("sac_depth")
    B = 16
    L = make_learner(cfg, vn, B, params)
    p, opt = {n: a.copy() for n, a in params.items()}, R.OptState.zeros(params)
    for it in range(2):
        raw, norm, eps = make_batch(vn, B, seed=100 + it)
        out = L.step_explicit(raw["obs"], raw["act"], raw["rew"], raw["next_obs"], raw["done"], eps, lr=LR)
        ref, _, p, opt = R.sac_step(p, opt, norm, eps, LR, cfg, torch.float64)
        p = {n: a.astype(np.float32) for n, a in p.items()}
        # step 2 starts from parameters that already differ by fp32 noise in near-zero-gradient
        # entries (see _check_step), so Q/V are held to 1e-4 and logp to 5e-4 here
        for k, bar in (("q1", TOL), ("q2", TOL), ("v", TOL), ("logp", 5 * TOL)):
            assert rel_err(out[k], np.asarray(ref[k]).reshape(-1)) <= bar, (it, k, rel_err(out[k], np.asarray(ref[k]).reshape(-1)))
    m, v = L.get_adam("model/values_fn/cnn_fc1/w")
    assert rel_err(m, opt.m["model/values_fn/cnn_fc1/w"]) <= 1e-3
    assert rel_err(v, opt.v["model/values_fn/cnn_fc1/w"]) <= 1e-3
    got = L.get_parameters()
    tname = "target/values_fn/cnn_fc1/w"
    assert np.abs(got[tname] - p[tname]).max() <= 2 * cfg.tau * 2.1 * LR + 1e-6 * np.abs(p[tname]).max()
    assert out["n_updates"] == 2
    L.close()


def test_sampled_step_from_replay_and_policy_act():
    cfg, params, vn = load_case("sac_depth")
    B = 32
    raw, norm, eps = make_batch(vn, B)
    L = make_learner(cfg, vn, B, params, buffer_size=64)
    # a buffer holding ONE transition repeated: any index draw gives the same batch, so the
    # eps-independent outputs of the sampled step must equal the explicit step on that batch
    rep = {k: np.repeat(v[:1], 48, axis=0) for k, v in raw.items()}
    L.replay_add(rep["obs"], rep["act"], rep["rew"], rep["next_obs"], rep["done"])
    assert L.replay_size() == 48
    exp = L.step_explicit(*(np.repeat(raw[k][:1], B, axis=0) for k in ("obs", "act", "rew", "next_obs", "done")), eps, lr=LR,
                          apply_update=False)
    smp = L.step(1, lr=LR)
    for k in ("mean_q1", "mean_q2", "mean_v", "qf1_loss", "qf2_loss"):
        assert abs(smp[k] - exp[k]) <= 1e-5 * max(1.0, abs(exp[k])), (k, smp[k], exp[k])
    assert smp["n_updates"] == 1 and np.isfinite(list(v for v in smp.values())).all()
    assert L.launches_per_step() > 0
    # ring-buffer wrap
    L.replay_add(rep["obs"], rep["act"], rep["rew"], rep["next_obs"], rep["done"])
    assert L.replay_size() == 64
    # policy inference against the oracle (pre-update weights reloaded)
    L.load_parameters(params)
    a_gpu = L.act(raw["obs"][:5], deterministic=True)
    a_ref = R.policy_act(params, norm["obs"][:5], cfg, deterministic=True)
    assert np.abs(a_gpu - a_ref).max() <= 1e-5
    a_sto = L.act(raw["obs"][:5], deterministic=False)
    assert a_sto.shape == (5, 5) and np.abs(a_sto).max() <= 1.0 and np.abs(a_sto - a_gpu).max() > 0
    L.close()


@pytest.mark.parametrize("case,precision", [("sac_depth", 0), ("sac_depth", 1), ("sac_rgbd", 0)])
def test_replay_get_expands_compact_rows(case, precision):
    """Every CNN handle stores compact replay rows: the image planes and the one actuator value the policy reads (pixel [0,0]
    of the last plane).  replay_get returns the image planes bit-exact and the actuator plane as zeros except pixel [0,0],
    which holds the stored value -- also when the caller's actuator plane is constant over the image, as the environment's is.
    8 transitions into a 6-slot ring: slots 0 and 1 hold the wrapped ones."""
    vn = dict(np.load(f"{GOLD}/vecnorm_{case}.npz"))
    cfg = R.SACConfig(obs_shape=tuple(vn["obs_mean"].shape))
    raw, _, _ = make_batch(vn, 8)
    for k in ("obs", "next_obs"):
        raw[k][..., -1] = raw[k][:, :1, :1, -1]            # constant actuator plane
    L = make_learner(cfg, vn, 4, buffer_size=6, precision=precision)
    L.replay_add(raw["obs"], raw["act"], raw["rew"], raw["next_obs"], raw["done"])
    assert L.replay_size() == 6
    for s in range(6):
        t = s + 6 if s < 2 else s
        got = L.replay_get(s)
        for k in ("obs", "next_obs"):
            assert np.array_equal(got[k][..., :-1], raw[k][t][..., :-1]), (s, k)
            plane = got[k][..., -1]
            assert plane[0, 0] == raw[k][t][0, 0, -1] and not plane.reshape(-1)[1:].any(), (s, k)
        assert np.array_equal(got["act"], raw["act"][t]) and got["rew"] == raw["rew"][t] and got["done"] == raw["done"][t]
    L.close()


def test_pipelined_host_batch_path_equals_explicit_path():
    """b2g_sac_step_host_pipelined (copy/compute overlap, losses one step late) must produce the same
    parameters and losses as b2g_sac_step_explicit on the same two batches."""
    _check_pipelined_vs_explicit(16)


def _check_pipelined_vs_explicit(B, precision=0, cfg=None, params=None, vn=None):
    """Three batches through both paths; the depth case's trained weights unless (cfg, params, vn) are given."""
    if cfg is None:
        cfg, params, vn = load_case("sac_depth")
    batches = [make_batch(vn, B, seed=300 + i, n_act=cfg.n_act) for i in range(3)]
    A = make_learner(cfg, vn, B, params, precision=precision, hidden=cfg.layers[0])
    Bm = make_learner(cfg, vn, B, params, precision=precision, hidden=cfg.layers[0])
    outs_a, well = [], {}
    for r, _, e in batches:
        outs_a.append(A.step_explicit(r["obs"], r["act"], r["rew"], r["next_obs"], r["done"], e, lr=LR))
        for n, g in A.get_gradients().items():
            ok = np.abs(g) > 1e-4 * max(1e-30, float(np.abs(g).max()))
            well[n] = well.get(n, ok) & ok
    prev = [Bm.step_host_pipelined(r["obs"], r["act"], r["rew"], r["next_obs"], r["done"], e, lr=LR) for r, _, e in batches]
    assert prev[0] is None
    outs_b = prev[1:] + [Bm.pipeline_flush()]
    for a, b in zip(outs_a, outs_b):
        for k in ("policy_loss", "qf1_loss", "value_loss", "grad_norm_values", "n_updates"):
            assert abs(a[k] - b[k]) <= 2e-5 * max(1.0, abs(a[k])), (k, a[k], b[k])
    pa, pb = A.get_parameters(), Bm.get_parameters()
    for n in pa:
        # Element-wise where every step's gradient is well away from zero (the rule of _check_step's update check): the
        # engines accumulate with fp32 atomics, so two runs agree to summation-order noise (test_graph_path_fork_branches_
        # are_race_free), and Adam's first steps turn that noise in a near-zero element into a move of up to lr.
        d = np.abs(pa[n] - pb[n])[well.get(n, Ellipsis)]
        bar = 1e-6 + 1e-5 * np.abs(pa[n]).max()
        assert d.size == 0 or d.max() <= bar, (n, float(d.max()), bar)
    A.close(); Bm.close()
