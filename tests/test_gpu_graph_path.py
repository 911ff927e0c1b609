"""Parity of the BENCHMARKED path: CUDA-graph replay + forked leaf branch + in-kernel Philox replay slots +
BF16x3 tensor engine (what ``bench.py`` times as `value`), replayed step by step in the float64 oracle.

The graph path draws its own replay slots and policy noise on the device; ``b2g_get_last_batch`` hands both back
(plus the per-sample outputs), so the oracle can take the very same batch through SURVEY.md Appendix A.

Rows covered (SURVEY.md section 8): a1 (slot draw: range / uniformity / ring wrap), a10 (the step as one unit, on
the path the number comes from), cfg3 (RGB-D, B=1024).
"""
import dataclasses
import os

import numpy as np
import pytest
import torch

from b200grasp import synth
from oracle import sac_ref as R
from tests.util import load_case, make_learner, normalize, rel_err, GOLD

pytestmark = pytest.mark.gpu
TOL = 1e-4
LR = 3e-4
GRAD_BAR = 1e-3     # per-tensor gradient, relative L2
VECTORS = ("q1", "q2", "v", "logp", "v_targ", "q1_pi", "q2_pi", "pi")
SCALARS = ("policy_loss", "qf1_loss", "qf2_loss", "value_loss", "ent_coef_loss", "entropy", "grad_norm_pi", "grad_norm_values")


def _norm_batch(tr, idx, vn):
    return normalize(tr, vn, idx)


def _run_graph_steps(cfg, params, vn, tr, B, K, precision, seed=4321, keep_params=False):
    """K sampled steps (one b2g_sac_step call each) -> list of (metrics, last_batch[, parameters BEFORE the step]) + final parameters.
    The learner takes its action count from the transitions and its head width from cfg."""
    cfg = dataclasses.replace(cfg, n_act=tr["act"].shape[1])
    L = make_learner(cfg, vn, B, params, buffer_size=len(tr["rew"]), precision=precision, seed=seed, hidden=cfg.layers[0])
    L.replay_add(tr["obs"], tr["act"], tr["rew"], tr["next_obs"], tr["done"])
    rows = []
    for _ in range(K):
        pre = L.get_parameters() if keep_params else None
        m = L.step(1, lr=LR)
        rows.append((m, L.last_batch(), pre) if keep_params else (m, L.last_batch()))
    p = L.get_parameters()
    L.close()
    return rows, p


def _oracle_trajectory(cfg, params, vn, tr, rows, dtype):
    p, opt, out = dict(params), R.OptState.zeros(params), []
    for row in rows:
        m, lb = row[0], row[1]
        norm = _norm_batch(tr, lb["indices"].astype(np.int64), vn)
        ref, grads, p, opt = R.sac_step(p, opt, norm, lb["eps"], LR, cfg, dtype)
        p = {n: np.asarray(a, np.float32) for n, a in p.items()}
        out.append(ref)
    return out, p


def test_graph_path_ten_steps_vs_oracle_bf16x3_b256():
    """a10: 10 consecutive graph replays (bf16x3 parity mode, depth, B=256, 4096 distinct replay slots).

    (i) Every step's outputs -- per-sample Q/V/logp/pi, the five losses, both gradient norms -- against the float64 oracle
    evaluated on the SAME batch (the device reports its slots and noise) from the parameters the device held BEFORE that
    step: bar 1e-4, or 3x the fp32 oracle's own distance from float64 where fp32 arithmetic itself does not resolve 1e-4.
    (ii) The parameters after the 10 updates against the float64 oracle running its OWN trajectory (parameters + Adam
    state) through the same 10 batches."""
    cfg, params, vn = load_case("sac_depth")
    B, K, NS = 256, 10, 4096
    tr = synth.make_transitions(NS, vn["obs_mean"], vn["obs_var"], seed=9001)
    rows, p_gpu = _run_graph_steps(cfg, params, vn, tr, B, K, precision=1, keep_params=True)
    for m, lb, _ in rows:
        assert lb["indices"].min() >= 0 and lb["indices"].max() < NS
    assert len({int(i) for _, lb, _ in rows for i in lb["indices"]}) > 1500          # the batches really differ
    worst = {}
    for it, (m, lb, pre) in enumerate(rows):
        norm = _norm_batch(tr, lb["indices"].astype(np.int64), vn)
        r64, _, _, _ = R.sac_step(pre, R.OptState.zeros(pre), norm, lb["eps"], LR, cfg, torch.float64)
        r32, _, _, _ = R.sac_step(pre, R.OptState.zeros(pre), norm, lb["eps"], LR, cfg, torch.float32)
        for k in VECTORS:
            e = rel_err(lb[k].reshape(-1), np.asarray(r64[k]).reshape(-1))
            bar = max(TOL, 3 * rel_err(np.asarray(r32[k]).reshape(-1), np.asarray(r64[k]).reshape(-1)))
            worst[k] = max(worst.get(k, 0.0), e / bar)
            assert e <= bar, (it, k, e, bar)
        for k in SCALARS:
            e = abs(m[k] - float(r64[k])) / (abs(float(r64[k])) + 1e-30)
            bar = max(TOL, 3 * abs(float(r32[k]) - float(r64[k])) / (abs(float(r64[k])) + 1e-30))
            worst[k] = max(worst.get(k, 0.0), e / bar)
            assert e <= bar, (it, k, e, bar)
        assert m["n_updates"] == it + 1
    print("worst err/bar over 10 steps:", {k: f"{v:.2f}" for k, v in worst.items()})
    _, p64 = _oracle_trajectory(cfg, params, vn, tr, rows, torch.float64)
    # parameters after 10 updates: every Adam step moves an entry by at most ~lr, and entries whose gradient is
    # numerically zero take a step of either sign (lr*g/(|g|+eps)), so the bar is a fraction of the 10-step budget:
    # <= 5 % of K*lr on 99 % of the entries of every tensor, and never more than 2*K*lr
    stats = {}
    for n in params:
        d = np.abs(p_gpu[n].astype(np.float64) - p64[n].astype(np.float64)).reshape(-1)
        if n.startswith("target/"):
            assert d.max() <= 2 * cfg.tau * K * K * LR + 1e-6 * np.abs(p64[n]).max(), n
            continue
        assert d.max() <= 2 * K * LR + 1e-6 * np.abs(p64[n]).max(), (n, d.max())
        if d.size >= 1000:
            stats[n] = (float(np.quantile(d, 0.99)) / (K * LR), float(np.quantile(d, 0.999)) / (K * LR))
    print("param drift after 10 steps, q99 / q99.9 in units of K*lr:", {n: f"{a:.3f}/{b:.3f}" for n, (a, b) in stats.items()})
    for n, (q99, _) in stats.items():
        assert q99 <= 0.05, (n, q99)


def test_graph_path_fork_branches_are_race_free(monkeypatch):
    """The step graph runs its leaf work (gradient zeroing, weight planes, prep, bias sums, heads wgrad) on a second
    branch.  The same 6 steps with the branch folded back onto one stream (B2G_FORK=0) and without the graph
    (B2G_NO_GRAPH=1) must give the same batches (same Philox draws) and the same numbers: a missing dependency
    between the branches would show up as a difference.  (Split-R accumulation uses fp32 atomics, so two runs agree
    to fp32 summation-order noise, not bit for bit: bar 2e-6 relative on every per-sample output.)"""
    cfg, params, vn = load_case("sac_depth")
    B, K, NS = 256, 6, 1024
    tr = synth.make_transitions(NS, vn["obs_mean"], vn["obs_var"], seed=9002)
    base, p_base = _run_graph_steps(cfg, params, vn, tr, B, K, precision=1, keep_params=True)
    again, p_again = _run_graph_steps(cfg, params, vn, tr, B, K, precision=1, keep_params=True)
    monkeypatch.setenv("B2G_FORK", "0")
    nofork, p_nofork = _run_graph_steps(cfg, params, vn, tr, B, K, precision=1, keep_params=True)
    monkeypatch.setenv("B2G_NO_GRAPH", "1")
    nograph, p_nograph = _run_graph_steps(cfg, params, vn, tr, B, K, precision=1, keep_params=True)
    for name, other in (("rerun", again), ("B2G_FORK=0", nofork), ("B2G_FORK=0 B2G_NO_GRAPH=1", nograph)):
        for it, ((m0, b0, pre0), (m1, b1, pre1)) in enumerate(zip(base, other)):
            assert np.array_equal(b0["indices"], b1["indices"]), (name, it)
            assert np.array_equal(b0["eps"], b1["eps"]), (name, it)
            for k in VECTORS:
                # later steps inherit the (atomic-order) noise of earlier updates through Adam's normalised step
                assert rel_err(b1[k], b0[k]) <= 2e-6 * (1 + 10 * it), (name, it, k, rel_err(b1[k], b0[k]))
            for k in SCALARS:
                if abs(m1[k] - m0[k]) <= 2e-5 * abs(m0[k]) * (1 + it) + 1e-9:
                    continue
                assert k.startswith("grad_norm"), (name, it, k, m0[k], m1[k])
                # A gradient norm jumps where a ReLU input of the batch sits within fp32 rounding of zero, and the summation
                # order decides its side: then each run is held to the float64 oracle on one side or the other of those
                # inputs, from its own parameters (the rule of tests/test_gpu_batch_edges.py::_graph_steps_vs_oracle).
                norm = _norm_batch(tr, b0["indices"].astype(np.int64), vn)
                for m, pre in ((m0, pre0), (m1, pre1)):
                    e, kinks = _grad_norm_vs_oracle_either_side(pre, norm, b0["eps"], cfg, k, m[k])
                    print(f"{name} step {it}: {k} {m0[k]:.8f} vs {m1[k]:.8f}; {len(kinks)} ReLU inputs within fp32 rounding "
                          f"of zero (nearest {kinks[0] if kinks else None}); this run's err/bar against float64 on either "
                          f"side {e:.3f}")
                    assert kinks and e <= 1.0, (name, it, k, m0[k], m1[k], kinks, e)


def _grad_norm_vs_oracle_either_side(pre, norm, eps, cfg, k, value):
    """-> (smallest err/bar of `value` against the float64 oracle's `k` with the CNN ReLU inputs that fp32 cannot place on
    either side, the bars of _graph_steps_vs_oracle; those inputs)."""
    from tests.test_gpu_batch_edges import _other_side, _relu_kinks
    kinks = _relu_kinks(pre, norm, cfg)
    r32 = R.sac_step(pre, R.OptState.zeros(pre), norm, eps, LR, cfg, torch.float32)[0]
    r64 = R.sac_step(pre, R.OptState.zeros(pre), norm, eps, LR, cfg, torch.float64)[0]
    bar = max(TOL, 3 * abs(float(r32[k]) - float(r64[k])) / abs(float(r64[k])))
    refs = [float(r64[k])] + [float(R.sac_step(q, R.OptState.zeros(q), norm, eps, LR, cfg, torch.float64)[0][k])
                              for q in _other_side(pre, kinks)]
    return min(abs(value - r) / abs(r) for r in refs) / bar, kinks


def test_replay_slot_draw_range_uniformity_and_ring_wrap():
    """a1: ReplayBuffer.sample draws B x randint(0, len-1).  Here: ~1e6 slots drawn by the step's own in-kernel Philox
    draw (MLP policy: cheap steps, same gather kernel) over (i) a partially filled and (ii) a wrapped ring buffer;
    every slot in [0, size), chi-square uniform over `size` bins; the ring holds the newest `capacity` transitions."""
    cfg, params, vn = load_case("sac_encoder")
    B = 256
    for cap, n_add, steps in ((1000, 600, 3900), (257, 700, 3900)):
        L = make_learner(cfg, vn, B, params, buffer_size=cap, precision=0, seed=77)
        tr = synth.make_transitions(n_add, vn["obs_mean"], vn["obs_var"], seed=5)
        tr["rew"] = np.arange(n_add, dtype=np.float32)                       # transition id rides in the reward
        for i in range(0, n_add, 128):                                       # several adds: exercises the wrap split
            sl = slice(i, min(n_add, i + 128))
            L.replay_add(tr["obs"][sl], tr["act"][sl], tr["rew"][sl], tr["next_obs"][sl], tr["done"][sl])
        size = min(cap, n_add)
        assert L.replay_size() == size
        # ring contents: slot s holds the newest transition written there
        for s in (0, 1, size // 2, size - 1):
            expect = max(t for t in range(n_add) if t % cap == s)
            got = L.replay_get(s)
            assert got["rew"] == float(expect), (cap, s, got["rew"], expect)
            assert np.array_equal(got["obs"], tr["obs"][expect]) and np.array_equal(got["act"], tr["act"][expect])
        with pytest.raises(Exception):
            L.replay_get(size)
        counts = np.zeros(size, np.int64)
        for _ in range(steps):
            L.step_async(1, lr=LR)
            idx = L.last_batch()["indices"]
            assert idx.min() >= 0 and idx.max() < size
            counts += np.bincount(idx, minlength=size)
        n = counts.sum()
        assert n == steps * B
        expected = n / size
        chi2 = float(((counts - expected) ** 2 / expected).sum())
        dof = size - 1
        # chi2 ~ N(dof, 2 dof) for large dof: accept within 5 sigma (a biased scaling or an off-by-one range
        # moves it by hundreds of sigma)
        assert abs(chi2 - dof) <= 5 * np.sqrt(2 * dof), (cap, chi2, dof)
        assert counts.min() > 0
        L.close()


@pytest.mark.parametrize("precision", [1])
def test_rgbd_b1024_parity_cfg3(precision):
    """cfg3: SAC RGB-D perception (obs 64x64x5, cnn1/w (8,8,4,32) as in trained_models/SAC_full_rgbd), batch 1024,
    statistics from the shipped vecnormalize.pkl (tests/golden/vecnorm_sac_rgbd.npz), fresh init (the 8 MB trained RGB-D
    arrays are not committed).  Explicit step and graph-path step against the float64 oracle."""
    vn = dict(np.load(f"{GOLD}/vecnorm_sac_rgbd.npz"))
    cfg = R.SACConfig(obs_shape=(64, 64, 5))
    params = R.init_params(cfg, seed=21)
    B = 1024
    tr = synth.make_transitions(B, vn["obs_mean"], vn["obs_var"], seed=9003)
    eps = synth.make_eps(B, seed=9004)
    L = make_learner(cfg, vn, B, params, buffer_size=B, precision=precision, seed=5)
    out = L.step_explicit(tr["obs"], tr["act"], tr["rew"], tr["next_obs"], tr["done"], eps, lr=LR, apply_update=False)
    norm = _norm_batch(tr, np.arange(B), vn)
    ref, grads, _, _ = R.sac_step(params, R.OptState.zeros(params), norm, eps, LR, cfg, torch.float64)
    ref32, _, _, _ = R.sac_step(params, R.OptState.zeros(params), norm, eps, LR, cfg, torch.float32)
    for k in VECTORS:
        e = rel_err(out[k].reshape(-1), np.asarray(ref[k]).reshape(-1))
        bar = max(TOL, 3 * rel_err(np.asarray(ref32[k]).reshape(-1), np.asarray(ref[k]).reshape(-1)))
        assert e <= bar, (k, e, bar)
    for k in SCALARS:
        e = abs(out[k] - float(ref[k])) / (abs(float(ref[k])) + 1e-30)
        assert e <= max(TOL, 3 * abs(float(ref32[k]) - float(ref[k])) / (abs(float(ref[k])) + 1e-30)), (k, e)
    g = L.get_gradients()
    for n in ("model/pi/cnn1/w", "model/values_fn/cnn1/w", "model/values_fn/cnn_fc1/w", "model/pi/fc0/kernel"):
        assert rel_err(g[n], grads[n]) <= GRAD_BAR, (n, rel_err(g[n], grads[n]))
    # the same weights through the sampled graph path
    L.replay_add(tr["obs"], tr["act"], tr["rew"], tr["next_obs"], tr["done"])
    m = L.step(1, lr=LR)
    lb = L.last_batch()
    norm2 = _norm_batch(tr, lb["indices"].astype(np.int64), vn)
    ref2, _, _, _ = R.sac_step(params, R.OptState.zeros(params), norm2, lb["eps"], LR, cfg, torch.float64)
    for k in ("q1", "q2", "v", "v_targ"):
        assert rel_err(lb[k], np.asarray(ref2[k]).reshape(-1)) <= TOL, k
    for k in ("qf1_loss", "qf2_loss", "value_loss", "policy_loss", "grad_norm_pi", "grad_norm_values"):
        assert abs(m[k] - float(ref2[k])) <= TOL * abs(float(ref2[k])), (k, m[k], float(ref2[k]))
    L.close()
