"""The contraction engines at batch sizes and split-K settings where their tiles do not line up with the data.

Every problem of the fused bf16x3 engine (csrc/engine_v2.cu) cuts the batch its own way -- 128-row conv1 tiles, conv2 tiles
of 3 samples, conv3 tiles of 8, conv2-dgrad tiles of 2, wgrad K-chunks of 4 samples, 128-sample tiles of the dense layers,
64-row K-chunks of the cnn_fc1 wgrad -- and the last, partial tile of each relies on TMA zero fill, the `lim_rows` masks and
the clamp of the counter waits between fused layers.  The batch sizes here put every one of those tiles at every offset
against the end of the batch (`test_sweep_covers_every_tile_residue` keeps the set honest), and each is held to the float64
oracle with the bars of tests/test_gpu_parity.py (explicit step) and tests/test_gpu_graph_path.py (graph-path steps).

Each check prints its worst err/bar ratio; `pytest -s` shows them.
"""
import numpy as np
import pytest
import torch

from b200grasp import synth
from b200grasp._lib import B2GError
from oracle import bdq_ref as Q
from oracle import sac_ref as R
from tests.test_gpu_bdq import test_bdq_step_matches_oracle as _bdq_step_check
from tests.test_gpu_graph_path import LR, SCALARS, TOL, VECTORS, _norm_batch, _run_graph_steps
from tests.test_gpu_parity import _check_pipelined_vs_explicit, _check_step
from tests.util import GOLD, load_case, make_batch, make_learner, rel_err

# Batch sizes of the bf16x3 sweep.  Together: every residue mod 2, 3, 4 and 8; 1 and 63 mod 64; 1 and 127 mod 128; a single
# partial tile of every small period (B < 3, 4, 8); a second, partial 128-sample tile; and a batch past 256 that is no
# multiple of 128.
SWEEP = (1, 2, 3, 5, 6, 9, 24, 100, 129, 200, 255, 383)

# The ways the engines cut the batch (csrc/engine_v2.cu v2_create, csrc/tail.cu heads_wgrad_kernel), as
# (what, samples per tile or chunk, residues of B the sweep must hold; None = all of them).
TILE_PERIODS = (
    ("conv2 dgrad tile: 2 samples", 2, None),
    ("conv2 fwd / conv3 dgrad tile: 3 samples", 3, None),
    ("conv3 / conv2 wgrad K-chunk: 4 samples; heads_wgrad: 4 batch slices", 4, None),
    ("conv3 fwd tile: 8 samples", 8, None),
    ("cnn_fc1 wgrad K-chunk: 64 samples", 64, (1, 63)),
    ("cnn_fc1 / fc0 / heads dgrad tile: 128 samples", 128, (1, 127)),
)

# Split-K settings of the cnn_fc1 forward (16 K-chunks) and dgrad (8 K-chunks) tiles.  6 and 3 do not divide the chunk
# count (the last split is short: 3+3+3+3+3+1, 3+3+2); 8 gives the dgrad one chunk per split.
FC1_CHUNKS, FC1_DGRAD_CHUNKS = 16, 8
SPLIT_SETTINGS = {
    "fc1=1": {"B2G_SPLIT_FC1": "1"},
    "fc1=2": {"B2G_SPLIT_FC1": "2"},
    "dgrad=2": {"B2G_SPLIT_FC1_DGRAD": "2"},
    "dgrad=3": {"B2G_SPLIT_FC1_DGRAD": "3"},
    "dgrad=8": {"B2G_SPLIT_FC1_DGRAD": "8"},
    "fc1=6,dgrad=3": {"B2G_SPLIT_FC1": "6", "B2G_SPLIT_FC1_DGRAD": "3"},
}
# Counts that leave a split without chunks; create refuses them (B2G_EINVAL).
REFUSED_SPLITS = (("B2G_SPLIT_FC1", 5), ("B2G_SPLIT_FC1", 7), ("B2G_SPLIT_FC1", 20), ("B2G_SPLIT_FC1_DGRAD", 5))

RGBD_B = 77       # the RGB-D case: odd, and no multiple of 3, 4 or 8
NS = 512          # replay transitions behind the graph-path steps
K_GRAPH = 3       # a workspace or arrival counter left dirty by one step shows from the second step on


def _has_empty_split(chunks, splits):
    return (splits - 1) * -(-chunks // splits) >= chunks


# ================================================================================================ CPU: the sweep stays honest
def test_sweep_covers_every_tile_residue():
    for what, period, residues in TILE_PERIODS:
        seen = {B % period for B in SWEEP}
        need = set(range(period)) if residues is None else set(residues)
        assert need <= seen, (what, sorted(need - seen))
        if residues is None:
            assert min(SWEEP) < period, (what, "no batch with one partial tile")
    assert any(128 < B < 256 for B in SWEEP), "no second, partial 128-sample tile"
    assert any(B > 256 and B % 128 for B in SWEEP), "no batch past 256 that is a non-multiple of 128"
    assert all(RGBD_B % p for p in (2, 3, 4, 8)), "the RGB-D case should sit off every small tile period"


def test_split_settings_cover_ragged_splits():
    fc1 = {int(e["B2G_SPLIT_FC1"]) for e in SPLIT_SETTINGS.values() if "B2G_SPLIT_FC1" in e}
    dgrad = {int(e["B2G_SPLIT_FC1_DGRAD"]) for e in SPLIT_SETTINGS.values() if "B2G_SPLIT_FC1_DGRAD" in e}
    assert 1 in fc1 and dgrad                                                    # no split, and the dgrad path at all
    assert any(FC1_CHUNKS % s for s in fc1) and any(FC1_DGRAD_CHUNKS % s for s in dgrad)    # a short last split
    assert FC1_DGRAD_CHUNKS in dgrad                                             # one chunk per split
    assert any(len(e) == 2 for e in SPLIT_SETTINGS.values())                     # both switches at once
    assert not any(_has_empty_split(FC1_CHUNKS, s) for s in fc1)
    assert not any(_has_empty_split(FC1_DGRAD_CHUNKS, s) for s in dgrad)
    for var, s in REFUSED_SPLITS:
        assert _has_empty_split(FC1_CHUNKS if var == "B2G_SPLIT_FC1" else FC1_DGRAD_CHUNKS, s), (var, s)


# ================================================================================================ GPU
_U32 = 2.0 ** -24
_CNN_NETS = (("model/pi", "obs"), ("model/values_fn", "obs"), ("target/values_fn", "next_obs"))


def _relu_kinks(params, norm, cfg, max_n=6):
    """ReLU pre-activations of the CNNs whose sign fp32 arithmetic cannot decide: |z| (float64) below 4 sqrt(K) u32 sum|w x|.
    At such an element the reference is not differentiable -- its gradient takes one of two values depending on the side the
    sum lands on -- so a gradient computed in fp32 (the engine's, or the fp32 oracle's on another CPU) may be the other one.
    -> [(bias name, channel, float64 pre-activation)], nearest to zero first."""
    import torch.nn.functional as F
    found = []
    for net, key in _CNN_NETS:
        h = torch.tensor(np.asarray(norm[key]), dtype=torch.float64)[..., :cfg.c_img].permute(0, 3, 1, 2) / 255.0
        for name, stride in (("cnn1", 4), ("cnn2", 2), ("cnn3", 1), ("cnn_fc1", 0)):
            w = torch.tensor(params[f"{net}/{name}/w"], dtype=torch.float64)
            b = torch.tensor(params[f"{net}/{name}/b"], dtype=torch.float64).reshape(-1)
            if stride:
                w = w.permute(3, 2, 0, 1)
                z = F.conv2d(h, w, stride=stride) + b.reshape(1, -1, 1, 1)
                mag = F.conv2d(h.abs(), w.abs(), stride=stride) + b.abs().reshape(1, -1, 1, 1)
                fan_in, chan = w[0].numel(), 1
            else:
                h = h.permute(0, 2, 3, 1).reshape(h.shape[0], -1)
                z, mag, fan_in, chan = h @ w + b, h.abs() @ w.abs() + b.abs(), w.shape[0], 1
            close = (z.abs() <= 4 * np.sqrt(fan_in) * _U32 * mag).nonzero()
            for idx in close.tolist():
                found.append((f"{net}/{name}/b", idx[chan], float(z[tuple(idx)])))
            h = torch.relu(z)
    return sorted(found, key=lambda f: abs(f[2]))[:max_n]


def _other_side(params, kinks):
    """Parameter sets that put the pre-activations of `kinks` on their other side: the channel's bias moves by -2z (~1e-7,
    which moves every other output of the channel by as little): one set per kink, and one with all of them moved."""
    def moved(sel):
        q = {n: a.copy() for n, a in params.items()}
        for bname, c, z in sel:
            q[bname].reshape(-1)[c] -= np.float32(2 * z)
        return q
    sets = [moved([k]) for k in kinks]
    return sets + ([moved(kinks)] if len(kinks) > 1 else [])


def _graph_steps_vs_oracle(cfg, params, vn, B, data_seed=9101, precision=1):
    """K_GRAPH graph-path steps; every step's outputs against the float64 oracle on the batch the device reports, from the
    parameters it held before that step (the bars of test_graph_path_ten_steps_vs_oracle_bf16x3_b256).  -> the steps' rows"""
    tr = synth.make_transitions(NS, vn["obs_mean"], vn["obs_var"], seed=data_seed, n_act=cfg.n_act)
    rows, _ = _run_graph_steps(cfg, params, vn, tr, B, K_GRAPH, precision=precision, keep_params=True)
    worst = {}
    for it, (m, lb, pre) in enumerate(rows):
        assert lb["indices"].min() >= 0 and lb["indices"].max() < NS
        norm = _norm_batch(tr, lb["indices"].astype(np.int64), vn)
        r64, _, _, _ = R.sac_step(pre, R.OptState.zeros(pre), norm, lb["eps"], LR, cfg, torch.float64)
        r32, _, _, _ = R.sac_step(pre, R.OptState.zeros(pre), norm, lb["eps"], LR, cfg, torch.float32)
        for k in VECTORS:
            e = rel_err(lb[k].reshape(-1), np.asarray(r64[k]).reshape(-1))
            bar = max(TOL, 3 * rel_err(np.asarray(r32[k]).reshape(-1), np.asarray(r64[k]).reshape(-1)))
            worst[k] = max(worst.get(k, 0.0), e / bar)
            assert e <= bar, (B, it, k, e, bar)
        # The gradient norms jump where a ReLU input sits within fp32 rounding of zero: there they are held to the float64
        # oracle on either side of the kink (each within the same bar), not to the side the float64 sum happens to take.
        # (the other sides are evaluated only when the float64 reference misses)
        kinks, alt = None, None
        for k in SCALARS:
            e = abs(m[k] - float(r64[k])) / (abs(float(r64[k])) + 1e-30)
            bar = max(TOL, 3 * abs(float(r32[k]) - float(r64[k])) / (abs(float(r64[k])) + 1e-30))
            if e > bar and k.startswith("grad_norm"):
                if alt is None:
                    kinks = _relu_kinks(pre, norm, cfg)
                    alt = [R.sac_step(q, R.OptState.zeros(q), norm, lb["eps"], LR, cfg, torch.float64)[0] for q in _other_side(pre, kinks)]
                e = min([e] + [abs(m[k] - float(r[k])) / (abs(float(r[k])) + 1e-30) for r in alt])
                print(f"B={B} step {it}: {k} held to the other side of a ReLU input within fp32 rounding of zero "
                      f"({len(kinks)} such inputs, nearest {kinks[0] if kinks else None}): rel err {e:.2e}")
            worst[k] = max(worst.get(k, 0.0), e / bar)
            assert e <= bar, (B, it, k, e, bar, kinks)
        assert m["n_updates"] == it + 1
    k = max(worst, key=worst.get)
    print(f"B={B} graph path, {K_GRAPH} steps: worst err/bar {worst[k]:.3f} ({k})")
    return rows


@pytest.mark.gpu
@pytest.mark.parametrize("B", SWEEP)
def test_bf16x3_depth_batch_sweep(B):
    """The benchmarked engine (bf16x3, fused engine v2) on the depth case's trained weights: one explicit step with every
    per-sample vector, loss, gradient norm, per-tensor gradient and the Adam / Polyak update against the oracle, then three
    graph-path steps."""
    cfg, params, vn = load_case("sac_depth")
    _check_step(cfg, params, vn, B, precision=1)
    _graph_steps_vs_oracle(cfg, params, vn, B)


@pytest.mark.gpu
def test_bf16x3_rgbd_odd_batch():
    """RGB-D (5 channels: K1 = 256, two conv1-wgrad M tiles) at an odd batch that is no multiple of 3, 4 or 8."""
    vn = dict(np.load(f"{GOLD}/vecnorm_sac_rgbd.npz"))
    cfg = R.SACConfig(obs_shape=(64, 64, 5))
    params = R.init_params(cfg, seed=5)
    _check_step(cfg, params, vn, RGBD_B, precision=1)
    _graph_steps_vs_oracle(cfg, params, vn, RGBD_B)


_default_runs = {}


def _default_graph_run(cfg, params, vn, B, monkeypatch):
    """The graph-path steps of the default split settings at batch B (computed once per B)."""
    if B not in _default_runs:
        monkeypatch.delenv("B2G_SPLIT_FC1", raising=False)
        monkeypatch.delenv("B2G_SPLIT_FC1_DGRAD", raising=False)
        _default_runs[B] = _graph_steps_vs_oracle(cfg, params, vn, B)
    return _default_runs[B]


@pytest.mark.gpu
@pytest.mark.parametrize("B", [129, 256])
@pytest.mark.parametrize("setting", list(SPLIT_SETTINGS))
def test_split_k_switches(setting, B, monkeypatch):
    """Non-default K-splits of the cnn_fc1 forward and dgrad tiles (read at create): one explicit step and three graph steps
    against the oracle, and the same replay slots, noise and -- to fp32 summation-order noise, the bar of
    test_graph_path_fork_branches_are_race_free -- the same per-sample outputs as the default settings."""
    cfg, params, vn = load_case("sac_depth")
    base = _default_graph_run(cfg, params, vn, B, monkeypatch)
    for var, val in SPLIT_SETTINGS[setting].items():
        monkeypatch.setenv(var, val)
    print(f"{setting}:")
    _check_step(cfg, params, vn, B, precision=1)
    rows = _graph_steps_vs_oracle(cfg, params, vn, B)
    worst = 0.0
    for it, ((m0, b0, _), (m1, b1, _)) in enumerate(zip(base, rows)):
        assert np.array_equal(b0["indices"], b1["indices"]), it
        assert np.array_equal(b0["eps"], b1["eps"]), it
        for k in VECTORS:
            e, bar = rel_err(b1[k], b0[k]), 2e-6 * (1 + 10 * it)
            worst = max(worst, e / bar)
            assert e <= bar, (setting, it, k, e)
        for k in SCALARS:
            assert abs(m1[k] - m0[k]) <= 2e-5 * abs(m0[k]) * (1 + it) + 1e-9, (setting, it, k, m0[k], m1[k])
    print(f"{setting} B={B} vs default settings: worst err/bar {worst:.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("var,splits", REFUSED_SPLITS)
def test_split_leaving_an_empty_split_is_refused(var, splits, monkeypatch):
    """A split count that leaves a split without K-chunks would never finish its tiles (the empty split never arrives at
    the finalisation counter): create refuses it with B2G_EINVAL and names the counts that work."""
    cfg, params, vn = load_case("sac_depth")
    monkeypatch.setenv(var, str(splits))
    with pytest.raises(B2GError, match=rf"error -1: {var}={splits} leaves a K-split of \d+ chunks empty; use one of 1, 2, 3, 4"):
        make_learner(cfg, vn, 129, params, precision=1)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 65, 129])
def test_fp32_simt_depth_ragged_batch(B):
    """The fp32 engine (gg_simt, 64 x 64 tiles): one row past a tile, and a single row."""
    cfg, params, vn = load_case("sac_depth")
    _check_step(cfg, params, vn, B, precision=0)


# bf16x3 at B = 65 misses the per-tensor gradient bar on model/pi/fc0/kernel: relative error 1.071e-3 against a bar of 1e-3
# (the fp32 oracle's own error is 3.1e-4).  It is not a tile edge: the error is the same to four digits with the batch rolled
# so that row 64 sits at row 0, or at row 31, and in repeated runs; nor the saturated actions of the batch (with those rows
# replaced it is 1.5e-3 against fp32's 4.2e-4).  The bf16x3 backward of this tensor is ~3.5x the fp32 oracle's error, above
# the 3x rule.  Strict: the mark goes when the engine meets the bar.
_MLP_BF16X3_B65 = pytest.mark.xfail(strict=True, reason="bf16x3 gradient error on an ill-conditioned MLP tensor at B=65 is 3.4x "
                                                       "the fp32 oracle's own error (bar 3x)")


@pytest.mark.gpu
@pytest.mark.parametrize("precision,B", [(0, 1), (0, 65), (0, 129), (1, 1), pytest.param(1, 65, marks=_MLP_BF16X3_B65), (1, 129)])
def test_mlp_policy_ragged_batch(precision, B):
    cfg, params, vn = load_case("sac_encoder")
    _check_step(cfg, params, vn, B, precision=precision)


@pytest.mark.gpu
def test_bf16_fast_mode_ragged_batch():
    """Single-pass BF16 at B = 129, held to its measured tolerance (test_tcgen05_bf16_fast_mode_tolerance): Q-values and
    log-probabilities within 5e-3, gradient norms within 0.15 relative."""
    cfg, params, vn = load_case("sac_depth")
    B = 129
    raw, norm, eps = make_batch(vn, B)
    L = make_learner(cfg, vn, B, params, precision=2)
    out = L.step_explicit(raw["obs"], raw["act"], raw["rew"], raw["next_obs"], raw["done"], eps, lr=LR, apply_update=False)
    L.close()
    ref, _, _, _ = R.sac_step(params, R.OptState.zeros(params), norm, eps, LR, cfg, torch.float64)
    ratios = {}
    for k in ("q1", "q2", "v", "logp"):
        ratios[k] = rel_err(out[k], np.asarray(ref[k]).reshape(-1)) / 5e-3
    for k in ("grad_norm_pi", "grad_norm_values"):
        ratios[k] = abs(out[k] - ref[k]) / (0.15 * abs(ref[k]))
    print(f"B={B} precision=2 worst err/bar {max(ratios.values()):.3f}")
    assert max(ratios.values()) <= 1.0, ratios


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 65, 130])
def test_bdq_ragged_batch(B):
    """BDQ (fp32 FFMA engine) at the first configuration of test_bdq_step_matches_oracle, with its bars."""
    _bdq_step_check(Q.BDQConfig(100, 3, 8, (64, 64), 32, 32, 0.99), B)


@pytest.mark.gpu
@pytest.mark.parametrize("precision,tol", [(0, 1e-4), (1, 1e-4), (2, 5e-3)])
def test_act_in_chunks_of_the_batch(precision, tol):
    """act() runs n observations in chunks of the batch size (32 here).  Calls of one short chunk (31 rows) and of two chunks
    plus a short third (67 rows) against the oracle with the bars of test_policy_act_depth_cnn (relative L2 over the call's
    rows; the fast mode's 5e-3 is a figure over ~32 rows, single rows of it spread to 1.7e-2).  Every row of a shorter call --
    one row, one short chunk, each row on its own at the chunk edges -- must match the same row of the 67-row call: a row's
    action must not depend on where in the call it sits."""
    cfg, params, vn = load_case("sac_depth")
    B = 32
    n_full = 2 * B + 3
    raw, norm, _ = make_batch(vn, n_full)
    L = make_learner(cfg, vn, B, params, precision=precision)
    full = L.act(raw["obs"], deterministic=True)
    a_ref = R.policy_act(params, norm["obs"], cfg, deterministic=True)
    worst = 0.0
    for n, a_gpu in ((B - 1, L.act(raw["obs"][:B - 1], deterministic=True)), (n_full, full)):
        assert a_gpu.shape == (n, cfg.n_act)
        e = rel_err(a_gpu, a_ref[:n])
        worst = max(worst, e / tol)
        assert e <= tol, (n, e)
    for n in (1, B - 1):
        part = L.act(raw["obs"][:n], deterministic=True)
        assert part.shape == (n, cfg.n_act) and np.abs(part - full[:n]).max() <= 1e-6, n
    for k in (0, 1, B - 1, B, 2 * B, 2 * B + 2):
        one = L.act(raw["obs"][k:k + 1], deterministic=True)
        assert np.abs(one[0] - full[k]).max() <= 1e-6, (k, one[0], full[k])
    L.close()
    print(f"act precision={precision}: worst err/bar {worst:.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("B", [5, 129])
@pytest.mark.parametrize("precision", [0, 1])
def test_pipelined_host_batch_path_ragged_batch(precision, B):
    """test_pipelined_host_batch_path_equals_explicit_path at B = 5 and 129.  At precision 1 (engine v2) the observations
    are compacted on the host by B2G_HOST_THREADS (16) threads before the copy: at B = 5 some threads get no rows."""
    _check_pipelined_vs_explicit(B, precision)
