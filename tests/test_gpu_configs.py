"""The SAC step at the configurations the C ABI accepts beyond the three shipped ones: image-channel counts 1, 2, 3, 4 and 8,
action counts 1 to 8, head widths 64 to 256, the three engines, the clamps of the step (log_std, observation and reward clip,
saturated actions) and VecNormalize switched off.

Where the code has a path of its own for these values:
  * conv1 reads a space-to-depth copy of the image with Cp = 1 channel at Ci = 1 and Cp = 4 at Ci = 2 to 4, so Ci = 2 and 3
    leave 2 and 1 zero pad channels; the conv1 wgrad scatter is scaled by Ci, not Cp, and at Ci = 4 the two agree;
  * the feature rows are round8(513 + A) wide, the Q heads' fc0 planes have feat_dim + A rows, and the tail kernels loop
    over A actions up to AMAX = 8 (tail4_kernel at H = 64, tailw_kernel<H> with its 8-wide blocks above);
  * images with more than 4 channels, and precision 0, run the round-1 engines (gg_tc, gg_simt), as does act() at precision 1.

The CPU tests keep the matrix honest (it covers each of those paths), check that the edge batches really cross every clamp on
both sides, pin the synthetic data the golden vectors and the benchmark are built from, and check the ABI bounds of n_act.
The GPU tests hold each case to the float64 oracle with the bars of tests/test_gpu_parity.py: one explicit step (every output,
every gradient tensor, the Adam / Polyak update), three graph-path steps, and act() against the oracle's policy.  `pytest -s`
prints the worst err/bar of each check.
"""
import ctypes as C
import dataclasses
import hashlib

import numpy as np
import pytest
import torch

from b200grasp import _lib, synth
from oracle import sac_ref as R
from tests.test_gpu_batch_edges import NS, _graph_steps_vs_oracle
from tests.test_gpu_parity import _check_pipelined_vs_explicit
from tests.test_sac_widths import _check_step
from tests.util import GOLD, load_case, make_batch, make_learner, normalize, rel_err

GRAPH_DATA_SEED = 9101          # the transitions behind _graph_steps_vs_oracle


# ------------------------------------------------------------------------------------------------ the cases
def vecnorm_for(ci):
    """VecNormalize statistics for Ci image channels: the depth run's own at Ci = 1; otherwise the RGB-D run's, with colour
    planes chosen from its channels 0-2, depth from channel 3 and the actuator plane from channel 4."""
    if ci == 1:
        return dict(np.load(f"{GOLD}/vecnorm_sac_depth.npz"))
    vn = dict(np.load(f"{GOLD}/vecnorm_sac_rgbd.npz"))
    if ci == 4:
        return vn
    chans = [c % 3 for c in range(ci - 1)] + [3, 4]
    for k in ("obs_mean", "obs_var", "old_obs"):
        vn[k] = np.ascontiguousarray(vn[k][..., chans])
    return vn


def s2d_channels(ci):
    """Channels of conv1's space-to-depth input (csrc/sac_internal.cuh); None where engine v2 does not run."""
    return 1 if ci == 1 else 4 if ci <= 4 else None


@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    ci: int           # image channels (the observation has ci + 1 planes)
    A: int            # actions
    H: int            # head width
    precision: int
    B: int
    params: str = "fresh"      # "fresh" | "trained" (the depth run's weights restricted to A actions) | "edge" | "norm_off"
    seed: int = 0

    @property
    def cfg(self):
        return R.SACConfig(obs_shape=(64, 64, self.ci + 1), n_act=self.A, layers=(self.H, self.H),
                           target_entropy=-float(self.A))

    @property
    def engine(self):
        if self.precision == 0:
            return "gg_simt"
        return "engine_v2" if self.ci <= 4 else "gg_tc"

    @property
    def tail(self):
        return "tail4" if self.H == 64 else "tailw"


CASES = [
    Case("ci2_a5_h64", 2, 5, 64, 1, 77, seed=201),                      # two pad channels
    Case("ci3_a3_h64", 3, 3, 64, 1, 129, seed=202),                     # one pad channel, the simplified action count
    Case("ci3_a8_h256", 3, 8, 256, 1, 77, seed=203),                    # tailw at AMAX
    Case("ci2_a1_h128", 2, 1, 128, 1, 65, seed=204),
    Case("ci1_a3_trained", 1, 3, 64, 1, 129, params="trained"),         # trained weights restricted to 3 actions
    Case("ci1_a8_simt", 1, 8, 64, 0, 65, seed=206),                     # gg_simt and tail4 at AMAX
    Case("ci8_a5_tc", 8, 5, 64, 1, 32, seed=207),                       # round-1 engines at the u8-mask channel limit
    Case("ci8_a5_simt", 8, 5, 64, 0, 32, seed=207),
]
EDGE_CASES = [Case(f"edge_h{H}_p{p}", 1, 5, H, p, 129, params="edge", seed=300 + H + p) for H in (64, 256) for p in (1, 0)]
NORM_OFF_CASES = [Case(f"norm_off_p{p}", 4, 3, 64, p, 77, params="norm_off", seed=400 + p) for p in (1, 0)]
ALL_CASES = CASES + EDGE_CASES + NORM_OFF_CASES

# The edge batches: clip_obs != clip_reward, and a return variance that puts the -200 rewards past -clip_reward, the 100 .. 110
# ones (4.76 .. 5.24) on both sides of +clip_reward and the 10000 ones far past it.
EDGE_CLIP_OBS, EDGE_CLIP_REWARD, EDGE_RET_VAR = 10.0, 5.0, 21.0 ** 2
KINK = 1e-3        # no raw log_std this close to a clamp bound: fp32 could not decide its side (the ReLU-kink rule)


def _restricted_trained(A):
    """The depth run's trained parameters restricted to A actions: the first A columns of pi/dense*, the qf fc0 kernels
    without their last 5 - A action rows."""
    cfg5, trained, _ = load_case("sac_depth")
    cfg = R.SACConfig(obs_shape=cfg5.obs_shape, n_act=A, target_entropy=-float(A))
    return {n: np.array(trained[n][tuple(slice(0, d) for d in shape)], np.float32) for n, shape in R.param_specs(cfg)}


def _edge_vecnorm():
    """The depth statistics with pixels whose data sit past every clip: mean 3 m (the data ceiling is 2 m) or -1 m (floor
    0.02 m) with variance 1e-6 normalise to -clip / +clip; zero variance leaves epsilon alone; the actuator value (U(0, 1))
    with variance 1e-4 is clipped at both signs unless within 0.1 of its mean."""
    vn = vecnorm_for(1)
    mean, var = vn["obs_mean"].copy(), vn["obs_var"].copy()
    mean[:8, :8, 0], var[:8, :8, 0] = 3.0, 1e-6
    mean[56:, 56:, 0], var[56:, 56:, 0] = -1.0, 1e-6
    var[:8, 56:, 0] = 0.0
    var[0, 0, 1] = 1e-4
    vn.update(obs_mean=mean, obs_var=var, ret_var=np.float64(EDGE_RET_VAR), clip_obs=np.float64(EDGE_CLIP_OBS),
              clip_reward=np.float64(EDGE_CLIP_REWARD))
    return vn


def _pi_latent(params, obs_norm, cfg):
    """The policy MLP's output g (float64) for normalised observations."""
    tp = {n: torch.tensor(a, dtype=torch.float64) for n, a in params.items() if n.startswith("model/pi/")}
    x = torch.tensor(np.asarray(obs_norm), dtype=torch.float64) / 255.0
    with torch.no_grad():
        return R.mlp(R.features(x, tp, "model/pi", cfg), tp, "model/pi", len(cfg.layers)).numpy()


def _edge_latents(case, params, vn):
    """g for the explicit step's batch and for every observation the graph-path steps may draw."""
    cfg = case.cfg
    _, norm, eps = make_batch(vn, case.B, n_act=case.A)
    tr = synth.make_transitions(NS, vn["obs_mean"], vn["obs_var"], seed=GRAPH_DATA_SEED, n_act=case.A)
    return _pi_latent(params, norm["obs"], cfg), _pi_latent(params, normalize(tr, vn)["obs"], cfg), norm, eps


def _edge_params(case, vn):
    """Fresh parameters with per-action biases: action 0's raw log_std straddles LOG_STD_MAX and action 1's LOG_STD_MIN (each
    column of pi/dense_1 scaled to a spread of 2 over the batch, its bias centring the batch on the bound, nudged so that no
    observation of the batch or of the graph-path transitions lies within KINK of it); pi/dense bias 9 on action 2 puts about
    half of its actions into fp32 saturation, as the wide noise of action 0 does for some of its."""
    params = R.init_params(case.cfg, seed=case.seed)
    g_b, g_t, _, _ = _edge_latents(case, params, vn)
    k, b = params["model/pi/dense_1/kernel"], params["model/pi/dense_1/bias"]
    for a, bound in ((0, R.LOG_STD_MAX), (1, R.LOG_STD_MIN)):
        rb, rt = g_b @ k[:, a].astype(np.float64), g_t @ k[:, a].astype(np.float64)
        scale = np.float32(2.0 / rb.std())
        k[:, a] *= scale
        rb, rt = g_b @ k[:, a].astype(np.float64), g_t @ k[:, a].astype(np.float64)
        for nudge in np.arange(0.0, 0.2, 0.00125):
            b[a] = np.float32(bound - np.median(rb) + nudge)
            if min(np.abs(rb + b[a] - bound).min(), np.abs(rt + b[a] - bound).min()) >= 2 * KINK:
                break
        else:
            raise AssertionError(f"no bias keeps action {a} clear of {bound}")
    params["model/pi/dense/bias"][2] = 9.0
    return params


def build(case):
    """-> (cfg, params, vecnormalize stats)."""
    cfg = case.cfg
    if case.params == "edge":
        vn = _edge_vecnorm()
        return cfg, _edge_params(case, vn), vn
    vn = vecnorm_for(case.ci)
    if case.params == "norm_off":
        vn.update(norm_obs=np.bool_(False), norm_reward=np.bool_(False))
    params = _restricted_trained(case.A) if case.params == "trained" else R.init_params(cfg, seed=case.seed)
    return cfg, params, vn


# ================================================================================================ CPU
def _digest(tr):
    h = hashlib.sha256()
    for k in ("obs", "next_obs", "act", "rew", "done"):
        h.update(np.ascontiguousarray(tr[k]).tobytes())
    return h.hexdigest()


# sha256 of make_transitions for the depth and RGB-D statistics, taken before synth learnt other channel counts: the golden
# vectors' and the benchmark's batches come from these streams.
SYNTH_DIGESTS = {
    ("sac_depth", 64, synth.DATA_SEED): "62b2e47919200d19101223674004e87cbd0266ee7667cc5b060f18767705dc90",
    ("sac_depth", 512, 9101): "738083479cf42b70d731c63f113ecd75f5017ef79315e33221d68c830a639bb8",
    ("sac_rgbd", 64, synth.DATA_SEED): "51bc151b32e54ac2f7a7591924f463f47c8482152626597358973df4eeb3eb39",
    ("sac_rgbd", 512, 9101): "e1db9e846726fba7e42460b4972a96af8eb9f44070edcd0900d105dccaacab43",
}


@pytest.mark.parametrize("key,n,seed", list(SYNTH_DIGESTS))
def test_synth_depth_and_rgbd_streams_unchanged(key, n, seed):
    vn = np.load(f"{GOLD}/vecnorm_{key}.npz")
    assert _digest(synth.make_transitions(n, vn["obs_mean"], vn["obs_var"], seed=seed)) == SYNTH_DIGESTS[(key, n, seed)]


@pytest.mark.parametrize("ci", [1, 2, 3, 4, 8])
def test_synth_every_channel_count(ci):
    """The last image plane is depth (0.02 .. 2 m), the ones before it integer colour 0 .. 255, the actuator plane zero but
    for pixel [0, 0]."""
    vn = vecnorm_for(ci)
    assert vn["obs_mean"].shape == (64, 64, ci + 1)
    tr = synth.make_transitions(16, vn["obs_mean"], vn["obs_var"], n_act=3)
    assert tr["act"].shape == (16, 3)
    for k in ("obs", "next_obs"):
        o = tr[k]
        depth = o[..., ci - 1]
        assert depth.min() >= np.float32(0.02) and depth.max() <= 2.0 and np.any(depth != np.round(depth))
        colour = o[..., :ci - 1]
        assert np.array_equal(colour, np.round(colour)) and np.all((colour >= 0) & (colour <= 255))
        assert not o[:, 1:, :, ci].any() and not o[:, 0, 1:, ci].any()


def test_matrix_covers_every_config_path():
    """Like test_sweep_covers_every_tile_residue: the cases reach each path of the code sized by Ci, Cp, A, H and precision."""
    v2 = [c for c in ALL_CASES if c.engine == "engine_v2"]
    pads = {(s2d_channels(c.ci), s2d_channels(c.ci) - c.ci) for c in v2}
    assert {(1, 0), (4, 0), (4, 1), (4, 2)} <= pads, pads
    assert {1, 3, 8} <= {c.A for c in ALL_CASES}
    assert {"tail4", "tailw"} <= {c.tail for c in ALL_CASES}
    assert {(8, "tail4"), (8, "tailw")} <= {(c.A, c.tail) for c in ALL_CASES}, "AMAX on both tail kernels"
    assert {"engine_v2", "gg_tc", "gg_simt"} <= {c.engine for c in ALL_CASES}
    assert any(c.engine == "gg_tc" and c.ci == 8 for c in CASES), "the tensor-core round-1 engine at the u8-mask limit"
    assert any(c.precision == 1 for c in CASES), "act() at precision 1 runs on gg_tc"
    assert any(c.params == "trained" and c.A == 3 for c in CASES)
    assert {(c.H, c.precision) for c in EDGE_CASES} == {(64, 0), (64, 1), (256, 0), (256, 1)}
    assert {c.precision for c in NORM_OFF_CASES} == {0, 1}


@pytest.mark.parametrize("case", EDGE_CASES, ids=lambda c: c.name)
def test_edge_batches_cross_every_clamp(case):
    """In the float64 oracle's forward of the explicit step's batch: raw log_std on both sides of 2 and of -20 and never within
    KINK of either; normalised observations at +clip, -clip and inside; rewards clipped at both signs and unclipped;
    actions saturated in fp32 and not."""
    cfg, params, vn = build(case)
    assert float(vn["clip_obs"]) != float(vn["clip_reward"])
    g_b, g_t, norm, eps = _edge_latents(case, params, vn)
    raw, _, _ = make_batch(vn, case.B, n_act=case.A)
    for g in (g_b, g_t):
        ls_raw = g @ params["model/pi/dense_1/kernel"].astype(np.float64) + params["model/pi/dense_1/bias"]
        for bound in (R.LOG_STD_MAX, R.LOG_STD_MIN):
            assert np.abs(ls_raw - bound).min() >= KINK, bound
    ls_raw = g_b @ params["model/pi/dense_1/kernel"].astype(np.float64) + params["model/pi/dense_1/bias"]
    for bound in (R.LOG_STD_MAX, R.LOG_STD_MIN):
        assert (ls_raw > bound).any() and (ls_raw < bound).any(), bound
    assert (ls_raw > R.LOG_STD_MAX).sum() >= 4 and (ls_raw < R.LOG_STD_MIN).sum() >= 4
    clip_o, clip_r = float(vn["clip_obs"]), float(vn["clip_reward"])
    for k in ("obs", "next_obs"):
        o = norm[k]
        for plane in (o[..., 0], o[:, 0, 0, 1]):           # image and actuator value
            assert (plane == np.float32(clip_o)).any() and (plane == np.float32(-clip_o)).any(), k
            assert (np.abs(plane) < clip_o).any(), k
    r = norm["rew"]
    assert (r == np.float32(clip_r)).any() and (r == np.float32(-clip_r)).any(), np.unique(raw["rew"])
    assert (np.abs(r) < clip_r).any()
    mu = g_b @ params["model/pi/dense/kernel"].astype(np.float64) + params["model/pi/dense/bias"]
    u = mu + eps * np.exp(np.clip(ls_raw, R.LOG_STD_MIN, R.LOG_STD_MAX))
    sat = np.abs(np.tanh(u.astype(np.float32))) == 1.0
    assert sat.any() and not sat.all()
    assert sat[:, 2].any() and not sat[:, 2].all()


def test_norm_off_cases_switch_both_halves_off():
    for case in NORM_OFF_CASES:
        _, _, vn = build(case)
        assert not bool(vn["norm_obs"]) and not bool(vn["norm_reward"])
        raw, norm, _ = make_batch(vn, 8, n_act=case.A)
        assert np.array_equal(norm["obs"], raw["obs"]) and np.array_equal(norm["rew"], raw["rew"])


@pytest.mark.parametrize("n_act", [0, 9, -1])
def test_create_rejects_action_counts_outside_1_to_8(n_act):
    """b2g_sac_create validates n_act before it looks for a device: B2G_EINVAL (-1) on any machine."""
    lib = _lib.load()
    cfg = _lib.SacCfg()
    cfg.obs_h, cfg.obs_w, cfg.obs_c, cfg.obs_dim = 64, 64, 2, 0
    cfg.n_act, cfg.hidden, cfg.batch, cfg.buffer_capacity = n_act, 64, 8, 64
    cfg.gamma, cfg.tau, cfg.target_entropy, cfg.precision, cfg.nranks = 0.99, 0.005, -5.0, 1, 1
    h = C.c_void_p()
    assert lib.b2g_sac_create(C.byref(cfg), C.byref(h)) == -1
    assert not h.value
    assert "n_act must be in [1,8]" in lib.b2g_last_error().decode()


# ================================================================================================ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES + EDGE_CASES + NORM_OFF_CASES, ids=lambda c: c.name)
def test_step_vs_oracle(case):
    """One explicit step and three graph-path steps against the float64 oracle."""
    cfg, params, vn = build(case)
    print(f"{case.name}: Ci={case.ci} A={case.A} H={case.H} precision={case.precision} B={case.B} ({case.engine}, {case.tail})")
    _check_step(cfg, params, vn, case.B, precision=case.precision)
    _graph_steps_vs_oracle(cfg, params, vn, case.B, data_seed=GRAPH_DATA_SEED, precision=case.precision)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES + EDGE_CASES, ids=lambda c: c.name)
def test_act_vs_oracle(case):
    """act(): deterministic against the oracle's policy over a call of two chunks and a short third (batch 32, 67 rows), the
    same rows split across calls at other offsets, and stochastic with the noise the device drew for a one-chunk call.
    Deterministic bars: 1e-5 absolute on fresh heads (test_act_equals_oracle_and_is_row_position_independent); on trained
    weights, whose pre-tanh means are larger, 1e-4 relative L2 over the call (test_act_in_chunks_of_the_batch), and the
    restricted model's actions must be the full 5-action model's first A."""
    cfg, params, vn = build(case)
    raw, norm, _ = make_batch(vn, 67, n_act=case.A)
    L = make_learner(cfg, vn, 32, params, precision=case.precision, hidden=case.H)
    full = L.act(raw["obs"], deterministic=True)
    ref = R.policy_act(params, norm["obs"], cfg, deterministic=True)
    assert full.shape == (67, case.A)
    det, det_rel = float(np.abs(full - ref).max()), rel_err(full, ref)
    parts = np.concatenate([L.act(raw["obs"][:31], deterministic=True), L.act(raw["obs"][31:40], deterministic=True),
                            L.act(raw["obs"][40:], deterministic=True)])
    assert np.abs(parts - full).max() <= 1e-6
    a_sto = L.act(raw["obs"][:20], deterministic=False)
    eps = L.last_batch()["eps"][:20]
    s_ref = R.policy_act(params, norm["obs"][:20], cfg, deterministic=False, eps_noise=eps)
    sto = rel_err(a_sto, s_ref)
    L.close()
    print(f"{case.name} act: deterministic max err {det:.2e}, rel err {det_rel:.2e}; stochastic rel err {sto:.2e} (bar 1e-4)")
    assert np.abs(eps).max() > 0 and np.abs(a_sto - full[:20]).max() > 0
    if case.params == "trained":
        assert det_rel <= 1e-4
        cfg5, params5, _ = load_case("sac_depth")
        L5 = make_learner(cfg5, vn, 32, params5, precision=case.precision)
        a5 = L5.act(raw["obs"], deterministic=True)
        L5.close()
        print(f"{case.name} act: max |A={case.A} - first {case.A} of A=5| {np.abs(full - a5[:, :case.A]).max():.2e}")
        assert np.abs(full - a5[:, :case.A]).max() <= 2e-6
    else:
        assert det <= 1e-5
    assert sto <= 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("case", NORM_OFF_CASES, ids=lambda c: c.name)
def test_norm_off_host_pipelined_path(case):
    """Normalisation off through the host-pipelined step: the same losses and parameters as the explicit step."""
    cfg, params, vn = build(case)
    _check_pipelined_vs_explicit(case.B, case.precision, cfg=cfg, params=params, vn=vn)
