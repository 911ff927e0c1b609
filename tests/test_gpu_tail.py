"""The SAC head tail (csrc/tail.cu: tail4_kernel at H = 64, tailw_kernel<H> at H = 128, 192, 256) held element by element to
float64 of the inputs it read.

The step-level tests compare per-sample vectors and gradient tensors by relative norm; an error confined to one sample, one
column, one action, one of tailw's four-sample groups or the lo plane of dz0 moves those norms by less than their bars.  Here
one step runs per case and `b2g_debug_tensor` reads back what the tail read (z0 of the five heads, the replay actions in
F32/values, rew_n, done_n; the parameters and the policy noise come from the handle) and what it wrote, and:
  * bit for bit: a0/<head> = fp32 max(z0 + b0, 0); the BF16 planes of dz0 (engine v2): hi = RN(dz0), lo = RN(dz0 - hi);
    dz0 = 0 wherever the stored a0 is 0; dense_1's gradient column of an action clamped in every sample is 0;
  * within gamma_H sum|dz1||W1|: dz0_pi and dz0_v3 recomputed from the stored dz1 and a0 (no non-linearity in between);
  * within tests/tail_ref.py's running error bound: the per-sample outputs, pi, dz1 of the four heads, the loss and metric
    sums, and the output-layer and log_ent_coef gradients of the arena.
The ReLU sides the kernel reveals (a0 > 0; a non-zero dz1 entry) are the sides the bound is taken on, and each must be the
float64 side unless its input is within its bound of 0.  The sides no tensor shows (qf1 / qf2 at pi, the log_std clamp) must
be clear of their kinks by more than the bound: the case takes the next batch seed if one is not.

`pytest -s` prints the worst err/bar of every quantity of every case.
"""
import dataclasses

import numpy as np
import pytest

import b200grasp
from b200grasp import synth
from oracle import sac_ref as R
from tests import tail_ref as T
from tests import test_gpu_configs as G
from tests.gg_tc_ref import Report, bf16_split
from tests.test_gpu_contractions import read
from tests.util import load_case, make_batch, make_learner

NS = 256          # replay transitions behind the sampled case
TRIES = 6         # batch seeds a case may take to keep its hidden masks clear of their kinks


@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    B: int
    H: int = 64
    A: int = 5
    ci: int = 1
    precision: int = 1
    params: str = "trained"     # "trained" (the depth run) | "edge" (test_gpu_configs' edge construction) | "fresh" |
                                # "encoder" (the MLP policy's shipped weights) | "nature" (nature_cnn, the depth run's weights)
    sampled: bool = False       # one graph-path step sampled from the replay (else an explicit step)
    seed: int = 0

    @property
    def kernel(self):
        return "tail4" if self.H == 64 else f"tailw<{self.H}>"

    @property
    def v2(self):
        """engine v2 (the value heads' z0 in one [B][3H] block, dz0 BF16 planes) runs the CNN policies at bf16x3"""
        return self.precision == 1 and self.params != "encoder" and self.ci <= 4


TAILW = []
for H in (128, 192, 256):
    for i, B in enumerate((1, 2, 3, 4, 5, 77 if H != 192 else 78)):
        A = (1, 3, 8)[(i + H // 64) % 3]
        TAILW.append(Case(f"h{H}_a{A}_b{B}_p{i % 2 ^ 1}", B, H=H, A=A, precision=i % 2 ^ 1,
                          params="edge" if A >= 3 else "fresh", seed=700 + H + i))
CASES = [Case(f"depth_b{B}", B) for B in (1, 2, 3, 129, 383)] + [
    Case("ci3_a3_b77", 77, A=3, ci=3, params="fresh", seed=12),
    Case("a8_p0_b65", 65, A=8, precision=0, params="edge", seed=31),
    Case("a1_p0_b40", 40, A=1, precision=0, params="fresh", seed=32),
    Case("edge_a5_b129", 129, A=5, params="edge", seed=33),
] + TAILW + [
    Case("mlp_encoder_b64", 64, params="encoder"),
    Case("nature_a3_b64", 64, A=3, params="nature", seed=34),
    Case("sampled_b77", 77, sampled=True, seed=35),
]


def build(case):
    """-> (cfg, params, vecnormalize stats)"""
    if case.params == "trained":
        cfg, params, vn = load_case("sac_depth")
    elif case.params == "encoder":
        cfg, params, vn = load_case("sac_encoder")
    elif case.params == "nature":
        from tests.test_gpu_sac_nature_cnn import trained, vecnorm
        cfg, params = trained(case.A)
        vn = vecnorm(2)
    elif case.params == "edge":
        # the edge construction centres raw log_std on the clamps over a batch of 129 (a spread needs more than one sample)
        cfg, params, vn = G.build(G.Case(case.name, case.ci, case.A, case.H, case.precision, max(case.B, 129), "edge", case.seed))
    else:
        cfg, vn = R.SACConfig(obs_shape=(64, 64, case.ci + 1), n_act=case.A, layers=(case.H, case.H),
                              target_entropy=-float(case.A)), G.vecnorm_for(case.ci)
        params = R.init_params(cfg, seed=case.seed)
        rng = np.random.default_rng(case.seed)
        for k in [k for k in params if k.endswith("/b") or k.endswith("/bias")]:
            params[k] = (rng.standard_normal(params[k].shape) * 0.05).astype(np.float32)
        params["model/pi/dense_1/bias"] += np.float32(-1.0)
    if case.params != "trained":
        params["model/log_ent_coef"] = np.array(-0.6, np.float32)
    return cfg, params, vn


def _learner(case, cfg, vn, params, monkeypatch):
    if case.params == "nature":
        from tests.test_gpu_sac_nature_cnn import NatureLearner
        monkeypatch.setattr(b200grasp, "Learner", NatureLearner)
    kw = dict(buffer_size=NS) if case.sampled else dict(buffer_size=max(64, case.B))
    return make_learner(cfg, vn, case.B, params, precision=case.precision, hidden=case.H, **kw)


def run_step(case, cfg, params, vn, seed, monkeypatch):
    """One step; -> (tensors, gradients, parameters the tail read, metrics, last batch)."""
    L = _learner(case, cfg, vn, params, monkeypatch)
    try:
        P = {k: np.asarray(v, np.float32) for k, v in L.get_parameters().items()}
        if case.sampled:
            tr = synth.make_transitions(NS, vn["obs_mean"], vn["obs_var"], seed=seed, n_act=case.A)
            L.replay_add(tr["obs"], tr["act"], tr["rew"], tr["next_obs"], tr["done"])
            m = L.step(1, lr=3e-4)
        else:
            raw, _, eps = make_batch(vn, case.B, seed=seed, n_act=case.A)
            m = L.step_explicit(raw["obs"], raw["act"], raw["rew"], raw["next_obs"], raw["done"], eps, lr=3e-4, apply_update=False)
        heads = [f"{t}/{h}" for t in ("a0", "dz1") for h in T.HEADS]
        names = heads + ["dz0_pi", "dz0_v3", "z0/pi", "z0/target", "F32/values", "rew_n", "done_n"]
        names += ["z0v", "dz0pi", "dz0v"] if case.v2 else ["z0/vf", "z0/qf1", "z0/qf2"]
        Tn = {n: read(L, n)[0] if n not in ("dz0pi", "dz0v") else read(L, n) for n in names}
        Gr = {k: np.asarray(v, np.float64) for k, v in L.get_gradients().items()}
        last = L.last_batch()
    finally:
        L.close()
    return Tn, Gr, P, m, last


def check(case, cfg, Tn, Gr, P, m, last, rep):
    B, H, A = case.B, case.H, case.A
    feat_dim = cfg.feat_dim
    z0 = {"pi": Tn["z0/pi"].reshape(B, H), "target": Tn["z0/target"].reshape(B, H)}
    if case.v2:
        v3 = Tn["z0v"].reshape(B, 3 * H)
        for j, h in enumerate(("vf", "qf1", "qf2")):
            z0[h] = v3[:, j * H:(j + 1) * H]
    else:
        for h in ("vf", "qf1", "qf2"):
            z0[h] = Tn[f"z0/{h}"].reshape(B, H)
    a0 = {h: Tn[f"a0/{h}"].reshape(B, H) for h in T.HEADS}
    dz1 = {h: Tn[f"dz1/{h}"].reshape(B, H) for h in T.HEADS}
    dz0 = {"pi": Tn["dz0_pi"].reshape(B, H)}
    d3 = Tn["dz0_v3"].reshape(B, 3 * H)
    for j, h in enumerate(("vf", "qf1", "qf2")):
        dz0[h] = d3[:, j * H:(j + 1) * H]
    act = Tn["F32/values"].reshape(B, -1)[:, feat_dim:feat_dim + A]
    rew, done, eps = Tn["rew_n"], Tn["done_n"], last["eps"]
    # ---- bit for bit
    for h in T.HEADS:
        b0 = P[f"{T.PREFIX[h]}/fc0/bias"]
        rep.exact(f"a0/{h} = max(z0 + b0, 0)", a0[h], np.maximum(z0[h] + b0, np.float32(0)))
        rep.exact(f"dz0/{h} = 0 where a0 = 0", np.where(a0[h] > 0, 0, dz0[h]), np.zeros_like(dz0[h]))
    if case.v2:
        for name, v in (("dz0pi", dz0["pi"]), ("dz0v", d3)):
            hi, lo = bf16_split(v, 2)
            rep.exact(f"{name} hi plane", Tn[name][0].reshape(hi.shape), hi)
            rep.exact(f"{name} lo plane", Tn[name][1].reshape(lo.shape), lo)
    # ---- dz0 from the stored dz1 and a0: gamma_H sum|dz1||W1|
    for h in T.HEADS:
        W1 = P[f"{T.PREFIX[h]}/fc1/kernel"].astype(np.float64)
        d = dz1[h].astype(np.float64)
        ref = np.where(a0[h] > 0, d @ W1.T, 0.0)
        rep.hold(f"dz0/{h} (gamma_H)", dz0[h], ref, np.where(a0[h] > 0, np.abs(d) @ np.abs(W1).T, 0.0), T.SLACK * T.gamma(H))
    # ---- the restatement, on the sides the kernel revealed
    masks = {f"a0/{h}": a0[h] > 0 for h in T.HEADS}
    masks.update({f"a1/{h}": dz1[h] != 0 for h in T.HEADS})
    X = T.Bound(masks)
    o = T.tail(X, z0, P, act, eps, rew, done, cfg.gamma, cfg.target_entropy, feat_dim, pi_in=last["pi"])
    for key in masks:
        rep.exact(f"{key} side possible", X.bad[key], np.zeros_like(X.bad[key]))
    near = {k: int(X.near[k].sum()) for k in T.UNREVEALED if X.near[k].any()}

    def hold(name, got, ref):
        rep.hold(name, np.asarray(got, np.float64).reshape(ref.v.shape), ref.v, T.SLACK * ref.e, 1.0)

    for k in T.PER_SAMPLE:
        hold(k, last[k], o[k])
    hold("pi", last["pi"], o["pi"])
    for h in T.HEADS:
        hold(f"dz1/{h}", dz1[h], o[f"dz1/{h}"])
    for k in T.SUMS:
        hold(k, m[k], o[k])
    for k in T.GRADS:
        hold(f"grad {k}", Gr[k], o["g/" + k])
    # an action clamped (past either bound) in every sample takes no dense_1 gradient at all
    off = ~X.side["ls"] & ~X.near["ls/max"] & ~X.near["ls/min"]
    for a in np.flatnonzero(off.all(0)):
        rep.exact(f"dense_1 column {a} (clamped in every sample)", Gr["model/pi/dense_1/kernel"][:, a], np.zeros(H))
        rep.exact(f"dense_1 bias {a} (clamped in every sample)", Gr["model/pi/dense_1/bias"][a], 0.0)
    return X, near


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_tail_matches_float64_of_its_inputs(case, monkeypatch):
    cfg, params, vn = build(case)
    base = 9101 + case.seed if case.sampled else synth.DATA_SEED       # attempt 0: the batch the edge construction saw
    for attempt in range(TRIES):
        rep = Report(f"{case.name} ({case.kernel}, {'engine v2' if case.v2 else f'precision {case.precision}'})")
        Tn, Gr, P, m, last = run_step(case, cfg, params, vn, base + 1000 * attempt, monkeypatch)
        _, near = check(case, cfg, Tn, Gr, P, m, last, rep)
        if not near:
            break
        print(f"{case.name}: batch seed {base + 1000 * attempt} leaves hidden masks within their bound of a kink {near}")
    else:
        pytest.fail(f"{case.name}: no batch seed of {TRIES} keeps the hidden masks clear of their kinks")
    rep.finish()


def test_matrix_covers_every_tail_path():
    """Both kernels at every head width, AMAX on both, every B mod 4 on tailw (its four-sample groups) at every H, both z0
    layouts and both precisions on tailw, and (through the edge cases) raw log_std past both clamps."""
    assert {c.H for c in CASES} == {64, 128, 192, 256}
    assert {(8, "tail4"), (8, "tailw")} <= {(c.A, c.kernel[:5]) for c in CASES}
    assert 1 in {c.A for c in CASES}
    for H in (128, 192, 256):
        assert {c.B % 4 for c in CASES if c.H == H} == {0, 1, 2, 3}
        assert any(c.B >= 77 for c in CASES if c.H == H)
        assert {c.v2 for c in CASES if c.H == H} == {True, False}
    assert {1, 2, 3, 129, 383} <= {c.B for c in CASES if c.params == "trained" and not c.sampled}
    assert any(c.ci == 3 and c.A == 3 and c.B == 77 for c in CASES)
    assert {c.v2 for c in CASES if c.H == 64} == {True, False}
    assert {"encoder", "nature", "edge"} <= {c.params for c in CASES} and any(c.sampled for c in CASES)


@pytest.mark.parametrize("case", [c for c in CASES if c.params == "edge" and c.B >= 77], ids=lambda c: c.name)
def test_edge_cases_cross_both_clamps(case):
    """The float64 oracle's raw log_std over the case's batch lies past 2 and past -20 on some samples and inside on others."""
    cfg, params, vn = build(case)
    g_b, _, _, _ = G._edge_latents(G.Case(case.name, case.ci, case.A, case.H, case.precision, case.B, "edge", case.seed),
                                   params, vn)
    ls = g_b @ params["model/pi/dense_1/kernel"].astype(np.float64) + params["model/pi/dense_1/bias"]
    assert (ls > T.LOG_STD_MAX).any() and (ls < T.LOG_STD_MIN).any()
    assert ((ls > T.LOG_STD_MIN) & (ls < T.LOG_STD_MAX)).any()
