"""The BDQ learner (csrc/bdq.cu) at the shapes b2g_bdq_create accepts, on its sampled graph step, and the device random streams.

Where the code has a path of its own for these values:
  * the tail kernel loops over D <= 8 branches (A[3][8], dA[8], d_Aptr) and n <= 64 bins held at a row stride NBS = round4(n),
    so n = 64, 63, 2 and 33 leave 0, 1, 2 and 3 pad columns;
  * every layer runs on gg_simt (64 x 64 tiles, 16-deep K-steps): widths below 16 sit inside one K-step, widths of 64k + 4 put
    4 columns into a last tile, multiples of 64 fill their tiles;
  * the gather writes observation rows of obs_dim floats (128-bit path when obs_dim % 4 == 0, scalar path otherwise) followed
    by the D raw action indices into rows of XS = round8(obs_dim + D);
  * trunk_grad_rescale scales the trunk's incoming gradient by 1/(D+1) or not at all; prioritised replay (PER) replaces the
    uniform slots by the segment-tree draw and weights the loss (batch <= 1024).

The CPU tests keep the matrix honest, check the create refusals, and pin the Philox4x32-10 restatement (oracle/philox_ref.py)
with the Random123 known-answer vectors and the statistics of the Box-Muller noise.  The GPU tests hold act(), argmax ties,
the sampled graph step as a trajectory, observation / reward normalisation and the device's slots and noise to the float64
oracle and to the restated streams.  The explicit step at every case is tests/test_gpu_bdq.py::test_bdq_step_matches_oracle.
`pytest -s` prints each check's worst err/bar and the number of near-tie rows and ReLU kinks it met.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

import b200grasp
from b200grasp import _lib
from oracle import bdq_ref as Q
from oracle import philox_ref as PX
from oracle import sac_ref as R
from tests.util import load_case, make_learner, normalize, rel_err

TOL = 1e-4         # outputs, relative (or 3x the fp32 oracle's own distance from float64)
GTOL = 1e-3        # per-tensor gradients, relative L2 (or 3x the fp32 oracle's)
LR = 1e-3
U32 = 2.0 ** -24
PER_EPS = 1e-6


def _round(x, m):
    return (x + m - 1) // m * m


# ------------------------------------------------------------------------------------------------ the cases
@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    obs: int
    D: int
    n: int
    T0: int
    T1: int
    HB: int
    B: int
    gamma: float = 0.99
    rescale: bool = True
    per: bool = False
    all_done: bool = False
    seed: int = 1

    @property
    def cfg(self):
        return Q.BDQConfig(self.obs, self.D, self.n, (self.T0, self.T1), self.HB, self.HB, self.gamma, self.rescale)

    @property
    def NBS(self):
        return _round(self.n, 4)

    @property
    def XS(self):
        return _round(self.obs + self.D, 8)


CASES = [
    Case("tiny_d1_n2_b1", 1, 1, 2, 4, 8, 4, 1, seed=11),
    Case("d8_n64_b63", 24, 8, 64, 64, 68, 12, 63, seed=12),
    Case("d3_n63_b65", 13, 3, 63, 68, 64, 128, 65, seed=13),
    Case("per_d5_n33_b130", 100, 5, 33, 64, 64, 32, 130, per=True, seed=14),
    Case("norescale_d2_n8_b3", 7, 2, 8, 260, 12, 68, 3, rescale=False, seed=15),
    Case("gamma1_d3_n33_b36", 101, 3, 33, 512, 256, 128, 36, gamma=1.0, seed=16),
    Case("alldone_d4_n16_b5", 30, 4, 16, 12, 4, 516, 5, all_done=True, seed=17),
    Case("per_b1024", 100, 3, 33, 64, 64, 32, 1024, per=True, seed=18),
    Case("d6_n2_b22", 10, 6, 2, 132, 8, 64, 22, seed=19),
    Case("d8_n33_b7", 9, 8, 33, 4, 260, 4, 7, rescale=False, seed=20),
    Case("d1_n64_b200", 55, 1, 64, 128, 128, 8, 200, per=True, seed=21),
    Case("d2_n63_b9", 6, 2, 63, 8, 12, 260, 9, seed=22),
    Case("d3_n8_b42", 100, 3, 8, 64, 64, 32, 42, gamma=1.0, all_done=True, seed=23),
    Case("d7_n5_b11", 2, 7, 5, 68, 4, 12, 11, seed=24),
    Case("d4_n64_b76", 60, 4, 64, 16, 132, 64, 76, rescale=False, per=True, seed=25),
    Case("d5_n2_b13", 3, 5, 2, 4, 4, 4, 13, seed=26),
    Case("d2_n33_b254", 31, 2, 33, 64, 128, 68, 254, seed=27),
]
CASE_BY_NAME = {c.name: c for c in CASES}
# the sampled graph step as a trajectory: half of them with PER
TRAJ_CASES = ["d8_n64_b63", "norescale_d2_n8_b3", "per_d5_n33_b130", "d4_n64_b76"]


def case_for(cfg, B):
    """The matrix case with this configuration and batch, or a plain one (fresh weights, uniform replay)."""
    for c in CASES:
        if c.cfg == cfg and c.B == B:
            return c
    return Case(f"cfg_{cfg.obs_dim}_{cfg.n_branches}_{cfg.n_bins}", cfg.obs_dim, cfg.n_branches, cfg.n_bins, cfg.trunk[0],
                cfg.trunk[1], cfg.branch_hidden, B, cfg.gamma, cfg.trunk_grad_rescale)


def make_params(case):
    """Xavier weights, biases N(0, 0.1), and a target net 0.02 away from the online one."""
    params = Q.init_params(case.cfg, seed=case.seed)
    rng = np.random.default_rng(case.seed + 1000)
    for n in params:
        if n.endswith("biases"):
            params[n] = (rng.normal(size=params[n].shape) * 0.1).astype(np.float32)
        elif n.startswith("bdq/target_q_func") and n.endswith("weights"):
            params[n] = (params[n] + rng.normal(size=params[n].shape).astype(np.float32) * 0.02).astype(np.float32)
    return params


def make_batch(case, B, seed):
    rng = np.random.default_rng(seed)
    cfg = case.cfg
    bt = dict(obs=rng.normal(0.4, 0.2, (B, cfg.obs_dim)).astype(np.float32),
              next_obs=rng.normal(0.4, 0.2, (B, cfg.obs_dim)).astype(np.float32),
              act_idx=rng.integers(0, cfg.n_bins, (B, cfg.n_branches)),
              rew=(rng.choice([0.0, 1.0], B) * rng.uniform(0.2, 3.0, B)).astype(np.float32),
              done=(rng.random(B) < 0.2).astype(np.float32))
    if case.all_done:
        bt["done"][:] = 1.0
    return bt


def make_learner_bdq(case, buffer_size=256, freq=2, seed=0, **kw):
    cfg = case.cfg
    return b200grasp.BDQLearner(cfg.obs_dim, cfg.n_branches, cfg.n_bins, (cfg.trunk, (cfg.branch_hidden,), (cfg.value_hidden,)),
                                batch_size=case.B, buffer_size=buffer_size, gamma=cfg.gamma, target_network_update_freq=freq,
                                trunk_grad_rescale=cfg.trunk_grad_rescale, seed=seed, prioritized_replay=case.per,
                                prioritized_replay_eps=PER_EPS, **kw)


# ------------------------------------------------------------------------------------------------ fp32 resolution rules
def _t64(a):
    return torch.tensor(np.asarray(a, np.float64))


def relu_kinks(params, obs, cfg):
    """ReLU inputs of the online net at s whose sign fp32 cannot decide: |z| (float64) <= 4 sqrt(K) 2^-24 sum|w x| (the rule
    of tests/test_gpu_batch_edges.py::_relu_kinks).  -> [(bias name, unit, z)], nearest to zero first."""
    p = {n: _t64(a) for n, a in params.items() if n.startswith("bdq/model/")}
    found = []

    def layer(x, name):
        w, b = p[name + "/weights"], p[name + "/biases"]
        z, mag = x @ w + b, x.abs() @ w.abs() + b.abs()
        for r, c in (z.abs() <= 4 * np.sqrt(w.shape[0]) * U32 * mag).nonzero().tolist():
            found.append((name + "/biases", c, float(z[r, c])))
        return torch.relu(z)

    h = layer(_t64(obs), "bdq/model/common_net/fully_connected")
    h = layer(h, "bdq/model/common_net/fully_connected_1")
    layer(h, "bdq/model/state_value/fully_connected")
    for d in range(cfg.n_branches):
        layer(h, f"bdq/model/action_value/{Q._fc(2 * d)}")
    return sorted(found, key=lambda f: abs(f[2]))


def other_sides(params, kinks, max_n=6):
    """Parameter sets with the pre-activations of `kinks` moved to their other side (bias -= 2z): one per kink, and all."""
    kinks = kinks[:max_n]

    def moved(sel):
        q = {n: np.array(a, np.float32, copy=True) for n, a in params.items()}
        for bname, c, z in sel:
            q[bname].reshape(-1)[c] -= np.float32(2 * z)
        return q
    return [moved([k]) for k in kinks] + ([moved(kinks)] if len(kinks) > 1 else [])


def online_advantages(params, obs, cfg):
    """float64 advantages A [B, D, n] of the online net and their fp32 resolution 4 sqrt(HB) 2^-24 sum|w hb|."""
    p = {n: _t64(a) for n, a in params.items() if n.startswith("bdq/model/")}
    h = _t64(obs)
    for k in range(2):
        h = torch.relu(h @ p[f"bdq/model/common_net/{Q._fc(k)}/weights"] + p[f"bdq/model/common_net/{Q._fc(k)}/biases"])
    A, bound = [], []
    for d in range(cfg.n_branches):
        hb = torch.relu(h @ p[f"bdq/model/action_value/{Q._fc(2 * d)}/weights"] + p[f"bdq/model/action_value/{Q._fc(2 * d)}/biases"])
        w, b = p[f"bdq/model/action_value/{Q._fc(2 * d + 1)}/weights"], p[f"bdq/model/action_value/{Q._fc(2 * d + 1)}/biases"]
        A.append((hb @ w + b).numpy())
        bound.append((4 * np.sqrt(w.shape[0]) * U32 * (hb.abs() @ w.abs() + b.abs())).numpy())
    return np.stack(A, 1), np.stack(bound, 1)


def near_ties(params, obs, cfg):
    """(row, branch, [candidate bins]) where the top two online advantages are within fp32 resolution of each other.  Bins
    whose float64 advantage equals a lower bin's exactly (bit-equal columns) are no candidates: the first maximal bin wins."""
    A, bound = online_advantages(params, obs, cfg)
    out = []
    top = A.argmax(2)
    a_top = np.take_along_axis(A, top[..., None], 2)
    b_top = np.take_along_axis(bound, top[..., None], 2)
    close = a_top - A <= b_top + bound                    # [B, D, n]; the top bin itself always
    for b, d in zip(*np.nonzero(close.sum(2) > 1)):
        cand = np.nonzero(close[b, d])[0]
        vals = {}
        for k in cand:
            vals.setdefault(A[b, d, k], k)
        if len(vals) > 1:
            out.append((int(b), int(d), sorted(vals.values())))
    return out


def tie_variants(params, batch, cfg, ties):
    """a* overrides with the near-tie choices flipped: one per tie (its runner-up), and all of them."""
    if not ties:
        return []
    base = online_advantages(params, batch["next_obs"], cfg)[0].argmax(2)
    out = []
    for b, d, cand in ties:
        a = base.copy()
        a[b, d] = next(k for k in cand if k != base[b, d])
        out.append(a)
    if len(ties) > 1:
        a = base.copy()
        for b, d, cand in ties:
            a[b, d] = next(k for k in cand if k != base[b, d])
        out.append(a)
    return out


# ------------------------------------------------------------------------------------------------ holding a step to the oracle
def hold_step(pre, opt, batch, cfg, got, grads=None, label=""):
    """The outputs `got` (loss, mean_q, grad_norm, and td [B, D] or priorities [B]) and per-tensor `grads` of one step from the
    parameters `pre` and Adam state `opt` against the float64 oracle: bar 1e-4 (outputs) / 1e-3 (gradients), or 3x the fp32
    oracle's own distance from float64 where larger.  Where a check misses and the batch holds ReLU inputs or double-Q choices
    that fp32 cannot decide, the oracle is evaluated on their other sides too and the nearest is taken.
    -> (float64 outputs, grads, new params, new opt state), worst err/bar."""
    r64, g64, p64, o64 = Q.bdq_step(pre, opt, batch, LR, cfg, torch.float64)
    r32, g32, _, _ = Q.bdq_step(pre, opt, batch, LR, cfg, torch.float32)
    vecs = [k for k in ("td", "priorities") if got.get(k) is not None]

    def errs(r, g):
        e = {k: abs(got[k] - r[k]) / (abs(r[k]) + 1e-30) for k in ("loss", "mean_q", "grad_norm")}
        for k in vecs:
            e[k] = rel_err(got[k], np.asarray(r[k], np.float64) + (PER_EPS if k == "priorities" else 0.0))
        if grads is not None:
            e.update({n: rel_err(grads[n], g[n]) for n in g})
        return e

    bars = {k: max(TOL, 3 * abs(r32[k] - r64[k]) / (abs(r64[k]) + 1e-30)) for k in ("loss", "mean_q", "grad_norm")}
    bars.update({k: max(TOL, 3 * rel_err(r32[k], r64[k])) for k in vecs})
    if grads is not None:
        bars.update({n: max(GTOL, 3 * rel_err(g32[n], g64[n])) for n in g64})
    e = errs(r64, g64)
    kinks, ties = relu_kinks(pre, batch["obs"], cfg), near_ties(pre, batch["next_obs"], cfg)
    if any(e[k] > bars[k] for k in e) and (kinks or ties):
        alts = [Q.bdq_step(q, opt, batch, LR, cfg, torch.float64)[:2] for q in other_sides(pre, kinks)]
        alts += [Q.bdq_step(pre, opt, batch, LR, cfg, torch.float64, a_star=a)[:2] for a in tie_variants(pre, batch, cfg, ties)]
        for r, g in alts:
            ea = errs(r, g)
            e = {k: min(e[k], ea[k]) for k in e}
        print(f"{label}: held on either side of {len(kinks)} ReLU kinks / {len(ties)} near-tie choices")
    worst = max(e, key=lambda k: e[k] / bars[k])
    print(f"{label}: {len(ties)} near-tie rows, {len(kinks)} ReLU kinks; worst err/bar {e[worst] / bars[worst]:.3f} ({worst})")
    bad = {k: (e[k], bars[k]) for k in e if not e[k] <= bars[k]}
    assert not bad, (label, bad)
    return (r64, g64, p64, o64), e[worst] / bars[worst]


def check_adam_update(before, after, g_gpu, m_prev, v_prev, t, label=""):
    """Element-wise: `after` equals TF-Adam applied in float64 to the GPU's own gradients `g_gpu` from `before` with moments
    (m_prev, v_prev) at step t (the rule of tests/test_gpu_parity.py::_check_step).  -> new moments, worst err/bar."""
    lr_t = LR * np.sqrt(1 - Q.ADAM_B2 ** t) / (1 - Q.ADAM_B1 ** t)
    worst, m_new, v_new = 0.0, {}, {}
    for n, g in g_gpu.items():
        g = g.astype(np.float64)
        m = Q.ADAM_B1 * m_prev.get(n, 0.0) + (1 - Q.ADAM_B1) * g
        v = Q.ADAM_B2 * v_prev.get(n, 0.0) + (1 - Q.ADAM_B2) * g * g
        m_new[n], v_new[n] = m, v
        ref = before[n].astype(np.float64) - lr_t * m / (np.sqrt(v) + Q.ADAM_EPS)
        bar = 1e-4 * LR + 2.5e-7 * np.abs(ref) + 1e-12
        worst = max(worst, float((np.abs(after[n].astype(np.float64) - ref) / bar).max()))
    print(f"{label}: Adam update worst err/bar {worst:.3f}")
    assert worst <= 1.0, (label, worst)
    return m_new, v_new


def check_vs_oracle_update(after, p64, g_list, label="", frac=1e-4):
    """Against the oracle's own update where every gradient of the step(s) is well away from zero."""
    for n in g_list[0]:
        well = np.ones(after[n].shape, bool)
        for g in g_list:
            well &= np.abs(g[n]) > frac * max(1e-30, float(np.abs(g[n]).max()))
        if well.any():
            d = np.abs(after[n].astype(np.float64) - p64[n])[well]
            assert d.max() <= 2e-2 * LR + 1e-6 * np.abs(p64[n]).max(), (label, n, d.max())


def check_explicit(cfg, B, case=None):
    """Two explicit steps at (cfg, B) against the float64 oracle: outputs, every gradient tensor, the Adam update on the GPU's
    own gradients and against the oracle's own update, the hard target copy (every 2 updates), then one sampled step."""
    case = case or case_for(cfg, B)
    cfg = case.cfg
    params = make_params(case)
    L = make_learner_bdq(case, freq=2)
    assert set(L.param_shapes) == set(n for n, _ in Q.all_specs(cfg))
    L.load_parameters(params)
    back = L.get_parameters()
    for n in params:
        assert np.array_equal(back[n], np.asarray(params[n], np.float32)), n
    bt = make_batch(case, B, case.seed + 3)
    w = np.random.default_rng(case.seed + 4).uniform(0.5, 1.5, B).astype(np.float32)
    b1 = dict(bt, weights=w)
    out = L.step_explicit(bt["obs"], bt["act_idx"].astype(np.float32), bt["rew"], bt["next_obs"], bt["done"], weights=w, lr=LR)
    g1 = L.get_gradients()
    p1 = L.get_parameters()
    assert out["n_updates"] == 1
    (r64, g64, newp64, opt64), _ = hold_step(params, {"t": 0, "m": {}, "v": {}}, b1, cfg, out, g1, label=f"{case.name} step 1")
    m1, v1 = check_adam_update(params, p1, g1, {}, {}, 1, label=f"{case.name} step 1")
    check_vs_oracle_update(p1, newp64, [g64], label=f"{case.name} step 1")
    for n in params:                                     # one update: the target net is untouched
        if n.startswith("bdq/target_q_func/"):
            assert np.array_equal(p1[n], params[n]), n
    # second step from the GPU's parameters with the oracle's moments; the hard copy follows it
    bt2 = make_batch(case, B, case.seed + 5)
    out2 = L.step_explicit(bt2["obs"], bt2["act_idx"].astype(np.float32), bt2["rew"], bt2["next_obs"], bt2["done"], lr=LR)
    g2 = L.get_gradients()
    p2 = L.get_parameters()
    assert out2["n_updates"] == 2
    (_, g64b, newp64b, _), _ = hold_step(p1, opt64, bt2, cfg, out2, g2, label=f"{case.name} step 2")
    online = {n: p2[n] for n in p2 if n.startswith("bdq/model/")}
    check_adam_update({n: p1[n] for n in online}, online, g2, m1, v1, 2, label=f"{case.name} step 2")
    check_vs_oracle_update(online, newp64b, [g64, g64b], label=f"{case.name} step 2", frac=1e-2)
    for n in online:                                     # update 2: hard copy, bit for bit
        assert np.array_equal(p2[n.replace("bdq/model", "bdq/target_q_func/model")], p2[n]), n
    L.replay_add(bt["obs"], bt["act_idx"].astype(np.float32), bt["rew"], bt["next_obs"], bt["done"])
    m = L.step(1, lr=LR)
    assert m["n_updates"] == 3 and np.isfinite(m["loss"])
    L.close()


# ================================================================================================ CPU
def test_bdq_matrix_covers_every_shape_path():
    cs = CASES
    assert {1, 8} <= {c.D for c in cs}
    assert {2, 33, 63, 64} <= {c.n for c in cs}
    assert {c.NBS - c.n for c in cs} == {0, 1, 2, 3}
    for width in ("T0", "T1", "HB"):
        ws = {getattr(c, width) for c in cs}
        assert 4 in ws and any(w < 16 for w in ws), width                       # inside one K-step
        assert any(w % 64 == 4 and w > 64 for w in ws), width                   # one 4-step past a tile
        assert any(w % 64 == 0 for w in ws), width
        assert all(w % 4 == 0 and w >= 4 for w in ws), width
    assert {c.obs % 4 for c in cs} == {0, 1, 2, 3} and 1 in {c.obs for c in cs}
    assert {(c.obs + c.D) % 8 for c in cs} >= {0, 1}                             # XS exact, and one past
    assert any(c.B % 64 == 1 for c in cs) and any(c.B % 64 == 63 for c in cs)
    assert set(range(1, 16)) <= {c.B % 16 for c in cs}
    assert 1 in {c.B for c in cs}
    assert any(c.per and c.B == 1024 for c in cs)
    assert {c.rescale for c in cs} == {False, True}
    assert any(c.gamma == 1.0 for c in cs) and any(c.all_done for c in cs)
    assert {c.per for c in cs} == {False, True}
    assert len({(dataclasses.astuple(c.cfg), c.B) for c in cs}) == len(cs), "case_for() tells the cases apart by (cfg, B)"
    assert len({c.name for c in cs}) == len(cs)
    traj = [CASE_BY_NAME[n] for n in TRAJ_CASES]
    assert sum(c.per for c in traj) * 2 == len(traj)


def test_bdq_explicit_batches_kinks_and_ties():
    """The explicit step's first batch at every case: no double-Q choice fp32 cannot decide; the ReLU inputs within fp32
    rounding of zero are counted, and other_sides() really puts each of them on its other side."""
    total = 0
    for c in CASES:
        params = make_params(c)
        bt = make_batch(c, c.B, c.seed + 3)
        kinks, ties = relu_kinks(params, bt["obs"], c.cfg), near_ties(params, bt["next_obs"], c.cfg)
        print(f"{c.name}: {len(kinks)} ReLU kinks, {len(ties)} near-tie rows")
        assert not ties, (c.name, ties[:3])
        for (bname, unit, z), moved in zip(kinks, other_sides(params, kinks)):
            after = [f for f in relu_kinks(moved, bt["obs"], c.cfg) if f[:2] == (bname, unit)]
            assert any(np.sign(f[2]) == -np.sign(z) for f in after), (c.name, bname, z, after)
        total += len(kinks)
    assert total > 0, "no case exercises the kink rule"


def test_bdq_all_done_batches():
    for c in CASES:
        if c.all_done:
            assert make_batch(c, c.B, c.seed + 3)["done"].min() == 1.0


def _bdq_cfg(**kw):
    f = dict(obs_dim=100, n_branches=3, n_bins=8, trunk0=64, trunk1=64, branch_hidden=32, batch=64, buffer_capacity=256, gamma=0.99,
             target_update_freq=100, trunk_grad_rescale=1, seed=0, device=0, rank=0, nranks=1, nccl_id=None, nccl_lib=None,
             prioritized_replay=0, per_alpha=0.6, per_eps=1e-6)
    f.update(kw)
    return _lib.BdqCfg(*f.values())


@pytest.mark.parametrize("kw,msg", [
    (dict(n_branches=0), "n_branches in [1,8]"), (dict(n_branches=9), "n_branches in [1,8]"),
    (dict(n_bins=1), "n_bins in [2,64]"), (dict(n_bins=65), "n_bins in [2,64]"),
    (dict(trunk0=0), "positive multiples of 4"), (dict(trunk1=6), "positive multiples of 4"),
    (dict(branch_hidden=-4), "positive multiples of 4"),
    (dict(obs_dim=0), "obs_dim, batch, buffer_capacity must be positive"),
    (dict(prioritized_replay=1, batch=1025), "batch <= 1024"),
], ids=["d0", "d9", "n1", "n65", "t0_0", "t1_6", "hb_m4", "obs0", "per_b1025"])
def test_bdq_create_refusals(kw, msg):
    """b2g_bdq_create validates its configuration before it looks for a device: B2G_EINVAL (-1) on any machine."""
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.b2g_bdq_create(C.byref(_bdq_cfg(**kw)), C.byref(h)) == -1
    assert not h.value
    assert msg in lib.b2g_last_error().decode()


def test_bdq_unequal_hidden_widths_not_implemented():
    with pytest.raises(NotImplementedError, match="branch and state-value hidden widths must match"):
        b200grasp.BDQLearner(100, 3, 8, ((64, 64), (32,), (64,)), batch_size=8, buffer_size=16)


def test_philox_known_answers():
    """Random123 kat_vectors for Philox4x32-10: the restatement (numpy) and a pure-Python one of the device round."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]

    def pure(c, k):                 # csrc/common.cuh philox_round, word for word
        c, k = list(c), list(k)
        for _ in range(10):
            p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
            c = [(p1 >> 32) ^ c[1] ^ k[0], p1 & 0xFFFFFFFF, (p0 >> 32) ^ c[3] ^ k[1], p0 & 0xFFFFFFFF]
            k = [(k[0] + 0x9E3779B9) & 0xFFFFFFFF, (k[1] + 0xBB67AE85) & 0xFFFFFFFF]
        return tuple(c)
    for c, k, want in kat:
        assert pure(c, k) == want
        assert tuple(int(x) for x in PX.philox4x32_10(*c, *k)) == want


def test_philox_stream_layout():
    """Slots: lane b & 3 of block b >> 2, scaled by (v * size) >> 32; the keys of the training steps and of act()."""
    key = PX.train_seed(7, rank=1)
    assert key == (7 + 0x9E3779B97F4A7C15) & (2 ** 64 - 1)
    assert PX.act_seed(7) == 7 ^ 0xA5A5A5A5DEADBEEF
    step, B, size = (1 << 32) + 5, 11, 1000
    s = PX.slots(key, step, B, size)
    for b in range(B):
        r = PX.philox4x32_10(step & 0xFFFFFFFF, step >> 32, b >> 2, 0, key & 0xFFFFFFFF, key >> 32)
        assert s[b] == (int(r[b & 3]) * size) >> 32
    assert np.array_equal(PX.slots(key, step, B, size, ring_base=995, ring_cap=1000), (995 + s) % 1000)
    assert PX.slots(key, step, 4096, size).max() < size


def test_philox_noise_is_standard_normal():
    """2^20 restated Box-Muller draws: mean and variance of N(0, 1) within 5 sigma, a Kolmogorov-Smirnov test against the
    normal, and no correlation between the cos and sin lanes of a pair or between neighbouring samples."""
    from scipy import stats
    n = 1 << 20
    z = np.concatenate([PX.noise(PX.train_seed(3), step, n // 4) for step in range(4)])
    se = 1 / np.sqrt(n)
    assert abs(z.mean()) <= 5 * se, z.mean()
    assert abs(z.var() - 1) <= 5 * np.sqrt(2) * se, z.var()
    ks = stats.kstest(z, "norm")
    assert ks.pvalue > 1e-4, ks
    pairs = z.reshape(-1, 2)                              # (r0 cos, r0 sin) of one angle
    for a, b in ((pairs[:, 0], pairs[:, 1]), (z[:-1], z[1:])):
        rho = np.corrcoef(a, b)[0, 1]
        assert abs(rho) <= 5 / np.sqrt(len(a)), rho
    # the sin lanes take both signs equally often (a one-sided angle would make them all non-negative)
    assert abs((pairs[:, 1] > 0).mean() - 0.5) <= 5 * 0.5 / np.sqrt(len(pairs))
    print(f"noise: mean {z.mean():.2e} var {z.var():.5f} KS p {ks.pvalue:.3f}")


# ================================================================================================ GPU
def _check_acts(L, params, obs, cfg, label):
    """act() on obs against greedy_action, excluding rows with a near tie; -> device actions"""
    got = L.act(obs)
    assert got.shape == (len(obs), cfg.n_branches)
    ref, _ = Q.greedy_action(params, obs, cfg)
    skip = np.zeros(len(obs), bool)
    for b, _, _ in near_ties(params, obs, cfg):
        skip[b] = True
    bad = np.nonzero((got != ref).any(1) & ~skip)[0]
    print(f"{label} act({len(obs)}): {skip.sum()} near-tie rows excluded, {len(bad)} rows differ")
    assert len(bad) == 0, (label, bad[:5], got[bad[:5]], ref[bad[:5]])
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_bdq_act_vs_oracle(case):
    """act() on B - 1 and 2B + 3 rows (chunks of B, a short last one) against the oracle's greedy actions, before and after
    an update; every row of the shorter call equals the same row of the long call."""
    cfg, B = case.cfg, case.B
    params = make_params(case)
    L = make_learner_bdq(case)
    L.load_parameters(params)
    obs = np.random.default_rng(case.seed + 7).normal(0.4, 0.3, (2 * B + 3, cfg.obs_dim)).astype(np.float32)
    for stage in ("fresh", "updated"):
        p = L.get_parameters()
        full = _check_acts(L, p, obs, cfg, f"{case.name} {stage}")
        if B > 1:
            short = _check_acts(L, p, obs[:B - 1], cfg, f"{case.name} {stage}")
            assert np.array_equal(short, full[:B - 1])
        one = L.act(obs[B:B + 1])
        assert np.array_equal(one[0], full[B])
        bt = make_batch(case, B, case.seed + 3)
        L.step_explicit(bt["obs"], bt["act_idx"].astype(np.float32), bt["rew"], bt["next_obs"], bt["done"], lr=LR)
    L.close()


@pytest.mark.gpu
@pytest.mark.parametrize("j,k", [(1, 5), (0, 7), (6, 7)])
def test_bdq_argmax_exact_ties(j, k):
    """Two bit-equal online output columns j < k of branch 1 hold the maximum on every row; the target net values them
    differently.  act() returns j, and the explicit step's td matches the oracle, which also takes the first maximal bin."""
    case = Case("ties", 20, 3, 8, 64, 64, 32, 64, seed=31)
    cfg = case.cfg
    params = make_params(case)
    rng = np.random.default_rng(5)
    for net in ("bdq/model", "bdq/target_q_func/model"):
        w, b = params[f"{net}/action_value/fully_connected_3/weights"], params[f"{net}/action_value/fully_connected_3/biases"]
        w[:, k] = w[:, j]
        b[k] = b[j] = np.float32(3.0)
        if net != "bdq/model":
            w[:, k] += rng.normal(0, 0.3, w.shape[0]).astype(np.float32)
            b[k] = np.float32(-1.0)
    bt = make_batch(case, case.B, 33)
    A, _ = online_advantages(params, bt["next_obs"], cfg)
    assert (A[:, 1, j] == A[:, 1, k]).all() and (A[:, 1].argmax(1) == j).all()
    L = make_learner_bdq(case)
    L.load_parameters(params)
    a = L.act(bt["next_obs"])
    assert (a[:, 1] == j).all(), np.unique(a[:, 1])
    out = L.step_explicit(bt["obs"], bt["act_idx"].astype(np.float32), bt["rew"], bt["next_obs"], bt["done"], lr=LR,
                          apply_update=False)
    r, _, _, _ = Q.bdq_step(params, {"t": 0, "m": {}, "v": {}}, bt, LR, cfg, torch.float64)
    assert (r["a_star"][:, 1] == j).all()
    e = rel_err(out["td"], r["td"])
    r_k, _, _, _ = Q.bdq_step(params, {"t": 0, "m": {}, "v": {}}, bt, LR, cfg, torch.float64,
                              a_star=np.where(np.arange(cfg.n_branches) == 1, k, r["a_star"]))
    print(f"ties ({j}, {k}): td rel err {e:.2e} (taking bin {k} instead: {rel_err(out['td'], r_k['td']):.2e})")
    assert e <= TOL and rel_err(r_k["td"], r["td"]) > 100 * TOL
    L.close()


class PerMirror:
    """numpy mirror of the device sum / min trees (bdq.cu per_write_kernel / per_sample_kernel), driven by what the device
    reports: new transitions enter with the running maximum priority, sampled ones take sum_d |td_d| + eps."""

    def __init__(self, cap, alpha):
        self.cap, self.C = cap, 1
        while self.C < cap:
            self.C <<= 1
        self.raw = np.zeros(cap, np.float32)
        self.used = np.zeros(cap, bool)
        self.alpha = float(np.float32(alpha))
        self.max_prio = np.float32(1.0)
        self.pos = self.size = 0

    def add(self, n):
        s = (self.pos + np.arange(n)) % self.cap
        self.raw[s], self.used[s] = self.max_prio, True
        self.pos, self.size = (self.pos + n) % self.cap, min(self.cap, self.size + n)

    def update(self, slots, prio):
        for s in np.unique(slots):                    # a slot drawn twice carries the same |td| (same row, same net)
            assert np.unique(prio[slots == s]).size == 1, (s, prio[slots == s])
        self.raw[slots] = prio
        self.max_prio = max(self.max_prio, np.float32(prio.max()))

    def trees(self):
        tsum, tmin = np.zeros(2 * self.C), np.full(2 * self.C, np.inf)
        leaf = np.power(self.raw.astype(np.float64), self.alpha)
        tsum[self.C:self.C + self.cap][self.used] = leaf[self.used]
        tmin[self.C:self.C + self.cap][self.used] = leaf[self.used]
        lo = self.C
        while lo > 1:
            lo //= 2
            tsum[lo:2 * lo] = tsum[2 * lo:4 * lo:2] + tsum[2 * lo + 1:4 * lo:2]
            tmin[lo:2 * lo] = np.fmin(tmin[2 * lo:4 * lo:2], tmin[2 * lo + 1:4 * lo:2])
        return tsum, tmin

    def sample(self, key, step, B, beta):
        """-> slots, IS weights, and a mask of the draws within 1e-12 of the total of a prefix-sum boundary"""
        tsum, tmin = self.trees()
        total = tsum[1]
        mass = PX.per_masses(key, step, B, total)
        node = np.ones(B, np.int64)
        edge = np.zeros(B, bool)
        while node[0] < self.C:
            left = tsum[2 * node]
            edge |= np.abs(left - mass) <= 1e-12 * total
            go = left > mass
            mass = np.where(go, mass, mass - left)
            node = np.where(go, 2 * node, 2 * node + 1)
        idx = np.minimum(node - self.C, self.size - 1)
        beta = float(np.float32(beta))
        max_w = (tmin[1] / total * self.size) ** -beta
        w = (tsum[self.C + idx] / total * self.size) ** -beta / max_w
        return idx, w, edge


def _run_trajectory(case, tr, K, freq=3, adds=None, cap=None, beta=0.7, seed=5):
    """K sampled steps (one step(1) call each) after adding all of `tr`, or the plan `adds`: a list of (n_add, n_steps) into a
    ring of `cap` slots.  Checks every step's slots against the restated streams and the PER mirror, and the target copies.
    -> rows of (metrics, slots, weights, priorities (PER) or None, parameters before the step, ring contents), final parameters."""
    cap = cap or len(tr["rew"])
    L = make_learner_bdq(case, buffer_size=cap, freq=freq, seed=seed, prioritized_replay_alpha=0.6)
    L.load_parameters(make_params(case))
    if case.per:
        L.set_per_beta(beta)
    key = PX.train_seed(seed)
    mirror = PerMirror(cap, 0.6) if case.per else None
    ring = {k: np.zeros((cap,) + v.shape[1:], v.dtype) for k, v in tr.items()}
    plan = adds or [(len(tr["rew"]), K)]
    rows, added, n_sampled, n_edge = [], 0, 0, 0
    for n_add, n_steps in plan:
        sl = slice(added, added + n_add)
        L.replay_add(tr["obs"][sl], tr["act_idx"][sl].astype(np.float32), tr["rew"][sl], tr["next_obs"][sl], tr["done"][sl])
        for i in range(n_add):
            for k in ring:
                ring[k][(added + i) % cap] = tr[k][added + i]
        added += n_add
        if mirror:
            mirror.add(n_add)
        for _ in range(n_steps):
            pre = L.get_parameters()
            m = L.step(1, lr=LR)
            slots, w, prio = L.last_per()
            size = min(added, cap)
            assert slots.min() >= 0 and slots.max() < size
            if mirror:
                want, w_ref, edge = mirror.sample(key, n_sampled + 1, case.B, beta)
                n_edge += int(edge.sum())
                assert np.array_equal(slots[~edge], want[~edge]), (n_sampled, np.nonzero(slots != want)[0][:5])
                assert np.abs(w - w_ref).max() <= 2e-5 * max(1.0, w_ref.max())
                mirror.update(slots, prio)
            else:
                assert np.array_equal(slots, PX.slots(key, n_sampled, case.B, size)), n_sampled
                w, prio = np.ones(case.B, np.float32), None        # priorities are written by PER steps only
            n_sampled += 1
            post = L.get_parameters()
            for n in post:
                if n.startswith("bdq/model/"):
                    t = n.replace("bdq/model", "bdq/target_q_func/model")
                    if m["n_updates"] % freq == 0:
                        assert np.array_equal(post[t], post[n]), (m["n_updates"], t)
                    else:
                        assert np.array_equal(post[t], pre[t]), (m["n_updates"], t)
            rows.append((m, slots, w, prio, pre, {k: v.copy() for k, v in ring.items()}))
    if mirror:
        print(f"{case.name}: {n_edge} PER draws within 1e-12 of a prefix-sum boundary (exempt from the exact slot check)")
    p = L.get_parameters()
    L.close()
    return rows, p


def _traj_batch(ring, slots, w):
    return dict(obs=ring["obs"][slots], next_obs=ring["next_obs"][slots], act_idx=ring["act_idx"][slots], rew=ring["rew"][slots],
                done=ring["done"][slots], weights=w)


def _hold_trajectory(case, rows, p_gpu, freq=3):
    """Every step from its pre-step parameters, then the final parameters against the oracle's own trajectory (the bars of
    test_graph_path_ten_steps_vs_oracle_bf16x3_b256)."""
    cfg = case.cfg
    worst = 0.0
    for it, (m, slots, w, prio, pre, ring) in enumerate(rows):
        got = dict(loss=m["loss"], mean_q=m["mean_q"], grad_norm=m["grad_norm"], priorities=prio)
        _, r = hold_step(pre, {"t": 0, "m": {}, "v": {}}, _traj_batch(ring, slots, w), cfg, got, label=f"{case.name} sampled step {it}")
        worst = max(worst, r)
        assert m["n_updates"] == it + 1
    p, opt = {n: np.asarray(a, np.float64) for n, a in rows[0][4].items()}, {"t": 0, "m": {}, "v": {}}
    for it, (m, slots, w, prio, pre, ring) in enumerate(rows):
        _, _, p, opt = Q.bdq_step(p, opt, _traj_batch(ring, slots, w), LR, cfg, torch.float64)
        if (it + 1) % freq == 0:
            Q.hard_target_update(p)
    K = len(rows)
    for n in p_gpu:
        if n == "bdq/eps":
            continue
        d = np.abs(p_gpu[n].astype(np.float64) - p[n]).reshape(-1)
        assert d.max() <= 2 * K * LR + 1e-6 * np.abs(p[n]).max(), (n, d.max())
        if d.size >= 1000:
            assert np.quantile(d, 0.99) <= 0.05 * K * LR, (n, np.quantile(d, 0.99) / (K * LR))
    print(f"{case.name}: {K} sampled steps, worst err/bar {worst:.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", TRAJ_CASES)
def test_bdq_sampled_trajectory_vs_oracle(name):
    """Six step(1) calls with a hard copy every 3 updates: slots (uniform: the restated stream 0; PER: the mirror of the trees
    on stream 2), IS weights, every step's loss / mean_q / grad_norm / priorities from its pre-step parameters, the target
    copies bit for bit, and the final parameters against the oracle's own trajectory."""
    case = CASE_BY_NAME[name]
    tr = make_batch(case, 3 * case.B + 50, case.seed + 40)
    rows, p = _run_trajectory(case, tr, 6)
    _hold_trajectory(case, rows, p)


@pytest.mark.gpu
def test_bdq_per_ring_wraps_inside_the_tree():
    """PER with capacity 300 (a 512-leaf tree) and 450 transitions added in four calls with steps in between: the ring wraps,
    overwritten slots re-enter with the running maximum priority."""
    case = Case("per_wrap", 100, 3, 33, 64, 64, 32, 130, per=True, seed=41)
    tr = make_batch(case, 450, 42)
    rows, p = _run_trajectory(case, tr, None, adds=[(200, 2), (150, 2), (60, 1), (40, 2)], cap=300)
    assert max(int(s.max()) for _, s, *_ in rows[2:]) > 150 and min(int(s.min()) for _, s, *_ in rows[2:]) < 50
    _hold_trajectory(case, rows, p)


@pytest.mark.gpu
def test_bdq_target_copies_count_explicit_and_sampled_updates():
    """counters[3] counts every applied update, explicit or sampled; an explicit step with apply_update=0 is no update."""
    case = CASE_BY_NAME["d8_n64_b63"]
    tr = make_batch(case, 200, 50)
    L = make_learner_bdq(case, buffer_size=200, freq=3)
    L.load_parameters(make_params(case))
    L.replay_add(tr["obs"], tr["act_idx"].astype(np.float32), tr["rew"], tr["next_obs"], tr["done"])
    bt = make_batch(case, case.B, 51)
    seq = ["explicit", "sampled", "noapply", "sampled", "explicit", "sampled", "sampled"]
    n_up = 0
    for what in seq:
        pre = L.get_parameters()
        if what == "sampled":
            m = L.step(1, lr=LR)
        else:
            m = L.step_explicit(bt["obs"], bt["act_idx"].astype(np.float32), bt["rew"], bt["next_obs"], bt["done"], lr=LR,
                                apply_update=what == "explicit")
        n_up += what != "noapply"
        assert m["n_updates"] == n_up
        post = L.get_parameters()
        copied = what != "noapply" and n_up % 3 == 0
        for n in post:
            if n.startswith("bdq/model/"):
                t = n.replace("bdq/model", "bdq/target_q_func/model")
                assert np.array_equal(post[t], post[n] if copied else pre[t]), (what, n_up, t)
                if what == "noapply":
                    assert np.array_equal(post[n], pre[n])
    L.close()


@pytest.mark.gpu
def test_bdq_graph_and_eager_steps_agree(monkeypatch):
    """The same six sampled steps through the captured graph and launched one by one (B2G_NO_GRAPH=1): the same slots, and the
    same IS weights and outputs to fp32 summation-order noise (the priorities, and so the trees behind the weights, inherit
    it from the td errors)."""
    case = CASE_BY_NAME["per_d5_n33_b130"]
    tr = make_batch(case, 3 * case.B + 50, case.seed + 40)
    base, p0 = _run_trajectory(case, tr, 6)
    monkeypatch.setenv("B2G_NO_GRAPH", "1")
    eager, p1 = _run_trajectory(case, tr, 6)
    for it, (r0, r1) in enumerate(zip(base, eager)):
        assert np.array_equal(r0[1], r1[1]), it
        assert rel_err(r1[2], r0[2]) <= 2e-6 * (1 + 10 * it), (it, rel_err(r1[2], r0[2]))
        assert rel_err(r1[3], r0[3]) <= 2e-6 * (1 + 10 * it), (it, rel_err(r1[3], r0[3]))
        for k in ("loss", "mean_q", "grad_norm"):
            assert abs(r1[0][k] - r0[0][k]) <= 2e-5 * abs(r0[0][k]) * (1 + it) + 1e-9, (it, k, r0[0][k], r1[0][k])
    for n in p0:      # an entry with a near-zero gradient takes an Adam step of either sign: the trajectory bars
        d = np.abs(p1[n].astype(np.float64) - p0[n]).reshape(-1)
        assert d.max() <= 2 * 6 * LR and (d.size < 1000 or np.quantile(d, 0.99) <= 0.05 * 6 * LR), n


def _set_norm(L, mean, var, ret_var, clip_obs, clip_rew, eps, norm_obs, norm_reward):
    dp = C.POINTER(C.c_double)
    m = np.ascontiguousarray(mean, np.float64)
    v = np.ascontiguousarray(var, np.float64)
    _lib.check(L.lib.b2g_bdq_set_norm_stats(L.h, m.ctypes.data_as(dp), v.ctypes.data_as(dp), float(ret_var), float(clip_obs),
                                            float(clip_rew), float(eps), int(norm_obs), int(norm_reward)))


@pytest.mark.gpu
@pytest.mark.parametrize("obs_dim,norm_obs,norm_reward", [(13, 1, 1), (24, 1, 0), (24, 0, 1), (13, 0, 0), (24, 1, 1)])
def test_bdq_normalisation_in_the_gather(obs_dim, norm_obs, norm_reward):
    """b2g_bdq_set_norm_stats: statistics that push observations past +-clip_obs (and zero-variance features) and rewards past
    +-clip_reward.  An explicit step and three sampled steps against the oracle on sac_ref.normalize_obs / normalize_reward
    inputs; the action columns of the gathered row stay raw bin indices (a normalised index would change every td)."""
    case = Case(f"norm_{obs_dim}", obs_dim, 3, 8, 64, 64, 32, 37, seed=61)
    cfg = case.cfg
    clip_obs, clip_rew, eps, ret_var = 5.0, 2.0, 1e-8, 1.5 ** 2
    rng = np.random.default_rng(62)
    mean = rng.normal(0.4, 0.1, obs_dim)
    var = rng.uniform(0.01, 0.05, obs_dim)
    mean[0], var[0] = -2.0, 0.01          # -> +clip
    mean[1], var[1] = 3.0, 0.01           # -> -clip
    var[2] = 0.0                          # zero variance: 1/sqrt(eps), clipped both ways
    tr = make_batch(case, 300, 63)
    tr["rew"] = (tr["rew"] * np.where(rng.random(300) < 0.5, -1, 1) * 3).astype(np.float32)   # |r| / 1.5 up to 6: past clip

    def norm(bt):
        out = dict(bt)
        if norm_obs:
            out["obs"] = R.normalize_obs(bt["obs"], mean, var, clip=clip_obs, eps=eps)
            out["next_obs"] = R.normalize_obs(bt["next_obs"], mean, var, clip=clip_obs, eps=eps)
        if norm_reward:
            out["rew"] = R.normalize_reward(bt["rew"], ret_var, clip=clip_rew, eps=eps)
        return out
    n = norm(tr)
    if norm_obs:
        assert (n["obs"][:, 0] == clip_obs).all() and (n["obs"][:, 1] == -clip_obs).all()
        assert (n["obs"][:, 2] == clip_obs).any() and (n["obs"][:, 2] == -clip_obs).any() and (np.abs(n["obs"][:, 3:]) < clip_obs).any()
    if norm_reward:
        assert (n["rew"] == clip_rew).any() and (n["rew"] == -clip_rew).any() and (np.abs(n["rew"]) < clip_rew).any()
    params = make_params(case)
    L = make_learner_bdq(case, buffer_size=300, freq=1000, seed=3)
    L.load_parameters(params)
    _set_norm(L, mean, var, ret_var, clip_obs, clip_rew, eps, norm_obs, norm_reward)
    bt = {k: v[:case.B] for k, v in tr.items()}
    out = L.step_explicit(bt["obs"], bt["act_idx"].astype(np.float32), bt["rew"], bt["next_obs"], bt["done"], lr=LR)
    hold_step(params, {"t": 0, "m": {}, "v": {}}, norm(bt), cfg, out, L.get_gradients(), label=f"{case.name} {norm_obs}{norm_reward} explicit")
    L.replay_add(tr["obs"], tr["act_idx"].astype(np.float32), tr["rew"], tr["next_obs"], tr["done"])
    key = PX.train_seed(3)
    for it in range(3):
        pre = L.get_parameters()
        m = L.step(1, lr=LR)
        slots, _, _ = L.last_per()
        assert np.array_equal(slots, PX.slots(key, it, case.B, 300))
        got = dict(loss=m["loss"], mean_q=m["mean_q"], grad_norm=m["grad_norm"])
        sb = norm({k: v[slots] for k, v in tr.items()})
        hold_step(pre, {"t": 0, "m": {}, "v": {}}, sb, cfg, got, L.get_gradients(), label=f"{case.name} {norm_obs}{norm_reward} sampled {it}")
    L.close()


# ------------------------------------------------------------------------------------------------ the SAC streams on the device
def _assert_noise(eps, ref, label):
    """Within 8 fp32 ulps of the restatement (the device evaluates it with logf, sqrtf and sincospif)."""
    ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    r = np.abs(eps.astype(np.float64) - ref) / np.maximum(ulp, 2.0 ** -149)
    print(f"{label}: noise within {r.max():.1f} ulps of the restated stream")
    assert r.max() <= 8, (label, r.max())


@pytest.mark.gpu
@pytest.mark.parametrize("key,precision", [("sac_depth", 1), ("sac_encoder", 0)], ids=["engine_v2", "round1_gather"])
def test_sac_graph_path_slots_and_noise_are_the_restated_streams(key, precision):
    """Engine v2's gather2 and the round-1 gather draw the replay slots in-kernel (stream 0, philox_slot); prep_kernel draws the
    policy noise (stream 1).  Over four graph-path steps both equal the restatement at counters[4] = step index."""
    from b200grasp import synth
    cfg, params, vn = load_case(key)
    B, NS, seed = 37, 300, 77
    tr = synth.make_transitions(NS, vn["obs_mean"], vn["obs_var"], seed=5)
    L = make_learner(cfg, vn, B, params, buffer_size=512, precision=precision, seed=seed)
    L.replay_add(tr["obs"], tr["act"], tr["rew"], tr["next_obs"], tr["done"])
    k = PX.train_seed(seed)
    for step in range(4):
        L.step(1, lr=3e-4)
        lb = L.last_batch()
        assert np.array_equal(lb["indices"], PX.slots(k, step, B, NS, ring_base=0, ring_cap=512)), step
        _assert_noise(lb["eps"], PX.noise(k, step, B * cfg.n_act).reshape(B, cfg.n_act), f"{key} step {step}")
    L.close()


@pytest.mark.gpu
def test_sac_act_noise_is_the_restated_stream():
    """act(deterministic=False) draws its noise from the key seed ^ 0xA5A5A5A5DEADBEEF at the shared step counter; the
    actions equal the oracle's policy on that restated noise."""
    cfg, params, vn = load_case("sac_depth")
    from tests.util import make_batch as sac_batch
    B, seed = 16, 123
    raw, norm, _ = sac_batch(vn, B)
    L = make_learner(cfg, vn, B, params, buffer_size=64, precision=1, seed=seed)
    for step in range(2):
        a = L.act(raw["obs"], deterministic=False)
        ref_eps = PX.noise(PX.act_seed(seed), step, B * cfg.n_act).reshape(B, cfg.n_act)
        _assert_noise(L.last_batch()["eps"], ref_eps, f"act call {step}")
        want = R.policy_act(params, norm["obs"], cfg, deterministic=False, eps_noise=ref_eps.astype(np.float32))
        print(f"act call {step}: rel err {rel_err(a, want):.2e}")
        assert rel_err(a, want) <= 1e-4
    L.close()
