"""The DQN learner (csrc/dqn.cu, b200grasp.deepq.DQN) against the float64 oracle (oracle/dqn_ref.py) and the restated streams.

  * explicit steps at the shipped shape and at the limits b2g_dqn_create accepts (n_actions 2..64 with 0..3 pad columns, widths
    4 and 512, obs_dim 1 and 7, batch 1..1024, gamma 1 and 0.99, an all-done batch, a batch whose clip scales some tensors);
  * six sampled graph steps, uniform and prioritised, slot for slot against oracle/philox_ref.py and the mirrored trees;
  * the shipped DQN_simple_4pads.zip: greedy and softmax actions, Q rows;
  * DQN.learn's schedule (updates, target copies at num_timesteps % freq == 0), save / load, training state and the CLI.
Tolerances and the ReLU-kink / argmax-tie rules are those of tests/test_gpu_bdq_configs.py.
"""
import dataclasses
import os
import shutil

import numpy as np
import pytest
import torch
import yaml

import b200grasp
from b200grasp import deepq, train_cli
from b200grasp.spaces import Box, Discrete
from oracle import dqn_ref as DR
from oracle import philox_ref as PX
from tests.test_gpu_bdq_configs import PerMirror, check_adam_update
from tests.util import rel_err

TOL, GTOL, LR, U32 = 1e-4, 1e-3, 1e-3, 2.0 ** -24
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ZIP = os.path.join(GOLD, "DQN_simple_4pads.zip")


@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    obs: int
    n: int
    H0: int
    H1: int
    B: int
    gamma: float = 0.99
    per: bool = False
    all_done: bool = False
    obs_scale: float = 1.0
    seed: int = 1

    @property
    def cfg(self):
        return DR.DQNConfig(self.obs, self.n, (self.H0, self.H1), self.gamma)


CASES = [
    Case("shipped_b32_per", 100, 12, 64, 64, 32, gamma=1.0, per=True, seed=11),
    Case("n2_w4_512_obs1_b1", 1, 2, 4, 512, 1, seed=12),
    Case("n33_w512_4_obs7_b33", 7, 33, 512, 4, 33, seed=13),
    Case("n63_obs7_b130", 7, 63, 68, 132, 130, seed=14),
    Case("n64_b1024_per", 100, 64, 128, 64, 1024, gamma=1.0, per=True, seed=15),
    Case("alldone_n12_b5", 30, 12, 64, 64, 5, all_done=True, seed=16),
    Case("clip_n5_b9", 7, 5, 8, 12, 9, obs_scale=60.0, seed=17),
]


def make_params(case):
    """Xavier weights, biases N(0, 0.1), a target net 0.02 away from the online one"""
    p = DR.init_params(case.cfg, seed=case.seed)
    rng = np.random.default_rng(case.seed + 1000)
    for n in p:
        if n.endswith("biases"):
            p[n] = (rng.normal(size=p[n].shape) * 0.1).astype(np.float32)
        elif n.startswith(DR.TARGET) and n.endswith("weights"):
            p[n] = (p[n] + rng.normal(size=p[n].shape).astype(np.float32) * 0.02).astype(np.float32)
    return p


def make_batch(case, B, seed):
    rng = np.random.default_rng(seed)
    bt = dict(obs=(rng.normal(0.4, 0.2, (B, case.obs)) * case.obs_scale).astype(np.float32),
              next_obs=rng.normal(0.4, 0.2, (B, case.obs)).astype(np.float32), act=rng.integers(0, case.n, B),
              rew=(rng.choice([0.0, 1.0], B) * rng.uniform(1.5, 3.0, B)).astype(np.float32),     # |td| on both sides of 1
              done=(rng.random(B) < 0.2).astype(np.float32))
    if case.all_done:
        bt["done"][:] = 1.0
    return bt


def make_learner(case, buffer_size=256, seed=0):
    return deepq.DQNLearner(case.obs, case.n, (case.H0, case.H1), case.B, buffer_size, case.gamma, seed=seed,
                            prioritized_replay=case.per, prioritized_replay_alpha=0.6, prioritized_replay_eps=1e-6)


def _t64(a):
    return torch.tensor(np.asarray(a, np.float64))


def relu_kinks(params, obs):
    """ReLU inputs of the online net at s whose sign fp32 cannot decide (tests/test_gpu_bdq_configs.py::relu_kinks)"""
    p = {n: _t64(a) for n, a in params.items() if n.startswith(DR.ONLINE + "/")}
    found = []
    for tower in ("action_value", "state_value"):
        h = _t64(obs)
        for k in range(2):
            name = f"{DR.ONLINE}/{tower}/{DR._fc(k)}"
            w, b = p[name + "/weights"], p[name + "/biases"]
            z, mag = h @ w + b, h.abs() @ w.abs() + b.abs()
            for r, c in (z.abs() <= 4 * np.sqrt(w.shape[0]) * U32 * mag).nonzero().tolist():
                found.append((name + "/biases", c, float(z[r, c])))
            h = torch.relu(z)
    return sorted(found, key=lambda f: abs(f[2]))


def other_sides(params, kinks, max_n=6):
    kinks = kinks[:max_n]

    def moved(sel):
        q = {n: np.array(a, np.float32, copy=True) for n, a in params.items()}
        for bname, c, z in sel:
            q[bname].reshape(-1)[c] -= np.float32(2 * z)
        return q
    return [moved([k]) for k in kinks] + ([moved(kinks)] if len(kinks) > 1 else [])


def near_ties(params, obs):
    """rows whose top two online Q values at s' are within fp32 resolution -> [(row, [candidates])]"""
    _, q = DR.greedy_action(params, obs)
    bar = 64 * U32 * (1.0 + np.abs(q).max(1, keepdims=True))
    top = q.max(1, keepdims=True)
    out = []
    for b in np.nonzero(((top - q) <= bar).sum(1) > 1)[0]:
        out.append((int(b), [int(k) for k in np.nonzero(top[b] - q[b] <= bar[b])[0]]))
    return out


def tie_variants(params, next_obs, ties):
    if not ties:
        return []
    base = DR.greedy_action(params, next_obs)[0]
    out = []
    for b, cand in ties:
        a = base.copy()
        a[b] = next(k for k in cand if k != base[b])
        out.append(a)
    return out


def hold_step(pre, opt, batch, cfg, got, grads=None, label=""):
    """Outputs (loss, mean_q, mean_abs_td, grad_norm, td or priorities) and clipped per-tensor gradients of one step against the
    float64 oracle: bar 1e-4 / 1e-3 or 3x the fp32 oracle's own distance; ReLU kinks and double-Q near-ties on either side."""
    r64, g64, p64, o64 = DR.dqn_step(pre, opt, batch, LR, cfg, torch.float64)
    r32, g32, _, _ = DR.dqn_step(pre, opt, batch, LR, cfg, torch.float32)
    scal = ("loss", "mean_q", "mean_abs_td", "grad_norm")
    vecs = [k for k in ("td", "priorities") if got.get(k) is not None]

    def errs(r, g):
        e = {k: abs(got[k] - r[k]) / (abs(r[k]) + 1e-30) for k in scal}
        e.update({k: rel_err(got[k], r[k]) for k in vecs})
        if grads is not None:
            e.update({n: rel_err(grads[n], g[n]) for n in g})
        return e

    bars = {k: max(TOL, 3 * abs(r32[k] - r64[k]) / (abs(r64[k]) + 1e-30)) for k in scal}
    bars.update({k: max(TOL, 3 * rel_err(r32[k], r64[k])) for k in vecs})
    if grads is not None:
        bars.update({n: max(GTOL, 3 * rel_err(g32[n], g64[n])) for n in g64})
    e = errs(r64, g64)
    kinks, ties = relu_kinks(pre, batch["obs"]), near_ties(pre, batch["next_obs"])
    if any(e[k] > bars[k] for k in e) and (kinks or ties):
        alts = [DR.dqn_step(q, opt, batch, LR, cfg, torch.float64)[:2] for q in other_sides(pre, kinks)]
        alts += [DR.dqn_step(pre, opt, batch, LR, cfg, torch.float64, a_star=a)[:2] for a in tie_variants(pre, batch["next_obs"], ties)]
        for r, g in alts:
            ea = errs(r, g)
            e = {k: min(e[k], ea[k]) for k in e}
    worst = max(e, key=lambda k: e[k] / bars[k])
    print(f"{label}: {len(ties)} near-tie rows, {len(kinks)} ReLU kinks; worst err/bar {e[worst] / bars[worst]:.3f} ({worst})")
    bad = {k: (e[k], bars[k]) for k in e if not e[k] <= bars[k]}
    assert not bad, (label, bad)
    if "n_clipped" in got and all(abs(v - DR.GRAD_CLIP) > 1e-3 * DR.GRAD_CLIP for v in r64["norms"].values()):
        assert got["n_clipped"] == r64["n_clipped"], (label, got["n_clipped"], r64["n_clipped"])
    return r64, g64, p64, o64


# ================================================================================================ explicit steps
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_dqn_explicit_steps_vs_oracle(case):
    """Two explicit steps (the second from the GPU's parameters with the oracle's moments): outputs, every clipped gradient, the
    Adam update element-wise on the GPU's own gradients; the target copy is update_target's alone."""
    cfg, B = case.cfg, case.B
    params = make_params(case)
    L = make_learner(case)
    assert list(L.param_shapes) == [n for n, _ in DR.all_specs(cfg)]
    for n, shp in DR.all_specs(cfg):
        assert L.param_shapes[n] == tuple(shp), n
    L.load_parameters(params)
    back = L.get_parameters()
    for n in params:
        assert np.array_equal(back[n], np.asarray(params[n], np.float32)), n
    tds = []
    bt = make_batch(case, B, case.seed + 3)
    if B == 1:
        bt["rew"][:] = 2.5
    w = np.random.default_rng(case.seed + 4).uniform(0.5, 1.5, B).astype(np.float32) if case.per else None
    out = L.step_explicit(bt["obs"], bt["act"].astype(np.float32), bt["rew"], bt["next_obs"], bt["done"], weights=w, lr=LR)
    assert out["n_updates"] == 1
    g1, p1 = L.get_gradients(), L.get_parameters()
    b1 = dict(bt, weights=w) if w is not None else bt
    r64, _, _, opt64 = hold_step(params, {"t": 0, "m": {}, "v": {}}, b1, cfg, out, g1, label=f"{case.name} step 1")
    tds.append(np.abs(r64["td"]))
    if case.name.startswith("clip"):
        assert 0 < out["n_clipped"] < 12, out["n_clipped"]
    m1, v1 = check_adam_update({n: params[n] for n in g1}, {n: p1[n] for n in g1}, g1, {}, {}, 1, label=f"{case.name} step 1")
    for n in params:
        if n.startswith(DR.TARGET):
            assert np.array_equal(p1[n], params[n]), n
    bt2 = make_batch(case, B, case.seed + 5)
    if B == 1:
        bt2["rew"][:] = 0.0                   # step 1 has |td| > 1 (reward >= 1.5), step 2 |td| < 1
    out2 = L.step_explicit(bt2["obs"], bt2["act"].astype(np.float32), bt2["rew"], bt2["next_obs"], bt2["done"], lr=LR)
    g2, p2 = L.get_gradients(), L.get_parameters()
    r64b, *_ = hold_step(p1, opt64, bt2, cfg, out2, g2, label=f"{case.name} step 2")
    tds.append(np.abs(r64b["td"]))
    check_adam_update({n: p1[n] for n in g2}, {n: p2[n] for n in g2}, g2, m1, v1, 2, label=f"{case.name} step 2")
    at = np.concatenate(tds) if B == 1 else tds[0]
    assert (at < 1).any() and (at > 1).any(), case.name          # both branches of the Huber loss
    L.update_target()
    p3 = L.get_parameters()
    for n in g2:
        assert np.array_equal(p3[n.replace(DR.ONLINE, DR.TARGET)], p3[n]), n
    L.close()


# ================================================================================================ sampled trajectory
@pytest.mark.gpu
@pytest.mark.parametrize("per", [False, True], ids=["uniform", "per"])
def test_dqn_sampled_trajectory_vs_oracle(per):
    """Six step(1) calls (a target copy after the third): slots and IS weights against the restated streams and the mirrored
    trees, every step's loss / priorities from its pre-step parameters, the final parameters against the oracle's trajectory."""
    case = Case("traj", 100, 12, 64, 64, 32 if per else 40, gamma=1.0, per=per, seed=21)
    cfg, seed, beta = case.cfg, 5, 0.7
    tr = make_batch(case, 150, 22)
    cap = 150
    L = make_learner(case, buffer_size=cap, seed=seed)
    L.load_parameters(make_params(case))
    if per:
        L.set_per_beta(beta)
    L.replay_add(tr["obs"], tr["act"].astype(np.float32), tr["rew"], tr["next_obs"], tr["done"])
    key = PX.train_seed(seed)
    mirror = PerMirror(cap, 0.6) if per else None
    if mirror:
        mirror.add(cap)
    rows = []
    for k in range(6):
        pre = L.get_parameters()
        m = L.step(1, lr=LR)
        slots, w, prio = L.last_per()
        if mirror:
            want, w_ref, edge = mirror.sample(key, k + 1, case.B, beta)
            assert np.array_equal(slots[~edge], want[~edge]), k
            assert np.abs(w - w_ref).max() <= 2e-5 * max(1.0, w_ref.max())
            mirror.update(slots, prio)
        else:
            assert np.array_equal(slots, PX.slots(key, k, case.B, cap)), k
            w, prio = np.ones(case.B, np.float32), None
        assert m["n_updates"] == k + 1
        batch = dict(obs=tr["obs"][slots], next_obs=tr["next_obs"][slots], act=tr["act"][slots], rew=tr["rew"][slots],
                     done=tr["done"][slots], weights=w)
        got = dict(loss=m["loss"], mean_q=m["mean_q"], mean_abs_td=m["mean_abs_td"], grad_norm=m["grad_norm"], priorities=prio)
        hold_step(pre, {"t": 0, "m": {}, "v": {}}, batch, cfg, got, label=f"traj {k}")
        rows.append(batch)
        if k == 2:
            L.update_target()
    p_gpu = L.get_parameters()
    L.close()
    p, opt = {n: np.asarray(a, np.float64) for n, a in make_params(case).items()}, {"t": 0, "m": {}, "v": {}}
    for k, batch in enumerate(rows):
        _, _, p, opt = DR.dqn_step(p, opt, batch, LR, cfg, torch.float64)
        if k == 2:
            DR.hard_target_update(p)
    K = len(rows)
    for n in p_gpu:
        if n == "deepq/eps":
            continue
        d = np.abs(p_gpu[n].astype(np.float64) - p[n]).reshape(-1)
        assert d.max() <= 2 * K * LR + 1e-6 * np.abs(p[n]).max(), (n, d.max())
        if d.size >= 1000:
            assert np.quantile(d, 0.99) <= 0.05 * K * LR, (n, np.quantile(d, 0.99) / (K * LR))


# ================================================================================================ the shipped model
@pytest.mark.gpu
def test_shipped_zip_predicts_the_oracle():
    """DQN.load(DQN_simple_4pads.zip): greedy actions and Q rows on 1,000 observations in [-1, 1]^100, and the softmax(Q) draw of
    predict(deterministic=False) from a seeded generator."""
    from b200grasp import sb_io
    _, params = sb_io.load_sb_zip(ZIP)
    m = deepq.DQN.load(ZIP)
    assert m.learner.n_actions == 12 and m.learner.obs_dim == 100 and m.gamma == 1.0 and m.batch_size == 32 and m.buffer_size == 50000
    obs = np.random.default_rng(0).uniform(-1, 1, (1000, 100)).astype(np.float32)
    a_ref, q_ref = DR.greedy_action(params, obs)
    idx, q = m.learner.act(obs, with_q=True)
    assert rel_err(q, q_ref) <= 1e-5, rel_err(q, q_ref)
    srt = np.sort(q_ref, 1)
    clear = (srt[:, -1] - srt[:, -2]) > 1e-5 * (1 + np.abs(q_ref).max(1))
    assert clear.sum() >= 990
    assert np.array_equal(idx[clear], a_ref[clear])
    act, _ = m.predict(obs)
    assert np.array_equal(act, idx)
    assert m.predict(obs[0])[0] == idx[0]
    m.predict_rng = np.random.default_rng(7)
    st, _ = m.predict(obs, deterministic=False)
    u = np.random.default_rng(7).random(len(obs))
    want, prob = DR.softmax_action(q_ref, u)
    cdf = np.cumsum(prob, 1)
    safe = np.abs(cdf - u[:, None]).min(1) > 1e-5
    assert safe.sum() >= 990 and np.array_equal(st[safe], want[safe])
    assert len(np.unique(st)) > 1
    m.close()


# ================================================================================================ learn / save / load / state
class LineEnv:
    """Test-local discrete environment: obs 6 floats from (t, last action), 4 actions, reward 1 for action t % 4, episodes of
    10 steps; deterministic, so a resumed run sees the frames an uninterrupted one does."""
    observation_space = Box(-np.inf, np.inf, (6,))
    action_space = Discrete(4)

    def __init__(self, *a, **k):
        self.t, self.last = 0, 0

    def _obs(self):
        return np.array([self.t / 10.0, self.last / 4.0, np.sin(self.t), np.cos(self.t), 1.0, -0.5], np.float32)

    def reset(self):
        self.t, self.last = 0, 0
        return self._obs()

    def step(self, a):
        a = int(np.asarray(a).reshape(-1)[0])
        r = float(a == self.t % 4)
        self.t += 1
        self.last = a
        return self._obs(), r, self.t >= 10, {"is_success": r > 0}

    def close(self):
        pass


class Line100Env(LineEnv):
    """The shipped zip's spaces (Box 100, Discrete 12) for `train_cli run`."""
    observation_space = Box(-1.0, 1.0, (100,))
    action_space = Discrete(12)

    def _obs(self):
        return np.tile(super()._obs(), 17)[:100]


def make_env(config, evaluate=False, validate=False, test=False):
    return Line100Env() if config.get("dqn_env_100") else LineEnv()


KW = dict(batch_size=16, buffer_size=500, learning_starts=50, target_network_update_freq=40, prioritized_replay=True,
          exploration_fraction=0.3, policy_kwargs={"layers": [16, 16]}, seed=3)


@pytest.mark.gpu
def test_dqn_learn_schedule_and_save_load(tmp_path):
    model = deepq.DQN(deepq.policies.MlpPolicy, LineEnv(), **KW)
    L = model.learner
    copies, steps = [], []
    orig_copy, orig_step = L.update_target, L.step

    def rec_copy():
        orig_copy()
        p = L.get_parameters()
        for n in p:
            if n.startswith(DR.ONLINE + "/"):
                assert np.array_equal(p[n.replace(DR.ONLINE, DR.TARGET)], p[n]), n
        copies.append(model.num_timesteps)

    def rec_step(n=1, lr=5e-4):
        steps.append(model.num_timesteps)
        return orig_step(n, lr)
    L.update_target, L.step = rec_copy, rec_step
    model.learn(200)
    assert model.num_timesteps == 200 and L.replay_size() == 200
    assert steps == list(range(51, 201))
    assert copies == [80, 120, 160, 200]
    assert abs(float(L.get_parameters()["deepq/eps"]) - 0.02) < 1e-7
    obs = np.random.default_rng(1).normal(size=(50, 6)).astype(np.float32)
    a0, _ = model.predict(obs)
    path = str(tmp_path / "dqn_model")
    model.save(path)
    m2 = deepq.DQN.load(path)
    a1, _ = m2.predict(obs)
    assert np.array_equal(a0, a1)
    p0, p1 = model.get_parameters(), m2.get_parameters()
    for n in p0:
        assert np.array_equal(p0[n], p1[n]), n
    model.close()
    m2.close()


@pytest.mark.gpu
def test_dqn_training_state_round_trip_and_continue(tmp_path):
    """save_training_state -> load_training_state restores parameters, Adam moments, replay, trees and host state bit for bit:
    the next sampled step draws the same slots and IS weights.  learn(60, reset_num_timesteps=False) from the file then follows
    learn(60) -> learn(60, reset_num_timesteps=False) on one model: the same exploration draws and schedule, and parameters equal
    up to the engine's atomic summation order (as tests/test_gpu_resume.py holds BDQ and SAC)."""
    acts = {"a": [], "c": []}

    class Rec(LineEnv):
        def __init__(self, tag):
            super().__init__()
            self.tag = tag

        def step(self, a):
            acts[self.tag].append(int(np.asarray(a).reshape(-1)[0]))
            return super().step(a)

    a = deepq.DQN("MlpPolicy", Rec("a"), **KW)
    a.learn(60)
    d = str(tmp_path / "state")
    a.save_training_state(d)
    p60 = a.get_parameters()
    c = deepq.DQN.load_training_state(d, Rec("c"))
    assert c.num_timesteps == 60 and c.learner.replay_size() == 60
    pc = c.get_parameters()
    for n in p60:
        assert np.array_equal(p60[n].view(np.uint32), pc[n].view(np.uint32)), n
    assert c._rng.bit_generator.state == a._rng.bit_generator.state
    a.learn(60, reset_num_timesteps=False)          # the uninterrupted run
    c.learn(60, reset_num_timesteps=False)
    assert a.num_timesteps == c.num_timesteps == 120 and a.n_target_updates == c.n_target_updates == 2
    agree = np.mean(np.array(acts["a"][60:]) == np.array(acts["c"]))
    assert len(acts["c"]) == 60 and agree >= 0.95, agree
    pa, pc = a.get_parameters(), c.get_parameters()
    for n in pa:
        if n != "deepq/eps":
            assert np.abs(pa[n].astype(np.float64) - pc[n]).max() <= 1e-3 * max(1e-3, np.abs(pa[n]).max()), n
    # learner level: a handle restored from the file draws the same slots and weights on its next sampled step
    path = str(tmp_path / "dqn.state")
    a.learner.save_state(path)
    r = deepq.DQNLearner(6, 4, (16, 16), 16, 500, 0.99, seed=3, prioritized_replay=True)
    r.load_state(path)
    pa, pr = a.learner.get_parameters(), r.get_parameters()
    for n in pa:
        assert np.array_equal(pa[n].view(np.uint32), pr[n].view(np.uint32)), n
    for L in (a.learner, r):
        L.set_per_beta(0.9)
    ma, mr = a.learner.step(1, 5e-4), r.step(1, 5e-4)
    (sa, wa, qa), (sr, wr, qr) = a.learner.last_per(), r.last_per()
    assert ma["n_updates"] == mr["n_updates"] and np.array_equal(sa, sr) and np.array_equal(wa.view(np.uint32), wr.view(np.uint32))
    assert abs(ma["loss"] - mr["loss"]) <= 1e-6 * abs(ma["loss"]) and np.allclose(qa, qr, rtol=1e-5, atol=0)
    r.close()
    a.close()
    c.close()


@pytest.mark.gpu
def test_dqn_learn_and_predict_under_vec_normalize():
    """With a host VecNormalize: learn stores raw transitions and acts on the wrapper's output; afterwards predict takes
    normalised observations as they are (no second normalisation), and the replay gather of a step normalises raw rows with
    the wrapper's statistics."""
    from b200grasp.vec_env import DummyVecEnv, VecNormalize
    env = VecNormalize(DummyVecEnv([LineEnv]), norm_obs=True, norm_reward=True, clip_obs=10.0)
    model = deepq.DQN("MlpPolicy", env, **KW)
    model.learn(150)
    vn = model.get_vec_normalize_env()
    assert vn is env and vn.obs_rms.count > 100
    params = model.learner.get_parameters()
    rng = np.random.default_rng(2)
    raw = np.stack([np.array([t / 10.0, a / 4.0, np.sin(t), np.cos(t), 1.0, -0.5]) for t, a in
                    zip(rng.integers(0, 10, 300), rng.integers(0, 4, 300))]).astype(np.float32)
    raw += rng.normal(0, 0.05, raw.shape).astype(np.float32)
    norm = vn.normalize_obs(raw).astype(np.float32)
    assert np.abs(norm - raw).max() > 0.5                     # the statistics move the observations
    a_ref, q_ref = DR.greedy_action(params, norm)
    srt = np.sort(q_ref, 1)
    clear = (srt[:, -1] - srt[:, -2]) > 1e-5 * (1 + np.abs(q_ref).max(1))
    assert clear.sum() >= 280
    act, _ = model.predict(norm)
    assert np.array_equal(act[clear], a_ref[clear])
    _, q = model.learner.act(norm, with_q=True)
    assert rel_err(q, q_ref) <= 1e-5
    # an observation the wrapper hands out
    obs = env.reset()
    a1, _ = model.predict(obs)
    _, q1 = DR.greedy_action(params, np.asarray(obs, np.float32))
    assert np.sort(q1[0])[-1] - np.sort(q1[0])[-2] <= 1e-5 or a1[0] == int(q1[0].argmax())
    # the step's gather: raw rows normalised with the statistics learn last synced (obs and reward)
    L = model.learner
    model._sync_norm_stats()
    B = L.batch_size
    bt = dict(obs=raw[:B], next_obs=raw[B:2 * B], act=rng.integers(0, 4, B), rew=rng.choice([0.0, 1.0], B).astype(np.float32),
              done=(rng.random(B) < 0.2).astype(np.float32))
    out = L.step_explicit(bt["obs"], bt["act"].astype(np.float32), bt["rew"], bt["next_obs"], bt["done"], apply_update=False)
    ret_std = np.sqrt(float(vn.ret_rms.var) + vn.epsilon)
    nb = dict(bt, obs=vn.normalize_obs(bt["obs"]).astype(np.float32), next_obs=vn.normalize_obs(bt["next_obs"]).astype(np.float32),
              rew=np.clip(bt["rew"] / ret_std, -vn.clip_reward, vn.clip_reward).astype(np.float32))
    p = L.get_parameters()
    r64, *_ = DR.dqn_step(p, {"t": 0, "m": {}, "v": {}}, nb, LR, model_cfg(model), torch.float64)
    assert rel_err(out["td"], r64["td"]) <= 1e-4, rel_err(out["td"], r64["td"])
    model.close()


def model_cfg(model):
    return DR.DQNConfig(model.learner.obs_dim, model.learner.n_actions, tuple(model.layers), model.gamma)


@pytest.mark.gpu
def test_dqn_refuses_actions_outside_the_action_space():
    case = CASES[0]
    L = make_learner(case)
    bt = make_batch(case, case.B, 3)
    for bad in (12.0, -1.0, 2.5, np.nan):
        a = bt["act"].astype(np.float32)
        a[5] = bad
        with pytest.raises(b200grasp._lib.B2GError, match="action 5"):
            L.replay_add(bt["obs"], a, bt["rew"], bt["next_obs"], bt["done"])
        with pytest.raises(b200grasp._lib.B2GError, match="action 5"):
            L.step_explicit(bt["obs"], a, bt["rew"], bt["next_obs"], bt["done"], lr=LR)
    assert L.replay_size() == 0
    m = L.step_explicit(bt["obs"], bt["act"].astype(np.float32), bt["rew"], bt["next_obs"], bt["done"], lr=LR)
    assert m["n_updates"] == 1
    L.close()


@pytest.mark.gpu
def test_cli_train_and_run_dqn(tmp_path):
    cfg = {"DQN": {"batch_size": 16, "learning_rate": 0.001, "prioritized_replay": True, "total_timesteps": 1100},
           "discount_factor": 1.0, "robot": {"discrete": False}, "reward": {}, "normalize": False}
    cpath = tmp_path / "c.yaml"
    cpath.write_text(yaml.safe_dump(cfg))
    out = tmp_path / "run"
    model = train_cli.main(["train", "--config", str(cpath), "--algo", "DQN", "--model_dir", str(out), "--env",
                            "tests.test_gpu_dqn:make_env", "--eval_freq", "500", "--checkpoint_freq", "600", "--state_freq", "550"])
    assert model.num_timesteps == 1100 and model.learner.replay_size() == 1100
    assert os.path.exists(out / "final_model.zip") and os.path.exists(out / "best_model" / "best_model.zip")
    assert yaml.safe_load(open(out / "config.yaml"))["robot"]["discrete"] is True
    assert os.path.exists(out / "training_state" / "host.json")
    model.close()
    # run the shipped zip on a 100-float, 12-action environment
    rdir = tmp_path / "shipped"
    rdir.mkdir()
    shutil.copy(ZIP, rdir / "DQN_simple_4pads.zip")
    (rdir / "config.yaml").write_text(yaml.safe_dump({"algorithm": "dqn", "normalize": False, "dqn_env_100": True}))
    res = train_cli.main(["run", "--model", str(rdir / "DQN_simple_4pads.zip"), "--env", "tests.test_gpu_dqn:make_env", "--episodes", "3"])
    assert res["episodes"] == 3 and res["mean_steps"] == 10.0
    res = train_cli.main(["run", "--model", str(rdir / "DQN_simple_4pads.zip"), "--env", "tests.test_gpu_dqn:make_env", "--episodes", "2",
                          "-s"])
    assert res["episodes"] == 2
