"""The BDQ / DQN transition replay with frames (``replay_frames=`` / ``frame_capacity``, include/b200grasp.h b2g_bdq_create2):
same runs as the default layout, frame sharing, eviction, bytes and training state."""
import struct

import numpy as np
import pytest
import torch

from b200grasp import BDQ, _lib
from b200grasp.bdq import BDQLearner
from b200grasp.deepq import DQN
from b200grasp.dqn import DQNLearner
from b200grasp.learner import transition_replay_bytes
from b200grasp.spaces import Box, Discrete
from b200grasp.vec_env import DummyVecEnv, VecNormalize

pytestmark = pytest.mark.gpu

D, NB = 3, 9
LAYERS = [[32, 16], [8], [8]]


class Env:
    """Observations of obs_dim floats (a 64x64x2 depth + pad layout when obs_dim = 8192), episodes of `horizon` steps."""

    def __init__(self, seed, horizon, obs_dim, discrete=None):
        self.observation_space = Box(-np.inf, np.inf, (obs_dim,))
        self.action_space = Box(-1.0, 1.0, (D,)) if discrete is None else Discrete(discrete, seed=seed)
        self.rng = np.random.default_rng(seed)
        self.horizon, self.t, self.obs_dim = horizon, 0, obs_dim

    def _obs(self):
        return self.rng.normal(0.3, 1.0, self.obs_dim).astype(np.float32)

    def reset(self):
        self.t = 0
        return self._obs()

    def step(self, action):
        self.t += 1
        return self._obs(), float(self.rng.normal()), self.t >= self.horizon, {}

    def close(self):
        pass


def make_venv(n_envs, obs_dim, observe):
    venv = DummyVecEnv([(lambda i=i: Env(7 + 100 * i, 4 + i % 5, obs_dim)) for i in range(n_envs)])
    return VecNormalize(venv, norm_obs=True, norm_reward=True, clip_obs=10.0) if observe else venv


def bdq_model(n_envs, obs_dim, frames, per, observe, buffer_size=4096, venv=None, lr=1e-3):
    venv = venv or make_venv(n_envs, obs_dim, observe)
    return BDQ("MlpActPolicy", venv, buffer_size=buffer_size, batch_size=16, learning_starts=24, learning_rate=lr,
               prioritized_replay=per, num_actions_pad=NB, policy_kwargs={"layers": LAYERS}, seed=3, target_network_update_freq=50,
               device_obs_norm=observe, replay_frames=frames)


def sections(path):
    with open(path, "rb") as f:
        raw = f.read()
    n_fp, n_sec = struct.unpack_from("<II", raw, 16)
    out = {}
    for i in range(n_sec):
        tag, _, off, nb, _ = struct.unpack_from("<IIQQQ", raw, 32 + 40 * n_fp + 32 * i)
        out[tag.to_bytes(4, "little").decode()] = raw[off:off + nb]
    return out


def replay_rows(L):
    """(obs, act, rew, next_obs, done) of every live slot, in slot order"""
    info = L.replay_info()
    rows = {}
    for s in range(info["capacity"]):
        try:
            rows[s] = L.replay_get(s)
        except _lib.B2GError:
            pass
    assert len(rows) == info["size"]
    return rows


def run_record(model, steps):
    """learn(steps), recording every gradient step's sampled slots, weights and new priorities"""
    L, rec = model.learner, []
    step = L.step

    def recording_step(*a, **k):
        m = step(*a, **k)
        rec.append((m, *L.last_per()))
        return m
    L.step = recording_step
    model.learn(steps)
    L.step = step
    return rec


def spread(pa, pb):
    return max(float(np.abs(pa[k].astype(np.float64) - pb[k]).max()) for k in pa)


def compare(default, default2, framed, rec_d, rec_f, per):
    """frames against the default layout.  Two default runs already differ in the last bits of the parameters (the fp32
    engine's weight-gradient atomics add in a different order from run to run), and a draw that lands near a boundary can
    turn such a difference into a different batch: trained parameters are compared within max(4 s, 1e-3).  Every draw,
    weight, priority, stored row and loss is compared bit for bit when the default layout reproduces itself (s == 0, as
    with learning_rate 0; the gradient norm, summed by atomics, only to 1e-6)."""
    s = spread(default.learner.get_parameters(), default2.learner.get_parameters())
    got = spread(default.learner.get_parameters(), framed.learner.get_parameters())
    print(f"parameter spread: default vs default {s:.3g}, frames vs default {got:.3g}")
    assert got == 0 if s == 0 else got <= max(4 * s, 1e-3), (got, s)
    ra, rf = replay_rows(default.learner), replay_rows(framed.learner)
    assert ra.keys() == rf.keys()
    if s == 0:
        for k in ra:
            for f in ("obs", "act", "next_obs"):
                assert np.array_equal(ra[k][f], rf[k][f]), (k, f)
            assert ra[k]["rew"] == rf[k]["rew"] and ra[k]["done"] == rf[k]["done"]
        assert len(rec_d) == len(rec_f)
        for (ma, ia, wa, pa_), (mf, if_, wf, pf) in zip(rec_d, rec_f):
            assert {k: v for k, v in ma.items() if k != "grad_norm"} == {k: v for k, v in mf.items() if k != "grad_norm"}
            assert abs(ma["grad_norm"] - mf["grad_norm"]) <= 1e-6 * abs(ma["grad_norm"]) and np.array_equal(ia, if_)
            if per:
                assert np.array_equal(wa, wf) and np.array_equal(pa_, pf)
    return s


# ------------------------------------------------------------------------------------------------ 1. same run
@pytest.mark.parametrize("observe", [False, True])
@pytest.mark.parametrize("per", [False, True])
@pytest.mark.parametrize("n_envs", [1, 3, 16])
def test_bdq_frames_train_as_the_default_layout(n_envs, per, observe):
    steps = 400 if n_envs < 16 else 960
    models = [bdq_model(n_envs, 100, f, per, observe) for f in (None, None, 4096 + 4096 // 2 + n_envs)]
    recs = [run_record(m, steps) for m in models]
    compare(*models, recs[0], recs[2], per)
    info = models[2].learner.replay_info()
    assert info["evicted_early"] == 0 and info["frame_capacity"] == 4096 + 2048 + n_envs
    for m in models:
        m.close()


@pytest.mark.parametrize("observe", [False, True])
@pytest.mark.parametrize("per", [False, True])
@pytest.mark.parametrize("n_envs", [1, 3, 16])
def test_bdq_frames_run_bit_for_bit_as_the_default_layout_at_learning_rate_0(n_envs, per, observe):
    """learning_rate 0: parameters stay put, so the default layout reproduces itself bit for bit (actions, statistics, TD
    errors, priorities, draws) and the frame layout must match it exactly over the whole run"""
    models = [bdq_model(n_envs, 100, f, per, observe, lr=0.0) for f in (None, None, 4096 + 2048 + n_envs)]
    recs = [run_record(m, 400 if n_envs < 16 else 960) for m in models]
    assert compare(*models, recs[0], recs[2], per) == 0
    for m in models:
        m.close()


@pytest.mark.parametrize("observe", [False, True])
def test_bdq_frames_train_as_the_default_layout_on_depth_rows(observe):
    models = [bdq_model(3, 8192, f, True, observe, buffer_size=512) for f in (None, None, 512 + 256 + 3)]
    recs = [run_record(m, 300) for m in models]
    compare(*models, recs[0], recs[2], True)
    for m in models:
        m.close()


@pytest.mark.parametrize("per", [False, True])
def test_dqn_frames_train_as_the_default_layout(per):
    def model(frames):
        env = DummyVecEnv([lambda: Env(5, 6, 100, discrete=12)])
        return DQN("MlpPolicy", env, buffer_size=1024, batch_size=32, learning_starts=32, prioritized_replay=per, seed=1,
                   target_network_update_freq=40, policy_kwargs={"layers": [32, 32]}, replay_frames=frames)
    models = [model(f) for f in (None, None, 1024 + 512 + 1)]
    recs = [run_record(m, 400) for m in models]
    compare(*models, recs[0], recs[2], per)
    for m in models:
        m.close()


# ------------------------------------------------------------------------------------------------ 2. sharing
def stream(n_envs, steps, obs_dim, seed=0, horizon=5):
    """per step: obs, act, rew, next_obs, done, reset frames of an episodic stream (obs(t+1) = next_obs(t) within an episode)"""
    rng = np.random.default_rng(seed)
    cur = rng.normal(size=(n_envs, obs_dim)).astype(np.float32)
    t = np.zeros(n_envs, int)
    for _ in range(steps):
        nxt = rng.normal(size=(n_envs, obs_dim)).astype(np.float32)
        t += 1
        done = (t % (horizon + np.arange(n_envs)) == 0).astype(np.float32)
        act = rng.integers(0, NB, (n_envs, D)).astype(np.float32)
        rew = rng.normal(size=n_envs).astype(np.float32)
        reset = rng.normal(size=(n_envs, obs_dim)).astype(np.float32)
        yield cur.copy(), act, rew, nxt, done, reset
        cur = np.where(done[:, None] != 0, reset, nxt)


@pytest.mark.parametrize("observe", [False, True])
@pytest.mark.parametrize("obs_dim", [100, 8192])
def test_transitions_share_frames_and_rebuild_bit_for_bit(observe, obs_dim):
    n_envs, steps, cap = 3, 40, 1024
    L = BDQLearner(obs_dim, D, NB, tuple(tuple(l) for l in LAYERS), 16, cap, frame_capacity=cap + cap // 2 + n_envs)
    stored, ends = [], 0
    for i, (o, a, r, nx, d, reset) in enumerate(stream(n_envs, steps, obs_dim)):
        if observe:
            if i == 0:
                L.observe_act(o, update_stats=False, act=False)
            L.observe_add(a, r, nx, d, reset_obs=reset, update_stats=False)
        else:
            L.replay_add(o, a, r, nx, d)
        stored += [(o[k], a[k], r[k], nx[k], d[k]) for k in range(n_envs)]
        ends += int(d.sum()) if i < steps - 1 else 0          # the last call's reset frames are not stored yet
    info = L.replay_info()
    T = steps * n_envs
    # one frame per transition (its next_obs), one per first observation of an env and one per episode end (the reset frame)
    assert info["size"] == T and info["live_frames"] == T + n_envs + ends and info["evicted_early"] == 0
    prev_next = {}
    for t, (o, a, r, nx, d) in enumerate(stored):
        g = L.replay_get(t)
        assert np.array_equal(g["obs"], o) and np.array_equal(g["next_obs"], nx) and np.array_equal(g["act"], a)
        assert g["rew"] == r and g["done"] == d
        env = t % n_envs
        if env in prev_next:
            shared = prev_next[env][1] == 0.0
            assert (g["frames"][0] == prev_next[env][0]) == shared, t
        prev_next[env] = (g["frames"][1], d)
    # an obs that differs from the previous next_obs takes a frame of its own
    if not observe:
        o, a, r, nx, d, _ = next(stream(n_envs, 1, obs_dim, seed=9))
        L.replay_add(o, a, r, nx, d)
        assert L.replay_info()["live_frames"] == T + n_envs + ends + 2 * n_envs
        for k in range(n_envs):
            g = L.replay_get(T + k)
            assert g["frames"][0] != prev_next[k][0] and np.array_equal(g["obs"], o[k])
    L.close()


# ------------------------------------------------------------------------------------------------ 3. eviction
class HostRing:
    """SAC's eviction rule (csrc/frame_ring.cuh) restated: FIFO frame ids, the oldest transitions go when a new frame would
    overwrite one a live transition references."""

    def __init__(self, cap, fcap):
        self.cap, self.fcap, self.head, self.tail, self.next_fid, self.obs_frame = cap, fcap, 0, 0, 0, {}
        self.prev_next = {}

    def alloc(self):
        f = self.next_fid
        self.next_fid += 1
        while self.head > self.tail and min(self.obs_frame[t] for t in range(self.tail, self.head)) <= f - self.fcap:
            self.tail += 1
        return f

    def add(self, cand):
        if self.head - self.tail == self.cap:
            self.tail += 1
        share = self.fcap < 2 * self.cap and cand is not None and cand >= self.next_fid + 1 - self.fcap
        of = cand if share else self.alloc()
        nf = self.alloc()
        self.obs_frame[self.head] = of
        self.head += 1
        return nf


def test_eviction_follows_the_host_rule_and_sampling_skips_evicted_slots(tmp_path):
    cap, fcap, n_envs, obs_dim = 256, 300, 4, 100
    L = BDQLearner(obs_dim, D, NB, tuple(tuple(l) for l in LAYERS), 16, cap, prioritized_replay=True, frame_capacity=fcap)
    ring, live_ok = HostRing(cap, fcap), True
    rng = np.random.default_rng(4)
    prev = [None] * n_envs
    for i, (o, a, r, nx, d, _) in enumerate(stream(n_envs, 120, obs_dim, seed=2, horizon=2)):
        if i % 3 == 2:                   # every third call breaks the chain: obs differs from the previous next_obs
            o = o + np.float32(1.0)
        L.replay_add(o, a, r, nx, d)
        for k in range(n_envs):
            same = prev[k] is not None and np.array_equal(prev[k][1], o[k])
            prev[k] = (ring.add(prev[k][0] if same else None), nx[k])
        info = L.replay_info()
        assert info["size"] == ring.head - ring.tail, i
        live = {(ring.tail + u) % cap for u in range(ring.head - ring.tail)}
        if i > 10:
            L.step(1, lr=1e-4)
            slots, _, _ = L.last_per()
            live_ok &= all(int(s) in live for s in slots)
            # new priorities sit in the trees: the PERT leaves of evicted slots are empty and the root is the live sum
            if i % 20 == 0:
                p = str(tmp_path / f"s{i}.state")
                L.save_state(p)
                t = np.frombuffer(sections(p)["PERT"], np.float64)
                C2 = t.size // 2
                tsum, tmin = t[:C2], t[C2:]
                C = C2 // 2
                for s in range(C):
                    if s in live:
                        assert tsum[C + s] > 0, (i, s)
                    else:
                        assert tsum[C + s] == 0 and np.isinf(tmin[C + s]), (i, s)
                assert np.isclose(tsum[1], tsum[C:C + cap].sum(), rtol=1e-12, atol=0)
                assert tmin[1] == tmin[C:C + cap].min()
    assert live_ok
    assert L.replay_info()["evicted_early"] > 0
    L.close()


# ------------------------------------------------------------------------------------------------ 4. bytes
@pytest.mark.parametrize("obs_dim", [100, 8192])
def test_bytes_match_the_formula(obs_dim):
    cap, fcap = 1000, 1130
    L = BDQLearner(obs_dim, D, NB, tuple(tuple(l) for l in LAYERS), 16, cap, frame_capacity=fcap)
    row = (4 * obs_dim + 15) // 16 * 16
    want = fcap * row + 2 * cap * 4 + cap * (D + 2) * 4
    assert L.replay_info()["bytes"] == want == transition_replay_bytes(cap, obs_dim, D, fcap)
    L.close()
    Q = DQNLearner(obs_dim, 12, (32, 32), 32, cap, frame_capacity=fcap)
    assert Q.replay_info()["bytes"] == fcap * row + 2 * cap * 4 + cap * 3 * 4
    Q.close()
    # BDQ on the depth observation at 10^6 slots with --replay_spare 0.125: about 36.9 GB against 65.5 GB, not allocated
    f = int(1e6 * 1.125) + 1
    assert abs(transition_replay_bytes(10**6, 8192, D, f) / 1e9 - 36.9) < 0.05
    assert abs(transition_replay_bytes(10**6, 8192, D) / 1e9 - 65.5) < 0.1


def test_a_real_allocation_matches_mem_get_info():
    torch.cuda.init()
    cap, fcap = 10**5, int(10**5 * 1.125) + 1
    free0, _ = torch.cuda.mem_get_info(0)
    L = BDQLearner(8192, D, NB, tuple(tuple(l) for l in LAYERS), 16, cap, frame_capacity=fcap)
    free1, _ = torch.cuda.mem_get_info(0)
    want = L.replay_info()["bytes"]
    used = free0 - free1
    print(f"replay bytes {want}, device memory taken by the handle {used}")
    # the rest of the handle (network, staging) is a few MB; allocation granularity adds at most 2 MB per array
    assert want <= used <= want + (64 << 20)
    L.close()


# ------------------------------------------------------------------------------------------------ 5. training state
@pytest.mark.parametrize("observe", [False, True])
def test_save_load_continue_equals_an_uninterrupted_run(tmp_path, observe):
    fr = 64 + 2 + 3                   # below the ~1.2 frames per transition these episodes need: transitions go early
    env_b = make_venv(3, 100, observe)
    a, b = bdq_model(3, 100, fr, True, observe, buffer_size=64), bdq_model(3, 100, fr, True, observe, buffer_size=64, venv=env_b)
    a.learn(150)
    b.learn(150)
    assert a.learner.replay_info()["evicted_early"] > 0      # a budget that evicts: the window starts mid-ring
    state = b.save_training_state(str(tmp_path / "state"))
    b.close()
    b = BDQ.load_training_state(state, env_b)
    assert b.replay_frames == fr and b.learner.replay_info()["frame_capacity"] == fr
    a.learn(60, reset_num_timesteps=False)
    b.learn(60, reset_num_timesteps=False)
    pa, pb = a.learner.get_parameters(), b.learner.get_parameters()
    for nm in pa:
        np.testing.assert_allclose(pb[nm], pa[nm], rtol=0, atol=1e-6, err_msg=nm)
    for m, f in ((a, "a.state"), (b, "b.state")):
        m.learner.save_state(str(tmp_path / f))
    sa, sb = sections(str(tmp_path / "a.state")), sections(str(tmp_path / "b.state"))
    for tag in ("HOST", "ROFR", "RNFR", "RACT", "RREW", "RDON", "FRMS"):
        assert sa[tag] == sb[tag], tag
    a.close()
    b.close()


def test_files_do_not_cross_the_two_layouts(tmp_path):
    framed = BDQLearner(100, D, NB, tuple(tuple(l) for l in LAYERS), 16, 256, frame_capacity=300)
    plain = BDQLearner(100, D, NB, tuple(tuple(l) for l in LAYERS), 16, 256)
    for L, f in ((framed, "f.state"), (plain, "p.state")):
        for o, a, r, nx, d, _ in stream(2, 10, 100):
            L.replay_add(o, a, r, nx, d)
        L.save_state(str(tmp_path / f))
    for src, dst in (("f.state", plain), ("p.state", framed)):
        with pytest.raises(_lib.B2GError, match="replay_frames") as e:
            dst.load_state(str(tmp_path / src))
        assert e.value.code == _lib.B2G_EINVAL
    framed.load_state(str(tmp_path / "f.state"))       # its own file loads
    qf = DQNLearner(100, 12, (32, 32), 32, 256, frame_capacity=300)
    qp = DQNLearner(100, 12, (32, 32), 32, 256)
    qf.save_state(str(tmp_path / "qf.state"))
    with pytest.raises(_lib.B2GError, match="replay_frames"):
        qp.load_state(str(tmp_path / "qf.state"))
    for L in (framed, plain, qf, qp):
        L.close()


def test_refusals():
    with pytest.raises(_lib.B2GError, match="buffer_capacity \\+ 1"):
        BDQLearner(100, D, NB, tuple(tuple(l) for l in LAYERS), 16, 256, frame_capacity=256)
    with pytest.raises(_lib.B2GError, match="buffer_capacity \\+ 1"):
        DQNLearner(100, 12, (32, 32), 32, 256, frame_capacity=100)
    L = BDQLearner(100, D, NB, tuple(tuple(l) for l in LAYERS), 16, 256, frame_capacity=300)
    o, a, r, nx, d, _ = next(stream(200, 1, 100))
    with pytest.raises(_lib.B2GError, match="frame_capacity"):
        L.replay_add(o, a, r, nx, d)                     # 2 n rows > frame_capacity
    L.close()
