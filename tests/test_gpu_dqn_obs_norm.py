"""DQN with VecNormalize's observation statistics on the device and the epsilon-greedy actor fed from one upload per frame
(include/b200grasp.h: b2g_dqn_observe_act / _add, b2g_dqn_act_raw, b2g_dqn_obs_rms_set / _get; ``DQN(device_obs_norm=True)``),
held to the host RunningMeanStd, to b2g_dqn_act on host-normalised rows, to b2g_dqn_replay_add, to the encoder handle and to
the restated Philox stream 3."""
import numpy as np
import pytest

from b200grasp import _lib, synth
from b200grasp.deepq import DQN, DQNLearner
from b200grasp.encoders import SimpleAutoEncoder, keras_encoder_arrays
from b200grasp.spaces import Box, Discrete
from b200grasp.vec_env import DummyVecEnv, RunningMeanStd, VecNormalize
from oracle import dqn_ref as DR
from oracle import philox_ref as PX
from tests.test_dqn_obs_norm_cpu import explore_dqn
from tests.test_encoder_cpu import load_fixture
from tests.test_gpu_bdq_obs_norm import sections

pytestmark = pytest.mark.gpu

OBS, NA, B = 12, 6, 8
LAYERS = (32, 16)
U32 = 2.0 ** -24


def make_learner(frames=None, per=False, seed=5, obs=OBS, buffer_size=256):
    L = DQNLearner(obs, NA, LAYERS, B, buffer_size, 0.99, seed=seed, prioritized_replay=per, prioritized_replay_alpha=0.6,
                   frame_capacity=frames)
    L.load_parameters(make_params(obs))
    return L


def make_params(obs=OBS):
    p = DR.init_params(DR.DQNConfig(obs, NA, LAYERS), seed=21)
    rng = np.random.default_rng(22)
    for n in p:
        if n.endswith("biases"):
            p[n] = (rng.normal(size=p[n].shape) * 0.1).astype(np.float32)
    return p


def counter7(L, tmp_path):
    p = str(tmp_path / "c.state")
    L.save_state(p)
    return int(np.frombuffer(sections(p)["CNTR"], np.int64)[7])


def stats_table(L, clip):
    """obs_rms with a feature far past clip, a zero-variance one; the gather's scalars set for it."""
    rng = np.random.default_rng(3)
    mean, var = rng.normal(0.5, 1.0, OBS), rng.uniform(0.5, 4.0, OBS)
    mean[0], var[0] = -40.0, 1.0
    var[1] = 0.0
    L.obs_rms_set(mean, var, 10.0)
    L.set_norm_stats(None, None, 1.0, clip, 10.0, 1e-8, norm_obs=True, norm_reward=False)
    vn = VecNormalize(DummyVecEnv([lambda: FlatEnv(0)]), clip_obs=clip)
    vn.obs_rms.mean, vn.obs_rms.var = mean, var
    return vn


def raw_rows(n, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(0.5, 2.0, (n, OBS)).astype(np.float32)
    x[:, 1] = 2.0
    return x


def decided(params, xn):
    """Rows whose greedy action float64 Q decides beyond fp32 resolution and a one-ulp change of every input (the device
    normalises with 1/sqrt(var + eps), the host divides by sqrt(var + eps)): bound = propagated |dx| through |W| of each
    tower, dQ_k <= dV + dA_k + max dA."""
    _, q = DR.greedy_action(params, xn)
    dq = np.zeros_like(q)
    dv = None
    for tower in ("action_value", "state_value"):
        h = np.abs(np.asarray(xn, np.float64)) * 2.0 ** -23
        for k in range(3):
            h = h @ np.abs(np.asarray(params[f"{DR.ONLINE}/{tower}/{DR._fc(k)}/weights"], np.float64))
        if tower == "action_value":
            dq = h + h.max(1, keepdims=True)
        else:
            dv = h
    bar = 2 * (dq + dv).max(1) + 64 * U32 * (1.0 + np.abs(q).max(1))
    top2 = np.sort(q, 1)[:, -2:]
    return (top2[:, 1] - top2[:, 0]) > bar


class FlatEnv:
    """Flat observations with a feature that spikes far past clip_obs and a constant one; frames do not depend on the action;
    episodes of `horizon` steps."""

    def __init__(self, seed, horizon=4):
        self.observation_space = Box(-np.inf, np.inf, (OBS,))
        self.action_space = Discrete(NA)
        self.rng = np.random.default_rng(seed)
        self.horizon, self.t = horizon, 0

    def _obs(self):
        o = self.rng.normal(0.5, 2.0, OBS).astype(np.float32)
        o[0] = np.float32(400.0) if self.rng.random() < 0.05 else np.float32(self.rng.normal(0.0, 0.1))
        o[1] = np.float32(2.0)
        return o

    def reset(self):
        self.t = 0
        return self._obs()

    def step(self, action):
        self.t += 1
        return self._obs(), float(self.rng.normal(0.0, 3.0)), self.t >= self.horizon, {}


# ------------------------------------------------------------------------------------------------ statistics
def test_statistics_follow_the_host_running_mean_std():
    L = make_learner()
    rms = RunningMeanStd(shape=(OBS,))
    L.obs_rms_set(rms.mean, rms.var, rms.count)
    rng = np.random.default_rng(1)
    n = 3
    o = rng.normal(1.0, 3.0, (n, OBS)).astype(np.float32)
    L.observe_act(o, act=False)
    rms.update(o)
    for k in range(6):
        nx = rng.normal(1.0, 3.0, (n, OBS)).astype(np.float32)
        done = (rng.random(n) < 0.4).astype(np.float32)
        done[k % n] = 1.0
        reset = rng.normal(-2.0, 1.0, (n, OBS)).astype(np.float32)
        L.observe_add(rng.integers(0, NA, n).astype(np.float32), rng.normal(size=n), nx, done, reset_obs=reset)
        rms.update(np.where(done[:, None] != 0, reset, nx))      # a finished env's reset frame, never its terminal frame
    mean, var, count = L.obs_rms_get()
    assert count == rms.count
    assert np.abs(mean - rms.mean).max() <= 1e-12 * np.abs(rms.mean).max()
    assert np.abs(var - rms.var).max() <= 1e-12 * np.abs(rms.var).max()
    L.close()


# ------------------------------------------------------------------------------------------------ the actor
def test_actor_greedy_exploration_chunks_and_act_raw(tmp_path):
    L = make_learner()
    vn = stats_table(L, 5.0)
    key = PX.train_seed(5)
    n = 2 * B + 3
    raw = raw_rows(n, 4)
    xn = vn.normalize_obs(raw).astype(np.float32)
    assert (xn[:, 0] == 5.0).all()
    greedy = L.observe_act(raw, update_stats=False, eps=0.0)                 # acting call 0
    assert counter7(L, tmp_path) == 1
    ref = L.act(xn)                                                          # b2g_dqn_act on host-normalised rows
    ok = decided(make_params(), xn)
    assert ok.sum() >= n // 2
    assert np.array_equal(greedy[ok], ref[ok])
    # act_raw: the same greedy actions, and Q rows whose argmax they are
    a_raw, q_raw = L.act_raw(raw, with_q=True)
    assert np.array_equal(a_raw, greedy) and np.array_equal(np.argmax(q_raw, 1), greedy)
    # exploration against the restated stream 3; eps = 0 never explores
    seen = 0
    for step, eps in ((1, 1.0), (2, 0.3), (3, 0.3), (4, 0.0)):
        got = L.observe_act(None, n=n, eps=eps)
        go, acts = explore_dqn(key, step, n, NA, eps)
        assert np.array_equal(got[go], acts[go]) and np.array_equal(got[~go], greedy[~go]), step
        seen += int(go.sum())
        if eps in (0.0, 1.0):
            assert go.all() == (eps == 1.0) and go.any() == (eps == 1.0), step
    assert 0 < seen < 3 * n and counter7(L, tmp_path) == 5
    # n = B - 1 and 2B + 3 rows per call: the greedy action of every row as a single-row call gives it
    for m in (B - 1, 2 * B + 3):
        rows = raw_rows(m, 10 + m)
        many = L.observe_act(rows, update_stats=False, eps=0.0)
        one = np.array([L.observe_act(rows[i:i + 1], update_stats=False, eps=0.0)[0] for i in range(m)])
        assert np.array_equal(many, one), m
    L.close()


# ------------------------------------------------------------------------------------------------ replay
def _stream(n, k, seed):
    rng = np.random.default_rng(seed)
    o = rng.normal(size=(n, OBS)).astype(np.float32)
    out = []
    for _ in range(k):
        nx = rng.normal(size=(n, OBS)).astype(np.float32)
        done = (rng.random(n) < 0.3).astype(np.float32)
        reset = rng.normal(size=(n, OBS)).astype(np.float32)
        out.append((o, rng.integers(0, NA, n).astype(np.float32), rng.normal(size=n).astype(np.float32), nx, done, reset))
        o = np.where(done[:, None] != 0, reset, nx)
    return out


@pytest.mark.parametrize("frames", [None, 300])
def test_observe_add_stores_what_replay_add_stores(frames, tmp_path):
    n = 5
    dev, host = make_learner(frames, per=True), make_learner(frames, per=True)
    data = _stream(n, 12, 2)
    dev.observe_act(data[0][0], update_stats=False, act=False)
    for o, a, r, nx, d, reset in data:
        dev.observe_add(a, r, nx, d, reset_obs=reset if d.any() else None, update_stats=False)
        host.replay_add(o, a, r, nx, d)
    assert dev.replay_size() == host.replay_size() == n * len(data)
    for s in range(n * len(data)):
        t, u = dev.replay_get(s), host.replay_get(s)
        for k in ("obs", "act", "next_obs"):
            assert np.array_equal(t[k], u[k]), (s, k)
        assert t["rew"] == u["rew"] and t["done"] == u["done"], s
    if frames:     # linked: obs shares the previous next_obs frame, unless the env was reset (then a frame of its own)
        for k in range(1, len(data)):
            for i in range(n):
                f, g = dev.replay_get(k * n + i)["frames"], dev.replay_get((k - 1) * n + i)["frames"]
                if data[k - 1][4][i]:
                    assert f[0] != g[1] and f[0] >= 0, (k, i)
                else:
                    assert f[0] == g[1], (k, i)
    # PER: every new leaf at max_prio^alpha, as replay_add writes them
    pa, pb = str(tmp_path / "a.state"), str(tmp_path / "b.state")
    dev.save_state(pa)
    host.save_state(pb)
    sa, sb = sections(pa), sections(pb)
    assert sa["PERT"] == sb["PERT"] and sa["PERS"] == sb["PERS"]
    tsum = np.frombuffer(sa["PERT"], np.float64)
    C = tsum.size // 4
    max_prio = np.frombuffer(sa["PERS"], np.float32)[0]
    np.testing.assert_allclose(tsum[C:C + n * len(data)], np.float64(max_prio) ** np.float64(np.float32(0.6)), rtol=1e-15)
    # a sampled step from the same seed: the same slots and metrics (the backward's atomics may order the norm's sum apart)
    ma, mb = dev.step(1, lr=1e-3), host.step(1, lr=1e-3)
    assert np.array_equal(dev.last_per()[0], host.last_per()[0])
    assert ma["n_clipped"] == mb["n_clipped"]
    for k in ("loss", "mean_q", "mean_abs_td", "grad_norm"):
        assert ma[k] == pytest.approx(mb[k], rel=1e-6), k
    dev.close(), host.close()


# ------------------------------------------------------------------------------------------------ encoder
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_encoder_stage_equals_the_encoder_handle(precision):
    w, cfg = load_fixture()
    enc = SimpleAutoEncoder(cfg, max_batch=512, precision=precision)
    enc.set_weights(keras_encoder_arrays(w, len(cfg["network"])))
    D, tail, n, px = cfg["encoding_dim"], 1, 4, 64 * 64
    L = make_learner(obs=D + tail)
    L.set_obs_encoder(enc, tail)

    def raw(seed):
        rng = np.random.default_rng(seed)
        imgs = synth.make_depth_scenes(n, seed=seed) + rng.normal(0, 0.02, (n, 64, 64, 1)).astype(np.float32)
        return np.concatenate([imgs.reshape(n, px), rng.uniform(0, 1, (n, tail))], 1).astype(np.float32)

    def host(rows):
        return np.concatenate([enc.encode(rows[:, :px].reshape(-1, 64, 64, 1)), rows[:, px:]], 1)

    r0, r1, r2, reset = raw(1), raw(2), raw(3), raw(4)
    done = np.array([0, 1, 0, 1], np.float32)
    L.observe_act(r0, update_stats=False, act=False)
    L.observe_add(np.zeros(n, np.float32), np.zeros(n, np.float32), r1, done, reset_obs=reset, update_stats=False)
    L.observe_add(np.zeros(n, np.float32), np.zeros(n, np.float32), r2, np.zeros(n, np.float32), update_stats=False)
    staged = np.where(done[:, None] != 0, reset, r1)
    for i in range(n):
        t0, t1 = L.replay_get(i), L.replay_get(n + i)
        assert np.array_equal(t0["obs"], host(r0)[i]) and np.array_equal(t0["next_obs"], host(r1)[i]), i
        assert np.array_equal(t1["obs"], host(staged)[i]) and np.array_equal(t1["next_obs"], host(r2)[i]), i
    L.close()


# ------------------------------------------------------------------------------------------------ learn
def make_env(seed=0, horizon=4):
    return VecNormalize(DummyVecEnv([lambda: FlatEnv(seed, horizon)]), norm_obs=True, norm_reward=True, clip_obs=5.0)


def make_model(env, dev, **kw):
    args = dict(buffer_size=512, batch_size=B, learning_starts=20, learning_rate=1e-3, prioritized_replay=True, seed=3,
                target_network_update_freq=25, policy_kwargs={"layers": list(LAYERS)}, device_obs_norm=dev)
    args.update(kw)
    return DQN("MlpPolicy", env, **args)


def rows(L, k):
    return [L.replay_get(s) for s in range(k)]


def test_learn_stores_the_host_loop_transitions_and_statistics():
    T = 60
    env_h, env_d = make_env(), make_env()
    host, dev = make_model(env_h, False), make_model(env_d, True)
    assert env_d.learner_owns_obs_rms and dev.predict_takes_raw_obs
    host.learn(T)
    before = dev.learner.upload_bytes()["observe"]
    dev.learn(T)
    up = dev.learner.upload_bytes()["observe"] - before
    rh, rd = rows(host.learner, T), rows(dev.learner, T)
    n_done = 0
    for s, (a, b) in enumerate(zip(rh, rd)):
        for k in ("obs", "next_obs"):
            assert np.array_equal(a[k], b[k]), (s, k)
        assert a["rew"] == b["rew"] and a["done"] == b["done"], s
        n_done += int(b["done"])
    assert n_done == T // 4
    m, v, c = dev.learner.obs_rms_get()
    assert c == env_h.obs_rms.count
    assert np.abs(m - env_h.obs_rms.mean).max() <= 1e-12 * np.abs(env_h.obs_rms.mean).max()
    assert np.abs(v - env_h.obs_rms.var).max() <= 1e-12 * np.abs(env_h.obs_rms.var).max()
    # one frame per env step (the reset frame of a finished env is its next_obs: it crosses again as reset_obs), the reset
    # frame, and act / rew / done
    E = OBS * 4
    assert up == E + T * (E + 3 * 4) + n_done * E, up
    # predict on raw rows normalises on the device: the greedy action of act_raw
    x = raw_rows(3, 9)
    assert np.array_equal(dev.predict(x)[0], dev.learner.act_raw(x))
    host.close(), dev.close()
    assert not env_d.learner_owns_obs_rms


# ------------------------------------------------------------------------------------------------ resume
def test_save_load_continue_equals_an_uninterrupted_run(tmp_path):
    env_a, env_b = make_env(11), make_env(11)
    a, b = make_model(env_a, True), make_model(env_b, True)
    a.learn(40)
    b.learn(40)
    state = b.save_training_state(str(tmp_path / "state"))
    b.close()
    b = DQN.load_training_state(state, env_b)
    assert b.device_obs_norm and env_b.learner_owns_obs_rms
    a.learn(40, reset_num_timesteps=False)
    b.learn(40, reset_num_timesteps=False)
    for m, f in ((a, "a.state"), (b, "b.state")):
        m.learner.save_state(str(tmp_path / f))
    sa, sb = sections(str(tmp_path / "a.state")), sections(str(tmp_path / "b.state"))
    for tag in ("ORMS", "ROBS", "RNXT", "RACT", "RREW", "RDON"):
        assert sa[tag] == sb[tag], tag
    ca, cb = np.frombuffer(sa["CNTR"], np.int64), np.frombuffer(sb["CNTR"], np.int64)
    assert ca[7] == cb[7] == 80
    x = raw_rows(5, 1)
    a.learner.set_norm_stats(None, None, 1.0, 5.0, 10.0, 1e-8, norm_obs=True, norm_reward=False)
    b.learner.set_norm_stats(None, None, 1.0, 5.0, 10.0, 1e-8, norm_obs=True, norm_reward=False)
    np.testing.assert_allclose(b.learner.act_raw(x, with_q=True)[1], a.learner.act_raw(x, with_q=True)[1], rtol=0, atol=1e-5)
    # a handle without device statistics: no obs_rms section, its own file loads; files do not cross the difference
    plain = make_model(make_env(11), False)
    plain.learn(30)
    plain.learner.save_state(str(tmp_path / "plain.state"))
    assert "ORMS" not in sections(str(tmp_path / "plain.state"))
    plain.learner.load_state(str(tmp_path / "plain.state"))
    for src, dst in ((str(tmp_path / "a.state"), plain), (str(tmp_path / "plain.state"), a)):
        with pytest.raises(_lib.B2GError, match="obs_rms") as e:
            dst.learner.load_state(src)
        assert e.value.code == _lib.B2G_EINVAL
    for m in (a, b, plain):
        m.close()


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals():
    L = make_learner()
    x = raw_rows(3, 0)
    cases = [(lambda: L.observe_add(np.zeros(3), np.zeros(3), x, np.zeros(3), update_stats=False), _lib.B2G_ESTATE),
             (lambda: L.observe_act(x, update_stats=True, act=False), _lib.B2G_ESTATE),
             (lambda: L.act_raw(x), _lib.B2G_ESTATE),
             (lambda: L.obs_rms_get(), _lib.B2G_ESTATE)]
    for f, code in cases:
        with pytest.raises(_lib.B2GError) as e:
            f()
        assert e.value.code == code
    L.observe_act(x, update_stats=False, act=False)
    for f in (lambda: L.observe_act(None, n=3, eps=1.5),
              lambda: L.observe_act(None, n=2, eps=0.5),
              lambda: L.observe_add(np.zeros(2), np.zeros(2), x[:2], np.zeros(2), update_stats=False),
              lambda: L.observe_add(np.array([0, NA, 1], np.float32), np.zeros(3), x, np.zeros(3), update_stats=False),
              lambda: L.observe_add(np.array([0, 0.5, 1], np.float32), np.zeros(3), x, np.zeros(3), update_stats=False)):
        with pytest.raises(_lib.B2GError) as e:
            f()
        assert e.value.code == _lib.B2G_EINVAL
    assert L.replay_size() == 0
    L.close()
