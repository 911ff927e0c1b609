"""PPO2 / TRPO with VecNormalize's obs_rms on the device (``device_obs_norm=True``, b2g_ppo_observe_act / b2g_trpo_observe_act):
the float64 statistics against a host RunningMeanStd, every stored rollout row bit for bit against VecNormalize.normalize_obs
of the device's own statistics, learn() against the host-VecNormalize run fed the same statistics, predict, the encoder's
pass-raw stack, the upload counts, the training-state file and the refusals."""
import ctypes as C
import os

import numpy as np
import pytest

import b200grasp  # noqa: F401
from b200grasp import _lib, training_state
from b200grasp.encoders import SimpleAutoEncoder
from b200grasp.ppo2 import PPO2, PPO2Learner
from b200grasp.trpo_mpi import TRPO, TRPOLearner
from b200grasp.vec_env import DummyVecEnv, RunningMeanStd, VecEncodeDepth, VecNormalize, unwrap_encode_depth
from tests.deferred_env import PIXELS, FakeDeferredEnv
from tests.fake_env import FakeFlatEnv
from tests.test_encoder_cpu import load_fixture

pytestmark = pytest.mark.gpu


def _dbg(L, name):
    lib = _lib.load()
    n, eb = C.c_int64(), C.c_int32()
    _lib.check(getattr(lib, f"b2g_debug_{L._abi}_tensor_info")(L.h, name.encode(), C.byref(n), C.byref(eb)))
    out = np.empty(n.value, np.float32 if eb.value == 4 else np.int64)
    _lib.check(getattr(lib, f"b2g_debug_{L._abi}_tensor")(L.h, name.encode(), out.ctypes.data_as(C.c_void_p), out.nbytes))
    return out


def _learner(algo, D, E, T):
    if algo == "ppo":
        return PPO2Learner(D, 2, (8, 8), n_envs=E, n_steps=T, nminibatches=1, noptepochs=1, seed=7)
    return TRPOLearner(D, 2, (8, 8), timesteps_per_batch=T, vf_iters=0, seed=7)


def _update(L, algo, E, T):
    if algo == "ppo":
        return L.update(None, np.arange(E * T, dtype=np.int32)[None], 1e-3, 0.2, -1.0)
    return L.update(None, np.empty((0, T), np.int32))


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


CASES = [("ppo", E, D) for E in (1, 3, 16, 128) for D in (1, 5, 100, 8192)] + [("trpo", 1, D) for D in (1, 5, 100, 8192)]


@pytest.mark.parametrize("algo,E,D", CASES)
def test_statistics_and_stored_rows(algo, E, D):
    T, clip, eps = 3, 3.0, 1e-8
    L = _learner(algo, D, E, T)
    rng = np.random.default_rng(E * 10007 + D)
    host = RunningMeanStd(shape=(D,))
    host.mean, host.var, host.count = rng.normal(0, 1, D), rng.uniform(0.5, 2.0, D), 5.0
    L.obs_rms_set(host.mean, host.var, host.count)
    L.set_norm_stats(clip, eps, True)
    XS = (D + 3) // 4 * 4

    def frames():
        f = rng.normal(0, 1, (E, D)).astype(np.float32)
        f[rng.random((E, D)) < 0.05] *= 50.0          # some elements more than clip_obs standard deviations out
        return f

    def check(row, f, upd):
        if upd:
            host.update(f)
        m, v, c = L.obs_rms_get()
        np.testing.assert_allclose(m, host.mean, rtol=1e-12, atol=1e-300)
        np.testing.assert_allclose(v, host.var, rtol=1e-12, atol=1e-300)
        assert c == host.count
        want = np.float32(np.clip((f.astype(np.float64) - m) / np.sqrt(v + eps), -clip, clip))
        got = _dbg(L, "r_obs").reshape(T + 1, E, XS)[row]
        assert np.array_equal(_bits(got[:, :D]), _bits(want)), row
        assert not got[:, D:].any()                   # the pad columns stay zero
        return got[:, :D].copy()

    f = frames()
    assert L.observe_act(f, update_stats=True, act=False) is None
    rows = [check(0, f, True)]
    for t in range(T):
        a = L.observe_act(None)
        assert a.shape == (E, 2) and np.isfinite(a).all()
        f = frames()
        upd = t % 2 == 0
        L.observe_act(f, update_stats=upd, act=False)                   # after step t: row t + 1 (the last: row T)
        rows.append(check(t + 1, f, upd))
        L.rollout_reward(np.zeros(E, np.float32), np.zeros(E, np.float32))
    up = L.upload_bytes()
    assert up["observe"] == 2 * D * 8 + (T + 1) * E * D * 4             # obs_rms_set, then n * D * 4 per observe
    _update(L, algo, E, T)
    assert L.upload_bytes()["observe"] == up["observe"]                  # update(None) uploads no observation
    r = _dbg(L, "r_obs").reshape(T + 1, E, XS)
    assert np.array_equal(_bits(r[0, :, :D]), _bits(rows[T]))            # the next rollout starts from row T (TRPO: carried)
    if algo == "trpo":      # step 0 after the update: the boundary action drawn before it, on the carried row
        act0 = _dbg(L, "r_act").reshape(T + 1, 2)[0].copy()
        assert np.array_equal(L.observe_act(None).reshape(-1), act0)
    L.close()


class ScaledEnv(FakeFlatEnv):
    """FakeFlatEnv with frames spread over [-40, 40): statistics far from VecNormalize's initial ones."""

    def reset(self):
        return super().reset() * 80.0 - 40.0

    def step(self, action):
        o, r, d, i = super().step(action)
        return o * 80.0 - 40.0, r, d, i


class ReplayVecNormalize(VecNormalize):
    """A host VecNormalize whose obs_rms is overwritten, before every normalisation, with the statistics a device run had
    at that point."""
    queue = None

    def normalize_obs(self, obs):
        if self.queue is not None:
            self.obs_rms.mean, self.obs_rms.var = self.queue.pop(0)
        return super().normalize_obs(obs)


def _model(algo, device, queue=None):
    """A model on ScaledEnv's under a ReplayVecNormalize -> (model, the statistics after every device merge, the update
    metrics)."""
    E, D = (16, 100) if algo == "ppo" else (1, 100)
    venv = DummyVecEnv([lambda s=s: ScaledEnv(seed=s, horizon=6, obs_dim=D, n_act=2) for s in range(E)])
    vn = ReplayVecNormalize(venv)
    vn.queue = queue
    if algo == "ppo":
        m = PPO2("MlpPolicy", vn, n_steps=8, nminibatches=4, noptepochs=2, seed=3, policy_kwargs={"layers": [32, 16]},
                 device_obs_norm=device)
    else:
        m = TRPO("MlpPolicy", vn, timesteps_per_batch=256, vf_iters=2, seed=3, policy_kwargs={"layers": [32, 16]},
                 device_obs_norm=device)
    L, stats, metrics = m.learner, [], []
    if device:      # the statistics right after every merge, which the host run is then fed
        observe = L.observe_act

        def recording(obs, update_stats=True, act=True):
            out = observe(obs, update_stats=update_stats, act=act)
            if obs is not None:
                mean, var, _ = L.obs_rms_get()
                stats.append((mean.reshape(vn.observation_space.shape), var.reshape(vn.observation_space.shape)))
            return out
        L.observe_act = recording
    update = L.update
    L.update = lambda *a: metrics.append(update(*a)) or metrics[-1]
    return m, stats, metrics


def _learn(m, seed):
    """One rollout and update, the permutations drawn after np.random.seed(seed)."""
    np.random.seed(seed)
    m.learn(m.n_envs * 8 if isinstance(m, PPO2) else 256, reset_num_timesteps=False)
    return m


def _run(algo, device):
    m, stats, metrics = _model(algo, device)
    _learn(m, 11), _learn(m, 12)
    return m, stats, metrics


@pytest.mark.parametrize("algo", ["ppo", "trpo"])
def test_learn_is_the_host_run_fed_the_same_statistics(algo):
    d, stats, md = _model(algo, True)
    h, _, mh = _model(algo, False, queue=stats)     # consumed as the device run appends to it
    _learn(d, 11), _learn(h, 11)
    # up to the first optimiser step everything is a function of the same inputs: bit for bit.  PPO2's update metrics are
    # means over its minibatches' first forward passes; TRPO's iteration steps (CG, line search, value Adam) before it reports,
    # and then writes row 0's value under the updated value tower, so those agree to the rounding of the engine's atomics.
    assert len(md) == len(mh) == 1 and not stats
    if algo == "ppo":
        assert md == mh
    else:
        for k, v in md[0].items():
            np.testing.assert_allclose(v, mh[0][k], rtol=1e-4, atol=1e-6, err_msg=k)
    rd_, rh_ = d.learner.rollout_get(), h.learner.rollout_get()
    for k, v in rd_.items():
        skip = 1 if algo == "trpo" and k == "values" else 0
        bad = np.argwhere(_bits(v[skip:]) != _bits(rh_[k][skip:]))
        assert not bad.size, (k, bad[:5].tolist())
    for name in ("r_act", "r_val", "r_nlp", "r_rew", "r_done"):
        skip = 1 if algo == "trpo" and name == "r_val" else 0
        assert np.array_equal(_bits(_dbg(d.learner, name)[skip:]), _bits(_dbg(h.learner, name)[skip:])), name
    T, E = (8, 16) if algo == "ppo" else (256, 1)
    rd, rh = (_dbg(m.learner, "r_obs").reshape(T + 1, E, -1) for m in (d, h))
    assert np.array_equal(_bits(rd[1:]), _bits(rh[1:]))          # row 0: the device run already holds the next rollout's
    assert np.array_equal(_bits(rd[0]), _bits(rd[T]))
    # a second update: the engine's split-R and column-sum atomics make two runs agree to rounding once the optimiser has
    # stepped (test_gpu_ppo.py's bar for a continued run)
    _learn(d, 12), _learn(h, 12)
    assert len(mh) == 2 and not stats
    for k, v in d.learner.get_parameters().items():
        dd = np.abs(v.astype(np.float64) - h.learner.get_parameters()[k])
        assert np.quantile(dd, 0.99) <= 1e-5 and dd.max() <= 1e-3, (k, np.quantile(dd, 0.99), dd.max())
    assert np.array_equal(d.get_vec_normalize_env().ret_rms.var, h.get_vec_normalize_env().ret_rms.var)
    d.close(), h.close()


@pytest.mark.parametrize("algo", ["ppo", "trpo"])
def test_predict_normalises_as_the_wrapper_then_predicts(algo, tmp_path):
    m, _, _ = _run(algo, True)
    vn, L = m.get_vec_normalize_env(), m.learner
    assert m.predict_takes_raw_obs
    raw = np.random.default_rng(2).uniform(-60, 60, (5, 100)).astype(np.float32)
    low, high = m.action_space.low, m.action_space.high
    for det in (True, False):
        L.save_state(str(tmp_path / "s"))              # the noise counter, so both arms draw the same stream-1 noise
        a_dev = m.predict(raw, deterministic=det)[0]
        L.load_state(str(tmp_path / "s"))
        a_host = np.clip(L.act(np.asarray(vn.normalize_obs(raw), np.float32), deterministic=det)[0], low, high)
        assert np.array_equal(_bits(a_dev), _bits(a_host)), det
    # evaluate_policy through a host-normalising evaluation wrapper hands the raw copy to such a model
    from b200grasp.evaluation import evaluate_policy
    from b200grasp.vec_env import sync_envs_normalization
    ev = VecNormalize(DummyVecEnv([lambda: ScaledEnv(seed=9, horizon=4, obs_dim=100, n_act=2)]), training=False)
    sync_envs_normalization(vn, ev)
    r, n = evaluate_policy(m, ev, n_eval_episodes=2, return_episode_rewards=True)
    assert n == [4, 4]
    m.close()


def _stack(algo, enc, tail=1):
    E = 4 if algo == "ppo" else 1
    venv = DummyVecEnv([(lambda i=i: FakeDeferredEnv(seed=i, horizon=5, tail=tail, n_act=3)) for i in range(E)])
    return VecNormalize(VecEncodeDepth(venv, enc), norm_obs=True, norm_reward=True)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
@pytest.mark.parametrize("algo", ["ppo", "trpo"])
def test_encoder_pass_raw_is_the_host_mode_run(algo, precision):
    from b200grasp.encoders import keras_encoder_arrays
    w, cfg = load_fixture()
    enc = SimpleAutoEncoder(cfg, max_batch=16, precision=precision)
    enc.set_weights(keras_encoder_arrays(w, len(cfg["network"])))
    models = []
    for raw in (True, False):
        env = _stack(algo, enc)
        if algo == "ppo":
            m = PPO2("MlpPolicy", env, n_steps=8, nminibatches=2, noptepochs=2, seed=1, device_obs_norm=True)
        else:
            m = TRPO("MlpPolicy", env, timesteps_per_batch=128, vf_iters=1, seed=1, device_obs_norm=True)
        assert unwrap_encode_depth(env).pass_raw and unwrap_encode_depth(env).encoder_owner is m.learner
        if not raw:         # the same stack encoding in the wrapper: the learner keeps the statistics
            m.learner.set_obs_encoder(None)
            unwrap_encode_depth(env).take_encoder_back()
        np.random.seed(5)
        m.learn(2 * m.n_envs * (8 if algo == "ppo" else 128))
        models.append(m)
    p, h = models
    for x, y in zip(p.learner.obs_rms_get(), h.learner.obs_rms_get()):
        assert np.array_equal(x, y)
    # the stored rows are bit for bit the host-mode rows (the frames do not depend on the actions); the parameters after two
    # updates agree to the rounding of the engine's atomics (test_learn_is_the_host_run_fed_the_same_statistics)
    assert np.array_equal(_bits(_dbg(p.learner, "r_obs")), _bits(_dbg(h.learner, "r_obs")))
    for k, v in p.learner.get_parameters().items():
        dd = np.abs(v.astype(np.float64) - h.learner.get_parameters()[k])
        assert np.quantile(dd, 0.99) <= 1e-5 and dd.max() <= 1e-3, (k, np.quantile(dd, 0.99), dd.max())
    # only raw frames cross on the observe path: (reset + one per step) x n_envs raw rows, after obs_rms_set
    D = cfg["encoding_dim"] + 1
    steps = 2 * (8 if algo == "ppo" else 128)
    assert p.learner.upload_bytes()["observe"] == 2 * D * 8 + (1 + steps) * p.n_envs * (PIXELS + 1) * 4
    for m in models:
        m.close()


@pytest.mark.parametrize("algo", ["ppo", "trpo"])
def test_training_state_round_trip_and_cross_kind_refusal(algo, tmp_path):
    m, _, _ = _run(algo, True)
    m.save_training_state(str(tmp_path / "st"))
    mean, var, count = m.learner.obs_rms_get()
    E = m.n_envs
    venv = DummyVecEnv([lambda s=s: ScaledEnv(seed=s, horizon=6, obs_dim=100, n_act=2) for s in range(E)])
    cls = PPO2 if algo == "ppo" else TRPO
    r = cls.load_training_state(str(tmp_path / "st"), VecNormalize(venv))
    assert r.device_obs_norm and r.get_vec_normalize_env().obs_rms_owner is r.learner
    m2, v2, c2 = r.learner.obs_rms_get()
    assert np.array_equal(m2, mean) and np.array_equal(v2, var) and c2 == count
    r.learn(r.n_envs * (8 if algo == "ppo" else 256), reset_num_timesteps=False)
    assert r.learner.obs_rms_get()[2] > count
    # a handle without device statistics refuses the file, naming obs_rms; and the reverse
    if algo == "ppo":
        plain = PPO2Learner(100, 2, (32, 16), n_envs=E, n_steps=8, nminibatches=4, noptepochs=2, seed=3)
    else:
        plain = TRPOLearner(100, 2, (32, 16), timesteps_per_batch=256, vf_iters=2, seed=3)
    with pytest.raises(_lib.B2GError, match="obs_rms"):
        plain.load_state(os.path.join(str(tmp_path / "st"), training_state.STATE_FILE))
    plain.save_state(str(tmp_path / "plain.state"))
    with pytest.raises(_lib.B2GError, match="obs_rms"):
        r.learner.load_state(str(tmp_path / "plain.state"))
    plain.close(), r.close(), m.close()


@pytest.mark.parametrize("algo", ["ppo", "trpo"])
def test_refusals(algo):
    lib = _lib.load()
    E, T, D = (3, 2, 5) if algo == "ppo" else (1, 2, 5)
    L = _learner(algo, D, E, T)
    fn = getattr(lib, f"b2g_{algo}_observe_act")
    obs = np.zeros((E + 1, D), np.float32)
    fp = obs.ctypes.data_as(C.POINTER(C.c_float))
    assert fn(L.h, None, E, 0, None) == _lib.B2G_EINVAL                       # nothing to do
    assert fn(L.h, fp, E + 1, 0, None) == _lib.B2G_EINVAL                     # n != n_envs
    assert fn(L.h, fp, E, 1, None) == _lib.B2G_ESTATE                         # update_stats without device statistics
    assert L.steps()[2] == 0 and L.upload_bytes()["observe"] == 0             # refused before any upload
    for _ in range(T):      # a full rollout through the host path: nothing staged in the bootstrap row
        L.rollout_act(obs[:E] if algo == "ppo" else obs[0])
        L.rollout_reward(np.zeros(E, np.float32), np.zeros(E, np.float32))
    with pytest.raises(_lib.B2GError) as e:
        _update(L, algo, E, T)
    assert e.value.code == _lib.B2G_EINVAL
    w, cfg = load_fixture()
    from b200grasp.encoders import keras_encoder_arrays
    enc = SimpleAutoEncoder(cfg, max_batch=4)
    enc.set_weights(keras_encoder_arrays(w, len(cfg["network"])))
    with pytest.raises(_lib.B2GError) as e:                                    # encoding_dim + tail != obs_dim
        L.set_obs_encoder(enc, 1)
    assert e.value.code == _lib.B2G_EINVAL
    L.close()
