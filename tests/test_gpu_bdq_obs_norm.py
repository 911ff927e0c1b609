"""BDQ with VecNormalize's observation statistics on the device and the epsilon-greedy actor fed from one upload per frame
(include/b200grasp.h: b2g_bdq_observe_act / _add, b2g_bdq_obs_rms_set / _get; ``BDQ(device_obs_norm=True)``), held to the
host RunningMeanStd / VecNormalize, to the explicit step on host-normalised rows, and to the restated Philox stream 3."""
import struct

import numpy as np
import pytest

from b200grasp import BDQ, _lib
from b200grasp.spaces import Box
from b200grasp.vec_env import DummyVecEnv, RunningMeanStd, VecNormalize
from oracle import philox_ref as PX
from tests.test_bdq_obs_norm_cpu import explore
from tests.test_gpu_bdq_configs import Case, make_learner_bdq, make_params, near_ties
from tests.util import rel_err

pytestmark = pytest.mark.gpu

OBS, D, NB = 12, 3, 9
LAYERS = [[32, 16], [8], [8]]


# ------------------------------------------------------------------------------------------------ fixtures
class FlatEnv:
    """Flat observations with a feature that spikes far past clip_obs, a constant (zero-variance) one, and rewards that
    reach past clip_reward; episodes of `horizon` steps."""

    def __init__(self, seed, horizon):
        self.observation_space = Box(-np.inf, np.inf, (OBS,))
        self.action_space = Box(-1.0, 1.0, (D,))
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
        return self._obs(), float(self.rng.normal(0.0, 30.0)), self.t >= self.horizon, {}


class Recorder:
    """A VecEnv in front of DummyVecEnv that keeps every array it hands to VecNormalize."""

    def __init__(self, venv):
        self.venv, self.num_envs = venv, venv.num_envs
        self.observation_space, self.action_space = venv.observation_space, venv.action_space
        self.resets, self.steps = [], []

    def reset(self):
        o = self.venv.reset()
        self.resets.append(o.copy())
        return o

    def step_async(self, a):
        self.venv.step_async(a)

    def step_wait(self):
        o, r, d, infos = self.venv.step_wait()
        self.steps.append((o.copy(), r.copy(), d.copy(), [dict(i) for i in infos]))
        return o, r, d, infos

    @property
    def buf_infos(self):
        return self.venv.buf_infos


def make_env(n_envs, seed=0, clip_obs=10.0, clip_reward=10.0):
    rec = Recorder(DummyVecEnv([(lambda i=i: FlatEnv(seed + 100 * i, 3 + i % 5)) for i in range(n_envs)]))
    return VecNormalize(rec, norm_obs=True, norm_reward=True, clip_obs=clip_obs, clip_reward=clip_reward), rec


def make_model(env, **kw):
    args = dict(buffer_size=2048, batch_size=16, learning_starts=24, learning_rate=1e-3, prioritized_replay=True,
                num_actions_pad=NB, policy_kwargs={"layers": LAYERS}, seed=3, target_network_update_freq=50, device_obs_norm=True)
    args.update(kw)
    return BDQ("MlpActPolicy", env, **args)


def sections(path):
    """{tag: bytes} of a training-state file (csrc/state.cu: 32-byte header, 40-byte fingerprint fields, 32-byte entries)."""
    with open(path, "rb") as f:
        raw = f.read()
    n_fp, n_sec = struct.unpack_from("<II", raw, 16)
    out = {}
    for i in range(n_sec):
        tag, _, off, nb, _ = struct.unpack_from("<IIQQQ", raw, 32 + 40 * n_fp + 32 * i)
        out[tag.to_bytes(4, "little").decode()] = raw[off:off + nb]
    return out


def replay_rows(L, tmp_path, cap):
    p = str(tmp_path / "rows.state")
    L.save_state(p)
    s = sections(p)
    f = lambda k: np.frombuffer(s[k], np.float32)
    return dict(obs=f("ROBS").reshape(-1, OBS), next_obs=f("RNXT").reshape(-1, OBS), act=f("RACT").reshape(cap, D), rew=f("RREW"),
                done=f("RDON")), s


def host_statistics(rec):
    """VecNormalize's own rule on the host: reset frames, then every frame step_wait returned (a finished env's reset frame)."""
    rms = RunningMeanStd(shape=(OBS,))
    for o in rec.resets:
        rms.update(o)
    for o, *_ in rec.steps:
        rms.update(o)
    return rms


def assert_stats(L, rms):
    mean, var, count = L.obs_rms_get()
    assert count == rms.count
    assert np.abs(mean - rms.mean).max() <= 1e-12 * np.abs(rms.mean).max()
    assert np.abs(var - rms.var).max() <= 1e-12 * np.abs(rms.var).max()


# ------------------------------------------------------------------------------------------------ statistics, replay, uploads
@pytest.mark.parametrize("n_envs", [1, 3, 16])
def test_learn_merges_vecnormalize_frames_and_stores_raw_transitions(n_envs, tmp_path):
    env, rec = make_env(n_envs)
    model = make_model(env)
    L = model.learner
    acts = []
    orig = L.observe_act

    def rec_act(*a, **k):
        out = orig(*a, **k)
        if out is not None:
            acts.append(out.copy())
        return out
    L.observe_act = rec_act
    iters = 96 // n_envs + 5
    model.learn(iters * n_envs)
    assert env.learner_owns_obs_rms and len(acts) == iters == len(rec.steps)
    assert_stats(L, host_statistics(rec))
    # the replay: the env's original arrays, the terminal observation as a finished env's next_obs
    cap = 2048
    rows, _ = replay_rows(L, tmp_path, cap)
    assert L.replay_size() == iters * n_envs
    cur = rec.resets[0]
    n_done = 0
    for k, (o, r, d, infos) in enumerate(rec.steps):
        for i in range(n_envs):
            s = k * n_envs + i
            nxt = infos[i]["terminal_observation"] if d[i] else o[i]
            assert np.array_equal(rows["obs"][s], cur[i]), (k, i)
            assert np.array_equal(rows["next_obs"][s], nxt), (k, i)
            assert np.array_equal(rows["act"][s], acts[k][i].astype(np.float32)), (k, i)
            assert rows["rew"][s] == np.float32(r[i]) and rows["done"][s] == float(d[i]), (k, i)
        n_done += int(d.sum())
        cur = o
    assert n_done > 0
    # uploads: the statistics once, the reset frames, one frame per env step, one per finished env, and act / rew / done
    E = OBS * 4
    up = L.upload_bytes()
    assert up["observe"] == 2 * OBS * 8 + n_envs * E + iters * n_envs * (E + (D + 2) * 4) + n_done * E, up
    assert up["other"] % 64 == 0
    model.close()
    assert not env.learner_owns_obs_rms


# ------------------------------------------------------------------------------------------------ sample-time normalisation
def test_sampled_step_normalises_with_the_statistics_of_that_step(tmp_path):
    """Sampled steps of the device path against the explicit step on the same rows normalised on the host with
    VecNormalize.normalize_obs / normalize_reward and the statistics current at that step: observations past both clips, a
    zero-variance feature, rewards past clip_reward.  The statistics move on between the steps."""
    env, _ = make_env(4, seed=7, clip_obs=1.0, clip_reward=0.3)
    model = make_model(env, learning_starts=10 ** 9)
    model.learn(4 * 40)
    L = model.learner
    var = np.array(env.obs_rms.var, copy=True)
    var[1] = 0.0                                   # a zero-variance feature (count kept)
    env.obs_rms.var = var
    for it in range(3):
        model._sync_norm_stats()
        rows, _ = replay_rows(L, tmp_path, 2048)
        pre = L.get_parameters()
        m = L.step(1, lr=1e-3)
        g_dev = L.get_gradients()
        slots, w, prio = L.last_per()
        x, xn = env.normalize_obs(rows["obs"][slots]), env.normalize_obs(rows["next_obs"][slots])
        r = env.normalize_reward(rows["rew"][slots])
        assert (x == 1.0).any() and (x == -1.0).any() and (np.abs(x) < 1.0).any()
        assert (np.abs(r) == 0.3).any() and (np.abs(r) < 0.3).any()
        post = L.get_parameters()
        L.load_parameters(pre)
        L.set_norm_stats(norm_obs=False, norm_reward=False)      # the explicit batch arrives normalised
        out = L.step_explicit(x, rows["act"][slots], r, xn, rows["done"][slots], weights=w, lr=1e-3, apply_update=False)
        g_exp = L.get_gradients()
        L.load_parameters(post)
        for k in ("loss", "mean_q"):
            assert abs(out[k] - m[k]) <= 1e-4 * abs(out[k]), (it, k, out[k], m[k])
        np.testing.assert_allclose(prio, np.abs(out["td"]).sum(1) + 1e-6, rtol=1e-4)
        for nm in g_exp:
            assert rel_err(g_dev[nm], g_exp[nm]) <= 1e-3, (it, nm)
        model.learn(4 * 3, reset_num_timesteps=False)
    model.close()


# ------------------------------------------------------------------------------------------------ the actor
def _actor_learner(B=8):
    case = Case("actor", OBS, D, NB, 32, 16, 8, B, seed=71)
    L = make_learner_bdq(case, buffer_size=256, seed=5)
    params = make_params(case)
    L.load_parameters(params)
    return L, case, params


def test_actor_greedy_and_exploration_follow_the_host_and_stream_3():
    L, case, params = _actor_learner()
    rng = np.random.default_rng(3)
    mean, var = rng.normal(0.5, 1.0, OBS), rng.uniform(0.5, 4.0, OBS)
    mean[0], var[0] = -40.0, 1.0                  # -> past +clip
    var[1] = 0.0                                  # zero variance
    L.obs_rms_set(mean, var, 10.0)
    L.set_norm_stats(None, None, 1.0, 5.0, 10.0, 1e-8, norm_obs=True, norm_reward=False)
    vn = VecNormalize(DummyVecEnv([lambda: FlatEnv(0, 3)]), clip_obs=5.0)
    vn.obs_rms.mean, vn.obs_rms.var = mean, var
    key = PX.train_seed(5)
    n = 21                                        # three chunks of the batch of 8, a short last one
    raw = rng.normal(0.5, 2.0, (n, OBS)).astype(np.float32)
    raw[:, 1] = 2.0
    xn = vn.normalize_obs(raw).astype(np.float32)
    assert (xn[:, 0] == 5.0).all()
    greedy = L.observe_act(raw, update_stats=False, eps=0.0)          # acting call 0
    L.set_norm_stats(None, None, 1.0, 5.0, 10.0, 1e-8, norm_obs=False, norm_reward=False)
    ref = L.act(xn)                                                   # b2g_bdq_act on host-normalised observations
    L.set_norm_stats(None, None, 1.0, 5.0, 10.0, 1e-8, norm_obs=True, norm_reward=False)
    ties = {(b, d): c for b, d, c in near_ties(params, xn, case.cfg)}
    for b in range(n):
        for d in range(D):
            if (b, d) in ties:
                assert greedy[b, d] in ties[(b, d)] and ref[b, d] in ties[(b, d)]
            else:
                assert greedy[b, d] == ref[b, d], (b, d)
    seen = 0
    for step, eps in ((1, 1.0), (2, 0.3), (3, 0.3), (4, 0.0)):
        got = L.observe_act(None, n=n, eps=eps)
        go, bins = explore(key, step, n, D, NB, eps)
        assert np.array_equal(got[go], bins[go]), step
        assert np.array_equal(got[~go], greedy[~go]), step
        seen += int(go.sum())
        if eps == 1.0:
            assert go.all()
    assert 0 < seen < 3 * n * D
    L.close()


# ------------------------------------------------------------------------------------------------ prioritised replay
def test_new_rows_enter_the_trees_at_the_running_max_priority(tmp_path):
    """After observe_add the new leaves of the sum and min trees hold max_prio^alpha, as replay_add writes them; once a
    sampled step has raised max_prio the next rows take the new value."""
    per = Case("actor_per", OBS, D, NB, 32, 16, 8, 8, per=True, seed=71)
    L2 = make_learner_bdq(per, buffer_size=256, seed=5, prioritized_replay_alpha=0.6)
    R2 = make_learner_bdq(per, buffer_size=256, seed=5, prioritized_replay_alpha=0.6)
    rng = np.random.default_rng(8)
    n = 10
    o0 = rng.normal(size=(n, OBS)).astype(np.float32)
    L2.observe_act(o0, update_stats=False, act=False)
    cur = o0
    for k in range(3):
        nx = rng.normal(size=(n, OBS)).astype(np.float32)
        a = rng.integers(0, NB, (n, D)).astype(np.float32)
        r, d = rng.normal(size=n).astype(np.float32), np.zeros(n, np.float32)
        L2.observe_add(a, r, nx, d, update_stats=False)
        R2.replay_add(cur, a, r, nx, d)
        cur = nx
        pa, pb = str(tmp_path / "a.state"), str(tmp_path / "b.state")
        L2.save_state(pa)
        R2.save_state(pb)
        sa, sb = sections(pa), sections(pb)
        # the same rows; before any sampled step the same trees (afterwards each learner's own td errors drive them)
        for tag in ("ROBS", "RNXT", "RACT", "RREW", "RDON") + (("PERT", "PERS") if k == 0 else ()):
            assert sa[tag] == sb[tag], (k, tag)
        tsum = np.frombuffer(sa["PERT"], np.float64)
        C = tsum.size // 4
        max_prio = np.frombuffer(sa["PERS"], np.float32)[0]
        leaves = tsum[C + k * n:C + (k + 1) * n]
        np.testing.assert_allclose(leaves, np.float64(max_prio) ** np.float64(np.float32(0.6)), rtol=1e-15)
        for x in (L2, R2):
            x.step(1, lr=1e-3)
    assert np.frombuffer(sections(pa)["PERS"], np.float32)[0] > 1.0
    L2.close()
    R2.close()


# ------------------------------------------------------------------------------------------------ resume
def test_save_load_continue_equals_an_uninterrupted_run(tmp_path):
    env_a, _ = make_env(3, seed=11)
    env_b, _ = make_env(3, seed=11)
    a, b = make_model(env_a), make_model(env_b)
    a.learn(60)
    b.learn(60)
    state = b.save_training_state(str(tmp_path / "state"))
    b.close()
    b = BDQ.load_training_state(state, env_b)
    assert b.device_obs_norm and env_b.learner_owns_obs_rms
    a.learn(60, reset_num_timesteps=False)
    b.learn(60, reset_num_timesteps=False)
    pa, pb = a.learner.get_parameters(), b.learner.get_parameters()
    for nm in pa:
        np.testing.assert_allclose(pb[nm], pa[nm], rtol=0, atol=1e-6, err_msg=nm)
    for m, f in ((a, "a.state"), (b, "b.state")):
        m.learner.save_state(str(tmp_path / f))
    sa, sb = sections(str(tmp_path / "a.state")), sections(str(tmp_path / "b.state"))
    assert sa["ORMS"] == sb["ORMS"] and sa["CNTR"][:8 * 6] == sb["CNTR"][:8 * 6] and sa["CNTR"][56:] == sb["CNTR"][56:]
    for tag in ("ROBS", "RNXT", "RACT", "RREW", "RDON"):
        assert sa[tag] == sb[tag], tag
    np.testing.assert_allclose(np.frombuffer(sb["PERT"], np.float64), np.frombuffer(sa["PERT"], np.float64), rtol=1e-5)
    # a default handle writes no obs_rms and loads its own file; files do not cross the fingerprint difference
    plain = make_model(make_env(3, seed=11)[0], device_obs_norm=False)
    plain.learn(30)
    plain.learner.save_state(str(tmp_path / "plain.state"))
    assert "ORMS" not in sections(str(tmp_path / "plain.state"))
    before = plain.learner.get_parameters()
    plain.learner.load_state(str(tmp_path / "plain.state"))
    for nm, v in plain.learner.get_parameters().items():
        assert np.array_equal(v, before[nm])
    for src, dst in ((str(tmp_path / "a.state"), plain), (str(tmp_path / "plain.state"), a)):
        with pytest.raises(_lib.B2GError, match="obs_rms") as e:
            dst.learner.load_state(src)
        assert e.value.code == _lib.B2G_EINVAL
    for m in (a, b, plain):
        m.close()


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals():
    plain_env = DummyVecEnv([lambda: FlatEnv(0, 4)])
    m = make_model(plain_env)
    with pytest.raises(RuntimeError, match="VecNormalize"):
        m.learn(8)
    m.close()
    env, _ = make_env(2)
    owner = make_model(env)
    second = make_model(env)
    assert env.obs_rms_owner is owner.learner
    with pytest.raises(RuntimeError, match="owned by another"):
        second.learn(8)
    second.close()
    assert env.obs_rms_owner is owner.learner
    L = owner.learner
    with pytest.raises(_lib.B2GError) as e:
        L.observe_act(None, n=2, eps=1.5)
    assert e.value.code == _lib.B2G_EINVAL
    owner.close()
    L2, _, _ = _actor_learner()
    with pytest.raises(_lib.B2GError) as e:
        L2.obs_rms_get()
    assert e.value.code == _lib.B2G_ESTATE
    with pytest.raises(_lib.B2GError) as e:
        L2.observe_act(np.zeros((2, OBS), np.float32), update_stats=True, act=False)
    assert e.value.code == _lib.B2G_ESTATE
    L2.close()
