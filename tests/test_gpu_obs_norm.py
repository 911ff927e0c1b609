"""VecNormalize's observation statistics on the device and the actor loop fed from one upload per frame
(include/b200grasp.h: b2g_sac_observe_act / _add, b2g_obs_rms_set / _get; ``SAC(device_obs_norm=True)``), held to the host
RunningMeanStd / VecNormalize and to the default ``learn`` path on a real GPU."""
import os

import numpy as np
import pytest

import b200grasp
from b200grasp import _lib
from b200grasp.sac_model import SAC, CnnPolicy
from b200grasp.vec_env import DummyVecEnv, RunningMeanStd, VecNormalize, sync_envs_normalization
from tests.fake_env import FakeGraspEnv
from tests.util import GOLD

pytestmark = pytest.mark.gpu

N_ACT = 5


def _learner(obs_shape, B=8, cap=64, **kw):
    L = b200grasp.Learner(obs_shape, n_act=N_ACT, batch_size=B, buffer_size=cap, seed=3, **kw)
    L.set_norm_stats(norm_obs=False, norm_reward=False)
    return L


def _frames(rng, obs_shape, n, u8=()):
    """Observations in the environment's layout: image planes (integers in [0, 255] on the 8-bit ones), and for images an
    actuator plane that is zero except pixel [0, 0]."""
    if len(obs_shape) == 1:
        return (rng.normal(3.0, 2.0, (n,) + obs_shape)).astype(np.float32)
    o = np.zeros((n,) + obs_shape, np.float32)
    o[..., :-1] = rng.uniform(0.0, 200.0, (n,) + obs_shape[:2] + (obs_shape[2] - 1,))
    for c in u8:
        o[..., c] = np.rint(o[..., c])
    o[:, 0, 0, -1] = rng.uniform(0, 1, n)
    return o


def _close(a, b):
    np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-300)


# ------------------------------------------------------------------------------------------------ 1. statistics
@pytest.mark.parametrize("obs_shape,u8,start", [((64, 64, 2), (), "zero"), ((64, 64, 2), (), "golden"),
                                                ((64, 64, 5), (0, 1, 2), "zero"), ((101,), (), "zero")])
def test_device_statistics_follow_running_mean_std(obs_shape, u8, start):
    rng = np.random.default_rng(11)
    pool = _frames(rng, obs_shape, 256, u8)
    host = RunningMeanStd(epsilon=0.0, shape=obs_shape)
    if start == "golden":
        g = np.load(os.path.join(GOLD, "vecnorm_sac_depth.npz"))
        host.mean, host.var, host.count = g["obs_mean"].copy(), g["obs_var"].copy(), float(g["obs_count"])
    L = _learner(obs_shape, u8_planes=u8, frame_capacity=64 + 64 if u8 else None)
    L.obs_rms_set(host.mean, host.var, host.count)
    for k in range(201):
        n = (1, 8, 128)[k % 3]
        batch = pool[rng.integers(0, len(pool), n)]
        host.update(batch)
        L.observe_act(batch, update_stats=True, act=False)
    mean, var, count = L.obs_rms_get()
    assert count == host.count
    _close(mean, host.mean)
    _close(var, host.var)
    # update_stats off: staged, not merged
    L.observe_act(pool[:4], update_stats=False, act=False)
    assert L.obs_rms_get()[2] == host.count
    L.close()


# ------------------------------------------------------------------------------------------------ 2. a whole run, 5. uploads
def _make_env(n_envs=4):
    venv = DummyVecEnv([(lambda i=i: FakeGraspEnv(seed=10 + i, horizon=20)) for i in range(n_envs)])
    return VecNormalize(venv, norm_obs=True, norm_reward=True, clip_obs=10.0)


def _run(device, steps, lr, replay_frames=None, learning_starts=100):
    """learn(steps) on 4 fake envs; returns the model, the actions the actor produced and the losses of every update."""
    model = SAC(CnnPolicy, _make_env(), policy_kwargs={"cnn_extractor": "augmented_nature_cnn"}, buffer_size=1000, batch_size=64,
                learning_rate=lr, learning_starts=learning_starts, seed=7, precision="fp32", replay_frames=replay_frames,
                device_obs_norm=device)
    acts, losses = [], []
    L = model.learner
    name = "observe_act" if device else "act"
    orig_act, orig_step = getattr(L, name), L.step_async

    def rec_act(*a, **k):
        out = orig_act(*a, **k)
        if out is not None:
            acts.append(out.copy())
        return out

    def rec_step(n, lr_):
        orig_step(n, lr_)
        losses.append(L.step(0, lr_))

    setattr(L, name, rec_act)
    L.step_async = rec_step
    model.learn(steps)
    return model, acts, losses


@pytest.mark.parametrize("replay_frames", [None, 1200])
def test_learn_is_the_same_run_with_the_statistics_on_the_device(replay_frames):
    host, a_h, _ = _run(False, 300, 0.0, replay_frames)
    dev, a_d, _ = _run(True, 300, 0.0, replay_frames)
    assert dev.get_vec_normalize_env().learner_owns_obs_rms and not host.get_vec_normalize_env().learner_owns_obs_rms
    # the same action at every step the actor decided
    assert len(a_h) == len(a_d) == (300 - 100) // 4
    for x, y in zip(a_h, a_d):
        np.testing.assert_allclose(x, y, rtol=0, atol=1e-6)
    # the same replay: raw frames, and the terminal observation in a finished env's transition
    Lh, Ld = host.learner, dev.learner
    ih, idv = Lh.replay_info(), Ld.replay_info()
    assert ih["size"] == idv["size"] == 300 and ih["live_frames"] == idv["live_frames"]
    n_done = 0
    for s in range(300):
        th, td = Lh.replay_get(s), Ld.replay_get(s)
        for k in ("obs", "next_obs", "act"):
            assert np.array_equal(th[k], td[k]), (s, k)
        assert th["rew"] == td["rew"] and th["done"] == td["done"]
        n_done += int(td["done"])
        if td["done"] and s + 4 < 300:        # the env's next transition starts from the reset frame, not the terminal one
            assert not np.array_equal(Ld.replay_get(s + 4)["obs"], td["next_obs"])
    assert n_done == 12
    # the same statistics
    rh, rd = host.get_vec_normalize_env().obs_rms, dev.get_vec_normalize_env().obs_rms
    assert rh.count == rd.count
    _close(rd.mean, rh.mean)
    _close(rd.var, rh.var)
    # the same sampled step: same Philox draw, same normalised batch through the same parameters
    host._sync_norm_stats()
    dev._sync_norm_stats()
    Lh.step(1, 0.0)
    Ld.step(1, 0.0)
    bh, bd = Lh.last_batch(), Ld.last_batch()
    assert np.array_equal(bh["indices"], bd["indices"]) and np.array_equal(bh["eps"], bd["eps"])
    for k in ("q1", "q2", "v", "logp", "v_targ"):
        np.testing.assert_allclose(bd[k], bh[k], rtol=1e-5, atol=1e-6)
    # uploads: every new frame crossed once (reset frames, one next_obs per env step, one reset frame per episode end) ...
    E, n_env, iters = 64 * 64 * 2, 4, 75
    up = Ld.upload_bytes()
    frames = n_env + iters * n_env + n_done
    assert up["observe"] == 2 * E * 8 + frames * E * 4 + iters * n_env * (N_ACT + 2) * 4
    assert up["other"] % 64 == 0 and up["other"] <= 64 * (2 * iters + 8)          # ... and the scalars of set_norm_stats
    # the default path: obs for the actor, obs and next_obs for the replay, float64 statistics twice a step
    assert Lh.upload_bytes()["observe"] == 0 and Lh.upload_bytes()["other"] > 2 * iters * n_env * E * 4 + 50 * n_env * E * 4
    host.close()
    dev.close()


def test_training_starts_like_the_default_path():
    """Default learning rate: both runs make the same updates and their first nine give the same losses.  Later updates are
    not compared: from the tenth on, two runs of the default path itself can separate (the step sums its gradients with
    atomics, and Adam's first steps are sensitive to their order).  The lr = 0 test above is the equivalence of the two paths
    with the parameters held still."""
    host, a_h, l_h = _run(False, 64 + 4 * 20, 3e-4, learning_starts=64)
    dev, a_d, l_d = _run(True, 64 + 4 * 20, 3e-4, learning_starts=64)
    assert len(l_h) == len(l_d) >= 20
    assert [m["n_updates"] for m in l_h] == [m["n_updates"] for m in l_d]
    for mh, md in zip(l_h[:9], l_d[:9]):
        for k in ("policy_loss", "qf1_loss", "qf2_loss", "value_loss"):
            assert abs(mh[k] - md[k]) <= 1e-5 * max(abs(mh[k]), 1e-3), (k, mh[k], md[k])
    host.close()
    dev.close()


# ------------------------------------------------------------------------------------------------ loaded models, predict, evaluation
def test_loaded_and_second_models_on_a_wrapped_env_predict_like_the_host_wrapper(tmp_path):
    from b200grasp.evaluation import evaluate_policy
    model, _, _ = _run(True, 120, 3e-4, learning_starts=64)
    vn = model.get_vec_normalize_env()
    zip_path, pkl = str(tmp_path / "m.zip"), str(tmp_path / "vecnormalize.pkl")
    model.save(zip_path)
    vn.save(pkl)
    raw = _frames(np.random.default_rng(5), (64, 64, 2), 1)

    # the model itself: its wrapper hands out raw observations and predict takes them as they are
    assert model.predict_takes_raw_obs
    ref = model.learner.act(raw, deterministic=True)
    np.testing.assert_allclose(model._scale_action(model.predict(raw[0])[0]), ref[0], rtol=0, atol=1e-6)

    # (the loads name the fp32 engine the run above trained with: across engines the actor agrees to 1e-5 only)
    # a second model on the owned env (train --load's parameter donor) reads the owner's statistics and leaves them in place
    donor = SAC.load(zip_path, model.get_env(), buffer_size=1, precision="fp32")
    assert donor.device_obs_norm and vn.obs_rms_owner is model.learner
    np.testing.assert_allclose(donor._scale_action(donor.predict(raw[0])[0]), ref[0], rtol=0, atol=1e-6)
    with pytest.raises(RuntimeError, match="owned by another"):
        donor.learn(8)
    donor.close()
    assert vn.obs_rms_owner is model.learner and vn.obs_rms.count == model.learner.obs_rms_get()[2]

    # the stable-baselines sequence: VecNormalize.load, SAC.load(zip, env), predict(env.reset()) -- against a model that keeps
    # the host wrapper
    def wrapped():
        e = VecNormalize.load(pkl, DummyVecEnv([lambda: FakeGraspEnv(seed=3, horizon=20)]))
        e.training = False
        return e

    env_d, env_h = wrapped(), wrapped()
    on_dev = SAC.load(zip_path, env_d, precision="fp32")
    on_host = SAC.load(zip_path, env_h, device_obs_norm=False, precision="fp32")
    assert env_d.learner_owns_obs_rms and not env_h.learner_owns_obs_rms
    o_d, o_h = env_d.reset(), env_h.reset()
    np.testing.assert_array_equal(o_d, env_h.get_original_obs())            # raw from the owned wrapper, normalised from the other
    np.testing.assert_allclose(on_dev.predict(o_d)[0], on_host.predict(o_h)[0], rtol=0, atol=1e-6)
    # evaluation on a host wrapper (EvalCallback's eval_env) with a model that owns its statistics
    ev_d, ev_h = wrapped(), wrapped()
    sync_envs_normalization(env_d, ev_d)
    r_d = evaluate_policy(on_dev, ev_d, n_eval_episodes=2, return_episode_rewards=True)
    r_h = evaluate_policy(on_host, ev_h, n_eval_episodes=2, return_episode_rewards=True)
    assert r_d == r_h
    # closing hands the statistics back: the wrapper works on, and saves, without the learner
    mean = env_d.obs_rms.mean.copy()
    on_dev.close()
    assert not env_d.learner_owns_obs_rms and type(env_d.obs_rms) is RunningMeanStd and np.array_equal(env_d.obs_rms.mean, mean)
    env_d.save(str(tmp_path / "after.pkl"))
    on_host.close()
    model.close()
    assert not vn.learner_owns_obs_rms


# ------------------------------------------------------------------------------------------------ 3. the auto-reset rule
def test_finished_env_stores_terminal_frame_merges_and_stages_reset_frame():
    shape = (64, 64, 2)
    rng = np.random.default_rng(4)
    o0, nxt, rst, nxt2 = (_frames(rng, shape, 2) for _ in range(4))
    L = _learner(shape, frame_capacity=64 + 16)
    host = RunningMeanStd(shape=shape)
    L.obs_rms_set(host.mean, host.var, host.count)
    L.set_norm_stats(None, None, 1.0, 10.0, 10.0, 1e-8, norm_obs=True, norm_reward=False)
    L.observe_act(o0, update_stats=True, act=False)
    host.update(o0)
    act = rng.uniform(-1, 1, (2, N_ACT)).astype(np.float32)
    L.observe_add(act, [1.0, 2.0], nxt, [0.0, 1.0], reset_obs=rst, update_stats=True)       # env 1 finishes on this step
    host.update(np.stack([nxt[0], rst[1]]))                # what the VecEnv returned: the reset frame, not the terminal one
    mean, var, count = L.obs_rms_get()
    assert count == host.count
    _close(mean, host.mean)
    _close(var, host.var)
    t0, t1 = L.replay_get(0), L.replay_get(1)
    assert np.array_equal(t0["obs"], o0[0]) and np.array_equal(t0["next_obs"], nxt[0]) and t0["done"] == 0.0
    assert np.array_equal(t1["obs"], o0[1]) and np.array_equal(t1["next_obs"], nxt[1]) and t1["done"] == 1.0      # terminal frame
    # the actor sees the staged frames: env 0 its next_obs, env 1 the reset frame
    a = L.observe_act(None, n=2, deterministic=True)
    ref = L.act(np.stack([nxt[0], rst[1]]), deterministic=True)
    np.testing.assert_allclose(a, ref, rtol=0, atol=1e-6)
    L.observe_add(act, [0.0, 0.0], nxt2, [0.0, 0.0], update_stats=True)
    t2, t3 = L.replay_get(2), L.replay_get(3)
    assert np.array_equal(t2["obs"], nxt[0]) and np.array_equal(t3["obs"], rst[1]) and np.array_equal(t3["next_obs"], nxt2[1])
    # env 0's frame was linked, env 1's reset frame stored: 2 + 2 frames for the first call, 1 + 2 for the second
    assert L.replay_info()["live_frames"] == 7
    L.close()


# ------------------------------------------------------------------------------------------------ 4. persistence
def test_vecnormalize_files_sync_and_training_state_carry_the_device_statistics(tmp_path):
    model, _, _ = _run(True, 160, 3e-4, replay_frames=1200, learning_starts=64)
    vn = model.get_vec_normalize_env()
    mean, var, count = model.learner.obs_rms_get()
    assert abs(count - (1e-4 + 4 + 160)) < 1e-9
    vn.save(str(tmp_path / "vecnormalize.pkl"))
    back = VecNormalize.load(str(tmp_path / "vecnormalize.pkl"), _make_env().venv)
    assert type(back.obs_rms) is RunningMeanStd and back.obs_rms.count == count
    assert np.array_equal(back.obs_rms.mean, mean) and np.array_equal(back.obs_rms.var, var)
    ev = _make_env()
    sync_envs_normalization(vn, ev)
    assert np.array_equal(ev.obs_rms.mean, mean) and ev.obs_rms.count == count and vn.learner_owns_obs_rms
    # a stopped run continues with the same statistics and the same actor
    state = model.save_training_state(str(tmp_path / "state"))
    again = SAC.load_training_state(state, _make_env())
    assert again.device_obs_norm and again.get_vec_normalize_env().learner_owns_obs_rms
    m2, v2, c2 = again.learner.obs_rms_get()
    assert c2 == count and np.array_equal(m2, mean) and np.array_equal(v2, var)
    probe = _frames(np.random.default_rng(9), (64, 64, 2), 4)
    np.testing.assert_allclose(model.learner.act(probe, deterministic=True), again.learner.act(probe, deterministic=True), rtol=0, atol=1e-6)
    a1 = model.learner.observe_act(probe, update_stats=True, deterministic=True)
    a2 = again.learner.observe_act(probe, update_stats=True, deterministic=True)
    np.testing.assert_allclose(a1, a2, rtol=0, atol=1e-6)
    _close(again.learner.obs_rms_get()[0], model.learner.obs_rms_get()[0])
    # files and handles with and without obs_rms do not mix; a default handle reads a default file as before
    plain, _, _ = _run(False, 80, 3e-4, replay_frames=1200, learning_starts=64)
    plain.learner.save_state(str(tmp_path / "plain.state"))
    for src, dst in ((os.path.join(state, "learner.state"), plain), (str(tmp_path / "plain.state"), again)):
        with pytest.raises(_lib.B2GError, match="obs_rms") as e:
            dst.learner.load_state(src)
        assert e.value.code == _lib.B2G_EINVAL
    before = plain.learner.act(probe, deterministic=True)
    plain.learner.load_state(str(tmp_path / "plain.state"))
    np.testing.assert_allclose(plain.learner.act(probe, deterministic=True), before, rtol=0, atol=1e-6)
    for m in (model, again, plain):
        m.close()


# ------------------------------------------------------------------------------------------------ refusals
def test_bad_arguments_return_codes():
    shape = (64, 64, 4)
    L = _learner(shape, u8_planes=(0,), frame_capacity=80)
    rng = np.random.default_rng(1)
    f = _frames(rng, shape, 2, u8=(0,))
    act = np.zeros((2, N_ACT), np.float32)

    def code(fn, *a, **k):
        with pytest.raises(_lib.B2GError) as e:
            fn(*a, **k)
        assert str(e.value).split(": ", 1)[1]              # a message comes with the code
        return e.value.code

    assert code(L.observe_add, act, [0, 0], f, [0, 0], update_stats=False) == _lib.B2G_ESTATE        # nothing staged yet
    assert code(L.observe_act, None, n=2) == _lib.B2G_ESTATE
    assert code(L.observe_act, f, update_stats=True, act=False) == _lib.B2G_ESTATE                     # no device statistics
    assert code(L.obs_rms_get) == _lib.B2G_ESTATE
    big = np.zeros((257,) + shape, np.float32)
    assert code(L.observe_act, big, update_stats=False, act=False) == _lib.B2G_EINVAL               # more than the staging
    ones = np.ones(shape)
    assert code(L.obs_rms_set, ones, ones, -1.0) == _lib.B2G_EINVAL
    neg = ones.copy()
    neg[3, 3, 1] = -0.5
    assert code(L.obs_rms_set, ones, neg, 1.0) == _lib.B2G_EINVAL
    assert code(L.obs_rms_set, ones * np.nan, ones, 1.0) == _lib.B2G_EINVAL
    L.obs_rms_set(0 * ones, ones, 1e-4)
    bad = f.copy()
    bad[1, 5, 5, 0] = 0.5                                   # not a byte value on the 8-bit plane
    assert code(L.observe_act, bad, update_stats=True, act=False) == _lib.B2G_EINVAL
    assert L.obs_rms_get()[2] == 1e-4                       # a refused call merged nothing
    L.observe_act(f, update_stats=True, act=False)
    assert code(L.observe_add, act, [0, 0], bad, [0, 0]) == _lib.B2G_EINVAL
    assert code(L.observe_add, act, [0, 1], f, [0, 1], reset_obs=None) == _lib.B2G_EINVAL            # finished, no reset frame
    assert code(L.observe_add, act[:1], [0], f[:1], [0]) == _lib.B2G_EINVAL                          # n differs from the staged
    assert L.replay_size() == 0 and L.obs_rms_get()[2] == 1e-4 + 2
    L.observe_add(act, [0, 0], f, [0, 0])
    assert L.replay_size() == 2
    L.close()
