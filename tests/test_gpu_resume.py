"""Training state on a real GPU (include/b200grasp.h: b2g_sac_state_save / _load, b2g_bdq_state_save / _load; training_state.py):
a restored learner holds bitwise the state of the one that saved it and takes the same next step, bad files are refused before
anything changes, and SAC / BDQ runs continue through save_training_state / load_training_state."""
import os

import numpy as np
import pytest

import b200grasp
from b200grasp import _lib
from tests.fake_env import FakeGraspEnv
from tests.test_gpu_replay_frames import N_ACT, _episodic_stream, _learner, _same_row
from tests.util import rel_err

pytestmark = pytest.mark.gpu

LR = 3e-4


def _fill(L, obs_shape, cap, lanes, u8, seed, steps_every=5):
    """An episodic stream with frequent episode ends through the learner, with graph-path steps along the way; returns the
    stream, positioned after the last call."""
    rng = np.random.default_rng(seed)
    stream = _episodic_stream(rng, obs_shape, lanes, 10 ** 6, p_done=0.3, u8=u8)
    for t in range(3 * cap // lanes):
        L.replay_add(*next(stream))
        if t >= 8 and t % steps_every == 0:
            L.step(2, lr=LR)
    return stream


def _assert_same_state(L, R, cap):
    pl, pr = L.get_parameters(), R.get_parameters()
    for n in pl:
        assert np.array_equal(pl[n].view(np.uint32), pr[n].view(np.uint32)), n
        if not n.startswith("target/"):
            (ml, vl), (mr, vr) = L.get_adam(n), R.get_adam(n)
            assert np.array_equal(ml.view(np.uint32), mr.view(np.uint32)) and np.array_equal(vl.view(np.uint32), vr.view(np.uint32)), n
    assert L.replay_info() == R.replay_info()
    n_live = 0
    for s in range(cap):
        try:
            a = L.replay_get(s)
        except _lib.B2GError:
            with pytest.raises(_lib.B2GError):
                R.replay_get(s)
            continue
        assert _same_row(a, R.replay_get(s)), s
        n_live += 1
    assert n_live == L.replay_size()


def _assert_same_engine_losses(mL, mR, bL, bR, B):
    """The first step of two handles in the same state, on the same batch and engine.  Their per-sample outputs differ only
    by the order in which the forward's fp32 atomics add (the same-engine bar of tests/test_gpu_graph_path.py, 2e-6).  Each
    loss is the sum of B per-sample terms, which the tail kernel also adds with fp32 atomics in either order, so two runs
    may differ by 2 (B + 6) 2^-24 sum|terms| (both runs' summation orders and each term's own roundings) plus what the
    per-sample differences move the loss by: to first order, by Cauchy-Schwarz, sqrt(2 L) rms(de) for a loss
    L = mean(e^2) / 2, and mean|d term| for the policy and entropy-coefficient losses."""
    f = {k: (bL[k].astype(np.float64), bR[k].astype(np.float64)) for k in ("q1", "q2", "v", "logp", "v_targ", "q1_pi", "q2_pi", "pi")}
    for k, (a, b) in f.items():
        assert rel_err(b, a) <= 2e-6, k
    d = {k: np.abs(a - b).reshape(B, -1).max(1) for k, (a, b) in f.items()}
    rms = lambda x: float(np.sqrt(np.mean(np.square(x))))
    alpha = float(mL["ent_coef"])
    log_alpha = float(np.log(np.float64(alpha)))
    logp, q1p = f["logp"][0], f["q1_pi"][0]
    te = -float(N_ACT)                                 # the Learner's default target entropy, -n_act
    de = {"qf1_loss": d["q1"] + d["v_targ"], "qf2_loss": d["q2"] + d["v_targ"],
          "value_loss": d["v"] + np.maximum(d["q1_pi"], d["q2_pi"]) + alpha * d["logp"]}
    terms = {k: abs(mL[k]) for k in de}               # these three sum non-negative terms
    move = {k: np.sqrt(2 * abs(mL[k])) * rms(de[k]) + 0.5 * float(np.mean(np.square(de[k]))) for k in de}
    terms["policy_loss"] = float(np.mean(np.abs(alpha * logp - q1p)))
    move["policy_loss"] = float(np.mean(alpha * d["logp"] + d["q1_pi"]))
    terms["ent_coef_loss"] = abs(log_alpha) * float(np.mean(np.abs(logp + te)))
    move["ent_coef_loss"] = abs(log_alpha) * float(np.mean(d["logp"]))
    for k in ("policy_loss", "qf1_loss", "qf2_loss", "value_loss", "ent_coef_loss"):
        bar = 1.01 * (2 * (B + 6) * 2.0 ** -24 * terms[k] + move[k])
        assert abs(mL[k] - mR[k]) <= bar, (k, mL[k], mR[k], bar)


def _resume_case(tmp_path, obs_shape, u8, prec_save, prec_load):
    cap, lanes, B = 64, 3, 16
    fc = cap + cap // 8 + lanes                       # tight: with an episode end every ~3 steps, transitions go early
    L = _learner(obs_shape, B, cap, prec_save, frame_capacity=fc, u8_planes=u8)
    stream = _fill(L, obs_shape, cap, lanes, u8, seed=7)
    info = L.replay_info()
    assert info["evicted_early"] > 0 and info["size"] > B
    path = str(tmp_path / "learner.state")
    L.save_state(path)
    R = _learner(obs_shape, B, cap, prec_load, frame_capacity=fc, u8_planes=u8)
    R.load_state(path)
    _assert_same_state(L, R, cap)
    before = L.get_parameters()
    mL, mR = L.step(1, lr=LR), R.step(1, lr=LR)
    bL, bR = L.last_batch(), R.last_batch()
    assert np.array_equal(bL["indices"], bR["indices"]) and np.array_equal(bL["eps"].view(np.uint32), bR["eps"].view(np.uint32))
    assert mL["n_updates"] == mR["n_updates"]
    same_engine = prec_save == prec_load
    if same_engine:
        _assert_same_engine_losses(mL, mR, bL, bR, B)
    else:
        for k in ("policy_loss", "qf1_loss", "qf2_loss", "value_loss", "ent_coef_loss"):   # the parity bar of test_gpu_parity.py
            assert abs(mL[k] - mR[k]) <= 1e-4 * max(abs(mL[k]), 1e-3), (k, mL[k], mR[k])
    if same_engine:
        # The two runs may sum the engine's atomics in another order, so their gradients agree only to rounding: within 1e-4
        # of each tensor's largest.  Adam (whose moments were bitwise equal before the step) carries a gradient that differs
        # in its last bits into an update that differs by lr_t * |m_L / (sqrt(v_L) + eps) - m_R / (sqrt(v_R) + eps)|, which is
        # large where the gradient is small; the stored weight can then round the other way (one ulp).  Every parameter must
        # lie within that, plus 1e-4 of its tensor's largest move.
        gL, gR = L.get_gradients(), R.get_gradients()
        for n in gL:
            assert np.abs(gL[n].astype(np.float64) - gR[n]).max() <= 1e-4 * np.abs(gL[n]).max(), n
        t = mL["n_updates"]
        lr_t = LR * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
        aL, aR = L.get_parameters(), R.get_parameters()
        for n in aL:
            moved = float(np.abs(aL[n].astype(np.float64) - before[n]).max())
            allow = 1e-4 * moved + np.spacing(np.abs(aL[n])).astype(np.float64)
            if n in gL:
                (m1, v1), (m2, v2) = (tuple(a.astype(np.float64) for a in X.get_adam(n)) for X in (L, R))
                allow = allow + 1.01 * lr_t * np.abs(m1 / (np.sqrt(v1) + 1e-8) - m2 / (np.sqrt(v2) + 1e-8))
            over = np.abs(aL[n].astype(np.float64) - aR[n]) - allow
            assert float(over.max()) <= 0, (n, float(over.max()), moved)
    else:
        for k in ("q1", "q2", "v", "logp"):
            assert rel_err(bR[k], bL[k]) <= 1e-4, k
    # the next call of the same episodes shares its obs frames on both handles alike
    row = next(stream)
    L.replay_add(*row)
    R.replay_add(*row)
    assert L.replay_info()["live_frames"] == R.replay_info()["live_frames"]
    assert L.replay_info() == R.replay_info()
    L.close()
    R.close()


def test_sac_depth_bf16x3_state_round_trip(tmp_path):
    _resume_case(tmp_path, (64, 64, 2), (), 1, 1)


def test_sac_rgbd_u8_planes_state_round_trip(tmp_path):
    _resume_case(tmp_path, (64, 64, 5), (0, 1, 2), 1, 1)


def test_sac_mlp_state_saved_at_bf16x3_loads_into_fp32(tmp_path):
    _resume_case(tmp_path, (101,), (), 1, 0)


def _bdq(seed=9, hidden=32):
    return b200grasp.BDQLearner(100, 3, 8, ((64, 64), (hidden,), (hidden,)), batch_size=32, buffer_size=256, gamma=0.99,
                                target_network_update_freq=7, prioritized_replay=True, prioritized_replay_alpha=0.6,
                                prioritized_replay_eps=1e-6, seed=seed)


def _bdq_rows(rng, n):
    return (rng.standard_normal((n, 100)).astype(np.float32), rng.integers(0, 8, (n, 3)).astype(np.float32),
            rng.standard_normal(n).astype(np.float32), rng.standard_normal((n, 100)).astype(np.float32),
            (rng.random(n) < 0.1).astype(np.float32))


def test_bdq_prioritized_state_round_trip(tmp_path):
    rng = np.random.default_rng(3)
    L = _bdq()
    for i in range(6):                                # 330 rows: the ring wraps
        L.replay_add(*_bdq_rows(rng, 55))
        L.set_per_beta(0.4 + 0.1 * i)
        L.step(3, lr=1e-3)
    path = str(tmp_path / "bdq.state")
    L.save_state(path)
    R = _bdq()
    R.load_state(path)
    pl, pr = L.get_parameters(), R.get_parameters()
    for n in pl:
        assert np.array_equal(np.asarray(pl[n]).view(np.uint32), np.asarray(pr[n]).view(np.uint32)), n
    assert L.replay_size() == R.replay_size() == 256
    # new rows enter the trees at the restored max priority; the trees and beta then decide the next draws and weights
    row = _bdq_rows(rng, 5)
    L.replay_add(*row)
    R.replay_add(*row)
    mL, mR = L.step(1, lr=1e-3), R.step(1, lr=1e-3)
    assert mL["n_updates"] == mR["n_updates"] == 19
    (sl, wl, ql), (sr, wr, qr) = L.last_per(), R.last_per()
    assert np.array_equal(sl, sr) and np.array_equal(wl.view(np.uint32), wr.view(np.uint32))
    assert np.allclose(ql, qr, rtol=1e-5, atol=0)
    assert abs(mL["loss"] - mR["loss"]) <= 1e-6 * abs(mL["loss"])
    L.close()
    R.close()


def test_refusals(tmp_path):
    cap, lanes, B = 64, 3, 16
    L = _learner((64, 64, 2), B, cap, 1, frame_capacity=cap + 16)
    _fill(L, (64, 64, 2), cap, lanes, (), seed=2)
    path = str(tmp_path / "a.state")
    L.save_state(path)
    # another configuration: B2G_EINVAL naming the field, the handle untouched and still usable
    W = b200grasp.Learner((64, 64, 2), n_act=N_ACT, hidden=128, batch_size=B, buffer_size=cap, seed=11, precision=1,
                          frame_capacity=cap + 16)
    W.replay_add(*next(_episodic_stream(np.random.default_rng(1), (64, 64, 2), 20, 1, 0.1)))
    before = W.get_parameters()
    with pytest.raises(_lib.B2GError, match="hidden") as e:
        W.load_state(path)
    assert e.value.code == _lib.B2G_EINVAL
    after = W.get_parameters()
    assert all(np.array_equal(before[n].view(np.uint32), after[n].view(np.uint32)) for n in before)
    W.step(1, lr=LR)
    W.close()
    # a truncated file is refused before any write
    R = _learner((64, 64, 2), B, cap, 1, frame_capacity=cap + 16)
    R.replay_add(*next(_episodic_stream(np.random.default_rng(1), (64, 64, 2), 20, 1, 0.1)))
    before = R.get_parameters()
    data = open(path, "rb").read()
    short = str(tmp_path / "short.state")
    open(short, "wb").write(data[:-1000])
    with pytest.raises(_lib.B2GError, match="truncated") as e:
        R.load_state(short)
    assert e.value.code == _lib.B2G_EINVAL
    after = R.get_parameters()
    assert all(np.array_equal(before[n].view(np.uint32), after[n].view(np.uint32)) for n in before)
    R.step(1, lr=LR)
    # a checksum failure after the writes began leaves the handle unusable until a load succeeds
    bad = str(tmp_path / "bad.state")
    flipped = bytearray(data)
    flipped[-5] ^= 0xFF
    open(bad, "wb").write(bytes(flipped))
    with pytest.raises(_lib.B2GError, match="checksum"):
        R.load_state(bad)
    with pytest.raises(_lib.B2GError) as e:
        R.step(1, lr=LR)
    assert e.value.code == _lib.B2G_ESTATE
    R.load_state(path)
    _assert_same_state(L, R, cap)
    R.close()
    # a host-pipelined step whose losses were not collected
    rng = np.random.default_rng(4)
    o = rng.random((B, 64, 64, 2), dtype=np.float32)
    a = rng.uniform(-1, 1, (B, N_ACT)).astype(np.float32)
    L.step_host_pipelined(o, a, np.zeros(B, np.float32), o, np.zeros(B, np.float32), rng.standard_normal((B, N_ACT)).astype(np.float32))
    with pytest.raises(_lib.B2GError, match="pipeline_flush") as e:
        L.save_state(path)
    assert e.value.code == _lib.B2G_ESTATE
    L.pipeline_flush()
    L.save_state(path)
    L.close()


def test_sac_learn_save_load_continue(tmp_path):
    def make(seed):
        return b200grasp.VecNormalize(b200grasp.DummyVecEnv([lambda: FakeGraspEnv(seed, horizon=8)]), norm_obs=True, norm_reward=True,
                                      clip_obs=10.0)
    env = make(1)
    model = b200grasp.SAC(b200grasp.CnnPolicy, env, policy_kwargs={"layers": [64, 64], "cnn_extractor": None}, buffer_size=200,
                          batch_size=16, learning_starts=30, seed=3, replay_frames=240)
    model.learn(total_timesteps=60)
    d = str(tmp_path / "run" / "training_state")
    model.save_training_state(d)
    assert sorted(os.listdir(d)) == ["host.json", "learner.state", "model.zip", "vecnormalize.pkl"]
    model.save_training_state(d)                      # replaces the previous checkpoint
    assert sorted(os.listdir(tmp_path / "run")) == ["training_state"]
    env2 = make(5)
    m2 = b200grasp.SAC.load_training_state(d, env2)
    assert m2.num_timesteps == 60 and m2.n_updates == model.n_updates == 31
    for a, b in ((env.obs_rms, env2.obs_rms), (env.ret_rms, env2.ret_rms)):
        assert np.array_equal(a.mean, b.mean) and np.array_equal(a.var, b.var) and a.count == b.count
    assert m2.learner.replay_info() == model.learner.replay_info()
    assert m2._rng.bit_generator.state == model._rng.bit_generator.state
    assert m2.replay_frames == 240 and m2.episode_rewards == model.episode_rewards

    def no_sample():
        raise AssertionError("random exploration after the resume")
    m2.action_space.sample = no_sample
    m2.learn(total_timesteps=20, reset_num_timesteps=False)
    assert m2.num_timesteps == 80 and m2.n_updates == 51
    assert m2.learner.replay_size() == 80
    model.close()
    m2.close()


def test_bdq_learn_save_load_continue(tmp_path):
    from b200grasp.spaces import Box

    class Env:
        observation_space = Box(-np.inf, np.inf, (100,))
        action_space = Box(-1.0, 1.0, (3,))

        def __init__(self, seed):
            self.rng = np.random.default_rng(seed); self.t = 0

        def reset(self):
            self.t = 0
            return self.rng.normal(size=100).astype(np.float32)

        def step(self, a):
            self.t += 1
            return self.rng.normal(size=100).astype(np.float32), float(a[0] > 0), self.t >= 10, {}

    kw = dict(policy_kwargs={"layers": [[64, 64], [32], [32]]}, num_actions_pad=8, batch_size=32, buffer_size=500, learning_starts=40,
              target_network_update_freq=20, prioritized_replay=True, exploration_fraction=0.5, seed=1)
    model = b200grasp.BDQ("MlpActPolicy", Env(0), **kw)
    model.learn(100)
    d = str(tmp_path / "state")
    model.save_training_state(d)
    m2 = b200grasp.BDQ.load_training_state(d, Env(1))
    assert m2.num_timesteps == 100 and m2.learner.replay_size() == 100
    seen = []
    eps_fn = m2._epsilon
    m2._epsilon = lambda t, total: seen.append((t, total)) or eps_fn(t, total)
    m2.learn(50, reset_num_timesteps=False)
    assert seen[0] == (100, 150) and seen[-1] == (149, 150) and m2.num_timesteps == 150
    # the schedule is the one a 150-step run follows: epsilon at step 100 of 150 with exploration over the first 75
    assert eps_fn(100, 150) == pytest.approx(kw.get("exploration_final_eps", 0.02))
    assert m2.learner.replay_size() == 150
    model.learner.close()
    m2.learner.close()
