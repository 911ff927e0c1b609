"""The perception encoder on the learners' observe path (b2g_sac_set_obs_encoder / b2g_bdq_set_obs_encoder, VecEncodeDepth's
pass-raw mode): the device stage encodes exactly what the encoder handle encodes, reads only what it must, uploads only raw
frames, and SAC.learn / BDQ.learn run the same as on host-encoded observations."""
import json
import os

import numpy as np
import pytest
import torch
import yaml

import b200grasp  # noqa: F401
from b200grasp import BDQ, SAC, _lib, synth, train_cli
from b200grasp.bdq import BDQLearner
from b200grasp.encoders import SimpleAutoEncoder, keras_encoder_arrays, keras_layer_names
from b200grasp.learner import Learner
from b200grasp.sac_model import MlpPolicy
from b200grasp.vec_env import DummyVecEnv, VecEncodeDepth, VecNormalize, unwrap_encode_depth
from oracle import encoder_ref as ER
from tests.deferred_env import PIXELS, FakeDeferredEnv
from tests.test_encoder_cpu import load_fixture

pytestmark = pytest.mark.gpu

TOL = 1e-4        # relative to the largest encoding magnitude (fp32 FMA chain vs float64 oracle)
OTHER = {"network": [{"filters": 8, "kernel_size": 3, "strides": 1}, {"filters": 16, "kernel_size": 4, "strides": 2},
                     {"filters": 12, "kernel_size": 5, "strides": 3}], "encoding_dim": 20, "alpha": 0.2}


def _encoder(geometry, max_batch=512):
    if geometry == "shipped":
        w, cfg = load_fixture()
        arr = keras_encoder_arrays(w, len(cfg["network"]))
    else:
        cfg = OTHER
        rng = np.random.default_rng(5)
        arr, c, hw = [], 1, 64
        for l in cfg["network"]:
            arr.append((rng.normal(0, 0.2, (l["kernel_size"], l["kernel_size"], c, l["filters"])).astype(np.float32),
                        rng.normal(0, 0.1, l["filters"]).astype(np.float32)))
            c, hw = l["filters"], -(-hw // l["strides"])
        arr.append((rng.normal(0, 0.05, (hw * hw * c, cfg["encoding_dim"])).astype(np.float32),
                    rng.normal(0, 0.1, cfg["encoding_dim"]).astype(np.float32)))
    enc = SimpleAutoEncoder(cfg, max_batch=max_batch)
    enc.set_weights(arr)
    return enc, arr, cfg


def _raw(n, tail, seed):
    rng = np.random.default_rng(seed)
    imgs = synth.make_depth_scenes(n, seed=seed) + rng.normal(0, 0.02, (n, 64, 64, 1)).astype(np.float32)
    return np.concatenate([imgs.reshape(n, PIXELS), rng.uniform(0, 1, (n, tail))], axis=1).astype(np.float32)


def _host(enc, rows):
    """What the host-mode wrapper returns for raw rows: the encoder handle's encodings + the tail."""
    rows = np.asarray(rows, np.float32)
    return np.concatenate([enc.encode(rows[:, :PIXELS].reshape(-1, 64, 64, 1)), rows[:, PIXELS:]], axis=1)


def _done(kind, n):
    if kind == "none":
        return np.zeros(n, np.float32)
    if kind == "all":
        return np.ones(n, np.float32)
    return (np.arange(n) % 3 == 1).astype(np.float32)


CASES = [("shipped", n, t, k) for n in (1, 3, 128, 256) for t in (0, 1, 2) for k in ("some", "none", "all")] + \
        [("other", n, t, k) for n in (3, 256) for t in (0, 2) for k in ("some", "all")]


@pytest.mark.parametrize("geometry,n,tail,kind", CASES)
def test_sac_stage_encodes_what_the_encoder_handle_encodes(geometry, n, tail, kind):
    enc, arr, cfg = _encoder(geometry)
    D = cfg["encoding_dim"]
    L = Learner((D + tail,), n_act=2, batch_size=64, buffer_size=2 * n, precision=_lib.B2G_PREC_FP32_SIMT)
    L.set_obs_encoder(enc, tail)
    assert L.frame_elems == PIXELS + tail
    r0, r1, r3 = _raw(n, tail, 1), _raw(n, tail, 2), _raw(n, tail, 3)
    done = _done(kind, n)
    reset = np.full_like(r1, np.nan)                    # rows of envs that did not finish are never read
    reset[done != 0] = _raw(n, tail, 4)[done != 0]
    act, rew = np.zeros((n, 2), np.float32), np.zeros(n, np.float32)
    L.observe_act(r0, update_stats=False, act=False)
    before = L.upload_bytes()["observe"]
    L.observe_add(act, rew, r1, done, reset_obs=reset if done.any() else None, update_stats=False)
    n_done = int(done.sum())
    assert L.upload_bytes()["observe"] - before == (n + n_done) * (PIXELS + tail) * 4 + n * 2 * 4 + n * 4 + n * 4
    L.observe_add(act, rew, r3, np.zeros(n, np.float32), update_stats=False)
    staged = np.where(done[:, None] != 0, reset, r1)
    want_obs0, want_next0 = _host(enc, r0), _host(enc, r1)
    want_obs1, want_next1 = _host(enc, staged), _host(enc, r3)
    for i in range(n):
        t0, t1 = L.replay_get(i), L.replay_get(n + i)
        assert np.array_equal(t0["obs"], want_obs0[i]) and np.array_equal(t0["next_obs"], want_next0[i]), i
        assert np.array_equal(t1["obs"], want_obs1[i]) and np.array_equal(t1["next_obs"], want_next1[i]), i
        assert np.array_equal(t1["obs"][D:], staged[i, PIXELS:])            # the tail, copied exactly
    ref = ER.encode(staged[:, :PIXELS].reshape(-1, 64, 64, 1), arr, [l["strides"] for l in cfg["network"]], cfg["alpha"],
                    torch.float64)
    assert np.abs(want_obs1[:, :D] - ref).max() <= TOL * np.abs(ref).max()
    L.close()


def test_bdq_stage_feeds_statistics_actor_and_replay_like_host_encoded_rows():
    enc, _, cfg = _encoder("shipped")
    n, tail = 128, 1
    E = cfg["encoding_dim"] + tail
    mk = lambda: BDQLearner(E, 2, 4, ((64, 64), (32,), (32,)), 16, 1024, seed=3)
    A, B = mk(), mk()
    for L in (A, B):
        L.obs_rms_set(np.zeros(E), np.ones(E), 1e-4)
    B.load_parameters(A.get_parameters())
    A.set_obs_encoder(enc, tail)
    r0, r1 = _raw(n, tail, 5), _raw(n, tail, 6)
    done = _done("some", n)
    reset = np.full_like(r1, np.nan)
    reset[done != 0] = _raw(n, tail, 7)[done != 0]
    reset_enc = np.full((n, E), np.nan, np.float32)
    reset_enc[done != 0] = _host(enc, reset[done != 0])
    a0 = A.observe_act(r0, eps=0.0)
    b0 = B.observe_act(_host(enc, r0), eps=0.0)
    assert np.array_equal(a0, b0)
    before = A.upload_bytes()["observe"]
    A.observe_add(a0.astype(np.float32), np.ones(n), r1, done, reset_obs=reset)
    n_done = int(done.sum())
    assert A.upload_bytes()["observe"] - before == (n + n_done) * (PIXELS + tail) * 4 + n * 2 * 4 + n * 4 + n * 4
    B.observe_add(b0.astype(np.float32), np.ones(n), _host(enc, r1), done, reset_obs=reset_enc)
    for x, y in zip(A.obs_rms_get(), B.obs_rms_get()):
        assert np.array_equal(x, y)
    assert np.array_equal(A.observe_act(None, n=n, eps=0.0), B.observe_act(None, n=n, eps=0.0))     # staged rows
    A.close(), B.close()


def _stack(n_envs, enc, tail=1, seed0=0):
    venv = DummyVecEnv([(lambda i=i: FakeDeferredEnv(seed=seed0 + i, horizon=5, tail=tail, n_act=3)) for i in range(n_envs)])
    return VecNormalize(VecEncodeDepth(venv, enc), norm_obs=True, norm_reward=True)


def _host_mode(model):
    """The same stack and model, but encoding in the wrapper: detach the learner's encoder, hand it back to the wrapper."""
    model.learner.set_obs_encoder(None)
    unwrap_encode_depth(model.env).take_encoder_back()


@pytest.mark.parametrize("learning", [False, True])
def test_sac_learn_pass_raw_is_the_host_mode_run(learning):
    enc, _, _ = _encoder("shipped")
    models = []
    for raw in (True, False):
        env = _stack(4, enc)
        m = SAC(MlpPolicy, env, batch_size=16, buffer_size=256, learning_starts=8 if learning else 10 ** 6, seed=0,
                precision="fp32", device_obs_norm=True)
        assert unwrap_encode_depth(env).pass_raw
        if not raw:
            _host_mode(m)
        m.learn(80)
        models.append(m)
    p, h = models
    for s in range(p.learner.replay_size()):
        tp, th = p.learner.replay_get(s), h.learner.replay_get(s)
        for k in ("obs", "next_obs", "act"):
            if learning:
                np.testing.assert_allclose(tp[k], th[k], rtol=0, atol=1e-6)
            else:
                assert np.array_equal(tp[k], th[k]), (s, k)
    for x, y in zip(p.learner.obs_rms_get(), h.learner.obs_rms_get()):
        if learning:
            np.testing.assert_allclose(x, y, rtol=1e-12, atol=1e-300)
        else:
            assert np.array_equal(x, y)
    a_p = p.learner.observe_act(None, n=4, deterministic=True)
    a_h = h.learner.observe_act(None, n=4, deterministic=True)
    if learning:        # the bars of test_gpu_obs_norm.py: actions, and one more sampled step on the same draw
        np.testing.assert_allclose(a_p, a_h, rtol=0, atol=1e-6)
        for m in models:
            m._sync_norm_stats()
            m.learner.step(1, 0.0)
        bp, bh = p.learner.last_batch(), h.learner.last_batch()
        assert np.array_equal(bp["indices"], bh["indices"]) and np.array_equal(bp["eps"], bh["eps"])
        for k in ("q1", "q2", "v", "logp", "v_targ"):
            np.testing.assert_allclose(bp[k], bh[k], rtol=1e-5, atol=1e-6)
    else:
        assert np.array_equal(a_p, a_h)
    for m in models:
        m.close()


@pytest.mark.parametrize("learning", [False, True])
def test_bdq_learn_pass_raw_is_the_host_mode_run(learning):
    enc, _, _ = _encoder("shipped")
    models = []
    for raw in (True, False):
        env = _stack(4, enc)
        m = BDQ("MlpActPolicy", env, batch_size=16, buffer_size=256, learning_starts=8 if learning else 10 ** 6, num_actions_pad=5,
                seed=0, device_obs_norm=True)
        if not raw:
            _host_mode(m)
        m.learn(80)
        models.append(m)
    p, h = models
    for x, y in zip(p.learner.obs_rms_get(), h.learner.obs_rms_get()):
        if learning:
            np.testing.assert_allclose(x, y, rtol=1e-12, atol=1e-300)
        else:
            assert np.array_equal(x, y)
    if learning:        # the bar of test_gpu_bdq_obs_norm.py's continued run
        for k, v in p.learner.get_parameters().items():
            np.testing.assert_allclose(v, h.learner.get_parameters()[k], rtol=0, atol=1e-6, err_msg=k)
    else:
        assert np.array_equal(p.learner.observe_act(None, n=4, eps=0.0), h.learner.observe_act(None, n=4, eps=0.0))
    for m in models:
        m.close()


def test_refusals():
    enc, _, cfg = _encoder("shipped")
    D = cfg["encoding_dim"]
    L = Learner((D + 1,), n_act=2, batch_size=16, buffer_size=64)
    for tail, code in ((0, _lib.B2G_EINVAL), (2, _lib.B2G_EINVAL), (-1, _lib.B2G_EINVAL)):
        with pytest.raises(_lib.B2GError) as e:
            L.set_obs_encoder(enc, tail)
        assert e.value.code == code
    unloaded = SimpleAutoEncoder(cfg, max_batch=4)
    with pytest.raises(_lib.B2GError) as e:
        L.set_obs_encoder(unloaded, 1)
    assert e.value.code == _lib.B2G_ESTATE
    L.close()
    cnn = Learner((64, 64, 2), n_act=5, batch_size=16, buffer_size=64)
    with pytest.raises(_lib.B2GError) as e:
        cnn.set_obs_encoder(enc, 1)
    assert e.value.code == _lib.B2G_EINVAL
    cnn.close()
    B = BDQLearner(D, 2, 4, ((64, 64), (32,), (32,)), 16, 64)
    with pytest.raises(_lib.B2GError) as e:
        B.set_obs_encoder(enc, 1)
    assert e.value.code == _lib.B2G_EINVAL
    with pytest.raises(_lib.B2GError) as e:
        B.set_obs_encoder(unloaded, 0)
    assert e.value.code == _lib.B2G_ESTATE
    B.close()
    if torch.cuda.device_count() > 1:               # an encoder on another device
        e1 = SimpleAutoEncoder(cfg, max_batch=4, device=1)
        e1.set_weights(keras_encoder_arrays(load_fixture()[0], 3))
        L = Learner((D + 1,), n_act=2, batch_size=16, buffer_size=64)
        with pytest.raises(_lib.B2GError) as e:
            L.set_obs_encoder(e1, 1)
        assert e.value.code == _lib.B2G_EINVAL
        L.close()


def test_attach_clears_staged_observations_and_detach_restores_the_encoded_layout():
    enc, _, cfg = _encoder("shipped")
    E = cfg["encoding_dim"] + 1
    L = Learner((E,), n_act=2, batch_size=16, buffer_size=64)
    L.observe_act(np.zeros((2, E), np.float32), update_stats=False, act=False)
    L.set_obs_encoder(enc, 1)
    with pytest.raises(_lib.B2GError):
        L.observe_act(None, n=2)                    # nothing staged any more
    L.observe_act(_raw(2, 1, 0), update_stats=False, act=False)
    L.set_obs_encoder(None)
    assert L.frame_elems == E
    with pytest.raises(_lib.B2GError):
        L.observe_act(None, n=2)
    L.observe_act(np.zeros((2, E), np.float32), update_stats=False, act=True)
    L.close()


def _write_encoder_dir(d):
    w, cfg = load_fixture()
    names = keras_layer_names(len(cfg["network"]))
    enc = SimpleAutoEncoder(cfg, max_batch=4)
    enc.set_model_weights([(w[f"{n}/kernel"], w[f"{n}/bias"]) for n in names])
    os.makedirs(d, exist_ok=True)
    enc.save_weights(os.path.join(d, "model.h5"))
    with open(os.path.join(d, "config.yaml"), "w") as f:
        yaml.safe_dump({k: cfg[k] for k in ("network", "encoding_dim", "alpha")}, f)
    enc.close()


def test_training_state_round_trip_and_digest_refusal(tmp_path):
    enc, _, cfg = _encoder("shipped")
    env = _stack(2, enc)
    m = SAC(MlpPolicy, env, batch_size=16, buffer_size=128, learning_starts=8, seed=1, precision="fp32", device_obs_norm=True)
    m.learn(30)
    m.save_training_state(str(tmp_path / "st"))
    host = json.load(open(tmp_path / "st" / "host.json"))
    assert host["obs_encoder"]["digest"] == enc.weights_digest()
    m.close()
    back = SAC.load_training_state(str(tmp_path / "st"), _stack(2, enc))
    assert unwrap_encode_depth(back.env).pass_raw and back.learner.raw_obs_elems == PIXELS + 1
    back.learn(10, reset_num_timesteps=False)
    back.close()
    other, _, _ = _encoder("shipped")
    k, b = other._encoder_arrays[-1]
    other.set_weights(other._encoder_arrays[:-1] + [(k, b + 1.0)])
    fresh = _stack(2, other)
    with pytest.raises(ValueError, match="encoder weights"):
        SAC.load_training_state(str(tmp_path / "st"), fresh)
    assert not fresh.learner_owns_obs_rms and not unwrap_encode_depth(fresh).pass_raw      # nothing written


def test_cli_device_encode_train_then_run(tmp_path):
    _write_encoder_dir(str(tmp_path / "enc"))
    cfg = {"sensor": {"encoder_dir": str(tmp_path / "enc")}, "robot": {}, "reward": {"shaped": False}, "normalize": True,
           "discount_factor": 0.99, "simplified": False, "algorithm": "sac",
           "SAC": {"layers": [64, 64], "buffer_size": 256, "batch_size": 16, "step_size": 3e-4, "total_timesteps": 40}}
    cp = tmp_path / "config.yaml"
    cp.write_text(yaml.safe_dump(cfg))
    md = tmp_path / "run"
    model = train_cli.main(["train", "--config", str(cp), "--algo", "SAC", "--model_dir", str(md), "--device_encode", "--device_norm",
                            "--env", "tests.deferred_env:make_env", "--n_envs", "1", "--eval_freq", "20", "--precision", "fp32"])
    assert model.observation_space.shape == (101,)
    from b200grasp import sb_io
    data, params = sb_io.load_sb_zip(str(md / "final_model.zip"))
    assert data["observation_space"]["shape"] == [101] and params["model/pi/fc0/kernel"].shape[0] == 101
    from b200grasp.sb_io import load_vecnormalize
    assert load_vecnormalize(str(md / "vecnormalize.pkl"))["obs_mean"].shape == (101,)
    out = train_cli.main(["run", "--model", str(md / "final_model.zip"), "--env", "tests.deferred_env:make_env", "--episodes", "2",
                          "--precision", "fp32"])
    assert out["episodes"] == 2
