"""Host side of ``SAC(device_obs_norm=True)``: the merge rule the device kernel restates, VecNormalize with its ``obs_rms``
owned by a learner, the ABI symbols and the CLI flag.  Needs no GPU."""
import copy
import ctypes
import os
import pickle

import numpy as np
import pytest

from b200grasp import _lib, train_cli
from b200grasp.vec_env import (DeviceRunningMeanStd, DummyVecEnv, RunningMeanStd, VecNormalize, sync_envs_normalization)
from tests.fake_env import FakeGraspEnv


def merge(mean, var, count, frames):
    """obs_rms_update_kernel in numpy float64: frames summed in order 0 .. n-1, then the parallel-moments rule."""
    n = frames.shape[0]
    s = np.zeros_like(mean)
    for f in frames:
        s = s + f.astype(np.float64)
    bm = s / n
    q = np.zeros_like(mean)
    for f in frames:
        d = f.astype(np.float64) - bm
        q = q + d * d
    bv = q / n
    delta = bm - mean
    tot = count + n
    return mean + delta * n / tot, (var * count + bv * n + delta * delta * count * n / tot) / tot, tot


@pytest.mark.parametrize("count0", [1e-4, 0.0])
def test_merge_rule_equals_running_mean_std(count0):
    rng = np.random.default_rng(5)
    shape = (6, 5, 3)
    rms = RunningMeanStd(epsilon=count0, shape=shape)
    mean, var, count = np.zeros(shape), np.ones(shape), count0
    for k in range(60):
        n = (1, 3, 128)[k % 3]
        frames = rng.uniform(0, 255, (n,) + shape).astype(np.float32)
        rms.update(frames)
        mean, var, count = merge(mean, var, count, frames)
        assert count == rms.count
    np.testing.assert_allclose(mean, rms.mean, rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(var, rms.var, rtol=1e-12, atol=1e-300)


class FakeOwner:
    """Stands in for a Learner: keeps (mean, var, count) and counts the fetches."""

    def __init__(self):
        self.obs_rms_version, self.fetches, self.stats = 0, 0, None

    def obs_rms_set(self, mean, var, count):
        self.stats = (np.array(mean, np.float64), np.array(var, np.float64), float(count))
        self.obs_rms_version += 1

    def obs_rms_get(self):
        self.fetches += 1
        return tuple(np.copy(x) for x in self.stats[:2]) + (self.stats[2],)


def owned_env(n_envs=3, horizon=4):
    venv = DummyVecEnv([(lambda i=i: FakeGraspEnv(seed=i, horizon=horizon)) for i in range(n_envs)])
    return VecNormalize(venv, norm_obs=True, norm_reward=True, clip_obs=10.0)


def test_learner_owned_vecnormalize_returns_raw_obs_and_keeps_the_reward_side():
    host, dev = owned_env(), owned_env()
    owner = FakeOwner()
    dev.give_obs_rms_to(owner)
    assert dev.learner_owns_obs_rms and not host.learner_owns_obs_rms
    assert owner.stats[2] == 1e-4 and np.all(owner.stats[1] == 1.0)
    o_h, o_d = host.reset(), dev.reset()
    np.testing.assert_array_equal(o_d, dev.get_original_obs())
    np.testing.assert_array_equal(o_d, host.get_original_obs())
    assert not np.array_equal(o_h, o_d)
    act = np.zeros((3, 5), np.float32)
    for _ in range(6):                                  # crosses an episode end (horizon 4)
        _, r_h, d_h, _ = host.step(act)
        o_d, r_d, d_d, _ = dev.step(act)
        np.testing.assert_array_equal(o_d, host.get_original_obs())
        np.testing.assert_array_equal(r_h, r_d)
        np.testing.assert_array_equal(d_h, d_d)
    assert dev.ret_rms.count == host.ret_rms.count and dev.ret_rms.var == host.ret_rms.var
    assert owner.obs_rms_version == 1                   # the wrapper never touched the owner's statistics
    with pytest.raises(RuntimeError):
        dev.obs_rms.update(o_d)
    # explicit normalisation works from the fetched statistics
    owner.obs_rms_set(host.obs_rms.mean, host.obs_rms.var, host.obs_rms.count)
    np.testing.assert_array_equal(dev.normalize_obs(o_d), host.normalize_obs(o_d))


def test_device_running_mean_std_fetches_caches_and_writes_through():
    owner = FakeOwner()
    owner.obs_rms_set(np.full((2, 2), 3.0), np.full((2, 2), 4.0), 7.0)
    rms = DeviceRunningMeanStd(owner)
    assert rms.count == 7.0 and rms.mean[0, 0] == 3.0 and rms.var[1, 1] == 4.0
    assert owner.fetches == 1                           # cached until the version moves
    owner.obs_rms_set(np.zeros((2, 2)), np.ones((2, 2)), 8.0)
    assert rms.count == 8.0 and owner.fetches == 2
    rms.mean = np.full((2, 2), 5.0)                     # assignment writes through, the other two kept
    assert owner.stats[0][0, 0] == 5.0 and owner.stats[1][0, 0] == 1.0 and owner.stats[2] == 8.0
    snap = copy.deepcopy(rms)
    assert type(snap) is RunningMeanStd and snap.count == 8.0 and snap.mean[0, 0] == 5.0
    back = pickle.loads(pickle.dumps(rms))
    assert type(back) is RunningMeanStd and back.count == 8.0 and np.all(back.var == 1.0)


def test_owned_vecnormalize_pickles_and_syncs_like_a_host_one(tmp_path):
    dev = owned_env()
    owner = FakeOwner()
    dev.give_obs_rms_to(owner)
    rng = np.random.default_rng(2)
    owner.obs_rms_set(rng.uniform(0, 1, (64, 64, 2)), rng.uniform(0.5, 2, (64, 64, 2)), 321.0)
    dev.reset()
    for sb in (True, False):
        path = os.path.join(tmp_path, f"vn_{sb}.pkl")
        dev.save(path, sb_compatible=sb)
        if sb:
            with open(path, "rb") as f:
                assert b"stable_baselines.common.running_mean_std" in f.read()
            back = VecNormalize.load(path, owned_env().venv)
        else:
            with open(path, "rb") as f:
                back = pickle.load(f)
        assert type(back.obs_rms) is RunningMeanStd and back.obs_rms.count == 321.0
        np.testing.assert_array_equal(back.obs_rms.mean, owner.stats[0])
        np.testing.assert_array_equal(back.obs_rms.var, owner.stats[1])
    ev = owned_env()
    sync_envs_normalization(dev, ev)
    assert type(ev.obs_rms) is RunningMeanStd and ev.obs_rms.count == 321.0
    np.testing.assert_array_equal(ev.obs_rms.var, owner.stats[1])
    assert dev.learner_owns_obs_rms                     # saving and syncing leave the owner in place


def test_a_wrapper_has_one_owner_and_takes_its_statistics_back():
    dev = owned_env()
    first, second = FakeOwner(), FakeOwner()
    dev.give_obs_rms_to(first)
    dev.give_obs_rms_to(first)                          # the same owner again: nothing to do
    assert first.obs_rms_version == 1 and dev.obs_rms_owner is first
    with pytest.raises(RuntimeError, match="already owned"):
        dev.give_obs_rms_to(second)
    assert second.stats is None and dev.obs_rms_owner is first
    first.obs_rms_set(np.full((64, 64, 2), 2.0), np.full((64, 64, 2), 3.0), 9.0)
    dev.take_obs_rms_back()
    assert not dev.learner_owns_obs_rms and dev.obs_rms_owner is None and type(dev.obs_rms) is RunningMeanStd
    assert dev.obs_rms.count == 9.0 and np.all(dev.obs_rms.mean == 2.0)
    o = dev.reset()                                     # the wrapper updates and normalises again itself
    assert dev.obs_rms.count == 12.0 and not np.array_equal(o, dev.get_original_obs())
    dev.give_obs_rms_to(second)                         # and can be handed on
    assert second.stats[2] == 12.0


def test_evaluate_policy_feeds_raw_observations_to_a_model_that_owns_its_statistics():
    from b200grasp.evaluation import evaluate_policy

    class Model:
        def __init__(self, raw):
            self.predict_takes_raw_obs, self.seen = raw, []

        def predict(self, obs, state=None, deterministic=True):
            self.seen.append(np.array(obs))
            return np.zeros((1, 5), np.float32), None

    for raw in (True, False):
        ev = owned_env(n_envs=1)
        ev.training = False
        ev.obs_rms.mean = np.ones((64, 64, 2))            # normalised observations go negative, raw depth never does
        m = Model(raw)
        evaluate_policy(m, ev, n_eval_episodes=1)
        assert len(m.seen) == 4                         # horizon 4
        assert (m.seen[0].min() >= 0.0) == raw
    owner, ev, m = FakeOwner(), owned_env(n_envs=1), Model(True)
    ev.give_obs_rms_to(owner)                           # an evaluation wrapper that is itself learner-owned returns raw already
    owner.obs_rms_set(np.ones((64, 64, 2)), np.ones((64, 64, 2)), 1.0)
    evaluate_policy(m, ev, n_eval_episodes=1)
    assert m.seen[0].min() >= 0.0


def test_abi_symbols_and_argtypes():
    names = ("b2g_sac_observe_act", "b2g_sac_observe_add", "b2g_obs_rms_set", "b2g_obs_rms_get", "b2g_upload_bytes")
    lib = _lib.load()
    for n in names:
        assert n in _lib.SYMBOLS and hasattr(lib, n)
    assert len(lib.b2g_sac_observe_act.argtypes) == 6 and len(lib.b2g_sac_observe_add.argtypes) == 8
    assert lib.b2g_obs_rms_set.argtypes[3] is ctypes.c_double
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200grasp.h")).read()
    for n in names:
        assert f"int {n}(" in header


def test_null_handle_is_refused_without_a_device():
    lib = _lib.load()
    assert lib.b2g_sac_observe_act(None, None, 1, 0, 0, None) == _lib.B2G_EINVAL
    assert lib.b2g_obs_rms_get(None, None, None, None) == _lib.B2G_EINVAL
    assert lib.b2g_upload_bytes(None, None, None) == _lib.B2G_EINVAL
    assert b"NULL" in lib.b2g_last_error()


def test_cli_flag_parses():
    p = train_cli.build_parser()
    a = p.parse_args(["train", "--config", "c.yaml", "--algo", "SAC", "--model_dir", "m", "--device_norm"])
    assert a.device_norm is True
    assert p.parse_args(["train", "--config", "c.yaml"]).device_norm is False


def test_nranks_above_one_is_refused():
    from b200grasp.sac_model import SAC, CnnPolicy
    with pytest.raises(NotImplementedError, match="every rank would own different statistics"):
        SAC(CnnPolicy, None, nranks=2, device_obs_norm=True)
