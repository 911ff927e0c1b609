"""The per-step metrics ring on the device and the TensorBoard event files learn writes from it.

The ring row of a step equals the metrics b2g_*_step returns for it, on every SAC path (graph replay, host-pipelined,
device_obs_norm learn) and on BDQ and DQN; a handle with the ring trains what one without it trains (bit for bit where two
runs without it agree bit for bit, else within their spread); a ring that is not drained past its capacity reports the exact count it lost; learn writes one summary per gradient step (replay learners)
or per update (PPO2, TRPO) plus one episode_reward per finished episode; train --resume continues the same run directory."""
import os

import numpy as np
import pytest
import yaml

import b200grasp
from b200grasp import _lib, train_cli
from b200grasp.bdq import BDQ, BDQLearner
from b200grasp.deepq import DQN
from b200grasp.deepq.policies import MlpPolicy as DQNMlpPolicy
from b200grasp.dqn import DQNLearner
from b200grasp.ppo2 import PPO2
from b200grasp.trpo_mpi import TRPO
from b200grasp.common.policies import MlpPolicy
from b200grasp.vec_env import DummyVecEnv, VecNormalize
from tests.fake_env import FakeFlatEnv, FakeGraspEnv
from tests.test_gpu_dqn import LineEnv
from tests.test_tensorboard_cpu import event_files, read_events

pytestmark = pytest.mark.gpu

SAC_COLS = ("policy_loss", "qf1_loss", "qf2_loss", "value_loss", "ent_coef_loss", "entropy", "ent_coef")


def sac_learner(seed=0, B=32):
    L = b200grasp.Learner((101,), n_act=5, batch_size=B, buffer_size=512, seed=seed, precision=0)
    rng = np.random.default_rng(seed)
    n = 256
    L.replay_add(rng.normal(size=(n, 101)).astype(np.float32), rng.uniform(-1, 1, (n, 5)).astype(np.float32),
                 rng.normal(size=n).astype(np.float32), rng.normal(size=(n, 101)).astype(np.float32),
                 (rng.uniform(size=n) < 0.1).astype(np.float32))
    return L


def trains_the_same(plain, logged, control):
    """logged (ring on) trained what plain (ring off) trained.  control is a second ring-off run of the same steps: where the
    step is bit-reproducible (control == plain) the ring run must be bit-identical too; where the engine's fp32 atomics
    add in a different order from run to run, it must agree with plain as closely as the control does."""
    pa, pb, pc = plain.get_parameters(), logged.get_parameters(), control.get_parameters()
    exact = all(np.array_equal(pa[k], pc[k]) for k in pa)
    if exact:
        for k in pa:
            assert np.array_equal(pa[k], pb[k]), k
        return True
    for k in pa:
        spread = float(np.max(np.abs(pa[k] - pc[k]))) if pa[k].size else 0.0
        assert np.allclose(pa[k], pb[k], rtol=1e-4, atol=max(1e-6, 4 * spread)), k
    return False


def clone_params(src, *dst):
    p = src.get_parameters()
    for d in dst:
        d.load_parameters(p)


def expect_rows(rows, metrics, cols, lrs):
    assert len(rows) == len(metrics)
    for r, m, lr in zip(rows, metrics, lrs):
        assert [float(x) for x in r[:-1]] == [float(np.float32(m[c])) for c in cols]
        assert r[-1] == np.float32(lr)


def test_sac_graph_path_ring_rows_and_parameters():
    plain, logged, control = sac_learner(), sac_learner(), sac_learner()
    clone_params(plain, logged, control)
    logged.metrics_log(64)
    lrs = [3e-4 * (1 - 0.1 * i) for i in range(6)]
    got = []
    for lr in lrs:
        plain.step_async(1, lr)
        control.step_async(1, lr)
        got.append(logged.step(1, lr))           # one graph replay per call, its metrics read back each time
    first, rows, lost = logged.metrics_drain()
    assert first == 1 and lost == 0
    expect_rows(rows, got, SAC_COLS, lrs)
    # n_steps > 1 in one call: every replay appends its row
    plain.step_async(3, 1e-4)
    control.step_async(3, 1e-4)
    m = logged.step(3, 1e-4)
    first, rows, lost = logged.metrics_drain()
    assert first == 7 and len(rows) == 3 and lost == 0
    expect_rows(rows[-1:], [m], SAC_COLS, [1e-4])
    plain.sync(); control.sync()
    trains_the_same(plain, logged, control)
    # turning the log off recaptures the step without the node
    logged.metrics_log(0)
    plain.step(2, 1e-4); logged.step(2, 1e-4); control.step(2, 1e-4)
    trains_the_same(plain, logged, control)
    plain.close(); logged.close(); control.close()


def test_sac_host_pipelined_path_ring_rows_and_parameters():
    plain, logged, control = sac_learner(1), sac_learner(1), sac_learner(1)
    clone_params(plain, logged, control)
    logged.metrics_log(16)
    rng = np.random.default_rng(5)
    B, lr = 32, 2e-4
    got = []
    for _ in range(5):
        b = [rng.normal(size=(B, 101)), rng.uniform(-1, 1, (B, 5)), rng.normal(size=B), rng.normal(size=(B, 101)),
             (rng.uniform(size=B) < 0.1), rng.normal(size=(B, 5))]
        b = [np.ascontiguousarray(x, np.float32) for x in b]
        plain.step_host_pipelined(*b, lr=lr)
        control.step_host_pipelined(*b, lr=lr)
        prev = logged.step_host_pipelined(*b, lr=lr)
        if prev is not None:
            got.append(prev)
    plain.pipeline_flush()
    control.pipeline_flush()
    got.append(logged.pipeline_flush())
    first, rows, lost = logged.metrics_drain()
    assert first == 1 and lost == 0
    expect_rows(rows, got, SAC_COLS, [lr] * 5)
    trains_the_same(plain, logged, control)
    plain.close(); logged.close(); control.close()


def test_ring_reports_exactly_what_it_lost():
    L = sac_learner(2)
    L.metrics_log(4)
    L.step_async(10, 3e-4)
    first, rows, lost = L.metrics_drain()
    assert (first, len(rows), lost) == (7, 4, 6)
    m = L.step(1, 3e-4)
    first, rows, lost = L.metrics_drain()
    assert (first, len(rows), lost) == (11, 1, 0)
    expect_rows(rows, [m], SAC_COLS, [3e-4])
    L.step_async(5, 3e-4)
    first, rows, lost = L.metrics_drain(max_rows=2)         # rows past max_rows wait for the next drain
    assert (first, len(rows), lost) == (13, 2, 1)
    first, rows, lost = L.metrics_drain()
    assert (first, len(rows), lost) == (15, 2, 0)
    L.close()


def _q_learner(kind, seed=0):
    rng = np.random.default_rng(seed)
    n, obs = 200, 12
    if kind == "bdq":
        L = BDQLearner(obs, n_branches=3, n_bins=5, batch_size=32, buffer_size=400, seed=seed)
        act = rng.integers(0, 5, (n, 3)).astype(np.float32)
    else:
        L = DQNLearner(obs, n_actions=4, batch_size=32, buffer_size=400, seed=seed)
        act = rng.integers(0, 4, n).astype(np.float32)
    L.replay_add(rng.normal(size=(n, obs)).astype(np.float32), act, rng.normal(size=n).astype(np.float32),
                 rng.normal(size=(n, obs)).astype(np.float32), (rng.uniform(size=n) < 0.1).astype(np.float32))
    return L


@pytest.mark.parametrize("kind", ["bdq", "dqn"])
def test_q_learners_ring_rows_and_parameters(kind):
    plain, logged, control = _q_learner(kind), _q_learner(kind), _q_learner(kind)
    clone_params(plain, logged, control)
    logged.metrics_log(32)
    cols = _lib.LOG_COLS[kind][:-1]
    lrs = [1e-3, 5e-4, 5e-4, 2e-4]
    got = []
    for lr in lrs:
        plain.step(1, lr)
        control.step(1, lr)
        got.append(logged.step(1, lr))
    first, rows, lost = logged.metrics_drain()
    assert first == 1 and lost == 0
    expect_rows(rows, got, cols, lrs)
    trains_the_same(plain, logged, control)
    plain.close(); logged.close(); control.close()


# ------------------------------------------------------------------ event files written by learn
def summaries(logdir):
    """(per-step summaries: [(step, {tag: value})], episode_reward count) of every event file under logdir"""
    steps, eps = [], 0
    for f in event_files(logdir):
        for e in read_events(f)[1:]:
            tags = dict(e["values"])
            if "episode_reward" in tags:
                eps += 1
            else:
                steps.append((e["step"], tags))
    return steps, eps


def test_sac_learn_writes_every_gradient_step(tmp_path):
    env = VecNormalize(DummyVecEnv([lambda: FakeGraspEnv(1, horizon=15)]), norm_obs=True, norm_reward=True, clip_obs=10.0)
    model = b200grasp.SAC(b200grasp.CnnPolicy, env, policy_kwargs={"layers": [64, 64], "cnn_extractor": None}, buffer_size=1000,
                          batch_size=32, learning_starts=40, tensorboard_log=str(tmp_path), seed=3, verbose=1)
    seen = []
    model.learn(total_timesteps=120, callback=lambda l, g: seen.append(l["writer"]) or True, log_interval=2)
    assert seen[0] is not None and seen[0]._fh is None            # the writer callbacks saw, closed at the end
    steps, eps = summaries(str(tmp_path / "SAC_1"))
    assert len(steps) == model.n_updates == 81
    assert eps == 120 // 15
    assert [s for s, _ in steps] == list(range(40, 121))
    assert set(steps[0][1]) == {"policy_loss", "qf1_loss", "qf2_loss", "value_loss", "entropy", "ent_coef_loss", "ent_coef",
                                "learning_rate"}
    assert all(np.isfinite(v) for _, t in steps for v in t.values())
    # a stop by a callback still drains what was enqueued
    model.learn(total_timesteps=1000, callback=lambda l, g: model.num_timesteps < 30, reset_num_timesteps=False)
    steps2, _ = summaries(str(tmp_path / "SAC_1"))
    assert len(steps2) == model.n_updates
    model.close()


def test_sac_device_obs_norm_learn_matches_and_logs(tmp_path):
    def run(log):
        env = VecNormalize(DummyVecEnv([lambda i=i: FakeFlatEnv(seed=i, horizon=9, obs_dim=20, n_act=3) for i in range(4)]))
        m = b200grasp.SAC(b200grasp.MlpPolicy, env, buffer_size=2000, batch_size=32, learning_starts=64, seed=7,
                          device_obs_norm=True, tensorboard_log=log, precision="fp32")
        m.learn(400)
        return m
    a, b, c = run(None), run(str(tmp_path)), run(None)
    assert a.n_updates == b.n_updates > 0
    trains_the_same(a.learner, b.learner, c.learner)
    steps, eps = summaries(str(tmp_path / "SAC_1"))
    assert len(steps) == b.n_updates and eps == 4 * (400 // 4 // 9)
    a.close(); b.close(); c.close()


def test_bdq_and_dqn_learn_write_every_gradient_step(tmp_path):
    env = DummyVecEnv([lambda: FakeFlatEnv(horizon=5, obs_dim=6, n_act=3)])
    m = BDQ("MlpActPolicy", env, policy_kwargs={"layers": [[32, 32], [16], [16]]}, batch_size=16, buffer_size=500, learning_starts=50,
            num_actions_pad=5, tensorboard_log=str(tmp_path), seed=1)
    calls = []
    orig = m.learner.step
    m.learner.step = lambda n=1, lr=1e-4: (calls.append(m.num_timesteps), orig(n, lr))[1]
    m.learn(200)
    steps, eps = summaries(str(tmp_path / "BDQ_1"))
    assert [s for s, _ in steps] == calls and len(calls) == 150
    assert set(steps[0][1]) == {"loss", "mean_q", "grad_norm", "learning_rate"} and eps == 200 // 5
    m.close()
    d = DQN(DQNMlpPolicy, LineEnv(), batch_size=16, buffer_size=500, learning_starts=50, policy_kwargs={"layers": [16, 16]}, seed=3,
            tensorboard_log=str(tmp_path))
    d.learn(200)
    steps, eps = summaries(str(tmp_path / "DQN_1"))
    assert [s for s, _ in steps] == list(range(51, 201))
    assert set(steps[0][1]) == {"loss", "mean_q", "mean_abs_td_error", "grad_norm"} and eps == 200 // 10
    d.close()


def test_ppo2_and_trpo_learn_write_every_update(tmp_path):
    env = DummyVecEnv([lambda i=i: FakeFlatEnv(seed=i, horizon=7) for i in range(2)])
    m = PPO2(MlpPolicy, env, n_steps=16, nminibatches=4, noptepochs=3, seed=5, tensorboard_log=str(tmp_path))
    m.learn(100)                                                  # n_batch 32: 3 updates
    steps, eps = summaries(str(tmp_path / "PPO2_1"))
    assert [s for s, _ in steps] == [32, 64, 96]
    assert "loss/approximate_kullback-leibler" in steps[0][1] and eps == 2 * (48 // 7)
    m.close()
    t = TRPO(MlpPolicy, VecNormalize(DummyVecEnv([lambda: FakeFlatEnv(horizon=7, obs_dim=6, n_act=3)])), timesteps_per_batch=128,
             seed=1, policy_kwargs={"layers": [16, 16]}, tensorboard_log=str(tmp_path))
    t.learn(300)                                                  # 3 iterations
    steps, eps = summaries(str(tmp_path / "TRPO_1"))
    assert [s for s, _ in steps] == [128, 256, 384]
    assert set(steps[0][1]) == {"policy_gradient_loss", "approximate_kullback-leibler", "entropy_loss", "value_function_loss"}
    assert eps == 384 // 7
    t.close()


def test_cli_resume_appends_to_the_same_run_directory(tmp_path, monkeypatch):
    from b200grasp import training_state
    monkeypatch.chdir(tmp_path)                     # sb_helper's rule: tensorboard_logs/<model_dir> under the working directory
    cfg = {"DQN": {"batch_size": 16, "prioritized_replay": False, "total_timesteps": 1300, "tensorboard_logs": "tensorboard_logs/dqn"},
           "discount_factor": 0.99, "robot": {"discrete": False}, "reward": {}, "normalize": False}
    (tmp_path / "c.yaml").write_text(yaml.safe_dump(cfg))
    args = ["--env", "tests.test_gpu_dqn:make_env", "--eval_freq", "5000", "--checkpoint_freq", "5000", "--state_freq", "650"]
    model = train_cli.main(["train", "--config", "c.yaml", "--algo", "DQN", "--model_dir", "run"] + args)
    assert model.tensorboard_log == "tensorboard_logs/run"
    model.close()
    log = os.path.join("tensorboard_logs", "run")
    assert os.listdir(log) == ["DQN_1"]
    steps, _ = summaries(os.path.join(log, "DQN_1"))
    assert [s for s, _ in steps] == list(range(1001, 1301))       # learning_starts 1000 (stable-baselines' default)
    run_cfg = yaml.safe_load(open("run/config.yaml"))
    run_cfg["DQN"]["total_timesteps"] = 1500
    yaml.safe_dump(run_cfg, open("run/config.yaml", "w"))
    done = int(training_state.read_host(training_state.resolve("run/training_state"))["num_timesteps"])
    model = train_cli.main(["train", "--resume", "run"] + args)
    assert model.num_timesteps == 1500
    model.close()
    assert os.listdir(log) == ["DQN_1"]
    files = event_files(os.path.join(log, "DQN_1"))
    assert len(files) == 2
    resumed = [e["step"] for f in files[1:] for e in read_events(f)[1:] if "episode_reward" not in dict(e["values"])]
    assert resumed == list(range(max(done, 1000) + 1, 1501))
