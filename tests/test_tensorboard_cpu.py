"""TensorBoard event files without tensorflow (b200grasp.tensorboard): checksums, framing, the Event / Summary encoding read
back by an independent reader, run-directory numbering, the tf.Summary stand-in under a success-rate callback, train_cli's
log directory and the metrics-ring ABI.  No GPU needed."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import b200grasp
from b200grasp import _lib, train_cli
from b200grasp import tensorboard as tb
from b200grasp.base_model import BaseModel
from b200grasp.callbacks import BaseCallback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------ an independent reader (bitwise CRC, hand-rolled protobuf)
def crc32c_bitwise(data: bytes) -> int:
    crc = 0xFFFFFFFF
    for b in data:
        crc ^= b
        for _ in range(8):
            crc = (crc >> 1) ^ (0x82F63B78 if crc & 1 else 0)
    return crc ^ 0xFFFFFFFF


def masked(crc: int) -> int:
    return ((((crc >> 15) | (crc << 17)) & 0xFFFFFFFF) + 0xA282EAD8) & 0xFFFFFFFF


def read_varint(b, i):
    v = s = 0
    while True:
        x = b[i]
        i += 1
        v |= (x & 0x7F) << s
        s += 7
        if not x & 0x80:
            return v, i


def parse_fields(b):
    """(field number, wire type, value) of one protobuf message."""
    i, out = 0, []
    while i < len(b):
        key, i = read_varint(b, i)
        f, wt = key >> 3, key & 7
        if wt == 0:
            v, i = read_varint(b, i)
        elif wt == 1:
            v = b[i:i + 8]; i += 8
        elif wt == 5:
            v = b[i:i + 4]; i += 4
        elif wt == 2:
            n, i = read_varint(b, i)
            v = b[i:i + n]; i += n
        else:
            raise AssertionError(f"wire type {wt}")
        out.append((f, wt, v))
    return out


def read_events(path):
    """[{wall_time, step, file_version | values: [(tag, value)]}] with every framing checksum verified."""
    data = open(path, "rb").read()
    i, events = 0, []
    while i < len(data):
        head = data[i:i + 8]
        (n,) = struct.unpack("<Q", head)
        assert struct.unpack("<I", data[i + 8:i + 12])[0] == masked(crc32c_bitwise(head))
        body = data[i + 12:i + 12 + n]
        assert struct.unpack("<I", data[i + 12 + n:i + 16 + n])[0] == masked(crc32c_bitwise(body))
        i += 16 + n
        ev = {"step": 0, "values": []}
        for f, _, v in parse_fields(body):
            if f == 1:
                ev["wall_time"] = struct.unpack("<d", v)[0]
            elif f == 2:
                ev["step"] = v
            elif f == 3:
                ev["file_version"] = v.decode()
            elif f == 5:
                for sf, _, sv in parse_fields(v):
                    assert sf == 1
                    d = {ff: vv for ff, _, vv in parse_fields(sv)}
                    ev["values"].append((d[1].decode(), struct.unpack("<f", d[2])[0]))
        events.append(ev)
    return events


def event_files(d):
    return sorted(os.path.join(d, f) for f in os.listdir(d) if f.startswith("events.out.tfevents."))


# ------------------------------------------------------------------ checksums
def test_crc32c_check_value_and_mask():
    assert tb.crc32c(b"123456789") == 0xE3069283
    c = 0xE3069283
    assert tb.masked_crc32c(b"123456789") == ((((c >> 15) | (c << 17)) + 0xA282EAD8) & 0xFFFFFFFF)
    assert tb.crc32c(b"") == 0


def test_crc32c_batch_matches_bitwise_for_ragged_records():
    rng = np.random.default_rng(0)
    recs = [bytes(rng.integers(0, 256, n, dtype=np.uint8)) for n in (0, 1, 7, 8, 33, 200, 5)]
    got = tb.crc32c_batch(recs)
    assert [int(x) for x in got] == [crc32c_bitwise(r) for r in recs]


# ------------------------------------------------------------------ writing and reading back
def test_writer_round_trip(tmp_path):
    w = tb.EventWriter(str(tmp_path))
    w.add_summary(tb.Summary(value=[tb.Summary.Value(tag="success_rate", simple_value=0.25)]), 7)
    rows = np.array([[1.5, -2.0], [3.25, 1e-3], [0.0, 7.0]], np.float32)
    w.add_scalars(["policy_loss", "learning_rate"], [10, 10, 300], rows)
    w.close()
    (path,) = event_files(str(tmp_path))
    ev = read_events(path)
    assert ev[0]["file_version"] == "brain.Event:2" and not ev[0]["values"]
    assert ev[1]["step"] == 7 and ev[1]["values"] == [("success_rate", 0.25)]
    assert [e["step"] for e in ev[2:]] == [10, 10, 300]
    for e, r in zip(ev[2:], rows):
        assert e["values"] == [("policy_loss", float(r[0])), ("learning_rate", float(r[1]))]
    assert all(abs(e["wall_time"] - ev[0]["wall_time"]) < 60 for e in ev)
    # a real tf.Summary-shaped object works too (any .value[i].tag / .simple_value)
    class V:
        tag, simple_value = "x", np.float64(2.0)

    class S:
        value = [V()]
    w2 = tb.EventWriter(str(tmp_path / "b"))
    w2.add_summary(S(), 2 ** 40)
    w2.close()
    assert read_events(event_files(str(tmp_path / "b"))[0])[1] == {"step": 2 ** 40, "values": [("x", 2.0)],
                                                                   "wall_time": pytest.approx(ev[0]["wall_time"], abs=60)}


def test_writer_against_tensorboards_reader_when_installed(tmp_path):
    loader_mod = pytest.importorskip("tensorboard.backend.event_processing.event_file_loader")
    event_pb2 = pytest.importorskip("tensorboard.compat.proto.event_pb2")
    w = tb.EventWriter(str(tmp_path))
    w.add_scalars(["a", "b"], [1, 2], [[0.5, 1.5], [2.5, 3.5]])
    w.close()
    # the raw loader checks the framing; the records are then parsed as Event protos (no simple_value -> tensor migration)
    evs = [event_pb2.Event.FromString(r) for r in loader_mod.RawEventFileLoader(event_files(str(tmp_path))[0]).Load()]
    assert evs[0].file_version == "brain.Event:2"
    vals = [(e.step, [(v.tag, v.simple_value) for v in e.summary.value]) for e in evs[1:]]
    assert vals == [(1, [("a", 0.5), ("b", 1.5)]), (2, [("a", 2.5), ("b", 3.5)])]


# ------------------------------------------------------------------ run directories
class _Model(BaseModel):
    def __init__(self, log):
        self.tensorboard_log = log


def test_run_directory_numbering_and_continuation(tmp_path):
    log = str(tmp_path / "logs")
    m = _Model(log)
    seen = []
    m._learn_logged("SAC", True, lambda w, s: seen.append((w.logdir, s)))
    m._learn_logged("SAC", True, lambda w, s: seen.append((w.logdir, s)))
    os.makedirs(os.path.join(log, "SAC_x"))             # not a run id
    os.makedirs(os.path.join(log, "SAC_b_9"))           # another name
    m._learn_logged("SAC", False, lambda w, s: seen.append((w.logdir, s)))     # reset_num_timesteps=False: the latest
    m._learn_logged("DQN", False, lambda w, s: seen.append((w.logdir, s)))
    assert [os.path.basename(d) for d, _ in seen] == ["SAC_1", "SAC_2", "SAC_2", "DQN_0"]
    assert all(s is None for _, s in seen)
    assert len(event_files(os.path.join(log, "SAC_2"))) == 2          # the continued run adds a file beside the first
    os.makedirs(os.path.join(log, "SAC_10"))
    assert tb.latest_run_id(log, "SAC") == 10
    # no log: no writer, no directory
    out = []
    _Model(None)._learn_logged("SAC", True, lambda w, s: out.append(w))
    assert out == [None]


def test_writer_is_closed_when_learn_raises(tmp_path):
    m = _Model(str(tmp_path))
    box = []

    def run(w, s):
        box.append(w)
        w.add_summary(tb.Summary([tb.Summary.Value("a", 1.0)]), 1)
        raise KeyboardInterrupt
    with pytest.raises(KeyboardInterrupt):
        m._learn_logged("PPO2", True, run)
    assert box[0]._fh is None
    assert read_events(box[0].path)[1]["values"] == [("a", 1.0)]


# ------------------------------------------------------------------ a success-rate callback against the stand-in
class SuccessRateCallback(BaseCallback):
    """What a tensorflow-era callback does with ``tf`` bound to b200grasp.tensorboard: a success_rate summary per new timestep."""

    def __init__(self, tf, rates):
        super().__init__()
        self.tf, self.rates, self.last = tf, rates, -1

    def _on_step(self):
        if self.num_timesteps != self.last:
            sr = self.rates[self.num_timesteps]
            summary = self.tf.Summary(value=[self.tf.Summary.Value(tag="success_rate", simple_value=sr)])
            self.locals["writer"].add_summary(summary, self.num_timesteps)
            self.last = self.num_timesteps
        return True


def test_success_rate_callback_writes_through_the_stand_in(tmp_path):
    from b200grasp import tensorboard as tf
    model = _Model(str(tmp_path))
    model.num_timesteps = 0
    model.get_env = lambda: None
    rates = {t: t / 10 for t in range(1, 6)}
    cb = SuccessRateCallback(tf, rates)

    def run(writer, _):
        cb.init_callback(model)
        cb.on_training_start({"self": model, "writer": writer}, {})
        for t in range(1, 6):
            model.num_timesteps = t
            cb.on_step()
    model._learn_logged("SAC", True, run)
    ev = read_events(event_files(str(tmp_path / "SAC_1"))[0])
    assert [(e["step"], e["values"]) for e in ev[1:]] == [(t, [("success_rate", pytest.approx(t / 10))]) for t in range(1, 6)]


def test_episode_reward_logger_follows_the_stable_baselines_rule(tmp_path):
    w = tb.EventWriter(str(tmp_path))
    lg = tb.EpisodeRewardLogger(2)
    rew = [[1, 10], [2, 20], [3, 30], [4, 40]]
    done = [[0, 0], [1, 0], [0, 1], [1, 0]]
    for k, (r, d) in enumerate(zip(rew, done)):
        lg(w, r, d, 2 * (k + 1))
    w.close()
    ev = [(e["step"], e["values"]) for e in read_events(event_files(str(tmp_path))[0])[1:]]
    # env 0 ends at steps 4 and 8: 1 (the ending reward 2 opens the next episode), then 2 + 3; env 1 ends at 6: 10 + 20
    assert ev == [(4, [("episode_reward", 1.0)]), (6, [("episode_reward", 30.0)]), (8, [("episode_reward", 5.0)])]
    assert lg.count == 3


# ------------------------------------------------------------------ train_cli
@pytest.mark.parametrize("section, expect", [({}, None), ({"tensorboard_logs": None}, None),
                                             ({"tensorboard_logs": "tensorboard_logs/ppo_5m"}, "tensorboard_logs/runs/a")])
def test_cli_log_directory_follows_sb_helper(section, expect):
    assert train_cli.tensorboard_log({"PPO": section}, "PPO", "runs/a") == expect
    assert train_cli.tensorboard_log({}, "PPO", "runs/a") is None


def test_cli_train_passes_the_log_directory(tmp_path, monkeypatch):
    import yaml
    seen = {}

    class Stop(Exception):
        pass

    def record(policy, env, **kw):
        seen.update(kw)
        raise Stop
    monkeypatch.setattr(train_cli, "PPO2", record)
    for i, logs in enumerate((None, "tensorboard_logs/ppo_5m")):
        cfg = {"discount_factor": 0.99, "normalize": False, "robot": {}, "reward": {}, "simplified": False,
               "PPO": {"learning_rate": 2.5e-4, "total_timesteps": 64, "tensorboard_logs": logs}}
        path = tmp_path / f"c{i}.yaml"
        yaml.safe_dump(cfg, open(path, "w"))
        mdir = str(tmp_path / f"run{i}")
        with pytest.raises(Stop):
            train_cli.main(["train", "--config", str(path), "--algo", "PPO", "--model_dir", mdir,
                            "--env", "tests.fake_env:make_env"])
        assert seen["tensorboard_log"] == (None if logs is None else "tensorboard_logs/" + mdir)


# ------------------------------------------------------------------ the metrics-ring ABI
NEW = ["b2g_sac_metrics_log", "b2g_sac_metrics_drain", "b2g_bdq_metrics_log", "b2g_bdq_metrics_drain",
       "b2g_dqn_metrics_log", "b2g_dqn_metrics_drain"]


def test_metrics_ring_abi_is_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "b200grasp.h")).read()
    for s in NEW:
        assert s in _lib.SYMBOLS and f"int {s}(" in header, s
    for k, n in (("SAC", 8), ("BDQ", 4), ("DQN", 6)):
        assert f"#define B2G_{k}_LOG_COLS {n}" in header and len(_lib.LOG_COLS[k.lower()]) == n
    if os.path.exists(_lib.LIB_PATH):
        lib = _lib.load()
        assert all(hasattr(lib, s) for s in NEW)


def test_metrics_log_compiles_for_sm90a(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not shutil.which(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "deep-rl-grasping_b200", "csrc", "metrics_log.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "m.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "metrics_log_append_kernel" in r.stderr and "spill" in r.stderr
    assert " 0 bytes spill stores" in r.stderr
