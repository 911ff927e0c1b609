"""Training-state directories without a GPU: host.json, the atomic directory swap and the CLI flags (training_state.py,
train_cli.py)."""
import os

import numpy as np
import pytest

from b200grasp import train_cli, training_state


class FakeLearner:
    def __init__(self, fail=False):
        self.fail = fail

    def save_state(self, path):
        with open(path, "wb") as f:
            f.write(b"half a replay")
        if self.fail:
            raise OSError("disk full")


class FakeModel:
    def __init__(self, tag, fail=False, seed=0):
        self.tag, self.learner = tag, FakeLearner(fail)
        self._rng = np.random.default_rng(seed)

    def save(self, path):
        with open(path, "w") as f:
            f.write(self.tag)

    def get_vec_normalize_env(self):
        return None

    def _host_state(self):
        return {"algo": "SAC", "num_timesteps": np.int64(123), "rng": training_state.rng_state(self._rng), "tag": self.tag}


def test_host_json_round_trips_the_generator_state(tmp_path):
    m = FakeModel("a", seed=42)
    m._rng.random(17)                                  # mid-stream, with a buffered 32-bit half pending
    m._rng.integers(0, 2 ** 31, dtype=np.uint32)
    d = training_state.save_training_state(m, str(tmp_path / "ts"))
    host = training_state.read_host(d)
    assert host["num_timesteps"] == 123 and host["format"] == training_state.FORMAT
    r = np.random.default_rng(0)
    training_state.set_rng_state(r, host["rng"])
    assert np.array_equal(r.random(50), m._rng.random(50))
    assert np.array_equal(r.integers(0, 9, 30), m._rng.integers(0, 9, 30))


def test_failed_write_keeps_the_previous_checkpoint(tmp_path):
    d = str(tmp_path / "ts")
    training_state.save_training_state(FakeModel("old"), d)
    with pytest.raises(OSError, match="disk full"):
        training_state.save_training_state(FakeModel("new", fail=True), d)
    assert open(os.path.join(d, "model.zip")).read() == "old"
    assert sorted(os.listdir(tmp_path)) == ["ts"]      # no half-written directory left behind
    assert training_state.resolve(d) == os.path.normpath(d)
    training_state.save_training_state(FakeModel("new"), d)
    assert open(os.path.join(d, "model.zip")).read() == "new"
    assert sorted(os.listdir(tmp_path)) == ["ts"]


def test_reader_finds_the_checkpoint_between_the_two_renames(tmp_path):
    d = str(tmp_path / "ts")
    training_state.save_training_state(FakeModel("old"), d)
    os.rename(d, d + ".old")
    assert training_state.resolve(d) == d + ".old"
    with pytest.raises(FileNotFoundError):
        training_state.resolve(str(tmp_path / "nothing"))


def test_cli_flags_parse():
    p = train_cli.build_parser()
    a = p.parse_args(["train", "--resume", "runs/sac", "--state_freq", "5000"])
    assert a.func is train_cli.train and a.resume == "runs/sac" and a.state_freq == 5000 and a.config is None
    a = p.parse_args(["train", "--config", "c.yaml", "--algo", "SAC", "--model_dir", "m", "--state_freq", "100"])
    assert a.state_freq == 100 and a.resume is None
    a = p.parse_args(["train", "--config", "c.yaml", "--algo", "SAC", "--model_dir", "m"])
    assert a.state_freq is None and a.resume is None
    with pytest.raises(SystemExit):
        train_cli.main(["train", "--algo", "SAC"])     # --config / --model_dir are still required without --resume
