"""CPU side of the BDQ / DQN replay frames (``replay_frames=``): ABI, host.json, the CLI's budget, refusals, sm_90a compile."""
import argparse
import inspect
import os
import shutil
import subprocess

import pytest

from b200grasp import BDQ, _lib, train_cli
from b200grasp.deepq import DQN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["b2g_bdq_create2", "b2g_bdq_replay_info", "b2g_bdq_replay_get", "b2g_dqn_create2", "b2g_dqn_replay_info", "b2g_dqn_replay_get"]


def test_abi_is_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "b200grasp.h")).read()
    for s in NEW:
        assert s in _lib.SYMBOLS and f"int {s}(" in header, s
    assert "int64_t b2g_transition_replay_bytes(" in header and "b2g_transition_replay_bytes" in _lib.SYMBOLS
    assert [f for f, _ in _lib.ReplayCfg._fields_] == ["frame_capacity", "u8_plane_mask"]
    if os.path.exists(_lib.LIB_PATH):
        lib = _lib.load()
        assert all(hasattr(lib, s) for s in NEW)


def test_replay_bytes_without_allocating():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    from b200grasp.learner import transition_replay_bytes
    for E in (100, 8192):
        row = (4 * E + 15) // 16 * 16
        assert transition_replay_bytes(1000, E, 3, 1130) == 1130 * row + 8 * 1000 + 1000 * 5 * 4
        assert transition_replay_bytes(1000, E, 3) == 8 * E * 1000 + 1000 * 5 * 4
    # the depth BDQ of config/gripper_grasp.yaml at 10^6 slots, --replay_spare 0.125 (one env): ~36.9 GB against 65.5 GB
    assert round(transition_replay_bytes(10**6, 8192, 3, int(10**6 * 1.125) + 1) / 1e9, 1) == 36.9
    assert 65.5 <= transition_replay_bytes(10**6, 8192, 3) / 1e9 < 65.6


def test_replay_spare_maps_to_replay_frames():
    a = argparse.Namespace(replay_spare=0.125)
    assert train_cli.replay_frames_kwargs(a, 10**6, 4) == {"replay_frames": 1125004}
    assert train_cli.replay_frames_kwargs(argparse.Namespace(replay_spare=None), 10**6, 4) == {}
    # DQN's budget starts from stable-baselines' default buffer_size, which sb_helper leaves in place
    assert inspect.signature(DQN).parameters["buffer_size"].default == 50000
    src = inspect.getsource(train_cli.train)
    assert src.count("replay_frames_kwargs(") == 3          # SAC, BDQ, DQN


def test_host_json_records_replay_frames():
    for cls, kw in ((BDQ, {}), (DQN, {})):
        m = cls("MlpActPolicy" if cls is BDQ else "MlpPolicy", None, replay_frames=5000, learning_rate=1e-3, **kw)
        init = m._host_state()["init"]
        assert init["replay_frames"] == 5000
        again = cls("MlpActPolicy" if cls is BDQ else "MlpPolicy", None, **init)
        assert again.replay_frames == 5000
        plain = cls("MlpActPolicy" if cls is BDQ else "MlpPolicy", None, learning_rate=1e-3)
        assert plain.replay_frames is None and "replay_frames" not in plain._host_state()["init"]


def test_refusals():
    with pytest.raises(NotImplementedError, match="replay_frames"):
        BDQ("MlpActPolicy", None, replay_frames=5000, nranks=2)


def test_touched_sources_compile_for_sm90a_without_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not shutil.which(nvcc):
        pytest.skip("nvcc not found")
    for f in ("per.cu", "bdq.cu", "dqn.cu"):          # (state.cu and q_learner.cu, also touched, hold no kernels)
        src = os.path.join(ROOT, "deep-rl-grasping_b200", "csrc", f)
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                            "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / (f + ".o"))], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        spills = [l for l in r.stderr.splitlines() if "spill" in l]
        assert spills and all(" 0 bytes spill stores" in l for l in spills), (f, spills)
