"""CPU tests (no GPU): oracle cross-checks and artefact pins, host logic, C-ABI symbol table."""
import json
import os
import pickle
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import b200grasp
from b200grasp import _lib, sb_io, synth
from b200grasp.callbacks import BaseCallback, as_callback
from b200grasp.vec_env import DummyVecEnv, RunningMeanStd, VecNormalize
from oracle import sac_ref as R
from oracle import sac_ref_np as N
from tests.fake_env import FakeGraspEnv
from tests.util import GOLD, load_case, make_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------ oracle: two restatements agree
@pytest.mark.parametrize("obs_shape", [(64, 64, 2), (64, 64, 5), (101,)])
def test_oracle_autograd_vs_hand_derived_backward(obs_shape):
    cfg = R.SACConfig(obs_shape=obs_shape)
    p = R.init_params(cfg, 1)
    rng = np.random.default_rng(0)
    for n in p:                      # non-zero biases so every ReLU pattern is exercised
        if n.endswith("/b") or n.endswith("bias"):
            p[n] = (rng.normal(size=p[n].shape) * 0.1).astype(np.float32)
    B = 3
    batch = dict(obs=(rng.normal(size=(B,) + obs_shape) * 3).clip(-10, 10).astype(np.float32),
                 next_obs=(rng.normal(size=(B,) + obs_shape) * 3).astype(np.float32),
                 act=rng.uniform(-1, 1, (B, 5)).astype(np.float32), rew=rng.normal(size=B).astype(np.float32),
                 done=(rng.random(B) < 0.3).astype(np.float32))
    eps = rng.normal(size=(B, 5)).astype(np.float32)
    res, g, _, _ = R.sac_step(p, R.OptState.zeros(p), batch, eps, 3e-4, cfg, torch.float64)
    out2, g2 = N.sac_grads(p, batch, eps, cfg)
    for k in ("q1", "q2", "v", "logp", "policy_loss", "qf1_loss", "qf2_loss", "value_loss", "ent_coef_loss", "entropy"):
        assert np.allclose(np.asarray(res[k]), np.asarray(out2[k]), rtol=1e-10, atol=1e-12), k
    for n in g:
        assert np.abs(g[n] - g2[n]).max() <= 1e-9 * max(1e-30, np.abs(g[n]).max()), n


# ------------------------------------------------------------------ oracle pinned by the reference's artefacts
def test_param_inventory_matches_shipped_zips():
    man = json.load(open(os.path.join(GOLD, "zip_manifest.json")))
    for key, shape in (("sac_depth", (64, 64, 2)), ("sac_rgbd", (64, 64, 5)), ("sac_encoder", (101,))):
        specs = R.param_specs(R.SACConfig(obs_shape=shape))
        z = man[key]["shapes"]
        assert set(n for n, _ in specs) == set(z.keys())
        for n, s in specs:
            assert list(s) == z[n], (key, n, s, z[n])
        assert sum(int(np.prod(s)) for _, s in specs) == man[key]["n_floats"]
    d = man["sac_depth"]["data"]
    assert d["tau"] == 0.005 and d["gamma"] == 0.99 and d["learning_starts"] == 100 and d["train_freq"] == 1
    assert d["ent_coef"] == "auto" and d["batch_size"] == 64 and d["buffer_size"] == 1000000
    assert man["sac_depth"]["n_floats"] == 1976751 and man["sac_rgbd"]["n_floats"] == 1995183 and man["sac_encoder"]["n_floats"] == 54991


def test_zip_parameter_order_is_the_oracles_order():
    raw = np.load(os.path.join(GOLD, "sac_depth_params.npz"))        # np.savez keeps the zip's parameter_list order
    assert [n for n, _ in R.param_specs(R.SACConfig())] == list(raw.keys())
    enc = np.load(os.path.join(GOLD, "sac_encoder_params.npz"))
    assert [n for n, _ in R.param_specs(R.SACConfig(obs_shape=(101,)))] == list(enc.keys())
    # trainable / target split of SURVEY Appendix B
    specs = R.param_specs(R.SACConfig())
    n_train = sum(int(np.prod(s)) for n, s in specs if R.group_of(n) != "target")
    assert n_train == 1342990 and sum(int(np.prod(s)) for n, s in specs if R.group_of(n) == "target") == 633761


def test_known_answer_ent_coef_trajectory():
    """logs.csv row 1 of SAC_full_rgbd: ent_coef = 0.9388962 at total_timesteps = 310, i.e. 210 entropy-Adam
    steps (learning_starts = 100) of constant sign: TF-Adam then moves log_alpha by ~lr per step."""
    logs = json.load(open(os.path.join(GOLD, "logs_head.json")))["sac_rgbd"]
    assert logs["total_timesteps"][0] == 310
    m = v = 0.0
    log_alpha, lr = 0.0, 3e-4
    rng = np.random.default_rng(0)
    for t in range(1, 211):
        g = 8.0 + rng.normal()           # d ent_coef_loss / d log_alpha = -(logp + H) > 0 early in training
        m = R.ADAM_B1 * m + (1 - R.ADAM_B1) * g
        v = R.ADAM_B2 * v + (1 - R.ADAM_B2) * g * g
        lr_t = lr * np.sqrt(1 - R.ADAM_B2 ** t) / (1 - R.ADAM_B1 ** t)
        log_alpha -= lr_t * m / (np.sqrt(v) + R.ADAM_EPS)
    assert abs(np.exp(log_alpha) - logs["ent_coef"][0]) < 2e-3
    assert abs(np.exp(-3e-4 * 210) - logs["ent_coef"][0]) < 1e-4


@pytest.mark.parametrize("run", ["sac_rgbd", "sac_depth"])
def test_known_answer_ent_coef_follows_unit_adam_steps_over_2000_updates(run):
    """Every logged row of the two shipped image runs (trained_models/SAC_full_rgbd, SAC_depth_1mbuffer logs.csv):
    ent_coef(t) = exp(-3e-4 * (t - 100)) to 1e-4 for t up to 2114.  That single curve pins, in the reference's own
    output, learning_starts = 100, ONE gradient step per environment step, and the TF1 Adam step the oracle and the
    CUDA optimiser implement: with a gradient of constant sign, lr_t * m_t / (sqrt(v_t) + eps) = lr at every t (the
    bias corrections cancel exactly), so log_alpha falls by lr per update.  (The vector run SAC_encoder_1mbuffer decays
    about 2 % faster -- its gradient magnitude trends -- and is left out.)"""
    logs = json.load(open(os.path.join(GOLD, "logs_head.json")))[run]
    for t_env, ec in zip(logs["total_timesteps"], logs["ent_coef"]):
        assert abs(np.log(ec) + 3e-4 * (t_env - 100)) < 2e-4, (t_env, ec)
    # the oracle's optimiser on a constant-sign gradient of varying size reproduces the unit step
    n_upd = logs["total_timesteps"][-1] - 100
    rng = np.random.default_rng(3)
    m = v = 0.0
    log_alpha = 0.0
    for t in range(1, n_upd + 1):
        g = 3.0 + 2.0 * rng.random()
        m = R.ADAM_B1 * m + (1 - R.ADAM_B1) * g
        v = R.ADAM_B2 * v + (1 - R.ADAM_B2) * g * g
        log_alpha -= 3e-4 * np.sqrt(1 - R.ADAM_B2 ** t) / (1 - R.ADAM_B1 ** t) * m / (np.sqrt(v) + R.ADAM_EPS)
    assert abs(log_alpha - np.log(logs["ent_coef"][-1])) < 0.03 * abs(np.log(logs["ent_coef"][-1]))


def test_known_answer_initial_entropy_and_logp_sign():
    """Same log row: entropy 6.513 => mean log_std = (6.513 - 5*0.5*ln(2*pi*e))/5 ~ -0.116; and
    ent_coef_loss / log(ent_coef) => mean logp ~ -3.46, which the oracle's squashed-Gaussian logp must
    reproduce for mu = 0 (sign and EPS placement of the tanh correction)."""
    logs = json.load(open(os.path.join(GOLD, "logs_head.json")))["sac_rgbd"]
    ls = (logs["entropy"][0] - 5 * 0.5 * np.log(2 * np.pi * np.e)) / 5
    assert -0.2 < ls < -0.05
    mean_logp_log = -logs["ent_coef_loss"][0] / np.log(logs["ent_coef"][0]) + 5.0     # L = -log_alpha*(logp - 5)
    eps = np.random.default_rng(1).standard_normal((200000, 5))
    std = np.exp(ls)
    u = eps * std
    logp = (-0.5 * ((u / (std + R.EPS)) ** 2 + 2 * ls + np.log(2 * np.pi))).sum(1) - np.log(1 - np.tanh(u) ** 2 + R.EPS).sum(1)
    assert abs(logp.mean() - mean_logp_log) < 0.35, (logp.mean(), mean_logp_log)


def test_vecnormalize_formula_on_the_real_frame():
    vn = dict(np.load(os.path.join(GOLD, "vecnorm_sac_depth.npz")))
    o = vn["old_obs"]
    n = R.normalize_obs(o, vn["obs_mean"], vn["obs_var"], float(vn["clip_obs"]), float(vn["epsilon"]))
    assert n.dtype == np.float32 and np.abs(n).max() <= 10.0
    # zero pad plane: (0 - 0)/sqrt(8.7e-11 + 1e-8) == 0 ; gripper-width pixel is finite
    assert np.all(n[0, 1:, :, 1] == 0) and np.isfinite(n[0, 0, 0, 1])
    assert float(vn["clip_obs"]) == 10.0 and float(vn["clip_reward"]) == 10.0 and float(vn["epsilon"]) == 1e-8 and float(vn["gamma"]) == 0.99
    r = R.normalize_reward(np.array([-200.0, 10000.0, 1e9]), float(vn["ret_var"]))
    assert r[2] == 10.0 and abs(r[0] + 200 / np.sqrt(float(vn["ret_var"]) + 1e-8)) < 1e-6


def test_golden_step_vector_is_reproducible():
    gold = np.load(os.path.join(GOLD, "golden_step_sac_depth_b32.npz"))
    cfg, params, vn = load_case("sac_depth")
    raw, norm, eps = make_batch(vn, 32)
    res, grads, _, _ = R.sac_step(params, R.OptState.zeros(params), norm, eps, 3e-4, cfg, torch.float32)
    for k in ("q1", "q2", "v"):
        assert np.allclose(np.asarray(res[k]).reshape(-1), gold[k].reshape(-1), rtol=2e-5, atol=1e-6), k
    assert abs(res["grad_norm_values"] - float(gold["grad_norm_values"])) <= 1e-4 * float(gold["grad_norm_values"])


def test_bdq_param_inventory_matches_shipped_zips():
    from oracle import bdq_ref as Q
    man = json.load(open(os.path.join(GOLD, "zip_manifest.json")))
    for key, cfg in (("bdq_8pads", Q.BDQConfig(100, 3, 8, (64, 64), 32, 32)), ("bdq_33big", Q.BDQConfig(100, 3, 33, (512, 256), 128, 128))):
        specs = dict(Q.all_specs(cfg))
        z = man[key]["shapes"]
        assert set(specs) == set(z), set(specs) ^ set(z)
        for n, shp in specs.items():
            assert list(shp) == z[n], (key, n)
        assert sum(int(np.prod(s)) for s in specs.values()) == man[key]["n_floats"]
    d = man["bdq_8pads"]["data"]
    assert d["double_q"] is True and d["target_network_update_freq"] == 1000 and d["num_actions_pad"] == 8 and d["batch_size"] == 64


# ------------------------------------------------------------------ C ABI
def test_shared_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "b200grasp.h")).read()
    declared = sorted(set(re.findall(r"\b(b2g_[a-z0-9_]+)\s*\(", hdr)) - {"b2g_sac_cfg", "b2g_sac_metrics"})
    assert set(declared) == set(_lib.SYMBOLS), set(declared) ^ set(_lib.SYMBOLS)
    lib = _lib.load()
    for s in declared:
        assert hasattr(lib, s), s
    assert lib.b2g_version() >= 100
    nm = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for s in declared:
        assert re.search(rf"\bT {s}\b", nm), s


def test_no_cpu_fallback_create_fails_loudly_without_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.B2GError) as e:
        b200grasp.Learner((64, 64, 2))
    assert "-2" in str(e.value) or "CUDA" in str(e.value)


def test_design_switch_table_lists_every_environment_switch():
    """DESIGN.md §4 documents exactly the B2G_* environment variables the library reads."""
    csrc = os.path.join(ROOT, "deep-rl-grasping_b200", "csrc")
    read = set()
    for f in os.listdir(csrc):
        with open(os.path.join(csrc, f)) as fh:
            read |= set(re.findall(r'getenv\("(B2G_[A-Z_0-9]+)"\)', fh.read()))
    with open(os.path.join(ROOT, "DESIGN.md")) as fh:
        design = fh.read()
    table = design.split("### Switches (environment variables")[1].split("\n\n")[1]
    documented = set()
    for row in table.splitlines()[2:]:
        documented |= set(re.findall(r"`(B2G_[A-Z_0-9]+)", re.split(r"(?<!\\)\|", row)[1]))     # first column; "\|" is a literal bar
    assert read and read == documented, (sorted(read - documented), sorted(documented - read))


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "deep-rl-grasping_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), f


# ------------------------------------------------------------------ host logic
def test_running_mean_std_and_vecnormalize_roundtrip(tmp_path):
    rng = np.random.default_rng(0)
    rms = RunningMeanStd(shape=(3,))
    data = rng.normal(2.0, 3.0, (1000, 3))
    for i in range(0, 1000, 50):
        rms.update(data[i:i + 50])
    assert np.allclose(rms.mean, data.mean(0), atol=1e-3) and np.allclose(rms.var, data.var(0), rtol=1e-3)
    env = VecNormalize(DummyVecEnv([lambda: FakeGraspEnv(0, obs_shape=(8, 8, 2))]), norm_obs=True, norm_reward=True, clip_obs=10.0)
    obs = env.reset()
    for _ in range(30):
        obs, r, d, info = env.step(np.zeros((1, 5), np.float32))
    assert obs.shape == (1, 8, 8, 2) and np.abs(obs).max() <= 10 and env.get_original_obs().shape == (1, 8, 8, 2)
    p = str(tmp_path / "vecnormalize.pkl")
    env.save(p)                                   # pickle naming stable_baselines' classes
    back = sb_io.load_vecnormalize(p)             # readable without stable_baselines
    assert np.allclose(back["obs_mean"], env.obs_rms.mean) and back["clip_obs"] == 10.0 and back["ret_var"] == float(env.ret_rms.var)
    vn2 = VecNormalize.load(p, env.venv)
    assert np.allclose(vn2.obs_rms.var, env.obs_rms.var)
    raw = pickle.dumps(0)
    assert b"stable_baselines.common.vec_env.vec_normalize" in open(p, "rb").read() and raw


def test_sb_zip_roundtrip(tmp_path):
    cfg = R.SACConfig(obs_shape=(101,))
    params = R.init_params(cfg, 2)
    p = str(tmp_path / "m.zip")
    sb_io.save_sb_zip(p, {"gamma": 0.99, "tau": 0.005, "fn": (lambda x: x)}, params)
    data, back = sb_io.load_sb_zip(p)
    assert list(back.keys()) == list(params.keys()) and data["gamma"] == 0.99
    for n in params:
        assert np.array_equal(back[n], params[n])
    import zipfile
    assert sorted(zipfile.ZipFile(p).namelist()) == ["data", "parameter_list", "parameters"]
    assert json.loads(zipfile.ZipFile(p).read("parameter_list"))[0].endswith(":0")


def test_callback_protocol_order():
    calls = []

    class C(BaseCallback):
        def _on_training_start(self):
            calls.append("start")

        def _on_rollout_start(self):
            calls.append("rs")

        def _on_step(self):
            calls.append("step")
            return self.n_calls < 2

        def _on_rollout_end(self):
            calls.append("re")

    class M:
        num_timesteps = 0

        def get_env(self):
            return "env"
    cb = as_callback([C(), lambda l, g: True])
    cb.init_callback(M())
    cb.on_training_start({"writer": None}, {})
    cb.on_rollout_start()
    assert cb.on_step() is True
    assert cb.on_step() is False
    cb.on_rollout_end()
    assert calls == ["start", "rs", "step", "step", "re"] and cb.callbacks[0].training_env == "env"


def test_synthetic_data_is_seeded_and_shaped():
    vn = dict(np.load(os.path.join(GOLD, "vecnorm_sac_depth.npz")))
    a = synth.make_transitions(4, vn["obs_mean"], vn["obs_var"])
    b = synth.make_transitions(4, vn["obs_mean"], vn["obs_var"])
    assert all(np.array_equal(a[k], b[k]) for k in a)
    assert a["obs"].shape == (4, 64, 64, 2) and a["obs"].dtype == np.float32
    assert np.all(a["obs"][:, 1:, :, 1] == 0) and np.all((a["obs"][..., 0] >= 0.02) & (a["obs"][..., 0] <= 2.0))
    assert synth.make_eps(4).shape == (4, 5) and synth.make_indices(8, 100).max() < 100


# ------------------------------------------------------------------ N > 1 host path on gloo (world size 2)
_WORKER = r'''
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, %r)
import b200grasp
from b200grasp import dist_utils
from oracle import sac_ref as R, sac_ref_np as N
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
nid = dist_utils.share_nccl_id(lambda: bytes(range(128)))
assert nid == bytes(range(128))
assert dist_utils.shard_seed(7, 0) != dist_utils.shard_seed(7, 1)
# data-parallel identity behind the design: mean over ranks of per-rank mean-loss gradients == full-batch gradient
cfg = R.SACConfig(obs_shape=(101,))
p = R.init_params(cfg, 3)
rng = np.random.default_rng(5)
B = 4
batch = dict(obs=rng.normal(size=(B, 101)).astype(np.float32), next_obs=rng.normal(size=(B, 101)).astype(np.float32),
             act=rng.uniform(-1, 1, (B, 5)).astype(np.float32), rew=rng.normal(size=B).astype(np.float32), done=np.zeros(B, np.float32))
eps = rng.normal(size=(B, 5)).astype(np.float32)
sl = slice(rank * B // world, (rank + 1) * B // world)
_, g_local = N.sac_grads(p, {k: v[sl] for k, v in batch.items()}, eps[sl], cfg)
_, g_full = N.sac_grads(p, batch, eps, cfg)
flat = torch.tensor(np.concatenate([g_local[n].reshape(-1) for n in g_local]))
dist.all_reduce(flat)                      # what ncclAllReduce(sum) + grad_scale = 1/world does on the device
flat /= world
ref = np.concatenate([g_full[n].reshape(-1) for n in g_full])
assert np.abs(flat.numpy() - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), np.abs(flat.numpy() - ref).max()
assert dist_utils.weak_scaling_value(100.0, world) == 200.0
dist.barrier(); dist.destroy_process_group(); print("ok " + str(rank), flush=True)
'''


def test_world_size_2_gloo_host_path(tmp_path):
    import socket
    script = tmp_path / "w.py"
    script.write_text(_WORKER % ROOT)
    with socket.socket() as sk:                 # a free port (a fixed one can sit in TIME_WAIT between runs)
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", str(port), str(script)], capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, OMP_NUM_THREADS="2"))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "ok 0" in r.stdout and "ok 1" in r.stdout


@pytest.mark.parametrize("cfull,threads", [(2, 1), (2, 7), (5, 4)])
def test_host_compaction_matches_numpy(cfull, threads):
    """b2g_sac_step_host_pipelined compacts observations on the host before the copy (the constant actuator plane never crosses
    PCIe): rows = image planes | value of the last plane at pixel [0,0] | three zeros -- the layout of the device replay
    (custom_obs_policy.py:20-23 reads that one pixel).  Host-only entry point, no device needed."""
    import ctypes as C
    from b200grasp import _lib
    lib = _lib.load()
    rng = np.random.default_rng(5)
    n, hw = 37, 64 * 64
    src = rng.standard_normal((n, hw, cfull)).astype(np.float32)
    dst = np.full((n, hw * (cfull - 1) + 4), np.nan, np.float32)
    rc = lib.b2g_debug_compact_host(src.ctypes.data_as(C.c_void_p), dst.ctypes.data_as(C.c_void_p), n, hw, cfull, threads)
    assert rc == 0
    ref = np.concatenate([src[:, :, :cfull - 1].reshape(n, -1), src[:, 0, cfull - 1:cfull], np.zeros((n, 3), np.float32)], axis=1)
    assert np.array_equal(dst, ref)
