"""The named-parameter table, the transition replay and the training-state skeleton shared by the BDQ, DQN and PPO2 handles.

For each learner: the parameter listing against the oracle's specs, bitwise set / get round trips (with and without ":0"), the
gradient names, the refusals of a bad name or size, the layout of a saved training-state file (header, fingerprint names,
section tags and lengths, parsed here from the format in csrc/state.cu), and the refusals of a load (another learner's file,
a truncated file, a flipped byte).
"""
import struct

import numpy as np
import pytest

from b200grasp import _lib
from b200grasp.bdq import BDQLearner
from b200grasp.dqn import DQNLearner
from b200grasp.learner import _fp
from b200grasp.ppo2 import PPO2Learner
from oracle import bdq_ref as BR
from oracle import dqn_ref as DR
from oracle import ppo_ref as PR

pytestmark = pytest.mark.gpu

OBS, CAP, B = 7, 48, 8
LR = 1e-3
KINDS = ("bdq", "bdq_per", "dqn", "dqn_per", "ppo")
KIND_CODE = {"bdq": 2, "dqn": 3, "ppo": 4}


def r32(n):
    return (n + 31) // 32 * 32


def r4(n):
    return (n + 3) // 4 * 4


class Case:
    """One small learner with what the test expects of it."""

    def __init__(self, kind, data_seed=0):
        self.kind, self.per = kind.split("_")[0], kind.endswith("_per")
        self.rng = np.random.default_rng(data_seed)
        if self.kind == "bdq":
            self.D, self.n, self.T0, self.T1, self.HB = 2, 5, 16, 12, 8
            self.L = BDQLearner(OBS, self.D, self.n, ((self.T0, self.T1), (self.HB,), (self.HB,)), batch_size=B, buffer_size=CAP,
                                prioritized_replay=self.per)
            cfg = BR.BDQConfig(obs_dim=OBS, n_branches=self.D, n_bins=self.n, trunk=(self.T0, self.T1), branch_hidden=self.HB,
                               value_hidden=self.HB)
            self.specs = BR.all_specs(cfg)
            self.trained = [n for n, _ in BR.param_specs(cfg, "bdq/model")]
            self.prefix = "b2g_bdq_"
        elif self.kind == "dqn":
            self.n, self.H0, self.H1 = 6, 16, 12
            self.L = DQNLearner(OBS, self.n, (self.H0, self.H1), batch_size=B, buffer_size=CAP, prioritized_replay=self.per)
            cfg = DR.DQNConfig(obs_dim=OBS, n_actions=self.n, layers=(self.H0, self.H1))
            self.specs = DR.all_specs(cfg)
            self.trained = [n for n, _ in DR.param_specs(cfg, DR.ONLINE)]
            self.prefix = "b2g_dqn_"
        else:
            self.A, self.H0, self.H1 = 3, 16, 12
            self.L = PPO2Learner(OBS, self.A, (self.H0, self.H1), n_envs=2, n_steps=4, nminibatches=1, noptepochs=1)
            self.specs = PR.param_specs(OBS, self.A, (self.H0, self.H1))
            self.trained = [n for n, _ in self.specs if not n.startswith("model/q/")]
            self.prefix = "b2g_ppo_"
        self.live = 0

    def fn(self, name):
        return getattr(self.L.lib, self.prefix + name)

    def batch(self):
        rng = self.rng
        obs, nxt = rng.standard_normal((B, OBS)).astype(np.float32), rng.standard_normal((B, OBS)).astype(np.float32)
        rew, done = rng.standard_normal(B).astype(np.float32), (rng.random(B) < 0.3).astype(np.float32)
        act = rng.integers(0, self.n, (B, self.D) if self.kind == "bdq" else B).astype(np.float32)
        return obs, act, rew, nxt, done

    def fill(self, rows):
        for _ in range(rows // B):
            self.L.replay_add(*self.batch())
        self.live = min(CAP, self.live + rows)

    def step(self):
        if self.kind == "ppo":
            M = self.L.minibatch
            rng = self.rng
            return self.L.train_step_explicit(rng.standard_normal((M, OBS)), rng.standard_normal(M), rng.standard_normal((M, self.A)),
                                              rng.standard_normal(M), rng.random(M) + 1.0, LR, 0.2, -1.0)
        return self.L.step_explicit(*self.batch(), lr=LR)

    # ---- the training-state file the parent commit writes
    def n_train(self):
        if self.kind == "bdq":
            NBS = r4(self.n)
            per_branch = r32(self.HB) + r32(self.T1 * self.HB) + r32(NBS) + r32(self.HB * NBS)
            return (self.D * per_branch + r32(self.T0) + r32(OBS * self.T0) + r32(self.T1) + r32(self.T0 * self.T1) + r32(self.HB) +
                    r32(self.T1 * self.HB) + r32(4) + r32(self.HB * 4))
        if self.kind == "dqn":
            tower = lambda so: r32(OBS * self.H0) + r32(self.H0) + r32(self.H0 * self.H1) + r32(self.H1) + r32(self.H1 * so) + r32(so)
            return tower(r4(self.n)) + tower(4)
        H0, H1, A = self.H0, self.H1, self.A
        return r32(OBS * 2 * H0) + r32(2 * H0) + 2 * (r32(H0 * H1) + r32(H1)) + r32(H1) + r32(1) + r32(H1 * A) + r32(A) + r32(A)

    def expected_layout(self):
        nt = self.n_train()
        if self.kind == "ppo":
            fp = ["obs_dim", "n_actions", "hidden0", "hidden1", "n_envs", "n_steps", "nminibatches", "noptepochs", "seed"]
            n_total = nt + r32(self.H1 * self.A) + r32(self.A)
            return 4, fp, [("HOST", 16), ("CNTR", 32), ("PARM", 4 * n_total), ("ADMM", 4 * nt), ("ADMV", 4 * nt)]
        if self.kind == "bdq":
            fp = ["obs_dim", "n_branches", "n_bins", "trunk0", "trunk1", "branch_hidden", "batch", "buffer_capacity", "gamma",
                  "target_update_freq", "trunk_grad_rescale", "seed", "prioritized_replay", "per_alpha", "per_eps"]
            width = self.D
        else:
            fp = ["obs_dim", "n_actions", "hidden0", "hidden1", "batch", "buffer_capacity", "gamma", "seed", "prioritized_replay",
                  "per_alpha", "per_eps"]
            width = 1
        C2 = 1 << (CAP - 1).bit_length()
        secs = [("HOST", 32), ("CNTR", 64), ("PARM", 8 * nt), ("ADMM", 4 * nt), ("ADMV", 4 * nt), ("ROBS", 4 * self.live * OBS),
                ("RNXT", 4 * self.live * OBS), ("RACT", 4 * CAP * width), ("RREW", 4 * CAP), ("RDON", 4 * CAP),
                ("PERT", 2 * 8 * 2 * C2 if self.per else 0), ("PERS", 8)]
        return KIND_CODE[self.kind], fp, secs


def parse_state(path):
    """(kind, fingerprint names, [(tag, offset, length)]) of a training-state file (StateHeader, FpField[], SecEntry[])."""
    data = open(path, "rb").read()
    magic, version, kind, n_fp, n_sec, file_bytes = struct.unpack_from("<8sIIIIQ", data, 0)
    assert magic == b"B2GSTATE" and version == 1 and file_bytes == len(data)
    names = [struct.unpack_from("<31s", data, 32 + 40 * i)[0].rstrip(b"\0").decode() for i in range(n_fp)]
    at = 32 + 40 * n_fp
    secs = []
    for i in range(n_sec):
        tag, _pad, off, nbytes, _sum = struct.unpack_from("<IIQQQ", data, at + 32 * i)
        secs.append((tag.to_bytes(4, "little").decode(), off, nbytes))
    return kind, names, secs


def bits(params):
    return {n: np.asarray(a, np.float32).view(np.uint32).copy() for n, a in params.items()}


def assert_same(a, b):
    assert a.keys() == b.keys()
    for n in a:
        assert np.array_equal(a[n], b[n]), n


def call_code(fn, *args):
    rc = fn(*args)
    assert rc < 0
    return rc


@pytest.fixture(params=KINDS)
def case(request):
    c = Case(request.param)
    yield c
    c.L.close()


def test_param_listing_and_round_trip(case):
    L = case.L
    assert [(n, tuple(s)) for n, s in L.param_shapes.items()] == [(n, tuple(s)) for n, s in case.specs]
    for suffix in ("", ":0"):
        want = {n: case.rng.standard_normal(s).astype(np.float32) for n, s in L.param_shapes.items()}
        for n, a in want.items():
            _lib.check(case.fn("set_param")(L.h, (n + suffix).encode(), _fp(a.reshape(-1)), a.size))
        got = {}
        for n, s in L.param_shapes.items():
            a = np.empty(s, np.float32)
            _lib.check(case.fn("get_param")(L.h, (n + suffix).encode(), _fp(a.reshape(-1)), a.size))
            got[n] = a
        assert_same(bits(want), bits(got))
        assert_same(bits(want), bits(L.get_parameters()))


def test_gradient_names_and_refusals(case):
    L = case.L
    if case.kind != "ppo":
        case.fill(2 * B)
    case.step()
    assert list(L.get_gradients()) == case.trained
    buf = np.zeros(4096, np.float32)
    name, shape = case.specs[-1]
    numel = int(np.prod(shape))
    # the last listed entry has no gradient: a target tensor, or PPO's q/b
    assert not name.startswith(("bdq/model/", "deepq/model/")) and name not in case.trained
    assert call_code(case.fn("get_grad"), L.h, name.encode(), _fp(buf), numel) == _lib.B2G_EINVAL
    if case.kind == "ppo":
        assert call_code(case.fn("get_grad"), L.h, b"model/q/w", _fp(buf), case.H1 * case.A) == _lib.B2G_EINVAL
    for fn in ("get_param", "set_param", "get_grad"):
        assert call_code(case.fn(fn), L.h, b"no/such/variable", _fp(buf), 1) == _lib.B2G_EINVAL
        n0, s0 = case.specs[1]
        assert call_code(case.fn(fn), L.h, n0.encode(), _fp(buf), int(np.prod(s0)) + 1) == _lib.B2G_EINVAL
    m = case.step()
    assert np.isfinite(m["grad_norm"])


def test_state_layout_and_refusals(case, tmp_path):
    if case.kind != "ppo":
        case.fill(3 * B)
    case.step()
    path = str(tmp_path / "a.state")
    case.L.save_state(path)
    kind, names, secs = parse_state(path)
    want_kind, want_fp, want_secs = case.expected_layout()
    assert kind == want_kind and names == want_fp
    assert [(t, n) for t, _, n in secs] == want_secs
    saved = bits(case.L.get_parameters())

    # another learner's file: refused before anything changes
    other = Case("dqn" if case.kind == "bdq" else "bdq")
    other_path = str(tmp_path / "other.state")
    other.L.save_state(other_path)
    other.L.close()
    R = Case(case.kind + ("_per" if case.per else ""), data_seed=1)
    R.L.load_parameters({n: R.rng.standard_normal(s).astype(np.float32) for n, s in R.L.param_shapes.items()})
    before = bits(R.L.get_parameters())
    with pytest.raises(_lib.B2GError) as e:
        R.L.load_state(other_path)
    assert e.value.code == _lib.B2G_EINVAL
    assert_same(before, bits(R.L.get_parameters()))
    # a truncated file
    data = open(path, "rb").read()
    short = str(tmp_path / "short.state")
    open(short, "wb").write(data[:-7])
    with pytest.raises(_lib.B2GError, match="truncated") as e:
        R.L.load_state(short)
    assert e.value.code == _lib.B2G_EINVAL
    assert_same(before, bits(R.L.get_parameters()))
    R.step()
    # a flipped byte in the parameter section fails its checksum after the writes began: unusable until a good load
    parm = next(off for t, off, _ in secs if t == "PARM")
    flipped = bytearray(data)
    flipped[parm + 5] ^= 0xFF
    bad = str(tmp_path / "bad.state")
    open(bad, "wb").write(bytes(flipped))
    with pytest.raises(_lib.B2GError, match="checksum") as e:
        R.L.load_state(bad)
    assert e.value.code == _lib.B2G_EINVAL
    with pytest.raises(_lib.B2GError) as e:
        R.step()
    assert e.value.code == _lib.B2G_ESTATE
    buf = np.zeros(1, np.float32)
    assert call_code(R.fn("get_param"), R.L.h, R.specs[0][0].encode(), _fp(buf), 1) == _lib.B2G_ESTATE
    R.L.load_state(path)
    assert_same(saved, bits(R.L.get_parameters()))
    R.step()
    R.L.close()
