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


# ---- the replay, normalisation, step and metrics-log entry points of the BDQ and DQN handles (one QLearner base)
Q_KINDS = ("bdq", "bdq_per", "dqn", "dqn_per")


@pytest.fixture(params=Q_KINDS)
def qcase(request):
    c = Case(request.param)
    yield c
    c.L.close()


@pytest.mark.parametrize("frames", [False, True])
@pytest.mark.parametrize("kind", Q_KINDS)
def test_replay_info_and_get(kind, frames):
    c = Case(kind)
    if frames:      # the same learner over a pool of frames
        c.L.close()
        per = c.per
        if c.kind == "bdq":
            c.L = BDQLearner(OBS, c.D, c.n, ((c.T0, c.T1), (c.HB,), (c.HB,)), batch_size=B, buffer_size=CAP, prioritized_replay=per,
                             frame_capacity=CAP + 16)
        else:
            c.L = DQNLearner(OBS, c.n, (c.H0, c.H1), batch_size=B, buffer_size=CAP, prioritized_replay=per, frame_capacity=CAP + 16)
    rows = [c.batch() for _ in range(3)]
    for r in rows:
        c.L.replay_add(*r)
    info = c.L.replay_info()
    assert info["capacity"] == CAP and info["size"] == 3 * B and info["evicted_early"] == 0 and info["bytes"] > 0
    if frames:
        assert info["frame_capacity"] == CAP + 16 and 0 < info["live_frames"] <= CAP + 16
    else:
        assert info["frame_capacity"] == 0 and info["live_frames"] == 0
    for k, (obs, act, rew, nxt, done) in enumerate(rows):
        for i in range(B):
            got = c.L.replay_get(k * B + i)
            assert np.array_equal(got["obs"], obs[i]) and np.array_equal(got["next_obs"], nxt[i])
            assert np.array_equal(got["act"], np.reshape(act[i], -1))
            assert got["rew"] == rew[i] and got["done"] == done[i]
            assert (min(got["frames"]) >= 0) if frames else got["frames"] == (-1, -1)
    c.L.close()


def test_q_refusals(qcase):
    L = qcase.L
    with pytest.raises(_lib.B2GError, match="replay buffer is empty") as e:
        L.step()
    assert e.value.code == _lib.B2G_ESTATE
    with pytest.raises(_lib.B2GError, match="norm_obs needs obs_mean/obs_var") as e:
        _lib.check(qcase.fn("set_norm_stats")(L.h, None, None, 1.0, 10.0, 10.0, 1e-8, 1, 0))
    assert e.value.code == _lib.B2G_EINVAL
    with pytest.raises(_lib.B2GError, match="bad argument") as e:
        L.metrics_log(-1)
    assert e.value.code == _lib.B2G_EINVAL


def test_last_per_after_sampled_step(qcase):
    qcase.fill(3 * B)
    qcase.L.step(1)
    slots, w, p = qcase.L.last_per()
    assert ((slots >= 0) & (slots < qcase.live)).all()
    if qcase.per:
        assert (np.isfinite(w) & (w > 0) & (w <= 1)).all()
        assert (np.isfinite(p) & (p > 0)).all()


@pytest.mark.parametrize("kind", Q_KINDS)
def test_sampled_step_matches_explicit_step_on_its_slots(kind):
    """A sampled step at learning rate 0 leaves the weights as they were; the explicit step on the slots it drew (and, with
    PER, on the importance weights it used) gives the same losses, bit for bit (one warp of samples: the loss sums have one
    order).  The sampled step's TD is read back only through PER's new priorities, sum_d |td_d| + eps in float32: with PER
    they must equal those of the explicit step's TD; with uniform replay no TD of a sampled step is readable."""
    c = Case(kind)
    c.fill(3 * B)
    m = c.L.step(1, lr=0.0)
    slots, w, prio = c.L.last_per()
    rows = [c.L.replay_get(int(s)) for s in slots]
    obs = np.stack([r["obs"] for r in rows])
    nxt = np.stack([r["next_obs"] for r in rows])
    act = np.stack([r["act"] for r in rows]).reshape((B, c.D) if c.kind == "bdq" else (B,))
    rew = np.array([r["rew"] for r in rows], np.float32)
    done = np.array([r["done"] for r in rows], np.float32)
    e = c.L.step_explicit(obs, act, rew, nxt, done, weights=w if c.per else None, lr=0.0, apply_update=False)
    keys = ("loss", "mean_q") + (("mean_abs_td",) if c.kind == "dqn" else ())
    for k in keys:
        assert np.float32(e[k]) == np.float32(m[k]), (k, e[k], m[k])
    td = np.asarray(e["td"], np.float32).reshape(B, -1)
    assert np.isfinite(td).all()
    if c.per:       # per_write_kernel's order: |td_0| + |td_1| + ... in float32, then + eps
        want = np.empty(B, np.float32)
        for i in range(B):
            s = np.float32(0)
            for v in td[i]:
                s = np.float32(s + np.abs(v))
            want[i] = np.float32(s + np.float32(1e-6))
        assert np.array_equal(want, prio), (want, prio)
    c.L.close()


def test_bdq_upload_bytes():
    c = Case("bdq")
    L, D, E, f, d = c.L, c.D, OBS, 4, 8
    up = lambda: (L.upload_bytes()["observe"], L.upload_bytes()["other"])
    assert up() == (0, 0)
    L.replay_add(*c.batch())
    other = B * (2 * E + D + 2) * f + 8
    assert up() == (0, other)
    L.set_norm_stats(np.zeros(E), np.ones(E))
    other += 2 * E * d + 8 * d
    assert up() == (0, other)
    L.set_norm_stats(norm_obs=False)
    other += 8 * d
    assert up() == (0, other)
    L.act(np.zeros((3, E), np.float32))
    other += 3 * E * f
    assert up() == (0, other)
    L.obs_rms_set(np.zeros(E), np.ones(E), 1.0)
    observe = 2 * E * d
    assert up() == (observe, other)
    L.set_norm_stats(np.zeros(E), np.ones(E))     # replaces the device statistics
    observe += 2 * E * d
    other += 8 * d
    assert up() == (observe, other)
    n = 5
    L.observe_act(np.ones((n, E), np.float32), eps=0.5)
    observe += n * E * f
    assert up() == (observe, other)
    done = np.array([0, 1, 0, 1, 0], np.float32)
    L.observe_add(np.zeros((n, D), np.float32), np.ones(n, np.float32), np.ones((n, E), np.float32), done,
                  reset_obs=np.zeros((n, E), np.float32))
    observe += n * E * f + n * D * f + 2 * n * f + 2 * E * f
    assert up() == (observe, other)
    L.close()
