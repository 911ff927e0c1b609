"""Replay frame pool (include/b200grasp.h, b2g_replay_cfg): observations shared between consecutive transitions and 8-bit
image planes must not change what the learner samples or computes, and what does not fit is dropped oldest-first."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import replay_budget  # noqa: E402

LR = 3e-4
N_ACT = 5


# ---------------------------------------------------------------------------------------------------- CPU: the arithmetic
def test_replay_bytes_of_the_shipped_configurations():
    rows = {r["run"]: r for r in replay_budget.table()}
    assert rows["SAC_full_rgbd"]["two_frames_per_slot_GB"] == pytest.approx(131.1, abs=0.1)
    assert rows["SAC_full_rgbd"]["shared_frames_GB"] == pytest.approx(32.3, abs=0.1)
    assert rows["table_clearing/SAC_real_2m_buffer_128"]["two_frames_per_slot_GB"] == pytest.approx(65.6, abs=0.1)
    assert rows["table_clearing/SAC_real_2m_buffer_128"]["shared_frames_GB"] == pytest.approx(36.9, abs=0.1)
    assert rows["SAC_depth_1mbuffer"]["shared_frames_GB"] == pytest.approx(18.5, abs=0.1)
    # 8-bit frames keep a 16-byte stride; fp32 frames are exactly the compact row
    assert replay_budget.frame_bytes((64, 64, 5), (0, 1, 2)) % 16 == 0
    assert replay_budget.frame_bytes((64, 64, 2)) == 4 * (64 * 64 + 4)
    assert replay_budget.frame_bytes((101,)) == 404


def test_train_cli_replay_spare_flag():
    from b200grasp import train_cli
    a = train_cli.build_parser().parse_args(["train", "--config", "c.yaml", "--algo", "SAC", "--model_dir", "m",
                                             "--replay_spare", "0.125"])
    assert a.replay_spare == 0.125
    a = train_cli.build_parser().parse_args(["train", "--config", "c.yaml", "--algo", "SAC", "--model_dir", "m"])
    assert a.replay_spare is None


# ---------------------------------------------------------------------------------------------------- GPU
def _learner(obs_shape, B, cap, precision, **kw):
    import b200grasp
    from tests.test_gpu_configs import vecnorm_for
    if len(obs_shape) == 1:
        vn = dict(np.load(os.path.join(ROOT, "tests", "golden", "vecnorm_sac_encoder.npz")))
    else:
        vn = vecnorm_for(obs_shape[2] - 1)
    L = b200grasp.Learner(obs_shape, n_act=N_ACT, batch_size=B, buffer_size=cap, seed=11, precision=precision, **kw)
    L.set_norm_stats(vn["obs_mean"], vn["obs_var"], float(vn["ret_var"]), float(vn["clip_obs"]), float(vn["clip_reward"]),
                     float(vn["epsilon"]))
    rng = np.random.default_rng(0)          # the same weights in every learner of a test
    L.load_parameters({n: (rng.standard_normal(s) / np.sqrt(np.prod(s[:-1]) if len(s) > 1 else 1.0)).astype(np.float32)
                       for n, s in L.param_shapes.items()})
    return L


def _fresh_obs(rng, obs_shape, n, u8=()):
    """n observations: integers 0..255 in exactly the 8-bit planes `u8`, floats in [0, 1) in the other image planes, a
    constant actuator plane; MLP: floats."""
    if len(obs_shape) == 1:
        return rng.standard_normal((n,) + tuple(obs_shape)).astype(np.float32)
    h, w, c = obs_shape
    o = rng.random((n, h, w, c), dtype=np.float32)
    if u8:
        o[..., sorted(u8)] = rng.integers(0, 256, (n, h, w, len(u8))).astype(np.float32)
    o[..., -1] = rng.random((n, 1, 1), dtype=np.float32)
    return o


def _episodic_stream(rng, obs_shape, lanes, calls, p_done, u8=()):
    """(obs, act, rew, next_obs, done) per call: lane i's next_obs is its obs of the next call unless the episode ended."""
    cur = _fresh_obs(rng, obs_shape, lanes, u8)
    for _ in range(calls):
        nxt = _fresh_obs(rng, obs_shape, lanes, u8)
        done = (rng.random(lanes) < p_done).astype(np.float32)
        act = rng.uniform(-1, 1, (lanes, N_ACT)).astype(np.float32)
        rew = rng.standard_normal(lanes).astype(np.float32)
        yield cur, act, rew, nxt, done
        cur = nxt.copy()
        ends = np.nonzero(done)[0]
        if len(ends):
            cur[ends] = _fresh_obs(rng, obs_shape, len(ends), u8)


def _same_row(a, b):
    return all(np.array_equal(a[k].view(np.uint32) if isinstance(a[k], np.ndarray) else np.float32(a[k]).view(np.uint32),
                              b[k].view(np.uint32) if isinstance(b[k], np.ndarray) else np.float32(b[k]).view(np.uint32))
               for k in ("obs", "act", "rew", "next_obs", "done"))


EXACT_CASES = [
    ((64, 64, 2), 1, ()),          # engine v2 gather (bf16x3)
    ((64, 64, 5), 1, (0, 1, 2)),   # engine v2 gather, 8-bit RGB
    ((64, 64, 5), 0, (0, 1, 2)),   # round-1 gather, fp32
    ((64, 64, 2), 2, ()),          # round-1 gather, bf16
    ((101,), 0, ()),               # MLP policy
    ((64, 64, 4), 1, (0, 1, 2)),   # engine v2 gather, every image plane 8-bit (no fp32 image block), one pad channel
    ((64, 64, 3), 1, (1,)),        # engine v2 gather, an 8-bit plane after an fp32 one, two pad channels
]


@pytest.mark.gpu
@pytest.mark.parametrize("obs_shape,precision,u8", EXACT_CASES)
def test_shared_frames_sample_and_compute_what_two_frames_do(obs_shape, precision, u8):
    from tests.util import rel_err
    cap, lanes, B = 96, 3, 16
    ref = _learner(obs_shape, B, cap, precision)
    bud = _learner(obs_shape, B, cap, precision, frame_capacity=cap + cap // 8 + lanes, u8_planes=u8)
    rng = np.random.default_rng(5)
    dones = []
    calls = 2 * cap // lanes + 40                    # the ring wraps more than twice
    bar = 5e-3 if precision == 2 else 1e-4           # test_gpu_parity.py: the bf16 fast mode's bar, the parity bar
    for t, (o, a, r, nx, d) in enumerate(_episodic_stream(rng, obs_shape, lanes, calls, p_done=0.04, u8=u8)):
        ref.replay_add(o, a, r, nx, d)
        bud.replay_add(o, a, r, nx, d)
        dones.extend(d.tolist())
        if t >= B and t % 23 == 0:
            m_ref, m_bud = ref.step(1, lr=LR), bud.step(1, lr=LR)
            b_ref, b_bud = ref.last_batch(), bud.last_batch()
            assert np.array_equal(b_ref["indices"], b_bud["indices"]), t
            for k in ("q1", "q2", "v", "logp", "v_targ", "q1_pi", "q2_pi"):
                assert rel_err(b_bud[k], b_ref[k]) <= bar, (t, k, rel_err(b_bud[k], b_ref[k]))
            for k in ("policy_loss", "qf1_loss", "qf2_loss", "value_loss"):
                assert abs(m_bud[k] - m_ref[k]) <= bar * max(1.0, abs(m_ref[k])), (t, k, m_bud[k], m_ref[k])
    assert ref.replay_size() == bud.replay_size() == cap
    for s in range(cap):
        assert _same_row(ref.replay_get(s), bud.replay_get(s)), s
    info = bud.replay_info()
    assert info["evicted_early"] == 0 and info["size"] == cap
    live_dones = int(np.sum(dones[-cap:]))
    assert cap <= info["live_frames"] <= cap + live_dones + 2 * lanes, (info, live_dones)
    assert info["bytes"] < ref.replay_info()["bytes"]
    assert ref.replay_info()["live_frames"] == 2 * cap and ref.replay_info()["evicted_early"] == 0
    ref.close()
    bud.close()


@pytest.mark.gpu
@pytest.mark.parametrize("obs_shape,precision", [((101,), 0), ((64, 64, 2), 1)])
def test_overflow_drops_the_oldest_transitions(obs_shape, precision):
    """Every transition terminal, every observation fresh: two frames per transition, so a budget of cap + cap // 8 frames
    holds about half the ring; the oldest transitions go early, and sampling stays inside the live ones."""
    cap, B = 64, 16
    fc = cap + cap // 8
    L = _learner(obs_shape, B, cap, precision, frame_capacity=fc)
    rng = np.random.default_rng(9)
    rows = []
    for _ in range(40):
        n = int(rng.integers(1, 5))
        o, nx = _fresh_obs(rng, obs_shape, n), _fresh_obs(rng, obs_shape, n)
        a = rng.uniform(-1, 1, (n, N_ACT)).astype(np.float32)
        r = rng.standard_normal(n).astype(np.float32)
        L.replay_add(o, a, r, nx, np.ones(n, np.float32))
        rows.extend(dict(obs=o[i], act=a[i], rew=float(r[i]), next_obs=nx[i], done=1.0) for i in range(n))
    info = L.replay_info()
    size = L.replay_size()
    assert info["evicted_early"] > 0 and info["size"] == size
    assert fc // 2 - 1 <= size <= fc // 2, (size, fc)
    total = len(rows)
    live = {(total - size + j) % cap: rows[total - size + j] for j in range(size)}
    for s in range(cap):
        if s in live:
            got = L.replay_get(s)
            for k in ("obs", "next_obs"):
                if len(obs_shape) == 3:
                    assert np.array_equal(got[k][..., :-1], live[s][k][..., :-1]), (s, k)
                    assert got[k][0, 0, -1] == live[s][k][0, 0, -1]
                else:
                    assert np.array_equal(got[k], live[s][k]), (s, k)
            assert np.array_equal(got["act"], live[s]["act"]) and got["rew"] == np.float32(live[s]["rew"])
        else:
            with pytest.raises(Exception):
                L.replay_get(s)
    for _ in range(30):
        L.step(1, lr=LR)
        idx = L.last_batch()["indices"]
        assert all(int(i) in live for i in idx), (sorted(set(idx.tolist()) - set(live)), sorted(live))
    L.close()


@pytest.mark.gpu
def test_refusals():
    import b200grasp
    from b200grasp import _lib
    cap, B = 32, 8
    L = _learner((64, 64, 5), B, cap, 0, frame_capacity=cap + cap // 8, u8_planes=(0, 1, 2))
    rng = np.random.default_rng(3)
    o, nx = _fresh_obs(rng, (64, 64, 5), 4, (0, 1, 2)), _fresh_obs(rng, (64, 64, 5), 4, (0, 1, 2))
    a, r, d = np.zeros((4, N_ACT), np.float32), np.zeros(4, np.float32), np.zeros(4, np.float32)
    L.replay_add(o, a, r, nx, d)
    assert L.replay_size() == 4
    for bad in (3.5, -1.0, 256.0, -0.0, float("nan")):
        for which in ("obs", "next_obs"):
            oo, nn = o.copy(), nx.copy()
            (oo if which == "obs" else nn)[2, 5, 7, 1] = bad
            with pytest.raises(_lib.B2GError):
                L.replay_add(oo, a, r, nn, d)
            assert L.replay_size() == 4, (bad, which)
    # non-integer depth and actuator values are fine: those planes stay fp32
    o2 = o.copy()
    o2[..., 3] += 0.25
    L.replay_add(o2, a, r, nx, d)
    assert L.replay_size() == 8
    # an oversized call: 2 n > frame_capacity
    big = (cap + cap // 8) // 2 + 1
    with pytest.raises(_lib.B2GError):
        L.replay_add(np.repeat(o[:1], big, 0), np.zeros((big, N_ACT), np.float32), np.zeros(big, np.float32),
                     np.repeat(nx[:1], big, 0), np.zeros(big, np.float32))
    assert L.replay_size() == 8
    L.close()
    with pytest.raises(_lib.B2GError):        # the actuator plane
        b200grasp.Learner((64, 64, 5), n_act=N_ACT, batch_size=B, buffer_size=cap, u8_planes=(4,))
    with pytest.raises(_lib.B2GError):        # the MLP policy has no image planes
        b200grasp.Learner((101,), n_act=N_ACT, batch_size=B, buffer_size=cap, u8_planes=(0,))
    with pytest.raises(_lib.B2GError):        # fewer frames than slots + 1
        b200grasp.Learner((64, 64, 2), n_act=N_ACT, batch_size=B, buffer_size=cap, frame_capacity=cap)
    # the C entry point itself: create2 with NULL is the default layout
    lib = _lib.load()
    cfg = _lib.SacCfg(obs_h=64, obs_w=64, obs_c=2, n_act=N_ACT, hidden=64, batch=B, buffer_capacity=cap, gamma=0.99,
                      tau=0.005, target_entropy=-5.0, nranks=1)
    h = C.c_void_p()
    _lib.check(lib.b2g_sac_create2(C.byref(cfg), None, C.byref(h)))
    vals = [C.c_int64() for _ in range(6)]
    _lib.check(lib.b2g_replay_info(h, *[C.byref(v) for v in vals]))
    assert vals[2].value == 2 * cap and vals[4].value == replay_budget.replay_bytes(cap, (64, 64, 2))
    lib.b2g_sac_destroy(h)
