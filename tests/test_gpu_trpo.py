"""TRPO on the device (csrc/trpo.cu) against the float64 restatement in tests/trpo_ref.py: the gradient and losses at theta_old,
Fisher-vector products, the conjugate-gradient step, the line search, the value step, rollouts and the TRPO front end."""
from collections import OrderedDict

import numpy as np
import pytest

from oracle import philox_ref, ppo_ref
from tests import trpo_ref as R
from tests.fake_env import FakeFlatEnv

pytestmark = pytest.mark.gpu

from b200grasp.common.policies import MlpPolicy  # noqa: E402
from b200grasp.trpo_mpi import TRPO, TRPOLearner, init_params  # noqa: E402
from b200grasp.vec_env import DummyVecEnv, VecNormalize  # noqa: E402


def short(params):
    return OrderedDict((k[len("pi/model/"):], np.asarray(v, np.float64)) for k, v in params.items() if k.startswith("pi/model/"))


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def make(D, A, layers, N, seed=0, **kw):
    L = TRPOLearner(D, A, layers, N, seed=seed, **kw)
    p = init_params(D, A, layers, seed)
    rng = np.random.default_rng(seed + 7)
    p["pi/model/pi/logstd"] = rng.normal(0, 0.2, p["pi/model/pi/logstd"].shape).astype(np.float32)
    p["pi/model/pi/w"] = (p["pi/model/pi/w"] * 30).astype(np.float32)
    L.load_parameters(p)
    return L, p


def batch(D, A, N, seed=1):
    """Observations of unit expected norm (zero-mean at large D, so that X^T X stays well conditioned), actions, advantages and
    returns."""
    rng = np.random.default_rng(seed)
    obs = rng.uniform(0, 1, (N, D)) if D < 1000 else rng.normal(0, 1, (N, D)) / np.sqrt(D)
    return (obs.astype(np.float32), rng.normal(0, 1, (N, A)).astype(np.float32),
            rng.normal(0, 1, N).astype(np.float32), rng.normal(0, 1, N).astype(np.float32))


def before(m):
    return np.array([m["optimgain"], m["meankl"], m["entbonus"], m["surrgain"], m["entropy"]], np.float64)


def after(m):
    return np.array([m["optimgain_after"], m["meankl_after"], m["entbonus_after"], m["surrgain_after"], m["entropy_after"]], np.float64)


def check_losses_at_old(m, L0):
    """At theta_old meankl is 0 and surrgain = mean(atarg), which is 0 up to rounding: those two are held absolutely, the
    entropy and the entropy bonus relatively."""
    got = before(m)
    assert got[1] == 0.0
    assert abs(got[3] - L0[3]) <= 1e-6 and abs(got[0] - L0[0]) <= 1e-6 + 1e-4 * abs(L0[2])
    assert abs(got[4] - L0[4]) <= 1e-4 * abs(L0[4]) and abs(got[2] - L0[2]) <= 1e-4 * abs(L0[2]) + 1e-12


def close(got, ref, rtol, atol):
    return np.all(np.abs(np.asarray(got, np.float64) - ref) <= rtol * np.abs(ref) + atol)


@pytest.mark.parametrize("D,A,layers,N,entcoeff", [(1, 1, (4, 4), 5, 0.0), (100, 3, (64, 64), 400, 0.0), (100, 16, (8, 256), 1, 0.0),
                                                   (8192, 5, (64, 64), 1024, 0.0), (20480, 3, (256, 256), 1024, 0.0),
                                                   (100, 3, (64, 64), 16384, 0.0), (100, 3, (64, 64), 400, 0.05), (8192, 5, (64, 64), 1024, 0.02)])
def test_gradient_losses_and_step(D, A, layers, N, entcoeff):
    # cg_damping 0.5 bounds F's condition number, so that ten fp32 and float64 CG iterations stay within 1e-3 of each other
    L, p = make(D, A, layers, N, cg_damping=0.5, entcoeff=entcoeff)
    obs, act, adv, ret = batch(D, A, N)
    perms = np.stack([np.random.default_rng(k).permutation(N) for k in range(3)]).astype(np.int32)
    m, g, x, f = L.step_explicit(obs, act, adv, ret, perms)
    P = short(p)
    atarg = R.standardize(adv)
    L0, g_ref = R.grad_at_old(P, obs, act, atarg, entcoeff)
    check_losses_at_old(m, L0)
    assert rel(g, g_ref) <= 1e-3, rel(g, g_ref)
    assert abs(m["grad_sq"] - g_ref.dot(g_ref)) <= 1e-3 * g_ref.dot(g_ref)
    new, rec = R.iteration(P, R.MpiAdam(), obs, act, adv, ret, perms, cg_damping=0.5, entcoeff=entcoeff)
    if rec["accepted"] == -2:
        assert m["accepted"] == -2
        return
    assert rel(x, rec["stepdir"]) <= 1e-3, rel(x, rec["stepdir"])
    assert rel(f, rec["fullstep"]) <= 1e-3
    assert abs(m["shs"] - rec["shs"]) <= 1e-3 * abs(rec["shs"])
    assert m["accepted"] == rec["accepted"]
    got = short(L.get_parameters())
    if m["accepted"] >= 0:         # the losses the line search reports at the accepted theta
        La = R.losses(got, P, obs, act, atarg, entcoeff)
        assert close(after(m), La, 1e-3, 1e-6), (after(m), La)
    for n in R.POLICY + R.VALUE:
        step = np.abs(new[n] - P[n]).max()
        assert np.abs(got[n] - new[n]).max() <= 0.05 * step + 1e-6, n
    old = L.get_parameters()
    for k, v in p.items():
        if k.startswith("pi/model/"):
            assert np.array_equal(old["oldpi/" + k[3:]], v)          # oldpi is theta at the start of the iteration
    assert np.array_equal(got["q/w"], P["q/w"])
    if rec["vf_loss"]:
        assert abs(m["vf_loss"] - rec["vf_loss"]) <= 1e-4 * rec["vf_loss"]
    L.close()


# ---- the line search: one fixture per outcome.  Each is checked in the oracle, at the device's own full step, to sit at least
# 10 % from every threshold that decides it (meankl against 1.5 max_kl; the improvement against 0, measured in units of the
# linear prediction 0.5^k expectedimprove), so that rounding cannot flip a decision.
def ls_fixture(kind):
    """(params, obs, actions, advantages, max_kl, expected decisions): K = rejected for KL, I = rejected for no improvement,
    A = accepted."""
    D, A = (4, 1) if kind == "imp" else (6, 2)
    rng = np.random.default_rng(0)
    p = init_params(D, A, (8, 8), 0)
    f32 = lambda a: np.asarray(a, np.float32)
    if kind == "imp":
        # every row sees the same observation, so the step moves one mean: 5 rows 1 sigma above it with advantage 3, 5 rows 2
        # sigma above it with advantage -1, 10 rows on it with advantage 0.  The surrogate is exp(z d - d^2 / 2)-weighted, so
        # the half step overshoots the first group's optimum and falls, although its KL is small.
        p["pi/model/pi/logstd"] = np.zeros((1, A), np.float32)
        N = 20
        obs = np.tile(rng.uniform(0, 1, (1, D)), (N, 1))
        mu = ppo_ref.forward(short(p), f32(obs))[0]
        z = np.r_[[1.0] * 5, [2.0] * 5, [0.0] * 10]
        act = mu + z[:, None]
        adv = np.r_[[3.0] * 5, [-1.0] * 5, [0.0] * 10]
        return p, f32(obs), f32(act), f32(adv), 1.0, "KIA"
    seed, scale, logstd, wmul, max_kl, want = {"zero": (0, 1, 0.0, 1, 1.0, "A"), "kl": (1, 1, 0.0, 30, 0.01, "KA"),
                                               "reject": (0, 1000.0, -3.0, 30, 0.01, "K" * 10)}[kind]
    p = OrderedDict((k, np.asarray(v, np.float32)) for k, v in p.items())
    rng = np.random.default_rng(seed)
    q = ppo_ref.init_params(D, A, (8, 8), rng)
    for k, v in q.items():
        p["pi/" + k] = np.asarray(v, np.float32)
    p["pi/model/pi/w"] = f32(p["pi/model/pi/w"] * wmul)
    p["pi/model/pi/logstd"] = np.full((1, A), logstd, np.float32)
    N = 40
    obs = rng.uniform(0, 1, (N, D))
    off = np.ones(N, bool)
    off[::5] = False
    obs[off] *= scale             # rows the Fisher matrix does not see: a large scale makes the true KL outgrow its model
    act = rng.normal(0, 1, (N, A)) * np.exp(logstd)
    adv = rng.normal(0, 1, N)
    return p, f32(obs), f32(act), f32(adv), max_kl, want


@pytest.mark.parametrize("kind", ["zero", "kl", "imp", "reject"])
def test_line_search_outcomes(kind):
    p, obs, act, adv, max_kl, want = ls_fixture(kind)
    D, A, N = obs.shape[1], act.shape[1], obs.shape[0]
    L = TRPOLearner(D, A, (8, 8), N, seed=0, max_kl=max_kl)
    L.load_parameters(p)
    m, g, x, f = L.step_explicit(obs, act, adv, adv, np.zeros((3, N), np.int32))
    P = short(p)
    atarg = R.standardize(adv)
    P0 = R.tensors(P)
    th0 = R.flat(P0)
    L0 = R.losses(P, P, obs, act, atarg)
    check_losses_at_old(m, L0)

    def at(k):                     # theta_old + 0.5^k fullstep, rounded as the device rounds it
        th = (np.float32(0.5 ** k) * f.astype(np.float32) + th0.astype(np.float32)).astype(np.float64)
        cand = dict(P)
        cand.update({n: t.numpy() for n, t in R.unflat(th, P0).items()})
        return cand
    table = np.stack([R.losses(at(k), P, obs, act, atarg) for k in range(10)])
    ei = float(g.astype(np.float64).dot(f.astype(np.float64)))
    got = ""
    for k in range(10):
        kl = table[k, 1] / (1.5 * max_kl)
        imp = (table[k, 0] - L0[0]) / (0.5 ** k * ei)
        assert np.isfinite(table[k]).all()
        assert kl >= 1.1 or kl <= 0.9, (k, kl)
        if kl >= 1.1:
            got += "K"
            continue
        assert imp >= 0.1 or imp <= -0.1, (k, imp)
        got += "A" if imp >= 0.1 else "I"
        if imp >= 0.1:
            break
    assert got == want, (got, want)
    k = want.find("A")
    assert m["accepted"] == k
    params = short(L.get_parameters())
    if k < 0:
        for n in R.POLICY:
            assert np.array_equal(params[n], P[n]), n      # theta_before restored
        assert np.array_equal(after(m), before(m))
    else:
        for n in R.POLICY:
            assert np.allclose(params[n], at(k)[n], rtol=1e-6, atol=1e-7), n
        assert close(after(m), table[k], 1e-3, 1e-6), (after(m), table[k])
    L.close()


@pytest.mark.parametrize("D,A,layers,N", [(7, 2, (8, 12), 23), (8192, 5, (64, 64), 1024)])
def test_fvp(D, A, layers, N):
    L, p = make(D, A, layers, N)
    obs = batch(D, A, N)[0]
    rng = np.random.default_rng(5)
    for _ in range(2):
        v = rng.normal(size=L.n_policy)
        got = L.fvp(obs, v)
        ref = R.fvp(short(p), obs[::5], v, 1e-2)
        assert rel(got, ref) <= 1e-3
    L.close()


def test_zero_gradient_trains_value_only():
    D, A, N = 10, 2, 256
    L, p = make(D, A, (16, 16), N)
    obs, act, _, ret = batch(D, A, N)
    perms = np.stack([np.random.default_rng(k).permutation(N) for k in range(3)]).astype(np.int32)
    m, *_ = L.step_explicit(obs, act, np.full(N, 1.5, np.float32), ret, perms)
    assert m["accepted"] == -2 and m["cg_iters"] == 0
    got = short(L.get_parameters())
    P = short(p)
    for n in R.POLICY:
        assert np.array_equal(got[n], P[n]), n
    new, rec = R.iteration(P, R.MpiAdam(), obs, act, np.full(N, 1.5), ret, perms)
    for n in R.VALUE:
        assert np.abs(got[n] - new[n]).max() <= 0.05 * np.abs(new[n] - P[n]).max() + 1e-6, n
    L.close()


def test_rollout_boundary_carry_and_gae():
    D, A, N = 6, 3, 8
    L, p = make(D, A, (16, 16), N, seed=3)
    rng = np.random.default_rng(2)
    obs = rng.uniform(0, 1, (N + 1, D)).astype(np.float32)
    rew, done = rng.normal(size=N).astype(np.float32), (rng.uniform(size=N) < 0.3).astype(np.float32)
    acts = []
    for t in range(N):
        acts.append(L.rollout_act(obs[t]))
        L.rollout_reward(rew[t], done[t])
    # the actions: mean + exp(logstd) * noise of stream 1 at steps 0..N-1
    P = short(p)
    mean, val = ppo_ref.forward(P, obs[:N])
    for t in range(N):
        z = np.asarray(philox_ref.noise(philox_ref.act_seed(3), t, A), np.float64).reshape(-1)
        assert np.allclose(acts[t], mean[t] + np.exp(P["pi/logstd"].reshape(-1)) * z, rtol=1e-4, atol=1e-5)
    m = L.update(obs[N], np.stack([np.random.default_rng(k).permutation(N) for k in range(3)]))
    r = L.rollout_get()
    vb = ppo_ref.forward(P, obs[N:N + 1])[1]
    adv, tdl = ppo_ref.gae(rew.reshape(N, 1), val.reshape(N, 1), np.r_[0, done[:-1]].reshape(N, 1), vb, done[-1:], 0.99, 0.98)
    assert rel(r["advantages"], adv.reshape(-1)) <= 1e-4 and rel(r["tdlamret"], tdl.reshape(-1)) <= 1e-4
    # the boundary action (drawn before the update) is row 0 of the next batch; its value comes from the updated tower
    a0 = L.rollout_act(obs[N])
    assert np.array_equal(a0, r["actions"][0])
    _, v_new = ppo_ref.forward(short(L.get_parameters()), obs[N:N + 1])
    assert abs(r["values"][0] - v_new[0]) <= 1e-4 * max(1.0, abs(v_new[0]))
    assert L.steps()[1] == N + 1 and m["n_iterations"] == 1
    L.close()


def test_learn_predict_save_load_and_resume(tmp_path):
    def env():
        return VecNormalize(DummyVecEnv([lambda: FakeFlatEnv(horizon=7, obs_dim=6, n_act=3)]))
    np.random.seed(0)
    m = TRPO(MlpPolicy, env(), timesteps_per_batch=256, seed=1, policy_kwargs={"layers": [32, 32]})
    m.learn(600)                                                # ceil(600 / 256) = 3 iterations
    assert m.num_timesteps == 768 and m.last_metrics["n_iterations"] == 3
    a, _ = m.predict(np.zeros(6, np.float32), deterministic=True)
    assert a.shape == (3,) and np.all(np.abs(a) <= 1)
    m.save(str(tmp_path / "t.zip"))
    m2 = TRPO.load(str(tmp_path / "t.zip"))
    for (k, x), (k2, y) in zip(m.get_parameters().items(), m2.get_parameters().items()):
        assert k == k2 and np.array_equal(x, y)
    m2.close()
    stopped = TRPO(MlpPolicy, env(), timesteps_per_batch=256, seed=1)
    stopped.learn(10000, callback=lambda _l, _g: stopped.num_timesteps < 300)
    assert stopped.num_timesteps == 300 and stopped.learner.steps()[0] == 3 * 2    # one iteration: 3 passes x 2 minibatches
    stopped.close()
    # resume: save at an iteration boundary, load, continue; against the uninterrupted run
    np.random.seed(5)
    a_env = env()
    ma = TRPO(MlpPolicy, a_env, timesteps_per_batch=128, seed=2, policy_kwargs={"layers": [16, 16]})
    ma.learn(256)
    ma.save_training_state(str(tmp_path / "st"))
    a_env.venv.envs[0].rng = np.random.default_rng(0)
    ma.learn(256, reset_num_timesteps=False)
    b_env = env()
    mb = TRPO.load_training_state(str(tmp_path / "st"), b_env)
    b_env.venv.envs[0].rng = np.random.default_rng(0)
    mb.learn(256, reset_num_timesteps=False)
    assert mb.num_timesteps == ma.num_timesteps == 512
    for (k, x), (_, y) in zip(ma.get_parameters().items(), mb.get_parameters().items()):
        assert np.allclose(x, y, rtol=1e-4, atol=1e-5), k
    for mm in (ma, mb, m):
        mm.close()


def test_train_cli_train_then_run(tmp_path):
    import yaml
    from b200grasp import train_cli
    cfg = {"discount_factor": 0.99, "normalize": True, "robot": {}, "reward": {}, "simplified": False,
           "TRPO": {"max_iters": 128, "step_size": 0.001, "total_timesteps": 256}}
    path = tmp_path / "c.yaml"
    yaml.safe_dump(cfg, open(path, "w"))
    d = tmp_path / "run"
    train_cli.main(["train", "--config", str(path), "--algo", "TRPO", "--model_dir", str(d), "--env", "tests.fake_env:make_env",
                    "--eval_freq", "100000", "--checkpoint_freq", "100000"])
    assert (d / "final_model.zip").exists()
    out = train_cli.main(["run", "--model", str(d / "final_model.zip"), "--env", "tests.fake_env:make_env", "--episodes", "2"])
    assert out["episodes"] == 2
