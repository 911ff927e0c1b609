"""PPO2 without a GPU: the float64 oracle (oracle/ppo_ref.py) against finite differences, a direct GAE loop and
scipy.stats.norm; the parameter list; the refusals that need no device; the command-line mapping."""
from collections import OrderedDict

import numpy as np
import pytest
import scipy.stats

import b200grasp
from b200grasp import train_cli
from b200grasp.common.policies import CnnPolicy, MlpPolicy
from b200grasp.ppo2 import PPO2, _check_policy_kwargs, _init_params
from b200grasp.spaces import Box, Discrete
from oracle import ppo_ref as R


def _case(seed, M=6, D=5, A=2, layers=(4, 3), spread=0.6):
    rng = np.random.default_rng(seed)
    p = R.as_float64(R.init_params(D, A, layers, rng))
    for k in p:
        if p[k].ndim == 1 or k.endswith("logstd"):
            p[k] = rng.uniform(-0.3, 0.3, p[k].shape)
    p["model/pi/w"] = p["model/pi/w"] * 60
    x = rng.normal(0, 1, (M, D))
    mean, v = R.forward(p, x)
    act = mean + rng.normal(0, 1, (M, A))
    nlp = R.neglogp(mean, p["model/pi/logstd"], act)
    return p, x, v + rng.normal(0, 1, M), act, v + rng.uniform(-0.5, 0.5, M), nlp + rng.uniform(-spread, spread, M)


def _loss(p, case, c, cvf):
    return R.loss_and_grads(p, *case, cliprange=c, cliprange_vf=cvf)[0]


@pytest.mark.parametrize("cvf", [None, 0.1, -1.0])
def test_oracle_gradient_matches_finite_differences(cvf):
    p, *case = _case(1)
    _, met, g = R.loss_and_grads(p, *case, cliprange=0.2, cliprange_vf=cvf)
    _, nlp_now = R.forward(p, case[0])
    ratio = np.exp(case[4] - R.neglogp(R.forward(p, case[0])[0], p["model/pi/logstd"], case[2]))
    assert (ratio > 1.2).any() and (ratio < 0.8).any()          # clipped on both sides
    h = 1e-6
    for k in g:
        flat = p[k].reshape(-1)
        for i in np.random.default_rng(3).choice(flat.size, min(6, flat.size), replace=False):
            q = OrderedDict((n, a.copy()) for n, a in p.items())
            q[k].reshape(-1)[i] += h
            lp = _loss(q, case, 0.2, cvf)
            q[k].reshape(-1)[i] -= 2 * h
            lm = _loss(q, case, 0.2, cvf)
            fd = (lp - lm) / (2 * h)
            assert abs(fd - g[k].reshape(-1)[i]) <= 1e-5 * max(1.0, abs(fd)), (k, i, fd, g[k].reshape(-1)[i])


def test_value_clip_default_is_cliprange():
    p, *case = _case(2)
    a = R.loss_and_grads(p, *case, cliprange=0.2, cliprange_vf=None)
    b = R.loss_and_grads(p, *case, cliprange=0.2, cliprange_vf=0.2)
    c = R.loss_and_grads(p, *case, cliprange=0.2, cliprange_vf=-1.0)
    assert a[0] == b[0] and a[1]["value_loss"] != c[1]["value_loss"]


@pytest.mark.parametrize("scale,clipped", [(1.0, True), (1e-4, False)])
def test_global_clip(scale, clipped):
    p, *case = _case(3)
    _, _, g = R.loss_and_grads(p, *case, cliprange=0.2)
    g = OrderedDict((k, v * scale) for k, v in g.items())
    gc, norm = R.clip_global(g, 0.5)
    assert (norm > 0.5) == clipped
    n2 = np.sqrt(sum((v * v).sum() for v in gc.values()))
    assert np.isclose(n2, 0.5 if clipped else norm)


def _gae_loop(r, v, starts, lastv, lastd, g, lam):
    T, E = r.shape
    adv = np.zeros((T, E))
    for e in range(E):
        acc = 0.0
        for t in range(T - 1, -1, -1):
            nd = lastd[e] if t == T - 1 else starts[t + 1, e]
            nv = lastv[e] if t == T - 1 else v[t + 1, e]
            acc = r[t, e] + g * nv * (1 - nd) - v[t, e] + g * lam * (1 - nd) * acc
            adv[t, e] = acc
    return adv


@pytest.mark.parametrize("pattern", ["first", "last", "consecutive", "many_envs"])
def test_gae_against_loop(pattern):
    rng = np.random.default_rng(4)
    T, E = 6, (5 if pattern == "many_envs" else 1)
    r, v, lastv = rng.normal(size=(T, E)), rng.normal(size=(T, E)), rng.normal(size=E)
    starts, lastd = np.zeros((T, E)), np.zeros(E)
    if pattern == "first":
        starts[0] = 1
    elif pattern == "last":
        lastd[:] = 1
    elif pattern == "consecutive":
        starts[2:5] = 1
    else:
        starts = (rng.random((T, E)) < 0.3).astype(float)
        lastd = (rng.random(E) < 0.5).astype(float)
    adv, ret = R.gae(r, v, starts, lastv, lastd, 0.99, 0.95)
    ref = _gae_loop(r, v, starts, lastv, lastd, 0.99, 0.95)
    assert np.allclose(adv, ref, rtol=0, atol=1e-12) and np.allclose(ret, ref + v, rtol=0, atol=1e-12)


def test_neglogp_and_entropy_against_scipy():
    rng = np.random.default_rng(5)
    mean, logstd, act = rng.normal(size=(7, 3)), rng.normal(size=(1, 3)) * 0.3, rng.normal(size=(7, 3))
    ref = -scipy.stats.norm.logpdf(act, mean, np.exp(logstd)).sum(1)
    assert np.allclose(R.neglogp(mean, logstd, act), ref, rtol=1e-12)
    assert np.isclose(R.entropy(logstd), scipy.stats.norm.entropy(0, np.exp(logstd)).sum(), rtol=1e-12)


@pytest.mark.parametrize("D,A", [(100, 3), (8192, 5)])
def test_parameter_list(D, A):
    specs = R.param_specs(D, A)
    assert [n for n, _ in specs] == ["model/" + n for n in ("pi_fc0/w", "pi_fc0/b", "vf_fc0/w", "vf_fc0/b", "pi_fc1/w", "pi_fc1/b",
                                                            "vf_fc1/w", "vf_fc1/b", "vf/w", "vf/b", "pi/w", "pi/b", "pi/logstd",
                                                            "q/w", "q/b")]
    assert dict(specs)["model/pi_fc0/w"] == (D, 64) and dict(specs)["model/pi/logstd"] == (1, A) and dict(specs)["model/vf/w"] == (64, 1)
    p = _init_params(D, A, (64, 64), 0)
    assert [(k, v.shape) for k, v in p.items()] == specs
    w = p["model/pi_fc1/w"].astype(np.float64)
    assert np.allclose(w.T @ w, 2.0 * np.eye(64), atol=1e-5)                  # orthogonal, scale sqrt(2)
    assert np.allclose(np.linalg.norm(p["model/pi/w"].astype(np.float64), axis=0), 0.01, atol=1e-6)
    assert not p["model/pi/logstd"].any() and not p["model/vf_fc0/b"].any()


class _Env:
    num_envs = 1
    observation_space = Box(-1.0, 1.0, (4,))
    action_space = Box(-1.0, 1.0, (2,))


def test_refusals_without_device():
    with pytest.raises(NotImplementedError, match="ppo2.PPO2"):
        b200grasp.PPO2
    with pytest.raises(NotImplementedError, match="ppo2.PPO2"):
        b200grasp.SAC(MlpPolicy, None)
    for bad in (CnnPolicy, "CnnPolicy", "MlpLstmPolicy", "MlpLnLstmPolicy"):
        with pytest.raises(NotImplementedError):
            PPO2(bad, None)
    for kw in ({"net_arch": [64, dict(pi=[64], vf=[64])]}, {"act_fun": np.abs}, {"layers": [64]}, {"layers": [8, 8, 8]},
               {"layer_norm": True}, {"net_arch": [dict(pi=[64, 64], vf=[32, 32])]}):
        with pytest.raises(NotImplementedError):
            PPO2(MlpPolicy, None, policy_kwargs=kw)
    with pytest.raises(NotImplementedError):
        PPO2(MlpPolicy, None, device_obs_norm=True)
    m = PPO2(MlpPolicy, None)
    class _D(_Env):
        action_space = Discrete(4)
    with pytest.raises(NotImplementedError, match="Box"):
        m._set_env(_D())
    m2 = PPO2(MlpPolicy, None, n_steps=10, nminibatches=4)
    with pytest.raises(ValueError, match="nminibatches"):
        m2._set_env(_Env())
    assert _check_policy_kwargs({"net_arch": [dict(pi=[32, 16], vf=[32, 16])]})[1] == [32, 16]


def test_defaults_are_stable_baselines():
    m = PPO2("MlpPolicy", None)
    assert (m.gamma, m.n_steps, m.ent_coef, m.learning_rate, m.vf_coef, m.max_grad_norm, m.lam, m.nminibatches, m.noptepochs,
            m.cliprange, m.cliprange_vf, m.layers) == (0.99, 128, 0.01, 2.5e-4, 0.5, 0.5, 0.95, 4, 4, 0.2, None, [64, 64])


def test_cli_mapping(tmp_path):
    cfg = {"PPO": {"learning_rate": 3e-4, "layers": [256, 256], "n_steps": 512, "total_timesteps": 10}, "discount_factor": 0.97}
    assert train_cli.ppo_kwargs(cfg) == {"verbose": 2, "gamma": 0.97, "learning_rate": 3e-4}
    for extra in (["--device_norm"], ["--load_dir", str(tmp_path / "x.zip")]):
        args = train_cli.build_parser().parse_args(["train", "--config", "c.yaml", "--algo", "PPO", "--model_dir", str(tmp_path / "m")] + extra)
        import yaml
        (tmp_path / "c.yaml").write_text(yaml.safe_dump(cfg))
        args.config = str(tmp_path / "c.yaml")
        with pytest.raises(NotImplementedError):
            train_cli.train(args)
        assert not (tmp_path / "m").exists()
