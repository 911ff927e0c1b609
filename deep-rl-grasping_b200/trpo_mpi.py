"""``TRPO`` -- the TRPO branch of the reference's training harness (/root/reference/manipulation_main/training/sb_helper.py:129-136,
train_stable_baselines.py:95-104): stable-baselines 2.10.1 ``trpo_mpi.TRPO`` with ``common.policies.MlpPolicy``, one environment
and its defaults.  The rollout, GAE, the natural-gradient step (Fisher-vector products, conjugate gradient, the line search)
and the value function's MpiAdam run on the GPU (csrc/trpo.cu); the algorithm is restated in tests/trpo_ref.py.  Import it as
``b200grasp.trpo_mpi.TRPO`` (the stable-baselines path ``stable_baselines.trpo_mpi.TRPO``).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _lib
from .actor_critic import ActorCriticLearner, ActorCriticModel, check_policy, check_policy_kwargs
from . import actor_critic
from .learner import _f32, _fp

PI, OLDPI = "pi/model/", "oldpi/model/"
#: the policy step's variables, in the flat order of its gradient and step (trpo_mpi.py var_list)
POLICY_VARS = ("pi_fc0/w", "pi_fc0/b", "pi_fc1/w", "pi_fc1/b", "pi/w", "pi/b", "pi/logstd")
_GAIL = ("expert_dataset", "hidden_size_adversary", "adversary_entcoeff", "g_step", "d_step", "d_stepsize", "using_gail")


class TRPOLearner(ActorCriticLearner):
    """numpy-facing wrapper of one ``b2g_trpo`` handle (maps 1:1 onto the C ABI)."""
    _abi = "trpo"

    def __init__(self, obs_dim, n_actions, layers=(64, 64), timesteps_per_batch=1024, gamma=0.99, lam=0.98, max_kl=0.01, cg_iters=10,
                 cg_damping=1e-2, entcoeff=0.0, vf_stepsize=3e-4, vf_iters=3, seed=0, device=0):
        self.lib = _lib.load()
        if len(layers) != 2:
            raise NotImplementedError(f"layers={list(layers)}: the TRPO learner builds two hidden layers")
        cfg = _lib.TrpoCfg(int(obs_dim), int(n_actions), int(layers[0]), int(layers[1]), int(timesteps_per_batch), int(cg_iters),
                           int(vf_iters), float(gamma), float(lam), float(max_kl), float(cg_damping), float(entcoeff), float(vf_stepsize),
                           int(seed) & 0xFFFFFFFFFFFFFFFF, int(device))
        self._create(cfg)
        self.obs_dim, self.n_actions, self.N = int(obs_dim), int(n_actions), int(timesteps_per_batch)
        self.vf_iters = int(vf_iters)
        self.n_policy = sum(int(np.prod(self._info[PI + n])) for n in POLICY_VARS)

    def _has_grad(self, name):
        return name.startswith(PI) and name[len(PI):] in POLICY_VARS

    def rollout_act(self, obs):
        """Rollout step: obs [obs_dim] -> the unclipped action [n_actions] (stored with its value)."""
        out = np.empty(self.n_actions, np.float32)
        _lib.check(self.lib.b2g_trpo_rollout_act(self.h, _fp(_f32(obs).reshape(self.obs_dim)), _fp(out)))
        return out

    def rollout_reward(self, rew, done):
        _lib.check(self.lib.b2g_trpo_rollout_reward(self.h, float(np.ravel(rew)[0]), float(np.ravel(done)[0])))

    def rollout_get(self):
        """advantages, tdlamret, values [N] and actions [N, n_actions]."""
        adv, ret, val = (np.empty(self.N, np.float32) for _ in range(3))
        act = np.empty((self.N, self.n_actions), np.float32)
        _lib.check(self.lib.b2g_trpo_rollout_get(self.h, _fp(adv), _fp(ret), _fp(val), _fp(act)))
        return dict(advantages=adv, tdlamret=ret, values=val, actions=act)

    def _perm(self, perms):
        p = np.ascontiguousarray(perms, np.int32).reshape(-1)
        assert p.size == self.vf_iters * self.N
        return p

    def update(self, last_obs, perms):
        """One iteration on a full rollout; perms [vf_iters, N] are the value passes' permutations.  ``last_obs=None``:
        the row observe_act staged after the last step is the boundary observation."""
        p = self._perm(perms)
        m = _lib.TrpoMetrics()
        lo = None if last_obs is None else _fp(_f32(last_obs).reshape(self.obs_dim))
        _lib.check(self.lib.b2g_trpo_update(self.h, lo, p.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(m)))
        return m.as_dict()

    def step_explicit(self, obs, actions, adv, tdlamret, perms):
        """The policy and value step on a caller's batch -> (metrics, g, stepdir, fullstep), vectors in var_list order."""
        p = self._perm(perms)
        m = _lib.TrpoMetrics()
        g, x, f = (np.empty(self.n_policy, np.float32) for _ in range(3))
        _lib.check(self.lib.b2g_trpo_step_explicit(
            self.h, _fp(_f32(obs).reshape(self.N, self.obs_dim)), _fp(_f32(actions).reshape(self.N, self.n_actions)),
            _fp(_f32(np.reshape(adv, -1))), _fp(_f32(np.reshape(tdlamret, -1))), p.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(m),
            _fp(g), _fp(x), _fp(f)))
        return m.as_dict(), g, x, f

    def fvp(self, obs, v):
        """F v over the rows [::5] of obs [N, obs_dim] at the current parameters, v and the result in var_list order."""
        out = np.empty(self.n_policy, np.float32)
        _lib.check(self.lib.b2g_trpo_fvp(self.h, _fp(_f32(obs).reshape(self.N, self.obs_dim)), _fp(_f32(v).reshape(self.n_policy)),
                                         _fp(out)))
        return out

    def act(self, obs, deterministic=True, raw=False):
        """-> actions [n, n_actions] (mean, or mean + std * noise of stream 1), values [n]; nothing is stored.  ``raw``: the
        observations are normalised with the device obs_rms first (b2g_trpo_act_raw)."""
        obs = _f32(obs).reshape(-1, self.obs_dim)
        n = obs.shape[0]
        a, v = np.empty((n, self.n_actions), np.float32), np.empty(n, np.float32)
        fn = self.lib.b2g_trpo_act_raw if raw else self.lib.b2g_trpo_act
        _lib.check(fn(self.h, _fp(obs), n, int(bool(deterministic)), _fp(a), _fp(v)))
        return a, v


def init_params(obs_dim, n_actions, layers, seed):
    """PPO2's initialisation rules for pi/model/... and then oldpi/model/..., drawn from one generator seeded with ``seed``."""
    rng = np.random.default_rng(seed)
    p = actor_critic.init_params(obs_dim, n_actions, layers, seed, rng=rng, scope=PI)
    p.update(actor_critic.init_params(obs_dim, n_actions, layers, seed, rng=rng, scope=OLDPI))
    return p


def value_minibatches(n, batch_size=128):
    """dataset.iterbatches(include_final_partial_batch=False): the [start, stop) of each full minibatch of one pass."""
    return [(s, s + batch_size) for s in range(0, n - batch_size + 1, batch_size)]


class TRPO(ActorCriticModel):
    """stable-baselines 2.10 ``TRPO(policy, env, ...)`` with its signature and defaults, plus ``device``: ``learn / predict /
    save / load / get_parameters / load_parameters / get_env / get_vec_normalize_env / close`` and
    ``save_training_state / load_training_state``.  One environment with a Box action space, as the reference's configs give."""
    _algo, _branch, _scope = "TRPO", "TRPO", PI
    _zip_hyper = ("gamma", "timesteps_per_batch", "max_kl", "cg_iters", "lam", "entcoeff", "cg_damping", "vf_stepsize", "vf_iters", "seed")

    def __init__(self, policy, env, gamma=0.99, timesteps_per_batch=1024, max_kl=0.01, cg_iters=10, lam=0.98, entcoeff=0.0,
                 cg_damping=1e-2, vf_stepsize=3e-4, vf_iters=3, verbose=0, tensorboard_log=None, _init_setup_model=True,
                 policy_kwargs=None, full_tensorboard_log=False, seed=None, n_cpu_tf_sess=1, device=0, device_obs_norm=False,
                 **unsupported):
        if unsupported:
            gail = sorted(set(unsupported) & set(_GAIL))
            if gail:
                raise NotImplementedError(f"{gail}: the GAIL path of TRPO is not built")
            raise TypeError(f"TRPO got unexpected keyword arguments {sorted(unsupported)}")
        # PPO2's observe path on one env (TRPOLearner.observe_act): the carried boundary row is the row as it was normalised
        self.device_obs_norm = bool(device_obs_norm)
        self._refuse_device_obs_norm_without_wrapper(env)
        check_policy(policy, "TRPO")
        self.policy_kwargs, self.layers = check_policy_kwargs(policy_kwargs, "TRPO")
        self.gamma, self.timesteps_per_batch, self.max_kl, self.cg_iters = gamma, int(timesteps_per_batch), max_kl, int(cg_iters)
        self.lam, self.entcoeff, self.cg_damping, self.vf_stepsize, self.vf_iters = lam, entcoeff, cg_damping, vf_stepsize, int(vf_iters)
        self.verbose, self.tensorboard_log, self.full_tensorboard_log = verbose, tensorboard_log, full_tensorboard_log
        self.seed, self.n_cpu_tf_sess, self.device = seed, n_cpu_tf_sess, device
        self.num_timesteps = 0
        self.n_envs = 1
        self.learner: Optional[TRPOLearner] = None
        self.ep_info_buf = []
        if env is not None:
            self._set_env(env)
            if _init_setup_model:
                self.setup_model()

    def _check_env(self):
        if self.n_envs != 1:
            raise ValueError("the model requires a non vectorized environment or a single vectorized environment")
        super()._check_env()

    def setup_model(self):
        obs_dim = int(np.prod(self.observation_space.shape))
        A = int(np.prod(self.action_space.shape))
        self.learner = TRPOLearner(obs_dim, A, tuple(self.layers), self.timesteps_per_batch, self.gamma, self.lam, self.max_kl,
                                   self.cg_iters, self.cg_damping, self.entcoeff, self.vf_stepsize, self.vf_iters, int(self.seed or 0),
                                   self.device)
        self.learner.load_parameters(init_params(obs_dim, A, self.layers, self.seed))
        self._attach_device()

    #: TensorBoard tag -> b2g_trpo_metrics field of the per-iteration summary (tensorboard.py)
    _update_tags = {"policy_gradient_loss": "optimgain", "approximate_kullback-leibler": "meankl", "entropy_loss": "entropy",
                    "value_function_loss": "vf_loss"}

    def learn(self, total_timesteps, callback=None, log_interval=100, tb_log_name="TRPO", reset_num_timesteps=True):
        """stable-baselines 2.10 TRPO.learn: iterations while timesteps_so_far < total_timesteps (ceil(total / N) full batches
        of N = timesteps_per_batch steps; clipped actions to the env, num_timesteps += 1, callback.on_step() False stops before
        the update), each followed by the policy step and vf_iters passes of np.random.shuffle'd value minibatches.  Every call
        starts from env.reset() with an empty rollout.  With tensorboard_log each iteration's metrics and every finished
        episode's reward are written (tensorboard.py)."""
        return self._learn_logged(tb_log_name, reset_num_timesteps,
                                  lambda writer, _: self._learn(total_timesteps, callback, log_interval, reset_num_timesteps, writer))

    def _learn(self, total_timesteps, callback, log_interval, reset_num_timesteps, writer):
        callback, ep_log, obs = self._learn_start(callback, reset_num_timesteps, writer, globals())
        N = self.timesteps_per_batch
        timesteps_so_far, iters_so_far = 0, 0
        while timesteps_so_far < total_timesteps:
            obs, stopped = self._rollout(obs, N, callback, writer, ep_log)
            if stopped:
                break
            perms = np.empty((self.vf_iters, N), np.int32)
            for k in range(self.vf_iters):
                inds = np.arange(N)
                np.random.shuffle(inds)
                perms[k] = inds
            metrics = self.learner.update(None if self.device_obs_norm else obs, perms)
            timesteps_so_far += N
            iters_so_far += 1
            self._update_done(metrics, writer)
            if self.verbose >= 1 and (iters_so_far % log_interval == 0 or iters_so_far == 1):
                print(f"| trpo iteration {iters_so_far} | total_timesteps {self.num_timesteps} | "
                      + " | ".join(f"{k} {v:.5g}" for k, v in self.last_metrics.items()))
        callback.on_training_end()
        return self

    def _data(self):
        return {"gamma": self.gamma, "timesteps_per_batch": self.timesteps_per_batch, "max_kl": self.max_kl, "cg_iters": self.cg_iters,
                "lam": self.lam, "entcoeff": self.entcoeff, "cg_damping": self.cg_damping, "vf_stepsize": self.vf_stepsize,
                "vf_iters": self.vf_iters, **self._space_data()}

    def _host_init(self):
        return dict(gamma=self.gamma, timesteps_per_batch=self.timesteps_per_batch, max_kl=self.max_kl, cg_iters=self.cg_iters, lam=self.lam,
                    entcoeff=self.entcoeff, cg_damping=self.cg_damping, vf_stepsize=self.vf_stepsize, vf_iters=self.vf_iters,
                    verbose=self.verbose, policy_kwargs=self.policy_kwargs, seed=self.seed, device=self.device)


__all__ = ["TRPO", "TRPOLearner", "POLICY_VARS", "init_params", "value_minibatches"]
