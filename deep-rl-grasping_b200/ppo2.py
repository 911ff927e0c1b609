"""``PPO2`` -- the PPO branch of the reference's training harness (/root/reference/manipulation_main/training/sb_helper.py:137-154,
train_stable_baselines.py:99-100): stable-baselines 2.10.1 ``PPO2`` with ``common.policies.MlpPolicy`` and its defaults.  The
rollout buffer, GAE and every minibatch step run on the GPU (csrc/ppo.cu); the algorithm is restated in oracle/ppo_ref.py.
Import it as ``b200grasp.ppo2.PPO2`` (the stable-baselines path ``stable_baselines.ppo2.PPO2``).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _lib
from .actor_critic import ActorCriticLearner, ActorCriticModel, check_policy, check_policy_kwargs
from .actor_critic import init_params as _init_params
from .learner import _f32, _fp

_SCOPE = "model/"


class PPO2Learner(ActorCriticLearner):
    """numpy-facing wrapper of one ``b2g_ppo`` handle (maps 1:1 onto the C ABI)."""
    _abi = "ppo"

    def __init__(self, obs_dim, n_actions, layers=(64, 64), n_envs=1, n_steps=128, nminibatches=4, noptepochs=4, gamma=0.99, lam=0.95,
                 ent_coef=0.01, vf_coef=0.5, max_grad_norm=0.5, seed=0, device=0):
        self.lib = _lib.load()
        if len(layers) != 2:
            raise NotImplementedError(f"layers={list(layers)}: the PPO2 learner builds two hidden layers")
        cfg = _lib.PpoCfg(int(obs_dim), int(n_actions), int(layers[0]), int(layers[1]), int(n_envs), int(n_steps), int(nminibatches),
                          int(noptepochs), float(gamma), float(lam), float(ent_coef), float(vf_coef), float(max_grad_norm),
                          int(seed) & 0xFFFFFFFFFFFFFFFF, int(device))
        self._create(cfg)
        self.obs_dim, self.n_actions, self.n_envs, self.n_steps = int(obs_dim), int(n_actions), int(n_envs), int(n_steps)
        self.nminibatches, self.noptepochs = int(nminibatches), int(noptepochs)
        self.n_batch = self.n_envs * self.n_steps
        self.minibatch = self.n_batch // self.nminibatches

    def _has_grad(self, name):
        return not name.startswith(_SCOPE + "q/")      # q has no gradient

    def rollout_act(self, obs):
        """Rollout step: obs [n_envs, obs_dim] -> unclipped actions [n_envs, n_actions] (stored with values and neglogp)."""
        obs = _f32(obs).reshape(self.n_envs, self.obs_dim)
        out = np.empty((self.n_envs, self.n_actions), np.float32)
        _lib.check(self.lib.b2g_ppo_rollout_act(self.h, _fp(obs), _fp(out)))
        return out

    def rollout_reward(self, rew, done):
        _lib.check(self.lib.b2g_ppo_rollout_reward(self.h, _fp(_f32(np.reshape(rew, -1))), _fp(_f32(np.reshape(done, -1)))))

    def rollout_get(self):
        """advantages, returns, values, neglogp [n_steps, n_envs] and actions [n_steps, n_envs, n_actions] (time-major)."""
        T, E = self.n_steps, self.n_envs
        adv, ret, val, nlp = (np.empty((T, E), np.float32) for _ in range(4))
        act = np.empty((T, E, self.n_actions), np.float32)
        _lib.check(self.lib.b2g_ppo_rollout_get(self.h, _fp(adv), _fp(ret), _fp(val), _fp(nlp), _fp(act)))
        return dict(advantages=adv, returns=ret, values=val, neglogp=nlp, actions=act)

    def update(self, last_obs, perms, lr, cliprange, cliprange_vf):
        """One update on a full rollout; perms [noptepochs, n_batch] are the epochs' permutations of the env-major batch.
        ``last_obs=None`` bootstraps from the row observe_act staged after the last step."""
        p = np.ascontiguousarray(perms, np.int32).reshape(-1)
        assert p.size == self.noptepochs * self.n_batch
        m = _lib.PpoMetrics()
        _lib.check(self.lib.b2g_ppo_update(self.h, None if last_obs is None else _fp(_f32(last_obs).reshape(self.n_envs, self.obs_dim)),
                                           p.ctypes.data_as(C.POINTER(C.c_int32)), float(lr), float(cliprange), float(cliprange_vf),
                                           C.byref(m)))
        return m.as_dict()

    def train_step_explicit(self, obs, returns, actions, values, neglogp, lr, cliprange, cliprange_vf, apply_update=True):
        M = self.minibatch
        m = _lib.PpoMetrics()
        _lib.check(self.lib.b2g_ppo_train_step_explicit(
            self.h, _fp(_f32(obs).reshape(M, self.obs_dim)), _fp(_f32(np.reshape(returns, -1))), _fp(_f32(actions).reshape(M, self.n_actions)),
            _fp(_f32(np.reshape(values, -1))), _fp(_f32(np.reshape(neglogp, -1))), float(lr), float(cliprange), float(cliprange_vf),
            int(bool(apply_update)), C.byref(m)))
        return m.as_dict()

    def act(self, obs, deterministic=True, raw=False):
        """-> actions [n, n_actions] (mean, or mean + std * noise of stream 1), values [n], neglogp [n]; nothing is stored.
        ``raw``: the observations are normalised with the device obs_rms first (b2g_ppo_act_raw)."""
        obs = _f32(obs).reshape(-1, self.obs_dim)
        n = obs.shape[0]
        a, v, nl = np.empty((n, self.n_actions), np.float32), np.empty(n, np.float32), np.empty(n, np.float32)
        fn = self.lib.b2g_ppo_act_raw if raw else self.lib.b2g_ppo_act
        _lib.check(fn(self.h, _fp(obs), n, int(bool(deterministic)), _fp(a), _fp(v), _fp(nl)))
        return a, v, nl


def _schedule(v):
    """stable-baselines' get_schedule_fn: a callable of frac, or a constant."""
    return v if callable(v) else (lambda _frac, _v=v: _v)


def _check_policy_kwargs(policy_kwargs):
    """check_policy_kwargs with PPO2's messages -> (policy_kwargs as a dict, [h0, h1])"""
    return check_policy_kwargs(policy_kwargs, "PPO2")


class PPO2(ActorCriticModel):
    """stable-baselines 2.10 ``PPO2(policy, env, ...)`` with its signature and defaults, plus ``device``: ``learn / predict /
    save / load / get_parameters / load_parameters / get_env / get_vec_normalize_env / close`` and
    ``save_training_state / load_training_state``.  Box action spaces only, as the reference's configs give."""
    _algo, _branch, _scope = "PPO2", "PPO", _SCOPE
    _zip_hyper = ("gamma", "n_steps", "vf_coef", "ent_coef", "max_grad_norm", "learning_rate", "lam", "nminibatches", "noptepochs",
                  "cliprange", "cliprange_vf", "seed")

    def __init__(self, policy, env, gamma=0.99, n_steps=128, ent_coef=0.01, learning_rate=2.5e-4, vf_coef=0.5, max_grad_norm=0.5,
                 lam=0.95, nminibatches=4, noptepochs=4, cliprange=0.2, cliprange_vf=None, verbose=0, tensorboard_log=None,
                 _init_setup_model=True, policy_kwargs=None, full_tensorboard_log=False, seed=None, n_cpu_tf_sess=None, device=0,
                 device_obs_norm=False, **unsupported):
        if unsupported:
            raise TypeError(f"PPO2 got unexpected keyword arguments {sorted(unsupported)}")
        # learn() uploads each raw frame once: a VecNormalize with norm_obs hands its obs_rms to the learner, which merges the
        # frame and stores it in the rollout normalised as the wrapper would have returned it (PPO2Learner.observe_act)
        self.device_obs_norm = bool(device_obs_norm)
        self._refuse_device_obs_norm_without_wrapper(env)
        check_policy(policy, "PPO2")
        self.policy_kwargs, self.layers = _check_policy_kwargs(policy_kwargs)
        self.gamma, self.n_steps, self.ent_coef, self.learning_rate = gamma, int(n_steps), ent_coef, learning_rate
        self.vf_coef, self.max_grad_norm, self.lam = vf_coef, max_grad_norm, lam
        self.nminibatches, self.noptepochs, self.cliprange, self.cliprange_vf = int(nminibatches), int(noptepochs), cliprange, cliprange_vf
        self.verbose, self.tensorboard_log, self.seed, self.device = verbose, tensorboard_log, seed, device
        self.num_timesteps = 0
        self.n_envs = 1
        self.learner: Optional[PPO2Learner] = None
        self.ep_info_buf = []
        if env is not None:
            self._set_env(env)
            if _init_setup_model:
                self.setup_model()

    def _check_env(self):
        super()._check_env()
        if (self.n_envs * self.n_steps) % self.nminibatches:
            # ppo2.py's assertion: "The number of minibatches (nminibatches) is not a factor of the total number of samples"
            raise ValueError(f"nminibatches={self.nminibatches} is not a factor of n_batch = n_envs * n_steps = {self.n_envs * self.n_steps}")

    def setup_model(self):
        obs_dim = int(np.prod(self.observation_space.shape))
        A = int(np.prod(self.action_space.shape))
        self.learner = PPO2Learner(obs_dim, A, tuple(self.layers), self.n_envs, self.n_steps, self.nminibatches, self.noptepochs,
                                   self.gamma, self.lam, self.ent_coef, self.vf_coef, self.max_grad_norm, int(self.seed or 0), self.device)
        self.learner.load_parameters(_init_params(obs_dim, A, self.layers, self.seed))
        self._attach_device()

    #: TensorBoard tag -> b2g_ppo_metrics field of the per-update summary (tensorboard.py)
    _update_tags = {"loss/policy_gradient_loss": "policy_loss", "loss/value_function_loss": "value_loss", "loss/entropy_loss": "entropy",
                    "loss/approximate_kullback-leibler": "approxkl", "loss/clip_factor": "clipfrac"}

    def learn(self, total_timesteps, callback=None, log_interval=1, tb_log_name="PPO2", reset_num_timesteps=True):
        """stable-baselines 2.10 PPO2.learn: n_updates = total_timesteps // n_batch rollouts of n_steps steps (clipped actions to
        the env, num_timesteps += n_envs, callback.on_step() False stops before the update), each followed by noptepochs epochs of
        np.random.shuffle'd minibatches.  Every call starts from env.reset() with an empty rollout.  With tensorboard_log each
        update's means and every finished episode's reward are written (tensorboard.py)."""
        return self._learn_logged(tb_log_name, reset_num_timesteps,
                                  lambda writer, _: self._learn(total_timesteps, callback, log_interval, reset_num_timesteps, writer))

    def _learn(self, total_timesteps, callback, log_interval, reset_num_timesteps, writer):
        callback, ep_log, obs = self._learn_start(callback, reset_num_timesteps, writer, globals())
        lr_fn, clip_fn = _schedule(self.learning_rate), _schedule(self.cliprange)
        cvf = self.cliprange_vf
        cvf_fn = clip_fn if cvf is None else _schedule(cvf)
        clip_vf_off = isinstance(cvf, (float, int)) and not isinstance(cvf, bool) and cvf < 0
        n_batch = self.n_envs * self.n_steps
        n_updates = total_timesteps // n_batch
        for update in range(1, n_updates + 1):
            frac = 1.0 - (update - 1.0) / n_updates
            lr_now, clip_now = lr_fn(frac), clip_fn(frac)
            cvf_now = -1.0 if clip_vf_off else cvf_fn(frac)
            obs, stopped = self._rollout(obs, self.n_steps, callback, writer, ep_log)
            if stopped:
                break
            inds = np.arange(n_batch)
            perms = np.empty((self.noptepochs, n_batch), np.int32)
            for e in range(self.noptepochs):
                np.random.shuffle(inds)
                perms[e] = inds
            last_obs = None if self.device_obs_norm else obs          # None: the row observed after the last step
            self._update_done(self.learner.update(last_obs, perms, lr_now, clip_now, cvf_now), writer,
                              (("input_info/learning_rate", lr_now), ("input_info/clip_range", clip_now)))
            if self.verbose >= 1 and (update % log_interval == 0 or update == 1):
                print(f"| ppo2 update {update}/{n_updates} | total_timesteps {self.num_timesteps} | "
                      + " | ".join(f"{k} {v:.5g}" for k, v in self.last_metrics.items()))
        callback.on_training_end()
        return self

    def _data(self):
        data = {"gamma": self.gamma, "n_steps": self.n_steps, "vf_coef": self.vf_coef, "ent_coef": self.ent_coef,
                "max_grad_norm": self.max_grad_norm, "learning_rate": self.learning_rate, "lam": self.lam,
                "nminibatches": self.nminibatches, "noptepochs": self.noptepochs, "cliprange": self.cliprange,
                "cliprange_vf": self.cliprange_vf, **self._space_data()}
        for k in ("learning_rate", "cliprange", "cliprange_vf"):
            if callable(data[k]):
                data[k] = None
        return data

    def _check_without_env(self):
        if self.n_steps % self.nminibatches:
            raise ValueError(f"nminibatches={self.nminibatches} is not a factor of n_batch = {self.n_steps}")

    def _host_init(self):
        for k in ("learning_rate", "cliprange", "cliprange_vf"):
            if callable(getattr(self, k)):
                raise NotImplementedError(f"save_training_state needs a constant {k}")
        return dict(gamma=self.gamma, n_steps=self.n_steps, ent_coef=self.ent_coef, learning_rate=self.learning_rate, vf_coef=self.vf_coef,
                    max_grad_norm=self.max_grad_norm, lam=self.lam, nminibatches=self.nminibatches, noptepochs=self.noptepochs,
                    cliprange=self.cliprange, cliprange_vf=self.cliprange_vf, verbose=self.verbose, policy_kwargs=self.policy_kwargs,
                    seed=self.seed, device=self.device)
