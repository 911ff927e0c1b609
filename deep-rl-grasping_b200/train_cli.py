"""``train`` / ``run`` command line of the reference, re-hosted on the H100 learner.

Mirrors /root/reference/manipulation_main/training/train_stable_baselines.py:26-148 (same sub-commands, flags,
``model_dir`` layout: ``config.yaml``, ``best_model/``, ``logs/rl_model_*`` checkpoints, ``vecnormalize.pkl``,
``log_file.monitor.csv``) and the SAC / TRPO / PPO / DQN / BDQ branches of ``SBPolicy.learn`` (sb_helper.py:69-165,175-247).  The
environment itself stays the reference's (PyBullet on host cores): ``--env module:callable`` names a factory
``f(config, evaluate=False, validate=False, test=False) -> gym.Env``; the default imports the reference package and
calls ``gym.make('gripper-env-v0', ...)`` exactly like the original script.

  python -m b200grasp.train_cli train --config config/gripper_grasp.yaml --algo SAC --model_dir out/sac_depth
  python -m b200grasp.train_cli run --model trained_models/SAC_depth_1mbuffer/best_model/best_model.zip -t
"""
from __future__ import annotations

import argparse
import importlib
import inspect
import logging
import os

import numpy as np
import yaml

from . import BDQ, SAC, training_state
from .bench import Monitor
from .callbacks import BaseCallback, CheckpointCallback, EvalCallback, TrainingStateCallback
from .deepq import DQN
from .deepq.policies import MlpPolicy as DQNMlpPolicy
from .common.policies import MlpPolicy as PPOMlpPolicy
from .ppo2 import PPO2
from .trpo_mpi import TRPO
from .sac_model import CnnPolicy, MlpPolicy
from .vec_env import DummyVecEnv, SubprocVecEnv, VecEncodeDepth, VecNormalize


def _default_factory(config, evaluate=False, validate=False, test=False):
    import gym                      # the reference's own dependency chain (gym + pybullet + manipulation_main)
    import manipulation_main        # noqa: F401  (registers gripper-env-v0)
    return gym.make("gripper-env-v0", config=config, evaluate=evaluate, validate=validate, test=test)


def _factory(spec):
    if not spec:
        return _default_factory
    mod, _, fn = spec.partition(":")
    return getattr(importlib.import_module(mod), fn)


class SaveVecNormalizeCallback(BaseCallback):
    """sb_helper.py:24-56: writes ``vecnormalize.pkl`` next to the (best) model."""

    def __init__(self, save_freq, save_path, name_prefix=None, verbose=0):
        super().__init__(verbose)
        self.save_freq, self.save_path, self.name_prefix = save_freq, save_path, name_prefix

    def _init_callback(self):
        os.makedirs(self.save_path, exist_ok=True)

    def _on_step(self):
        if self.n_calls % self.save_freq == 0:
            name = "vecnormalize.pkl" if self.name_prefix is None else f"{self.name_prefix}_{self.num_timesteps}_steps.pkl"
            vn = self.model.get_vec_normalize_env()
            if vn is not None:
                vn.save(os.path.join(self.save_path, name))
        return True


def _is_image_obs(env):
    return len(env.observation_space.shape) == 3


def device_encoder(config, n_envs):
    """The perception encoder of ``config['sensor']['encoder_dir']`` (the directory the reference sensor reads), for the
    frames and terminal observations of ``n_envs`` envs in one call, at the run's ``device_encode_precision`` (fp32 when
    the config has none)."""
    from .encoders import SimpleAutoEncoder
    model_dir = os.path.expanduser(config["sensor"]["encoder_dir"])
    with open(os.path.join(model_dir, "config.yaml")) as f:
        enc = SimpleAutoEncoder(yaml.safe_load(f), max_batch=2 * n_envs, precision=config.get("device_encode_precision", "fp32"))
    enc.load_weights(model_dir)
    return enc


def encode_depth(env, test_env, config, n_envs):
    """--device_encode: the training and evaluation envs hand out raw depth rows (encoders.DeferredEncodedDepthImgSensor);
    one VecEncodeDepth over each encodes them in this process.  A SAC / BDQ / PPO2 / TRPO model with device_obs_norm then takes the
    encoder and the training wrapper passes the rows through to the device; the evaluation wrapper stays in host mode."""
    encoder = device_encoder(config, n_envs)
    return VecEncodeDepth(env, encoder), VecEncodeDepth(test_env, encoder)


def _check_device_encode(config):
    if config.get("depth_observation", False) or config.get("full_observation", False):
        raise ValueError("--device_encode: the config observes images (depth_observation / full_observation); the encoder "
                         "feeds the encoded-depth observation only")


def train(args):
    if getattr(args, "resume", None):
        return resume(args)
    config = yaml.safe_load(open(args.config))
    algo = args.algo
    if args.device_encode:
        _check_device_encode(config)
        config["device_encode"] = True          # --resume and run rebuild the same stack
        config["device_encode_precision"] = args.encoder_precision or "fp32"
    if algo == "DQN":          # stable-baselines' DQN takes one environment; its statistics stay with the host VecNormalize
        if int(args.n_envs) > 1:
            raise ValueError("--algo DQN: DQN cannot be used with more than one environment (--n_envs 1)")
        if args.device_norm:
            raise NotImplementedError("--algo DQN: --device_norm is built for SAC, BDQ, PPO and TRPO only")
    if algo in ("PPO", "TRPO") and args.device_norm and not config.get("normalize", False):
        # PPO2 and TRPO store what VecNormalize returns: --device_norm moves its statistics to the learner, so it needs them
        raise NotImplementedError(f"--algo {algo}: --device_norm keeps VecNormalize's observation statistics on the GPU; the "
                                  "config has no normalize: true")
    if algo == "PPO":
        if args.load_dir:
            raise NotImplementedError("--algo PPO: --load_dir is not read by the reference's PPO branch (sb_helper.py:137-154)")
    if algo == "TRPO":         # TRPO trains on one environment
        if args.load_dir:
            raise NotImplementedError("--algo TRPO: --load_dir is not read by the reference's TRPO branch (sb_helper.py:129-136)")
        if int(args.n_envs) > 1:
            raise ValueError("--algo TRPO: the model requires a non vectorized environment or a single vectorized environment "
                             "(--n_envs 1)")
    os.mkdir(args.model_dir)                                   # like the reference: refuses to overwrite a run
    os.mkdir(os.path.join(args.model_dir, "best_model"))
    if args.simple:
        config["simplified"] = True
    if args.shaped:
        config["reward"]["shaped"] = True
    if args.timestep:
        config[algo]["total_timesteps"] = int(args.timestep)
    config["robot"]["discrete"] = algo == "DQN"
    config[algo]["save_dir"] = args.model_dir
    config["algorithm"] = algo.lower()
    make = _factory(args.env)
    n_envs = max(1, int(args.n_envs))
    if n_envs == 1:
        env = DummyVecEnv([lambda: Monitor(make(config), os.path.join(args.model_dir, "log_file"))])
    else:                                                      # BASELINE config 5: vectorised host actor loop
        env = SubprocVecEnv([(lambda i=i: Monitor(make(config), os.path.join(args.model_dir, f"log_file_{i}"))) for i in range(n_envs)])
    for sub in ("", "best_model"):
        yaml.safe_dump(config, open(os.path.join(args.model_dir, sub, "config.yaml"), "w"))
    test_env = DummyVecEnv([lambda: make(config, evaluate=True, validate=True)])
    if config.get("device_encode", False):
        env, test_env = encode_depth(env, test_env, config, n_envs)
    norm = bool(config.get("normalize", False))
    eval_path = os.path.join(args.model_dir, "best_model")
    if norm:
        test_env = VecNormalize(test_env, norm_obs=True, norm_reward=False, clip_obs=10.0)
    callbacks = [
        EvalCallback(test_env, best_model_save_path=eval_path, log_path=os.path.join(eval_path, "logs"), eval_freq=args.eval_freq,
                     n_eval_episodes=10, callback_on_new_best=SaveVecNormalizeCallback(1, eval_path), deterministic=True),
        CheckpointCallback(save_freq=args.checkpoint_freq, save_path=os.path.join(args.model_dir, "logs"), name_prefix="rl_model"),
    ]
    top = os.path.dirname(args.load_dir) if args.load_dir else None
    if norm:
        if args.load_dir:
            env = VecNormalize.load(os.path.join(top, "vecnormalize.pkl"), VecNormalize(env, training=True, norm_obs=False, norm_reward=False, clip_obs=10.0))
        else:
            env = VecNormalize(env, norm_obs=True, norm_reward=True, clip_obs=10.0)
    c = config[algo]
    tb = tensorboard_log(config, algo, args.model_dir)
    if algo == "SAC":
        simplified_image = _is_image_obs(env) and bool(config.get("simplified", False))
        if simplified_image:
            # sb_helper.py:92-94: CnnPolicy with policy_kwargs={}, i.e. stable-baselines' plain nature_cnn over every plane
            # and the default [64, 64] head, whatever the config's layers say
            policy, kw = CnnPolicy, {"cnn_extractor": "nature_cnn"}
        elif _is_image_obs(env):
            policy, kw = CnnPolicy, {"layers": c["layers"], "cnn_extractor": "augmented_nature_cnn"}
        else:
            policy, kw = MlpPolicy, {"layers": c["layers"], "layer_norm": False}
        replay = replay_frames_kwargs(args, c["buffer_size"], n_envs)
        if _is_image_obs(env) and config.get("full_observation", False) and not simplified_image:
            # RGB renders as uint8 (gripperEnv/sensor.py), depth stays fp32; the simplified observation is depth + pad even
            # under full_observation (robot.py:192-196), so it has no 8-bit planes
            replay["replay_u8_planes"] = (0, 1, 2)
        if args.device_norm:
            replay["device_obs_norm"] = True
        model = SAC(policy, env, policy_kwargs=kw, verbose=1, gamma=config["discount_factor"], buffer_size=c["buffer_size"],
                    batch_size=c["batch_size"], learning_rate=c["step_size"], precision=args.precision, tensorboard_log=tb, **replay)
        if args.load_dir:
            old = SAC.load(args.load_dir, env, buffer_size=1)
            model.load_parameters(old.get_parameters(), exact_match=False)
            old.close()
    elif algo == "BDQ":
        model = BDQ("MlpActPolicy", env, policy_kwargs={"layers": c["layers"]}, verbose=1, gamma=config["discount_factor"],
                    batch_size=c["batch_size"], buffer_size=c["buffer_size"], learning_rate=c["step_size"],
                    exploration_fraction=c.get("exploration_fraction", 0.1), exploration_final_eps=c.get("exploration_final_eps", 0.02),
                    num_actions_pad=c.get("num_actions_pad", 33), learning_starts=c.get("learning_starts", 1000),
                    target_network_update_freq=c.get("target_network_update_freq", 1000),
                    prioritized_replay=c.get("prioritized_replay", False), device_obs_norm=bool(args.device_norm), tensorboard_log=tb,
                    **replay_frames_kwargs(args, c["buffer_size"], n_envs))
        if args.load_dir:
            model.load_parameters(BDQ.load(args.load_dir, env).get_parameters())
    elif algo == "DQN":
        kw = dqn_kwargs(config)
        # sb_helper leaves DQN's buffer_size at stable-baselines' default, which DQN's signature holds
        kw.update(replay_frames_kwargs(args, inspect.signature(DQN).parameters["buffer_size"].default, n_envs))
        model = DQN(DQNMlpPolicy, env, tensorboard_log=tb, **kw)
        if args.load_dir:        # every parameter (sb_helper.py:183-199's partial load cannot run: tensorboard_file is undefined there)
            old = DQN.load(args.load_dir)
            model.load_parameters(old.get_parameters())
            old.close()
    elif algo == "PPO":
        model = PPO2(PPOMlpPolicy, env, tensorboard_log=tb, device_obs_norm=bool(args.device_norm), **ppo_kwargs(config))
    elif algo == "TRPO":
        model = TRPO(PPOMlpPolicy, env, tensorboard_log=tb, device_obs_norm=bool(args.device_norm), **trpo_kwargs(config))
    else:
        raise NotImplementedError(f"--algo {algo}: the H100 learner builds the SAC, TRPO, PPO, DQN and BDQ branches of SBPolicy.learn "
                                  "(sb_helper.py:85-226)")
    if args.state_freq:
        callbacks.append(TrainingStateCallback(args.state_freq, os.path.join(args.model_dir, STATE_DIR)))
        _learn_keeping_state(model, int(c["total_timesteps"]), callbacks, os.path.join(args.model_dir, STATE_DIR))
    else:
        model.learn(total_timesteps=int(c["total_timesteps"]), callback=callbacks)
    model.save(os.path.join(args.model_dir, "final_model" if algo != "BDQ" else "bdq_model"))   # sb_helper.py:228-247
    vn = model.get_vec_normalize_env()
    if vn is not None:
        vn.save(os.path.join(args.model_dir, "vecnormalize.pkl"))
    env.close()
    test_env.close()
    return model


STATE_DIR = "training_state"


def tensorboard_log(config, algo, model_dir):
    """sb_helper.py:84: no TensorBoard log when the algorithm's ``tensorboard_logs`` is missing or null, else
    ``"tensorboard_logs/" + model_dir`` (the directory name only, not the configured path), relative to the working
    directory."""
    if (config.get(algo) or {}).get("tensorboard_logs") is None:
        return None
    return "tensorboard_logs/" + model_dir


def replay_frames_kwargs(args, buffer_size, n_envs):
    """train --replay_spare F (SAC, BDQ, DQN): {"replay_frames": buffer_size * (1 + F) + n_envs}, or {} without the flag.  Every
    transition holds one frame of its own plus one per episode end; n_envs more for the rows in flight."""
    if args.replay_spare is None:
        return {}
    return {"replay_frames": int(buffer_size * (1.0 + args.replay_spare)) + n_envs}


def dqn_kwargs(config):
    """sb_helper.py:159-165: only gamma, batch_size and prioritized_replay come from the config; every other DQN setting stays at
    stable-baselines' default (the config's DQN learning_rate is not read there, and the shipped zip holds 5e-4)."""
    c = config["DQN"]
    return dict(verbose=2, gamma=config["discount_factor"], batch_size=c["batch_size"], prioritized_replay=c["prioritized_replay"])


def ppo_kwargs(config):
    """sb_helper.py:149-154: only gamma (discount_factor) and the PPO learning_rate come from the config, with verbose=2; every
    other PPO2 setting stays at stable-baselines' default.  The config's PPO ``layers`` and ``n_steps`` are not passed there,
    and the policy_kwargs sb_helper computes for image observations are dropped before the call, so the policy is always
    MlpPolicy with [64, 64]."""
    return dict(verbose=2, gamma=config["discount_factor"], learning_rate=config["PPO"]["learning_rate"])


def trpo_kwargs(config):
    """sb_helper.py:129-136: gamma (discount_factor), timesteps_per_batch (TRPO.max_iters) and vf_stepsize (TRPO.step_size) come
    from the config, with verbose=2; every other TRPO setting stays at stable-baselines' default."""
    c = config["TRPO"]
    return dict(verbose=2, gamma=config["discount_factor"], timesteps_per_batch=c["max_iters"], vf_stepsize=c["step_size"])


def _learn_keeping_state(model, total_timesteps, callbacks, state_dir, reset_num_timesteps=True):
    """model.learn; an interrupt (Ctrl-C) writes the training state before the run ends, as sb_helper.py:178-181 does
    for the model."""
    try:
        model.learn(total_timesteps=total_timesteps, callback=callbacks, reset_num_timesteps=reset_num_timesteps)
    except KeyboardInterrupt:
        model.save_training_state(state_dir)


def resume(args):
    """train --resume <model_dir>: continues the run whose config.yaml and training_state/ sit in model_dir for the
    remaining total_timesteps - num_timesteps steps.  The environment starts a fresh episode."""
    model_dir = args.resume
    config = yaml.safe_load(open(os.path.join(model_dir, "config.yaml")))
    algo = config["algorithm"].upper()
    if algo not in ("SAC", "BDQ", "DQN", "PPO", "TRPO"):
        raise NotImplementedError(f"--resume: algorithm '{algo}' has no training state")
    state_dir = training_state.resolve(os.path.join(model_dir, STATE_DIR))
    done = int(training_state.read_host(state_dir)["num_timesteps"])
    make = _factory(args.env)
    n_envs = max(1, int(args.n_envs))
    log = os.path.join(model_dir, f"log_file_resume_{done}")        # the original run's monitor file stays as it is
    if n_envs == 1:
        env = DummyVecEnv([lambda: Monitor(make(config), log)])
    else:
        env = SubprocVecEnv([(lambda i=i: Monitor(make(config), f"{log}_{i}")) for i in range(n_envs)])
    test_env = DummyVecEnv([lambda: make(config, evaluate=True, validate=True)])
    if config.get("device_encode", False):
        env, test_env = encode_depth(env, test_env, config, n_envs)
    eval_path = os.path.join(model_dir, "best_model")
    if config.get("normalize", False):
        test_env = VecNormalize(test_env, norm_obs=True, norm_reward=False, clip_obs=10.0)
        env = VecNormalize(env, norm_obs=True, norm_reward=True, clip_obs=10.0)     # statistics: the saved ones
    callbacks = [
        EvalCallback(test_env, best_model_save_path=eval_path, log_path=os.path.join(eval_path, "logs"), eval_freq=args.eval_freq,
                     n_eval_episodes=10, callback_on_new_best=SaveVecNormalizeCallback(1, eval_path), deterministic=True),
        CheckpointCallback(save_freq=args.checkpoint_freq, save_path=os.path.join(model_dir, "logs"), name_prefix="rl_model"),
    ]
    if args.state_freq:
        callbacks.append(TrainingStateCallback(args.state_freq, os.path.join(model_dir, STATE_DIR)))
    model = {"SAC": SAC, "BDQ": BDQ, "DQN": DQN, "PPO": PPO2, "TRPO": TRPO}[algo].load_training_state(state_dir, env)
    # the continued run writes into the latest run directory of the same log (learn(reset_num_timesteps=False))
    model.tensorboard_log = tensorboard_log(config, algo, model_dir)
    remaining = int(config[algo]["total_timesteps"]) - model.num_timesteps
    if remaining > 0:
        _learn_keeping_state(model, remaining, callbacks, os.path.join(model_dir, STATE_DIR), reset_num_timesteps=False)
    model.save(os.path.join(model_dir, "final_model" if algo != "BDQ" else "bdq_model"))
    vn = model.get_vec_normalize_env()
    if vn is not None:
        vn.save(os.path.join(model_dir, "vecnormalize.pkl"))
    env.close()
    test_env.close()
    return model



def run_agent(task, agent, stochastic=False, n_episodes=100):
    """manipulation_main/utils.py:14-76: roll out `n_episodes` and report success rate / reward / length."""
    rewards, steps, successes = [], [], []
    for _ in range(n_episodes):
        obs, done = task.reset(), np.array([False])
        ep_r, ep_n, info = 0.0, 0, {}
        while not done[0]:
            action = agent.predict(obs, deterministic=not stochastic)[0]
            obs, r, done, infos = task.step(action)
            rew = task.get_original_reward() if hasattr(task, "get_original_reward") else r
            ep_r += float(np.ravel(rew)[0]); ep_n += 1
            info = infos[0] if infos else {}
        rewards.append(ep_r); steps.append(ep_n)
        successes.append(bool(info.get("is_success", info.get("status", None) in ("SUCCESS", 1))))
    out = {"success_rate": float(np.mean(successes)), "mean_reward": float(np.mean(rewards)), "mean_steps": float(np.mean(steps)), "episodes": n_episodes}
    print(f"Finished {n_episodes} episodes: success rate {out['success_rate']:.3f}, mean reward {out['mean_reward']:.1f}, mean steps {out['mean_steps']:.1f}")
    return out


def run(args):
    top = os.path.dirname(args.model)
    config = yaml.safe_load(open(os.path.join(top, "config.yaml")))
    make = _factory(args.env)
    task = DummyVecEnv([lambda: make(config, evaluate=True, test=args.test)])
    if config.get("device_encode", False):         # the saved zip takes encoded observations: host mode
        task = VecEncodeDepth(task, device_encoder(config, 1))
    if config.get("normalize", False):
        task = VecNormalize.load(os.path.join(top, "vecnormalize.pkl"), VecNormalize(task, training=False, norm_obs=True, norm_reward=True, clip_obs=10.0))
        task.training = False
    algo = config["algorithm"]
    if algo == "sac":
        agent = SAC.load(args.model, precision=args.precision)
        agent._vec_normalize_env = task if isinstance(task, VecNormalize) else None     # predict() receives normalised observations
        if agent._vec_normalize_env is not None:
            agent._sync_norm_stats()
    elif algo == "bdq":
        agent = BDQ.load(args.model)
    elif algo == "dqn":
        agent = DQN.load(args.model)
    elif algo == "ppo":
        agent = PPO2.load(args.model)
    elif algo == "trpo":
        agent = TRPO.load(args.model)
    else:
        raise NotImplementedError(f"algorithm '{algo}': only sac / trpo / ppo / dqn / bdq zips run on the H100 learner")
    print("Run the agent")
    out = run_agent(task, agent, args.stochastic, n_episodes=args.episodes)
    task.close()
    return out


def build_parser():
    p = argparse.ArgumentParser(prog="b200grasp.train_cli")
    sub = p.add_subparsers()
    t = sub.add_parser("train")
    t.add_argument("--config", type=str)           # required unless --resume (checked in main)
    t.add_argument("--algo", type=str)
    t.add_argument("--model_dir", type=str)
    t.add_argument("--load_dir", type=str)
    t.add_argument("--timestep", type=str)
    t.add_argument("-s", "--simple", action="store_true")
    t.add_argument("-sh", "--shaped", action="store_true")
    t.add_argument("-v", "--visualize", action="store_true")
    t.add_argument("-tf", "--timefeature", action="store_true")
    t.add_argument("--env", type=str, default=None, help="module:callable environment factory (default: the reference's gripper-env-v0)")
    t.add_argument("--n_envs", type=int, default=1, help=">1: SubprocVecEnv actor loop on host cores feeding the device replay")
    t.add_argument("--precision", default="bf16x3", choices=["fp32", "bf16x3", "bf16"])
    t.add_argument("--replay_spare", type=float, default=None,
                   help="SAC / BDQ / DQN replay frame budget buffer_size * (1 + F) + n_envs (observations shared between "
                        "consecutive transitions; 0.125 covers episodes down to ~9 steps); default: two frames per replay slot; "
                        "--resume takes it from the saved run")
    t.add_argument("--device_norm", action="store_true",
                   help="keep VecNormalize's observation statistics on the GPU and upload every frame once "
                        "(SAC / BDQ / PPO / TRPO(device_obs_norm=True); not DQN); --resume takes it from the saved run")
    t.add_argument("--device_encode", action="store_true",
                   help="the env's sensor defers the depth encoding (encoders.DeferredEncodedDepthImgSensor): encode the "
                        "frames of all envs at once in this process, on the learner's device with --device_norm (SAC / BDQ / "
                        "PPO / TRPO)")
    t.add_argument("--encoder_precision", default=None, choices=["fp32", "bf16x3"],
                   help="with --device_encode: the encoder's arithmetic, fp32 on the CUDA cores (default) or bf16x3 on the tensor "
                        "cores (about 2^-16 relative per layer); recorded in config.yaml as device_encode_precision")
    t.add_argument("--eval_freq", type=int, default=50000)
    t.add_argument("--checkpoint_freq", type=int, default=25000)
    t.add_argument("--state_freq", type=int, default=None,
                   help="every N steps write the whole training state (replay, optimiser moments, counters) to "
                        "<model_dir>/training_state, keeping only the latest; an interrupt writes it too")
    t.add_argument("--resume", type=str, default=None, metavar="MODEL_DIR",
                   help="continue the run in MODEL_DIR from its training_state/ for the rest of its total_timesteps")
    t.set_defaults(func=train)
    r = sub.add_parser("run")
    r.add_argument("--model", type=str, required=True)
    r.add_argument("-v", "--visualize", action="store_true")
    r.add_argument("-t", "--test", action="store_true")
    r.add_argument("-s", "--stochastic", action="store_true")
    r.add_argument("--env", type=str, default=None)
    r.add_argument("--episodes", type=int, default=100)
    r.add_argument("--precision", default="bf16x3", choices=["fp32", "bf16x3", "bf16"])
    r.set_defaults(func=run)
    return p


def main(argv=None):
    logging.getLogger().setLevel(logging.INFO)
    parser = build_parser()
    args = parser.parse_args(argv)
    if not hasattr(args, "func"):
        build_parser().print_help()
        return None
    if args.func is train and args.encoder_precision is not None and not args.device_encode:
        parser._subparsers._group_actions[0].choices["train"].error("--encoder_precision needs --device_encode")
    if args.func is train and not args.resume:
        missing = [f"--{k}" for k in ("config", "algo", "model_dir") if getattr(args, k) is None]
        if missing:
            parser._subparsers._group_actions[0].choices["train"].error("the following arguments are required: " + ", ".join(missing))
    return args.func(args)


if __name__ == "__main__":
    main()
