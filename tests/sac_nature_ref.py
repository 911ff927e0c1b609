"""Float64 restatement of SAC with stable-baselines' plain ``nature_cnn`` extractor (the simplified environment's CnnPolicy,
sb_helper.py:92-94), for the tests.

The network is ``oracle/sac_ref.py``'s with two differences, both in ``NatureConfig``: conv1 reads every plane of the
observation (``c_img = C``), and there is no direct feature (``n_direct = 0``, so 512 features feed the heads).  Its
variables carry stable-baselines' names instead of ``create_augmented_nature_cnn``'s:

  model/pi/cnn1 .. cnn3, cnn_fc1  ->  model/pi/c1 .. c3, fc1        ([SB2] common/policies.py nature_cnn)
  model/pi/fc1/{kernel,bias}      ->  model/pi/fc1_1/{kernel,bias}  (TF1 uniquifies the actor's second dense layer, whose
                                                                     default name clashes with nature_cnn's 'fc1' scope)

So the oracle's own functions compute it, on parameters renamed with ``to_oracle`` / ``from_oracle``.  Parameter order is
TF creation order, the same as the augmented network's.
"""
from __future__ import annotations

import dataclasses
import re
from collections import OrderedDict

from oracle import sac_ref as R

_CNN = {"c1": "cnn1", "c2": "cnn2", "c3": "cnn3", "fc1": "cnn_fc1"}
_CNN_BACK = {v: k for k, v in _CNN.items()}
_SCOPES = "(model/pi|model/values_fn|target/values_fn)"


@dataclasses.dataclass
class NatureConfig(R.SACConfig):
    """obs_shape = (64, 64, C): every plane is an image plane."""
    obs_shape: tuple = (64, 64, 2)
    n_act: int = 3
    target_entropy: float = -3.0
    n_direct: int = 0

    @property
    def c_img(self) -> int:
        return self.obs_shape[2]


def nature_name(oracle_name: str) -> str:
    m = re.fullmatch(_SCOPES + r"/(cnn1|cnn2|cnn3|cnn_fc1)/(w|b)", oracle_name)
    if m:
        return f"{m.group(1)}/{_CNN_BACK[m.group(2)]}/{m.group(3)}"
    if re.fullmatch(r"model/pi/fc1/(kernel|bias)", oracle_name):
        return oracle_name.replace("model/pi/fc1/", "model/pi/fc1_1/")
    return oracle_name


def oracle_name(name: str) -> str:
    m = re.fullmatch(_SCOPES + r"/(c1|c2|c3|fc1)/(w|b)", name)
    if m:
        return f"{m.group(1)}/{_CNN[m.group(2)]}/{m.group(3)}"
    if re.fullmatch(r"model/pi/fc1_1/(kernel|bias)", name):
        return name.replace("model/pi/fc1_1/", "model/pi/fc1/")
    return name


def to_oracle(d):
    return OrderedDict((oracle_name(n), a) for n, a in d.items())


def from_oracle(d):
    return OrderedDict((nature_name(n), a) for n, a in d.items())


def param_specs(cfg: NatureConfig):
    """(name, shape) in stable-baselines' parameter_list order."""
    return [(nature_name(n), s) for n, s in R.param_specs(cfg)]


def init_params(cfg: NatureConfig, seed: int = 0):
    return from_oracle(R.init_params(cfg, seed=seed))


def sac_step(params, opt, batch, eps_noise, lr, cfg: NatureConfig, dtype):
    """R.sac_step on stable-baselines' names: -> (outputs, grads, new_params, new_opt)."""
    o = R.OptState(m=to_oracle(opt.m), v=to_oracle(opt.v), t=dict(opt.t))
    out, grads, newp, newopt = R.sac_step(to_oracle(params), o, batch, eps_noise, lr, cfg, dtype)
    return out, from_oracle(grads), from_oracle(newp), R.OptState(m=from_oracle(newopt.m), v=from_oracle(newopt.v), t=newopt.t)


def policy_act(params, obs_norm, cfg: NatureConfig, deterministic=True, eps_noise=None):
    return R.policy_act(to_oracle(params), obs_norm, cfg, deterministic=deterministic, eps_noise=eps_noise)
