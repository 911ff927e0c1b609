"""Public configurations that run on the round-1 tensor engine (csrc/gg_tc.cu) rather than the TMA-fed one:
policy inference at precision 1 and 2, bf16x3 training at an input size other than 64 x 64, and the bf16x3 MLP policy."""
import numpy as np
import pytest

from oracle import sac_ref as R
from tests.test_gpu_parity import _check_step
from tests.util import load_case, make_batch, make_learner, rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("precision,tol", [(1, 1e-4), (2, 5e-3)])
def test_policy_act_depth_cnn(precision, tol):
    """act() runs the pi forward through the round-1 groups; at precision 1 its conv activations live in planes the
    training engine shares.  Parity mode is held to 1e-4, the single-pass fast mode to its 5e-3 bar."""
    cfg, params, vn = load_case("sac_depth")
    B = 32
    raw, norm, _ = make_batch(vn, B)
    L = make_learner(cfg, vn, B, params, precision=precision)
    a_gpu = L.act(raw["obs"], deterministic=True)
    a_ref = R.policy_act(params, norm["obs"], cfg, deterministic=True)
    L.close()
    assert rel_err(a_gpu, a_ref) <= tol, rel_err(a_gpu, a_ref)


def test_bf16x3_step_60x60_input():
    """A 60 x 60 image still gives a 4 x 4 x 64 conv3 output, so the trained weights apply; bf16x3 trains on the round-1
    engine at this size.  The statistics are the depth case's, cropped to the image."""
    cfg, params, vn = load_case("sac_depth")
    vn60 = dict(vn, obs_mean=np.ascontiguousarray(vn["obs_mean"][:60, :60]), obs_var=np.ascontiguousarray(vn["obs_var"][:60, :60]))
    cfg60 = R.SACConfig(obs_shape=(60, 60, 2))
    _check_step(cfg60, params, vn60, 32, precision=1)


def test_bf16x3_step_mlp_policy():
    """The MLP (encoder) policy at bf16x3: its head contractions run on the round-1 engine without planes."""
    cfg, params, vn = load_case("sac_encoder")
    _check_step(cfg, params, vn, 64, precision=1)
