"""The graph-path step refreshes the BF16 weight planes in two launches: the forward layouts (W1T .. K0T) under the gather, and
the backward layouts (W2n .. K0n) alongside the tail, before bwd_fused reads them.  After several steps with updates, both
families must hold split3 of the weights the last step read, bit for bit: the weights before its update, not after it.  A
refresh moved behind the optimiser would leave split3 of the updated weights instead, which the parity tests cannot tell
apart from the right planes while one update barely moves the weights.

The second test catches a backward-plane refresh that runs after bwd_fused's reads but still before the optimiser (the end
state of the planes is then right): the step after a weight upload must produce the gradients of the uploaded weights, not of
the planes the previous step left.  Neither test can see a missing join whose refresh still happens to finish before
bwd_fused reads the planes; the event structure in issue_step (csrc/sac.cu) is what orders them."""
import numpy as np
import pytest
import torch

from b200grasp import synth
from oracle import sac_ref as R
from tests.test_gpu_contractions import NETS, Report, check_weight_planes, read
from tests.util import load_case, make_batch, make_learner, rel_err

PLANES = ["W1T/online", "W1T/target"] + [f"{t}/{n}" for t in ("W2T", "W3T", "WfT", "K0T") for n in NETS] + \
         [f"{t}/{n}" for t in ("W2n", "W3n", "Wfn", "K0n") for n in NETS[:2]]


@pytest.mark.gpu
def test_graph_steps_leave_both_plane_families_at_the_weights_the_step_read():
    cfg, params, vn = load_case("sac_depth")
    B, NS = 64, 512
    L = make_learner(cfg, vn, B, params, buffer_size=NS, precision=1)
    try:
        tr = synth.make_transitions(NS, vn["obs_mean"], vn["obs_var"], seed=21)
        L.replay_add(tr["obs"], tr["act"], tr["rew"], tr["next_obs"], tr["done"])
        L.step(4, lr=3e-3)
        read_by_last = {k: np.array(v) for k, v in L.get_parameters().items()}
        L.step(1, lr=3e-3)
        updated = {k: np.array(v) for k, v in L.get_parameters().items()}
        T = {n: read(L, n) for n in PLANES}
    finally:
        L.close()
    for scope in ("model/pi", "model/values_fn"):     # the last step moved the weights behind both families
        for w in ("cnn2/w", "cnn_fc1/w", "fc0/kernel" if scope == "model/pi" else "vf/fc0/kernel"):
            assert not np.array_equal(read_by_last[f"{scope}/{w}"], updated[f"{scope}/{w}"]), f"{scope}/{w} did not change"
    ci, A, H = cfg.obs_shape[-1] - 1, cfg.n_act, params["model/pi/fc0/kernel"].shape[1]
    rep = Report("graph path, last step's weights")
    check_weight_planes(rep, T, read_by_last, ci, A, H)
    rep.finish()
    stale = Report("graph path, updated weights")
    check_weight_planes(stale, T, updated, ci, A, H)
    for fam in ("WfT", "Wfn", "K0T", "K0n"):         # both families differ from split3 of the updated weights
        assert any(f.startswith(f"planes2/{fam}/") for f in stale.fail), fam


@pytest.mark.gpu
def test_step_after_an_upload_reads_backward_planes_of_the_uploaded_weights():
    cfg, trained, vn = load_case("sac_depth")
    other = R.init_params(cfg, seed=5)                  # far from the trained weights: stale planes move every conv gradient
    B, LR = 64, 3e-4
    raw, norm, eps = make_batch(vn, B)
    L = make_learner(cfg, vn, B, trained, precision=1)
    try:
        L.step_explicit(raw["obs"], raw["act"], raw["rew"], raw["next_obs"], raw["done"], eps, lr=LR, apply_update=False)
        L.load_parameters(other)                          # the planes now hold split3 of the trained weights
        L.step_explicit(raw["obs"], raw["act"], raw["rew"], raw["next_obs"], raw["done"], eps, lr=LR, apply_update=False)
        g = L.get_gradients()
    finally:
        L.close()
    _, g32, _, _ = R.sac_step(other, R.OptState.zeros(other), norm, eps, LR, cfg, torch.float32)
    _, g64, _, _ = R.sac_step(other, R.OptState.zeros(other), norm, eps, LR, cfg, torch.float64)
    names = [f"{scope}/{t}/{w}" for scope in ("model/pi", "model/values_fn") for t in ("cnn1", "cnn2", "cnn3", "cnn_fc1")
             for w in ("w", "b")]
    for n in names:                                       # the per-tensor bar of tests/test_gpu_parity.py
        bar = max(1e-3, 3.0 * rel_err(g32[n], g64[n]))
        assert rel_err(g[n], g64[n]) <= bar, (n, rel_err(g[n], g64[n]), bar)
