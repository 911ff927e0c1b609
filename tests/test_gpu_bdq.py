"""BDQ learner (SURVEY section 8 row a11) on the GPU against oracle/bdq_ref.py.  PARITY UNPINNED: the reference's
BDQ source is absent; shapes/names are pinned by the shipped zips (tests/test_host_cpu.py)."""
import numpy as np
import pytest
import torch

import b200grasp
from oracle import bdq_ref as Q
from tests.test_gpu_bdq_configs import CASES as BDQ_CASES
from tests.test_gpu_bdq_configs import check_explicit

pytestmark = pytest.mark.gpu


def _batch(cfg, B, seed):
    rng = np.random.default_rng(seed)
    return dict(obs=rng.normal(0.4, 0.2, (B, cfg.obs_dim)).astype(np.float32), next_obs=rng.normal(0.4, 0.2, (B, cfg.obs_dim)).astype(np.float32),
                act_idx=rng.integers(0, cfg.n_bins, (B, cfg.n_branches)), rew=rng.choice([0.0, 1.0], B).astype(np.float32),
                done=(rng.random(B) < 0.2).astype(np.float32))


@pytest.mark.parametrize("cfg,B", [(Q.BDQConfig(100, 3, 8, (64, 64), 32, 32, 0.99), 64),
                                   (Q.BDQConfig(100, 5, 33, (64, 64), 32, 32, 0.99), 64),
                                   (Q.BDQConfig(101, 3, 33, (512, 256), 128, 128, 1.0), 32)]
                         + [pytest.param(c.cfg, c.B, id=c.name) for c in BDQ_CASES])
def test_bdq_step_matches_oracle(cfg, B):
    """Two explicit steps against the float64 oracle (tests/test_gpu_bdq_configs.py::check_explicit): loss, mean_q, td and
    grad_norm within 1e-4 relative, every gradient tensor within 1e-3 (or 3x the fp32 oracle's own error where larger), the
    Adam update element-wise on the GPU's own gradients and against the oracle's update, the second step from the oracle's
    moments, and the hard target copy.  At the three shipped-size configurations and every case of the BDQ matrix."""
    check_explicit(cfg, B)


def test_bdq_front_end_learn_predict_save_load(tmp_path):
    from b200grasp.spaces import Box

    class Env:
        observation_space = Box(-np.inf, np.inf, (100,))
        action_space = Box(-1.0, 1.0, (3,))

        def __init__(self):
            self.rng = np.random.default_rng(0); self.t = 0

        def reset(self):
            self.t = 0
            return self.rng.normal(size=100).astype(np.float32)

        def step(self, a):
            self.t += 1
            return self.rng.normal(size=100).astype(np.float32), float(a[0] > 0), self.t >= 10, {}
    model = b200grasp.BDQ("MlpActPolicy", Env(), policy_kwargs={"layers": [[64, 64], [32], [32]]}, num_actions_pad=8, batch_size=32,
                          buffer_size=500, learning_starts=40, target_network_update_freq=20, seed=1)
    model.learn(100)
    assert model.learner.replay_size() == 100
    a, _ = model.predict(np.zeros(100, np.float32))
    assert a.shape == (3,) and np.all(np.abs(a) <= 1)
    path = str(tmp_path / "bdq")
    model.save(path)
    m2 = b200grasp.BDQ.load(path)
    a2, _ = m2.predict(np.zeros(100, np.float32))
    assert np.array_equal(a, a2)


def test_bdq_prioritized_replay_trees_weights_and_distribution():
    """f4: proportional prioritised replay on device segment trees ([SB2] PrioritizedReplayBuffer semantics: new transitions
    enter with max_priority^alpha; sample ~ p_i / sum; w_i = (N p_i / sum)^-beta / max_w with max_w from the MIN tree;
    update_priorities(sum_d |TD_d| + eps)).  A numpy mirror of the trees is driven by what the device reports and must
    predict the importance weights of the next step exactly; with frozen weights (lr = 0) the slot frequencies follow the
    stationary priorities (chi-square)."""
    cfg = Q.BDQConfig(100, 3, 8, (64, 64), 32, 32, 0.99)
    B, NSLOT, alpha, beta = 64, 200, 0.6, 0.7
    params = Q.init_params(cfg, seed=3)
    L = b200grasp.BDQLearner(cfg.obs_dim, cfg.n_branches, cfg.n_bins, (cfg.trunk, (cfg.branch_hidden,), (cfg.value_hidden,)), batch_size=B,
                             buffer_size=256, gamma=cfg.gamma, target_network_update_freq=10 ** 9, prioritized_replay=True,
                             prioritized_replay_alpha=alpha, prioritized_replay_eps=1e-6, seed=9)
    L.load_parameters(params)
    bt = _batch(cfg, NSLOT, 11)
    bt["rew"] = (bt["rew"] * np.random.default_rng(1).uniform(0.1, 5.0, NSLOT)).astype(np.float32)       # spread of TD errors
    for i in range(0, NSLOT, 70):                                                                         # several adds
        sl = slice(i, min(NSLOT, i + 70))
        L.replay_add(bt["obs"][sl], bt["act_idx"][sl].astype(np.float32), bt["rew"][sl], bt["next_obs"][sl], bt["done"][sl])
    L.set_per_beta(beta)
    prio = np.ones(NSLOT, np.float64)            # raw priorities; leaves hold prio ** alpha
    counts = np.zeros(NSLOT, np.int64)
    stationary_from = None
    for it in range(1500):
        L.step(1, lr=0.0)                        # lr = 0: the networks stay fixed, so every slot's TD error is a constant
        slots, w, newp = L.last_per()
        assert slots.min() >= 0 and slots.max() < NSLOT
        leaves = prio ** alpha
        p = leaves / leaves.sum()
        max_w = (leaves.min() / leaves.sum() * NSLOT) ** (-beta)
        w_ref = (p[slots] * NSLOT) ** (-beta) / max_w
        assert np.abs(w - w_ref).max() <= 2e-5 * max(1.0, w_ref.max()), (it, np.abs(w - w_ref).max())
        assert (newp > 0).all()
        prio[slots] = newp                       # update_priorities; duplicates of a slot carry the same |TD| (lr = 0)
        if stationary_from is None and (prio != 1.0).all() and it > 50:
            stationary_from = it + 1
        elif stationary_from is not None:
            counts += np.bincount(slots, minlength=NSLOT)
    assert stationary_from is not None
    n = counts.sum()
    leaves = prio ** alpha
    expect = n * leaves / leaves.sum()
    chi2 = float(((counts - expect) ** 2 / expect).sum())
    assert abs(chi2 - (NSLOT - 1)) <= 6 * np.sqrt(2 * (NSLOT - 1)), (chi2, NSLOT - 1)
    # priorities are the documented function of the TD errors: replay one slot through the explicit path
    s0 = int(np.argmax(counts))
    one = {k: np.repeat(v[s0:s0 + 1], B, axis=0) for k, v in bt.items()}
    out = L.step_explicit(one["obs"], one["act_idx"].astype(np.float32), one["rew"], one["next_obs"], one["done"], lr=0.0, apply_update=False)
    assert abs(np.abs(out["td"][0]).sum() + 1e-6 - prio[s0]) <= 1e-4 * prio[s0]
    L.close()


def test_bdq_two_rank_data_parallel_matches_oracle_on_concatenated_batch():
    """cfg4: BDQ data parallel -- every rank takes its half of a seeded batch, one NCCL all-reduce averages the gradients,
    the result equals the oracle's step on the concatenated batch and the replicas stay identical."""
    import os, subprocess, sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29541", os.path.join(root, "tests", "multi_gpu_bdq_worker.py")], capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0
