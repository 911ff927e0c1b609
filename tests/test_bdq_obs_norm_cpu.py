"""BDQ's device observation statistics without a GPU: the Philox stream-3 restatement the epsilon-greedy actor draws from
(``explore`` below, on the Philox4x32-10 of oracle/philox_ref.py), the exported entry points, and the refusals made before a
handle exists."""
import numpy as np
import pytest

from b200grasp import _lib
from oracle import philox_ref as PX

STREAM_EXPLORE = 3


def explore(key, step, n_env, n_branches, n_bins, eps):
    """Stream 3 of one acting b2g_bdq_observe_act call (csrc/bdq.cu bdq_explore_kernel): counter (step low word, step high
    word, env * n_branches + branch, 3) under the training key, step = counters[7] (the number of earlier acting calls).  Lane
    x explores when (x + 0.5) 2^-32 < eps (float64 of the fp32 eps), lane y gives the bin (y * n_bins) >> 32.
    -> (explore [n_env, n_branches] bool, random bin [n_env, n_branches] int64)."""
    step = int(step)
    blk = np.arange(n_env * n_branches, dtype=np.uint64)
    x, y, _, _ = PX.philox4x32_10(step & 0xFFFFFFFF, step >> 32, blk, STREAM_EXPLORE, key & 0xFFFFFFFF, key >> 32)
    go = (x.astype(np.float64) + 0.5) * (1.0 / 4294967296.0) < float(np.float32(eps))
    bins = (y.astype(np.uint64) * np.uint64(n_bins)) >> np.uint64(32)
    return go.reshape(n_env, n_branches), bins.astype(np.int64).reshape(n_env, n_branches)


def test_stream3_layout():
    """Block env * n_branches + branch at the call's step: lane x decides against eps, lane y picks the bin."""
    key, step, n_env, D, n = PX.train_seed(9), (1 << 32) + 3, 5, 3, 33
    go, bins = explore(key, step, n_env, D, n, 0.3)
    for e in range(n_env):
        for d in range(D):
            r = PX.philox4x32_10(step & 0xFFFFFFFF, step >> 32, e * D + d, 3, key & 0xFFFFFFFF, key >> 32)
            assert go[e, d] == ((int(r[0]) + 0.5) / 2 ** 32 < float(np.float32(0.3)))
            assert bins[e, d] == (int(r[1]) * n) >> 32
    assert explore(key, step, n_env, D, n, 0.0)[0].sum() == 0
    assert explore(key, step, n_env, D, n, 1.0)[0].all()
    # the next step: other words
    assert not np.array_equal(explore(key, step + 1, n_env, D, n, 0.5)[1], bins)


def test_stream3_is_uniform_and_independent():
    """2^18 (env, branch) draws over 16 calls: the exploration rate is eps within 5 sigma, the bins pass a chi-square test at
    n_bins = 33 and 2, and the decision does not correlate with the bin or with the neighbouring branch."""
    from scipy import stats
    key, eps = PX.train_seed(4), 0.3
    go, bins = zip(*[explore(key, s, 4096, 4, 33, eps) for s in range(16)])
    go, bins = np.concatenate(go).reshape(-1), np.concatenate(bins).reshape(-1)
    n = go.size
    assert abs(go.mean() - eps) <= 5 * np.sqrt(eps * (1 - eps) / n), go.mean()
    assert bins.min() == 0 and bins.max() == 32
    chi = stats.chisquare(np.bincount(bins, minlength=33))
    assert chi.pvalue > 1e-4, chi
    two = explore(key, 99, 1 << 16, 1, 2, eps)[1].reshape(-1)
    assert abs(two.mean() - 0.5) <= 5 * 0.5 / np.sqrt(two.size)
    for a, b in ((go.astype(float), bins.astype(float)), (go[:-1].astype(float), go[1:].astype(float))):
        rho = np.corrcoef(a, b)[0, 1]
        assert abs(rho) <= 5 / np.sqrt(n), rho


def test_entry_points_are_exported():
    lib = _lib.load()
    for name in ("b2g_bdq_observe_act", "b2g_bdq_observe_add", "b2g_bdq_obs_rms_set", "b2g_bdq_obs_rms_get", "b2g_bdq_upload_bytes"):
        assert name in _lib.SYMBOLS and hasattr(lib, name), name


def test_data_parallel_refused_before_any_device_work():
    from b200grasp import BDQ
    with pytest.raises(NotImplementedError, match="nranks > 1"):
        BDQ("MlpActPolicy", None, device_obs_norm=True, nranks=2)


def test_cli_passes_device_norm_to_bdq():
    import inspect
    from b200grasp import train_cli
    src = inspect.getsource(train_cli.train)
    bdq = src[src.index('elif algo == "BDQ"'):]
    assert "device_obs_norm=bool(args.device_norm)" in bdq[:bdq.index("else:")]
