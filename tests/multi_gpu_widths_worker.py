"""2-rank peer-memory data-parallel worker for 128-wide SAC heads (launched by tests/test_sac_widths.py):
   python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29531 tests/multi_gpu_widths_worker.py

Each rank takes its half of a seeded 2B batch (bf16x3 depth policy, fresh init, layers [128, 128]); the optimiser launch
reduces the gradients over NVLink peer memory and writes the updated parameters into both replicas.  The replicas must be
bit-identical afterwards and the update must equal the float64 oracle's single step on the concatenated batch."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import b200grasp  # noqa: E402
from oracle import sac_ref as R  # noqa: E402
from tests.util import make_batch, rel_err  # noqa: E402

H = 128


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    ids = [b200grasp.Learner.nccl_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, 0)
    vn = dict(np.load(os.path.join(ROOT, "tests", "golden", "vecnorm_sac_depth.npz")))
    cfg = R.SACConfig(obs_shape=(64, 64, 2), layers=(H, H))
    params = R.init_params(cfg, seed=61)
    B = 24
    raw, norm, eps = make_batch(vn, B * world)
    L = b200grasp.Learner(cfg.obs_shape, n_act=cfg.n_act, hidden=H, batch_size=B, buffer_size=64, device=local, rank=rank,
                          nranks=world, nccl_id=ids[0], precision=1)
    L.set_norm_stats(vn["obs_mean"], vn["obs_var"], float(vn["ret_var"]), float(vn["clip_obs"]), float(vn["clip_reward"]),
                     float(vn["epsilon"]))
    L.dp_connect_torch()
    L.load_parameters(params)
    sl = slice(rank * B, (rank + 1) * B)
    out = L.step_explicit(raw["obs"][sl], raw["act"][sl], raw["rew"][sl], raw["next_obs"][sl], raw["done"][sl], eps[sl], lr=3e-4)
    ref, grads, newp, _ = R.sac_step(params, R.OptState.zeros(params), norm, eps, 3e-4, cfg, torch.float64)
    ref32, _, _, _ = R.sac_step(params, R.OptState.zeros(params), norm, eps, 3e-4, cfg, torch.float32)
    # bars of tests/test_sac_widths.py: 1e-4 against float64, or 3x the fp32 oracle's own distance from float64 where fp32
    # arithmetic does not resolve 1e-4
    keys = ("policy_loss", "qf1_loss", "qf2_loss", "value_loss", "grad_norm_pi", "grad_norm_values")
    errs = {k: abs(out[k] - float(ref[k])) / abs(float(ref[k])) for k in keys}
    bars = {k: max(1e-4, 3 * abs(float(ref32[k]) - float(ref[k])) / abs(float(ref[k]))) for k in keys}
    # the first Adam step is sign-like: compare the update every entry received where the gradient is not ~0
    newd = L.get_parameters()
    upd_ref = np.concatenate([(np.asarray(newp[n], np.float64) - np.asarray(params[n], np.float64)).reshape(-1) for n in grads])
    upd_dev = np.concatenate([(newd[n].astype(np.float64) - np.asarray(params[n], np.float64)).reshape(-1) for n in grads])
    big = np.concatenate([np.abs(np.asarray(grads[n], np.float64)).reshape(-1) for n in grads]) > 1e-7
    gerr = float(np.linalg.norm((upd_dev - upd_ref)[big]) / np.linalg.norm(upd_ref[big]))
    mine = np.concatenate([a.reshape(-1) for a in newd.values()])
    allp = [None] * world
    dist.all_gather_object(allp, mine.tobytes())
    same = all(b == allp[0] for b in allp)
    q_err = rel_err(out["q1"], np.asarray(ref["q1"]).reshape(-1)[sl])
    q_bar = max(1e-4, 3 * rel_err(np.asarray(ref32["q1"]).reshape(-1)[sl], np.asarray(ref["q1"]).reshape(-1)[sl]))
    print(f"rank {rank}: H={H} err/bar {({k: round(errs[k] / bars[k], 3) for k in keys})} update-err {gerr:.2e} "
          f"q1 {q_err:.2e} (bar {q_bar:.2e}) replicas_identical {same}", flush=True)
    ok = all(errs[k] <= bars[k] for k in keys) and gerr <= 1e-3 and same and q_err <= q_bar
    L.close()
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
