"""Throughput of the SAC gradient step against the head width H (SAC.layers = [H, H], H = 64, 128, 192, 256) on one GPU.

Depth CNN policy (64x64x2, 5 actions), batch 256, bf16x3 (engine v2), CUDA-graph steps drawn from a device replay of
--replay-filled seeded transitions; fresh parameters (oracle.sac_ref.init_params) at every width.  Per width it prints
  * graph-path steps/s: the median over --regions timed regions of b2g_sac_step calls (CUDA events on the learner's stream,
    as bench.py times `value`);
  * the serial per-launch times of one step (b2g_profile_step: events between the launches, leaf branch folded onto the
    main stream), median over --profiles calls, for the head tail, heads_wgrad and the two fused cg_kernel launches;
  * the algorithmic FLOPs of one step, from shapes: the convolutions, cnn_fc1, the head fc0 / fc1 layers forward and
    backward (the H x A and H x 1 output layers are left out: < 0.1 %).
The card's name and power limit are read in the same run and printed first.

    python tools/sac_width_bench.py [--widths 64 128 192 256] [--steps 210] [--regions 7]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
LR = 3e-4
PROFILED = ("fwd_fused", "heads_tail", "heads_wgrad", "bwd_fused")


def step_flops(H, B=256, c_img=1, n_act=5):
    """Algorithmic FLOPs (2 x MAC) of one SAC step of the depth CNN policy with [H, H] heads."""
    fd = 512 + 1
    # (output rows per sample, reduction depth, output width) of conv1, conv2, conv3, cnn_fc1
    layers = [(225, 64 * c_img, 32), (36, 512, 64), (16, 576, 64), (1, 1024, 512)]
    fwd = sum(r * k * n for r, k, n in layers)
    mac = 3 * fwd                                             # pi, values, target CNNs forward
    mac += 2 * (2 * fwd - 225 * 64 * c_img * 32)              # pi, values backward: dgrad + wgrad, conv1 has no dgrad
    mac += (3 * fd + 2 * (fd + n_act)) * H                    # fc0 forward: pi, vf, target vf, qf1, qf2
    mac += (2 * fd + 2 * (fd + n_act)) * H + 4 * 512 * H      # fc0 wgrad of the four trained heads, dgrad into the features
    mac += 12 * H * H + 4 * H * H                             # fc1: the tail's 12 mat-vecs, the four kernel gradients
    return 2.0 * mac * B


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--widths", type=int, nargs="+", default=[64, 128, 192, 256])
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=210, help="timed steps per width, split into --regions regions")
    ap.add_argument("--regions", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--profiles", type=int, default=5)
    ap.add_argument("--replay-filled", type=int, default=16384)
    args = ap.parse_args()

    import torch
    import b200grasp
    from b200grasp import synth
    from oracle import sac_ref as R

    if not torch.cuda.is_available():
        raise SystemExit("sac_width_bench: no CUDA device (this measures the GPU; there is nothing to time without one)")
    print(json.dumps({"card": card()}), flush=True)
    vn = dict(np.load(os.path.join(GOLD, "vecnorm_sac_depth.npz")))
    tr = synth.make_transitions(2048, vn["obs_mean"], vn["obs_var"], seed=synth.DATA_SEED)
    B = args.batch
    per_region = [args.steps // args.regions + (1 if i < args.steps % args.regions else 0) for i in range(args.regions)]
    rows = []
    for H in args.widths:
        cfg = R.SACConfig(obs_shape=(64, 64, 2), layers=(H, H))
        L = b200grasp.Learner((64, 64, 2), n_act=5, hidden=H, batch_size=B, buffer_size=max(args.replay_filled, B), seed=1234,
                              precision=1)
        L.load_parameters(R.init_params(cfg, seed=5))
        L.set_norm_stats(vn["obs_mean"], vn["obs_var"], float(vn["ret_var"]), float(vn["clip_obs"]), float(vn["clip_reward"]),
                         float(vn["epsilon"]))
        for i in range(0, args.replay_filled, len(tr["rew"])):
            n = min(len(tr["rew"]), args.replay_filled - i)
            L.replay_add(tr["obs"][:n], tr["act"][:n], tr["rew"][:n], tr["next_obs"][:n], tr["done"][:n])
        L.step(args.warmup, lr=LR)
        torch.cuda.synchronize()
        ms_per_step = []
        for k in per_region:
            m = L.step(k, lr=LR)
            ms_per_step.append(L.last_step_ms() / k)
        assert np.isfinite(m["qf1_loss"]) and np.isfinite(m["policy_loss"]), m
        prof = [L.profile_step(lr=LR) for _ in range(args.profiles)]
        launch_ms = {name: float(np.median([p[name] for p in prof])) for name in PROFILED if name in prof[0]}
        L.close()
        ms = float(np.median(ms_per_step))
        fl = step_flops(H, B)
        row = {"H": H, "B": B, "steps_per_s": round(1e3 / ms, 1), "ms_per_step": round(ms, 4),
               "regions_ms_per_step": [round(x, 4) for x in ms_per_step], "serial_launch_ms": {k: round(v, 4) for k, v in launch_ms.items()},
               "algorithmic_gflop_per_step": round(fl / 1e9, 3), "achieved_tflops": round(fl / (ms * 1e-3) / 1e12, 2)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    print(f"{'H':>4} {'steps/s':>9} {'ms/step':>8} {'GFLOP/step':>11} {'TFLOP/s':>8}  " + "  ".join(f"{n:>11}" for n in PROFILED))
    for r in rows:
        print(f"{r['H']:>4} {r['steps_per_s']:>9} {r['ms_per_step']:>8} {r['algorithmic_gflop_per_step']:>11} {r['achieved_tflops']:>8}  "
              + "  ".join(f"{r['serial_launch_ms'].get(n, float('nan')):>11.4f}" for n in PROFILED))


if __name__ == "__main__":
    main()
