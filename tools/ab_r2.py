"""A/B of the design switches and precision modes on the benchmark workload (depth CNN, B=256, bf16x3, CUDA-graph step), one subprocess per
setting so that every switch is read at create time:   python tools/ab_r2.py > ab_r2.txt"""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r'''
import os, sys, numpy as np
sys.path.insert(0, %r)
import b200grasp
from b200grasp import synth
GOLD = os.path.join(%r, "tests", "golden")
vn = dict(np.load(os.path.join(GOLD, "vecnorm_sac_depth.npz")))
params = dict(np.load(os.path.join(GOLD, "sac_depth_params.npz")))
L = b200grasp.Learner((64, 64, 2), n_act=5, batch_size=256, buffer_size=8192, seed=1, precision=int(os.environ.get("PREC", "1")))
L.load_parameters(params)
L.set_norm_stats(vn["obs_mean"], vn["obs_var"], float(vn["ret_var"]), float(vn["clip_obs"]), float(vn["clip_reward"]), float(vn["epsilon"]))
for i in range(4):
    tr = synth.make_transitions(2048, vn["obs_mean"], vn["obs_var"], seed=1 + i)
    L.replay_add(tr["obs"], tr["act"], tr["rew"], tr["next_obs"], tr["done"])
L.step(20)
ms = []
for _ in range(5):
    L.step(100); ms.append(L.last_step_ms() / 100)
print("%%.1f us/step, %%d kernels/step" %% (float(np.median(ms)) * 1e3, L.launches_per_step()))
L.close()
''' % (ROOT, ROOT)
VARIANTS = [("default (TMA engine, fused launches, epilogue bias sums, CUDA-core head wgrads)", {}),
            ("B2G_FORK=0 (single-branch graph)", {"B2G_FORK": "0"}),
            ("precision fp32 (FFMA engine)", {"PREC": "0"}),
            ("precision bf16 single pass (fast mode, not a parity mode)", {"PREC": "2"})]
for name, env in VARIANTS:
    r = subprocess.run([sys.executable, "-c", CHILD], env=dict(os.environ, **env), capture_output=True, text=True, timeout=300)
    print(f"{name:90s} {r.stdout.strip() or ('FAILED: ' + r.stderr.strip().splitlines()[-1] if r.stderr.strip() else 'FAILED')}", flush=True)
