"""Device timeline of one SAC graph step in bench.py's configuration (depth CNN, 64x64x2, batch 256, bf16x3, one GPU).

  python tools/step_timeline.py [--steps 6] [--batch 256] [--out DIR]
  python tools/step_timeline.py --trace DIR/step_timeline.pt.trace.json      (re-reads a saved trace; no GPU needed)

Traces a few back-to-back graph replays of `Learner.step` with torch.profiler (CUDA activities) and prints, for the middle
replay, every kernel and memset with its start and end in microseconds from the step's first node, its stream and grid, and then:
  * the gap from the end of the gather to the start of the forward cg_kernel launch;
  * every node that runs while a cg_kernel launch starts (running at its start, or starting within --window us of it);
  * every pair of nodes that overlap, with the overlap in microseconds.
A closing line gives the median step length and gather -> fwd_fused gap over all traced replays. --out DIR also writes the
chrome trace there.  Needs a GPU; the numbers are only meaningful without other work on the device.
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
LR = 3e-4


def short(name):
    """Kernel name without template arguments and parameter lists: planes2_kernel, gather2_kernel, cg_kernel, ..."""
    n = name.replace("(anonymous namespace)::", "").split("(")[0].split("<")[0]
    return n.split("::")[-1].replace("void ", "").strip()


def device_nodes(trace):
    out = []
    for e in trace.get("traceEvents", []):
        if e.get("ph") != "X" or e.get("cat") not in ("kernel", "gpu_memset"):      # (the copies are the API calls' own)
            continue
        a = e.get("args", {})
        name = short(e["name"]) if e["cat"] == "kernel" else "memset"
        if name.startswith("memset"):          # memset nodes of a graph run as kernels named memset32 / memset8 ...
            name = "memset"
        out.append(dict(name=name, t0=float(e["ts"]), t1=float(e["ts"]) + float(e["dur"]), stream=a.get("stream"),
                        grid=a.get("grid"), bytes=a.get("bytes")))
    out.sort(key=lambda d: d["t0"])
    return out


def split_steps(nodes):
    """Graph replays on one stream run one after the other; the optimiser kernel is the last node of every step."""
    steps, cur = [], []
    for d in nodes:
        cur.append(d)
        if d["name"] in ("optim_kernel", "dp_optim_kernel"):
            steps.append(cur)
            cur = []
    return steps


def label(step):
    """Names the two fused launches and numbers repeated kernels in start order (planes2_kernel#0, #1, ...)."""
    seen = {}
    for d in step:
        k = d["name"]
        i = seen.get(k, 0)
        seen[k] = i + 1
        if k == "cg_kernel":
            d["label"] = ("fwd_fused", "bwd_fused")[i] if i < 2 else f"cg_kernel#{i}"
        else:
            d["label"] = k if k not in ("planes2_kernel", "memset") else f"{k}#{i}"
    return step


def first(step, name):
    return next((d for d in step if d["label"] == name or d["name"] == name), None)


def report(step, window):
    t00 = min(d["t0"] for d in step)
    lines = [f"{'node':<22} {'start':>8} {'end':>8} {'dur':>7}  stream  grid / bytes"]
    for d in step:
        extra = d["grid"] if d["grid"] is not None else (f"{d['bytes']} B" if d["bytes"] is not None else "")
        lines.append(f"{d['label']:<22} {d['t0'] - t00:8.1f} {d['t1'] - t00:8.1f} {d['t1'] - d['t0']:7.1f}  {str(d['stream']):>6}  {extra}")
    g, f = first(step, "gather2_kernel"), first(step, "fwd_fused")
    if g and f:
        lines.append(f"gather end -> fwd_fused start: {f['t0'] - g['t1']:+.1f} us")
    for cg in (d for d in step if d["name"] == "cg_kernel"):
        busy = [d for d in step if d is not cg and d["t0"] < cg["t0"] + window and d["t1"] > cg["t0"]]
        lines.append(f"running while {cg['label']} starts (+{window:g} us): " +
                     (", ".join(f"{d['label']} [{d['t0'] - t00:.1f}, {d['t1'] - t00:.1f}]" for d in busy) if busy else "none"))
    lines.append("overlapping pairs (us):")
    for i, a in enumerate(step):
        for b in step[i + 1:]:
            ov = min(a["t1"], b["t1"]) - max(a["t0"], b["t0"])
            if ov > 0:
                lines.append(f"  {a['label']:<22} {b['label']:<22} {ov:7.1f}")
    return "\n".join(lines)


def summarise(trace, window):
    steps = [label(s) for s in split_steps(device_nodes(trace))]
    if not steps:
        raise SystemExit("no step found in the trace (no optim_kernel)")
    print(f"{len(steps)} steps traced; step {len(steps) // 2}:")
    print(report(steps[len(steps) // 2], window))
    lens = [s[-1]["t1"] - min(d["t0"] for d in s) for s in steps]
    gaps = [first(s, "fwd_fused")["t0"] - first(s, "gather2_kernel")["t1"] for s in steps
            if first(s, "fwd_fused") and first(s, "gather2_kernel")]
    print(f"median over {len(steps)} steps: step {np.median(lens):.1f} us (first node to optimiser end), "
          f"gather end -> fwd_fused start {np.median(gaps) if gaps else float('nan'):+.1f} us")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6, help="graph replays traced (after a warm-up outside the trace)")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--replay-filled", type=int, default=65536)
    ap.add_argument("--buffer-size", type=int, default=1_000_000)
    ap.add_argument("--window", type=float, default=5.0, help="us after a cg_kernel start in which another node counts as co-resident")
    ap.add_argument("--out", default=None, help="directory for the chrome trace (default: a temporary directory, removed)")
    ap.add_argument("--trace", default=None, help="report on a chrome trace this tool wrote earlier instead of running")
    args = ap.parse_args()
    if args.trace:
        with open(args.trace) as fh:
            summarise(json.load(fh), args.window)
        return

    import torch
    from torch.profiler import ProfilerActivity, profile
    import b200grasp
    from b200grasp import synth

    if not torch.cuda.is_available():
        raise SystemExit("step_timeline.py needs a GPU")
    vn = dict(np.load(os.path.join(GOLD, "vecnorm_sac_depth.npz")))
    params = dict(np.load(os.path.join(GOLD, "sac_depth_params.npz")))
    L = b200grasp.Learner((64, 64, 2), n_act=5, batch_size=args.batch, buffer_size=args.buffer_size, seed=1234, precision=1)
    L.load_parameters(params)
    L.set_norm_stats(vn["obs_mean"], vn["obs_var"], float(vn["ret_var"]), float(vn["clip_obs"]), float(vn["clip_reward"]),
                     float(vn["epsilon"]))
    chunk, i = 2048, 0
    cache = []
    while i < args.replay_filled:
        k = (i // chunk) % 8
        if k >= len(cache):
            cache.append(synth.make_transitions(chunk, vn["obs_mean"], vn["obs_var"], seed=synth.DATA_SEED + k))
        n = min(chunk, args.replay_filled - i)
        tr = cache[k]
        L.replay_add(tr["obs"][:n], tr["act"][:n], tr["rew"][:n], tr["next_obs"][:n], tr["done"][:n])
        i += n
    L.step(20, lr=LR)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        L.step(args.steps, lr=LR)              # back-to-back graph replays, as bench.py times them
        torch.cuda.synchronize()
    out_dir = args.out or tempfile.mkdtemp(prefix="step_timeline_")
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "step_timeline.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as fh:
        trace = json.load(fh)
    if not args.out:
        os.remove(path)
        os.rmdir(out_dir)
    L.close()
    summarise(trace, args.window)


if __name__ == "__main__":
    main()
