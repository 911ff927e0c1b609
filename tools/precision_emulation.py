"""CPU emulation of the tensor engine's split-precision arithmetic on the REAL SAC step (oracle/sac_ref_np.py with every
matmul replaced), used to decide which operand split each contraction needs.

Every matmul operand is split into `n` BF16 (or scaled FP16) terms; the chosen products are summed in float64, i.e. with an
IDEAL accumulator, so what is measured is the operand split alone.  FWD / BWD select the mode of the forward and the
backward contractions separately.  The batch is the one the device drew in tests/test_gpu_graph_path.py
(gpurun_out/diag_batch.npz from tools/diag_gradnorm.py) when present, else a seeded one."""
import os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import sac_ref_np as N
from tests.util import load_case, rel_err
from tests.test_gpu_graph_path import _norm_batch
from b200grasp import synth

MODE = None


def rnd(x, kind):
    t = torch.from_numpy(np.asarray(x, np.float64)).float()
    return (t.bfloat16() if kind == "bf16" else t.half()).double().numpy()


def split(x, kind, n):
    parts, r = [], np.asarray(x, np.float64).astype(np.float32).astype(np.float64)   # operands are fp32 on the GPU
    for _ in range(n):
        h = rnd(r, kind); parts.append(h); r = r - h
    return parts


def mm(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if MODE is None:
        return a @ b
    kind, n, terms = MODE
    sa = sb = 1.0
    if kind == "fp16":      # per-tensor power-of-two scaling into the fp16 range
        sa = 2.0 ** np.floor(np.log2(8192.0 / max(np.abs(a).max(), 1e-30))); sb = 2.0 ** np.floor(np.log2(8192.0 / max(np.abs(b).max(), 1e-30)))
    pa, pb = split(a * sa, kind, n), split(b * sb, kind, n)
    return sum(pa[i] @ pb[j] for i, j in terms) / (sa * sb)


class SA(np.ndarray):
    def __matmul__(self, o): return mm(self.view(np.ndarray), np.asarray(o).view(np.ndarray)).view(SA)
    def __rmatmul__(self, o): return mm(np.asarray(o).view(np.ndarray), self.view(np.ndarray)).view(SA)


class FakeNP:
    def __getattr__(self, k): return getattr(np, k)
    def asarray(self, a, *args, **kw): return np.asarray(a, *args, **kw).view(SA)
    def ascontiguousarray(self, a, *args, **kw): return np.ascontiguousarray(a, *args, **kw).view(SA)


N.np = FakeNP()
FWD = BWD = None
_mb, _cb = N.mlp_bwd, N.cnn_bwd


def _wrap(fn):
    def w(*a, **k):
        global MODE
        MODE = BWD
        r = fn(*a, **k)
        MODE = FWD
        return r
    return w


N.mlp_bwd, N.cnn_bwd = _wrap(_mb), _wrap(_cb)

cfg, params, vn = load_case("sac_depth")
B = 256
tr = synth.make_transitions(4096, vn["obs_mean"], vn["obs_var"], seed=9001)
dpath = os.path.join(ROOT, "gpurun_out", "diag_batch.npz")
if os.path.exists(dpath):
    d = np.load(dpath); idx, eps = d["idx"], d["eps"]
else:
    idx, eps = np.random.default_rng(1).integers(0, 4096, B), synth.make_eps(B, seed=5)
norm = _norm_batch(tr, idx, vn)
ref, g64 = N.sac_grads(params, norm, eps, cfg)
gn = lambda gg, pre: np.sqrt(sum(float((np.asarray(gg[n], np.float64) ** 2).sum()) for n in gg if n.startswith(pre)))


def run(f, b, label):
    global FWD, BWD, MODE
    FWD, BWD, MODE = f, b, f
    p = {n: np.asarray(a, np.float64).view(SA) for n, a in params.items()}
    nb = {k: np.asarray(v, np.float64).view(SA) for k, v in norm.items()}
    out, g = N.sac_grads(p, nb, eps, cfg)
    MODE = None
    worst = max(rel_err(np.asarray(g[n]), g64[n]) for n in g64 if g64[n].size > 64)
    print(f"{label:46s} gn_pi {abs(gn(g,'model/pi/')-gn(g64,'model/pi/'))/gn(g64,'model/pi/'):.2e}  gn_v "
          f"{abs(gn(g,'model/values_fn/')-gn(g64,'model/values_fn/'))/gn(g64,'model/values_fn/'):.2e}  q1 {rel_err(out['q1'], ref['q1']):.1e}  "
          f"logp {rel_err(out['logp'], ref['logp']):.1e}  worst tensor {worst:.1e}", flush=True)


B2 = ("bf16", 2, [(0, 0), (0, 1), (1, 0)])
B5 = ("bf16", 3, [(0, 0), (0, 1), (1, 0), (0, 2), (2, 0)])
B6 = ("bf16", 3, [(0, 0), (0, 1), (1, 0), (1, 1), (0, 2), (2, 0)])
F2 = ("fp16", 2, [(0, 0), (0, 1), (1, 0)])
run(B2, B2, "fwd 2-plane bf16 (3 products) | bwd same")
run(B2, None, "fwd 2-plane bf16           | bwd exact")
run(None, B2, "fwd exact                  | bwd 2-plane bf16")
run(B6, B2, "fwd 3-plane bf16 (6 prod.)   | bwd 2-plane  [shipped]")
run(B5, B2, "fwd 3-plane bf16 (5 prod.)   | bwd 2-plane")
run(B6, B6, "fwd 3-plane bf16 (6 prod.)   | bwd same")
run(F2, F2, "fwd/bwd scaled fp16 2-plane (3 products)")
