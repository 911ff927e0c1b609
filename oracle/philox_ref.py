"""numpy restatement of the device random streams (TEST INFRASTRUCTURE ONLY, see ``oracle/__init__.py``).

Both learners draw from Philox4x32-10 (Salmon et al., SC'11; csrc/common.cuh ``philox4x32_10``).  A draw is the counter
(c0, c1, c2, c3) = (step low word, step high word, block, stream) under the key (seed low word, seed high word):

  stream 0  replay slots (prep_kernel, and philox_slot in gather_kernel / gather2_kernel): sample b takes element b & 3 of
            block b >> 2 and scales it to (v * size) >> 32; SAC then maps it into the ring, (counters[6] + u) mod capacity.
  stream 1  policy noise (prep_kernel): block i gives four samples 4i .. 4i + 3 of the flattened [B, A] noise by Box-Muller,
            u01(x) = ((x >> 8) + 0.5) 2^-24 (in fp32: see u01), r = sqrt(-2 log u01(x)), (r.x, r.y) -> (r0 cos 2 pi u01(r.y),
            r0 sin ...), and (r.z, r.w) likewise.
  stream 2  prioritised-replay masses (bdq.cu per_sample_kernel): (v + 0.5) 2^-32 tsum[1] in float64, v as for stream 0.

Keys.  Training steps use seed + 0x9E3779B97F4A7C15 * rank (mod 2^64); SAC's act() uses seed XOR 0xA5A5A5A5DEADBEEF.

The step word is the device counter counters[4], which every drawing step advances by one.  Which value a kernel sees:
  * prep_kernel reads counters[4] before it advances it (SAC act(deterministic=False) and every sampled step draw at the
    value the counter held when the call began);
  * SAC's graph path with the forked leaf branch (engine v2 and the round-1 gather) defers the advance to the optimiser
    kernel at the end of the step, so the in-kernel slot draw of the gather sees the same value prep_kernel sees;
  * BDQ's per_sample_kernel runs after prep_kernel has advanced the counter, so its masses use counters[4] + 1 of the
    step's uniform draw; the k-th sampled BDQ step (from 0) draws its uniform slots at k and its PER masses at k + 1.
"""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK32 = np.uint64(0xFFFFFFFF)
RANK_STRIDE = 0x9E3779B97F4A7C15
ACT_SEED_XOR = 0xA5A5A5A5DEADBEEF
STREAM_SLOTS, STREAM_NOISE, STREAM_PER = 0, 1, 2


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 of counters (c0..c3) under key (k0, k1), elementwise over broadcastable arrays -> four uint32 arrays."""
    c = [np.asarray(x, np.uint64) & MASK32 for x in np.broadcast_arrays(c0, c1, c2, c3)]
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]                       # < 2^64: exact in uint64
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & MASK32, p1 >> np.uint64(32), p1 & MASK32
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return tuple(x.astype(np.uint32) for x in c)


def train_seed(seed, rank=0):
    return (int(seed) + RANK_STRIDE * int(rank)) & 0xFFFFFFFFFFFFFFFF


def act_seed(seed):
    return (int(seed) ^ ACT_SEED_XOR) & 0xFFFFFFFFFFFFFFFF


def _blocks(key, step, n_blocks, stream):
    step = int(step)
    i = np.arange(n_blocks, dtype=np.uint64)
    r = philox4x32_10(step & 0xFFFFFFFF, step >> 32, i, stream, key & 0xFFFFFFFF, key >> 32)
    return np.stack(r, 1).reshape(-1)                      # element 4i + j is lane j of block i


def uniform_u32(key, step, n, stream):
    """The n words of `stream` at `step`: word b is lane b & 3 of block b >> 2."""
    return _blocks(key, step, (n + 3) // 4, stream)[:n]


def slots(key, step, B, size, ring_base=0, ring_cap=0):
    """Replay slots of stream 0: (v * size) >> 32, then (ring_base + u) mod ring_cap when ring_cap > 0."""
    u = ((uniform_u32(key, step, B, STREAM_SLOTS).astype(np.uint64) * np.uint64(size)) >> np.uint64(32)).astype(np.int64)
    return (ring_base + u) % ring_cap if ring_cap > 0 else u


def u01(x):
    """((x >> 8) + 0.5) 2^-24 in fp32 arithmetic, as the device forms it: for x >> 8 >= 2^23 the sum needs 25 bits and rounds
    to even, so the top half of the range lands on multiples of 2^-24, 1.0 included.  -> float64 of those fp32 values."""
    k = (np.asarray(x, np.uint32) >> np.uint32(8)).astype(np.float32)
    return ((k + np.float32(0.5)) * np.float32(2.0 ** -24)).astype(np.float64)


def noise(key, step, n):
    """The first n values of stream 1 in float64 (the device evaluates the same formula in fp32: logf, sqrtf, sincospif)."""
    r = _blocks(key, step, (n + 3) // 4, STREAM_NOISE).reshape(-1, 4)
    r0, r1 = np.sqrt(-2.0 * np.log(u01(r[:, 0]))), np.sqrt(-2.0 * np.log(u01(r[:, 2])))
    a0, a1 = 2.0 * np.pi * u01(r[:, 1]), 2.0 * np.pi * u01(r[:, 3])
    z = np.stack([r0 * np.cos(a0), r0 * np.sin(a0), r1 * np.cos(a1), r1 * np.sin(a1)], 1)
    return z.reshape(-1)[:n]


def per_masses(key, step, B, total):
    """Stream-2 masses (v + 0.5) 2^-32 total, float64, as per_sample_kernel forms them."""
    return (uniform_u32(key, step, B, STREAM_PER).astype(np.float64) + 0.5) * (1.0 / 4294967296.0) * total
