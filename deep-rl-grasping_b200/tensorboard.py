"""TensorBoard event files without tensorflow: what stable-baselines 2.10's ``TensorboardWriter`` gives ``learn`` as
``writer``, written with numpy only.

An event file is a sequence of TFRecord-framed ``Event`` protos: the ``file_version`` record ``brain.Event:2`` first, then
one ``Summary { Value { tag, simple_value } }`` per step.  Each record is framed as ``uint64 length``, the masked CRC32C of
those 8 bytes, the data, the masked CRC32C of the data.  The CRCs of a batch of records (a drained metrics ring) are
computed together, one byte column at a time across all records.

Directories follow ``TensorboardWriter``: ``<tensorboard_log>/<tb_log_name>_<N>``, N = the latest existing run id + 1 for a
new run, the latest id itself when ``learn(..., reset_num_timesteps=False)`` continues one.

Tags and step axis (chosen to follow stable-baselines 2.10; NOT checked against an event file stable-baselines wrote):

* SAC, one summary per gradient step: ``policy_loss``, ``qf1_loss``, ``qf2_loss``, ``value_loss``, ``entropy``,
  ``ent_coef_loss``, ``ent_coef``, ``learning_rate``.
* DQN, one summary per gradient step: ``loss``; besides stable-baselines' names ``mean_q``, ``mean_abs_td_error`` and
  ``grad_norm`` (the device accumulates |td|, so stable-baselines' signed ``td_error`` mean is not logged).
* BDQ, one summary per gradient step: ``loss``, ``mean_q``, ``grad_norm``, ``learning_rate``.
* The x value of a gradient-step summary is ``num_timesteps`` when the step was enqueued (several steps of one
  ``gradient_steps`` batch share it).
* SAC, BDQ, DQN, PPO2, TRPO: ``episode_reward`` per finished episode at ``num_timesteps`` (``total_episode_reward_logger``'s
  rule, which counts the reward of the step that ends an episode into the next one).
* PPO2, one summary per update at ``num_timesteps``: ``loss/policy_gradient_loss``, ``loss/value_function_loss``,
  ``loss/entropy_loss``, ``loss/approximate_kullback-leibler``, ``loss/clip_factor``, ``input_info/learning_rate``,
  ``input_info/clip_range``.
* TRPO, one summary per iteration at ``num_timesteps``: ``policy_gradient_loss`` (optimgain), ``approximate_kullback-leibler``
  (meankl), ``entropy_loss`` (entropy), ``value_function_loss`` (vf_loss).
"""
from __future__ import annotations

import glob
import os
import socket
import struct
import time
import warnings
from typing import Iterable, Optional, Sequence

import numpy as np

__all__ = ["Summary", "EventWriter", "TensorboardWriter", "crc32c", "masked_crc32c", "StepLog", "EpisodeRewardLogger"]


# ------------------------------------------------------------------ CRC32C (Castagnoli, reflected 0x82F63B78)
def _table() -> np.ndarray:
    t = np.arange(256, dtype=np.uint32)
    for _ in range(8):
        t = np.where(t & 1, (t >> 1) ^ np.uint32(0x82F63B78), t >> 1).astype(np.uint32)
    return t


_T = _table()


def crc32c_batch(records: Sequence[bytes]) -> np.ndarray:
    """CRC32C of every record, vectorised across records (one pass per byte column)."""
    n = len(records)
    if n == 0:
        return np.zeros(0, np.uint32)
    lens = np.fromiter((len(r) for r in records), np.int64, n)
    width = int(lens.max()) if n else 0
    buf = np.zeros((n, max(width, 1)), np.uint8)
    for i, r in enumerate(records):
        buf[i, :len(r)] = np.frombuffer(r, np.uint8)
    crc = np.full(n, 0xFFFFFFFF, np.uint32)
    for j in range(width):
        live = lens > j
        nxt = _T[(crc ^ buf[:, j]) & 0xFF] ^ (crc >> 8)
        crc = np.where(live, nxt, crc).astype(np.uint32)
    return crc ^ np.uint32(0xFFFFFFFF)


def crc32c(data: bytes) -> int:
    return int(crc32c_batch([bytes(data)])[0])


def _mask(crc):
    crc = np.asarray(crc, np.uint64)
    return (((crc >> np.uint64(15)) | (crc << np.uint64(17))) + np.uint64(0xA282EAD8)) & np.uint64(0xFFFFFFFF)


def masked_crc32c(data: bytes) -> int:
    """The TFRecord checksum: ((crc >> 15) | (crc << 17)) + 0xa282ead8, mod 2^32."""
    return int(_mask(crc32c(data)))


def frame_records(records: Sequence[bytes]) -> bytes:
    """TFRecord framing of a batch of serialised records, with all checksums computed together."""
    if not records:
        return b""
    heads = [struct.pack("<Q", len(r)) for r in records]
    crcs = _mask(crc32c_batch(heads + list(records)))
    n = len(records)
    out = []
    for i, r in enumerate(records):
        out += [heads[i], struct.pack("<I", int(crcs[i])), r, struct.pack("<I", int(crcs[n + i]))]
    return b"".join(out)


# ------------------------------------------------------------------ protobuf wire format of Event / Summary
def _varint(v: int) -> bytes:
    v &= (1 << 64) - 1
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _len_field(tag: int, payload: bytes) -> bytes:
    return bytes([tag]) + _varint(len(payload)) + payload


def _value_bytes(tag: str, value: float) -> bytes:
    # Summary.Value: 1 tag (string), 2 simple_value (float)
    return _len_field(0x0A, _len_field(0x0A, tag.encode()) + b"\x15" + struct.pack("<f", float(value)))


def event_bytes(wall_time: float, step: Optional[int] = None, values: Iterable = (), file_version: Optional[str] = None) -> bytes:
    """Event: 1 wall_time (double), 2 step (int64), 3 file_version (string), 5 summary (Summary: 1 repeated Value)."""
    out = b"\x09" + struct.pack("<d", wall_time)
    if step is not None:
        out += b"\x10" + _varint(int(step))
    if file_version is not None:
        out += _len_field(0x1A, file_version.encode())
    else:
        out += _len_field(0x2A, b"".join(_value_bytes(t, v) for t, v in values))
    return out


# ------------------------------------------------------------------ tf.Summary stand-in
class Summary:
    """The shape of ``tf.Summary`` that ``add_summary`` reads: ``Summary(value=[Summary.Value(tag=..., simple_value=...)])``.
    A callback written for tensorflow runs unchanged with ``from b200grasp import tensorboard as tf``."""

    class Value:
        def __init__(self, tag: str = "", simple_value: float = 0.0):
            self.tag, self.simple_value = tag, simple_value

    def __init__(self, value=()):
        self.value = list(value)


# ------------------------------------------------------------------ writer
class EventWriter:
    """Appends events to ``<logdir>/events.out.tfevents.<time>.<host>``; the ``writer`` a callback sees in ``locals``.
    Records are encoded as they come and framed in batches of up to ``batch`` records (their checksums computed together),
    at ``flush`` and at ``close``, so a summary per environment step costs its encoding only."""

    batch = 256

    def __init__(self, logdir: str):
        os.makedirs(logdir, exist_ok=True)
        self.logdir = logdir
        base = os.path.join(logdir, "events.out.tfevents.%010d.%s" % (int(time.time()), socket.gethostname()))
        path, k = base, 0
        while os.path.exists(path):          # a continued run in the same second keeps the earlier file
            k += 1
            path = f"{base}.{k}"
        self.path = path
        self._fh = open(path, "wb")
        self._fh.write(frame_records([event_bytes(time.time(), 0, file_version="brain.Event:2")]))
        self._fh.flush()
        self._pending = []

    def _add(self, recs):
        self._pending += recs
        if len(self._pending) >= self.batch:
            self._write()

    def _write(self):
        if self._pending:
            self._fh.write(frame_records(self._pending))
            self._pending = []

    def add_summary(self, summary, global_step=None):
        """``summary.value[i].tag / .simple_value`` (a ``tf.Summary`` or the stand-in) at ``global_step``."""
        vals = [(v.tag, float(v.simple_value)) for v in summary.value]
        self._add([event_bytes(time.time(), global_step, vals)])

    def add_scalars(self, tags: Sequence[str], steps, rows):
        """One event per row: rows[i, k] under tags[k] at steps[i]; the checksums of the batch are computed together."""
        rows = np.asarray(rows, np.float64).reshape(len(steps), len(tags))
        now = time.time()
        tag_b = [_len_field(0x0A, t.encode()) + b"\x15" for t in tags]
        recs = []
        for s, r in zip(np.asarray(steps, np.int64).tolist(), rows.tolist()):
            body = b"".join(_len_field(0x0A, tb + struct.pack("<f", v)) for tb, v in zip(tag_b, r))
            recs.append(b"\x09" + struct.pack("<d", now) + b"\x10" + _varint(s) + _len_field(0x2A, body))
        self._add(recs)

    def flush(self):
        if self._fh:
            self._write()
            self._fh.flush()

    def close(self):
        if self._fh:
            self._write()
            self._fh.close()
            self._fh = None


def latest_run_id(log_path: str, log_name: str) -> int:
    """The largest N of the ``<log_name>_<N>`` directories under log_path (0 when there is none)."""
    best = 0
    for path in glob.glob(os.path.join(glob.escape(log_path), glob.escape(log_name) + "_[0-9]*")):
        name = os.path.basename(path)
        head, _, ext = name.rpartition("_")
        if head == log_name and ext.isdigit() and int(ext) > best:
            best = int(ext)
    return best


class TensorboardWriter:
    """``with TensorboardWriter(tensorboard_log, tb_log_name, new_tb_log) as writer``: an EventWriter in
    ``<tensorboard_log>/<tb_log_name>_<N>`` (N = latest + 1 for a new run, the latest for a continued one), or None when
    tensorboard_log is None."""

    def __init__(self, tensorboard_log: Optional[str], tb_log_name: str, new_tb_log: bool = True):
        self.path, self.name, self.new = tensorboard_log, tb_log_name, new_tb_log
        self.writer = None

    def __enter__(self):
        if self.path is not None:
            n = latest_run_id(self.path, self.name) + (1 if self.new else 0)
            self.writer = EventWriter(os.path.join(self.path, f"{self.name}_{n}"))
        return self.writer

    def __exit__(self, *exc):
        if self.writer is not None:
            self.writer.close()
        return False


# ------------------------------------------------------------------ learner-side helpers
class StepLog:
    """Drains a replay learner's device metrics ring into ``writer``: one summary per gradient step, at the env step each
    step was enqueued at.  ``learn`` calls ``queued(n, x)`` after enqueuing n steps, ``maybe_drain()`` on its way and
    ``drain()`` at its log prints and at its end.  The ring drains once half full, so a run loses no row."""

    def __init__(self, learner, writer, tags: Sequence[str], columns: Sequence[int], capacity: int = 8192):
        self.learner, self.writer, self.tags, self.cols = learner, writer, list(tags), list(columns)
        self.capacity = int(capacity)
        self.pending = []            # env-step x of every gradient step enqueued since the last drain, in order
        self.lost = 0
        self.rows = 0
        learner.metrics_log(self.capacity)

    def queued(self, n: int, x: int):
        self.pending.extend([int(x)] * int(n))
        if len(self.pending) >= self.capacity // 2:
            self.drain()

    def drain(self):
        if not self.pending:
            return
        _, rows, lost = self.learner.metrics_drain(self.capacity)
        xs = self.pending[lost:lost + len(rows)]
        self.pending = self.pending[lost + len(rows):]
        if lost:
            self.lost += lost
            warnings.warn(f"tensorboard: {lost} gradient steps' metrics were overwritten before they were written")
        if len(rows):
            self.writer.add_scalars(self.tags, xs, rows[:, self.cols])
            self.rows += len(rows)
        self.writer.flush()

    def close(self):
        self.drain()
        self.learner.metrics_log(0)


class EpisodeRewardLogger:
    """stable-baselines' ``total_episode_reward_logger`` for one env step of n envs: an env whose episode ended writes its
    accumulated reward as ``episode_reward`` at x = steps; the ending step's reward opens the next accumulation."""

    def __init__(self, n_envs: int):
        self.acc = np.zeros(n_envs)
        self.count = 0

    def __call__(self, writer, rewards, dones, steps: int):
        rewards = np.asarray(rewards, np.float64).reshape(-1)
        dones = np.asarray(dones).reshape(-1)
        for i in range(len(rewards)):
            if dones[i]:
                writer.add_summary(Summary([Summary.Value("episode_reward", float(self.acc[i]))]), int(steps))
                self.count += 1
                self.acc[i] = rewards[i]
            else:
                self.acc[i] += rewards[i]
