"""Minimal HDF5 reader for Keras 2.2.4 weight files (h5py is not a dependency).

Handles exactly what ``keras.Model.save_weights`` / ``model.save`` produced for
/root/reference/encoder_files/*/model.h5: superblock version 0, version-1 object headers, groups as
symbol tables (B-tree ``TREE`` nodes + ``SNOD`` symbol nodes + local heaps), little-endian IEEE float
datasets with CONTIGUOUS layout.  Anything else raises ``NotImplementedError``.
"""
from __future__ import annotations

import struct
from typing import Dict

import numpy as np


class H5File:
    def __init__(self, path: str):
        self.b = open(path, "rb").read()
        if self.b[:8] != b"\x89HDF\r\n\x1a\n":
            raise ValueError("not an HDF5 file")
        if self.b[8] != 0:
            raise NotImplementedError(f"superblock version {self.b[8]}")
        self.so, self.sl = self.b[13], self.b[14]              # size of offsets / lengths
        if (self.so, self.sl) != (8, 8):
            raise NotImplementedError("only 8-byte offsets/lengths")
        # superblock v0: ... base addr, free-space addr, EOF addr, driver addr at 24.., root symbol-table entry at 56
        root = 24 + 4 * 8
        self.root_header = self._u64(root + 8)
        self.root_btree, self.root_heap = self._u64(root + 24), self._u64(root + 32)

    def _u64(self, o): return struct.unpack_from("<Q", self.b, o)[0]
    def _u32(self, o): return struct.unpack_from("<I", self.b, o)[0]
    def _u16(self, o): return struct.unpack_from("<H", self.b, o)[0]

    # ---- groups
    def _heap_data(self, heap_addr):
        assert self.b[heap_addr:heap_addr + 4] == b"HEAP"
        return self._u64(heap_addr + 24)

    def _name(self, heap_addr, off):
        d = self._heap_data(heap_addr) + off
        e = self.b.index(b"\x00", d)
        return self.b[d:e].decode()

    def _btree_entries(self, addr, heap):
        assert self.b[addr:addr + 4] == b"TREE", "bad B-tree node"
        level, n = self.b[addr + 5], self._u16(addr + 6)
        p = addr + 24
        out = {}
        for i in range(n):
            child = self._u64(p + 8)           # key_i (8) then child_i (8)
            p += 16
            if level > 0:
                out.update(self._btree_entries(child, heap))
            else:
                assert self.b[child:child + 4] == b"SNOD"
                ns = self._u16(child + 6)
                q = child + 8
                for _ in range(ns):
                    name_off, hdr = self._u64(q), self._u64(q + 8)
                    cache = self._u32(q + 16)
                    out[self._name(heap, name_off)] = (hdr, (self._u64(q + 24), self._u64(q + 32)) if cache == 1 else None)
                    q += 40
        return out

    def _messages(self, hdr):
        if self.b[hdr] != 1:
            raise NotImplementedError("object header version != 1")
        nmsg, size = self._u16(hdr + 2), self._u32(hdr + 8)
        blocks = [(hdr + 16, size)]
        msgs = []
        while blocks and len(msgs) < nmsg + 64:
            p, sz = blocks.pop(0)
            end = p + sz
            while p + 8 <= end:
                t, s = self._u16(p), self._u16(p + 2)
                body = p + 8
                if t == 0x10:                   # continuation
                    blocks.append((self._u64(body), self._u64(body + 8)))
                else:
                    msgs.append((t, body, s))
                p = body + s
        return msgs

    def _children(self, hdr, cached=None):
        if cached is not None:
            return self._btree_entries(cached[0], cached[1])
        for t, body, _ in self._messages(hdr):
            if t == 0x11:                       # symbol table message
                return self._btree_entries(self._u64(body), self._u64(body + 8))
        return None

    def _dataset(self, hdr):
        shape, dtype, addr = None, None, None
        for t, body, s in self._messages(hdr):
            if t == 0x01:                       # dataspace
                ver, rank = self.b[body], self.b[body + 1]
                o = body + (8 if ver == 1 else 4)
                shape = tuple(self._u64(o + 8 * i) for i in range(rank))
            elif t == 0x03:                     # datatype
                cls, size = self.b[body] & 0x0F, self._u32(body + 4)
                if cls != 1 or (self.b[body + 1] & 1):
                    raise NotImplementedError("only little-endian floating point datasets")
                dtype = {4: np.float32, 8: np.float64}[size]
            elif t == 0x08:                     # layout
                ver = self.b[body]
                if ver == 3:
                    if self.b[body + 1] != 1:
                        raise NotImplementedError("only contiguous layout")
                    addr = self._u64(body + 2)
                elif ver in (1, 2):
                    rank, lcls = self.b[body + 1], self.b[body + 2]
                    if lcls != 1:
                        raise NotImplementedError("only contiguous layout")
                    addr = self._u64(body + 8)
                else:
                    raise NotImplementedError(f"layout version {ver}")
        if shape is None or dtype is None or addr is None:
            return None
        n = int(np.prod(shape)) if shape else 1
        return np.frombuffer(self.b, dtype=dtype, count=n, offset=addr).reshape(shape).copy()

    def datasets(self) -> Dict[str, np.ndarray]:
        """All datasets, keyed by their full path (e.g. 'model_weights/conv2d_1/conv2d_1/kernel:0')."""
        out = {}

        def walk(hdr, cached, prefix):
            ch = self._children(hdr, cached)
            if ch is None:
                d = self._dataset(hdr)
                if d is not None:
                    out[prefix] = d
                return
            for name, (h2, c2) in ch.items():
                walk(h2, c2, f"{prefix}/{name}" if prefix else name)
        walk(self.root_header, (self.root_btree, self.root_heap), "")
        return out


def load_keras_weights(path: str) -> Dict[str, np.ndarray]:
    """{'conv2d_1/kernel': array, ...} from a Keras model.h5 / weights.h5."""
    ds = H5File(path).datasets()
    out = {}
    for k, v in ds.items():
        parts = k.split("/")
        if parts[-1].endswith(":0") and len(parts) >= 2:
            out[parts[-2] + "/" + parts[-1][:-2]] = v
    return out


# ---------------------------------------------------------------------------------------------------------- attributes
def _attr_value(f: H5File, body: int):
    """Decodes one attribute message (version 1): fixed- or variable-length strings and float arrays."""
    ver, nsz, tsz, ssz = f.b[body], f._u16(body + 2), f._u16(body + 4), f._u16(body + 6)
    if ver != 1:
        raise NotImplementedError(f"attribute message version {ver}")
    pad = lambda n: (n + 7) // 8 * 8
    name = f.b[body + 8:body + 8 + nsz - 1].decode()
    t = body + 8 + pad(nsz)
    s = t + pad(tsz)
    d = s + pad(ssz)
    rank = f.b[s + 1]
    shape = tuple(f._u64(s + 8 + 8 * i) for i in range(rank))
    n = int(np.prod(shape)) if shape else 1
    cls, size = f.b[t] & 0x0F, f._u32(t + 4)
    if cls == 3:                                   # fixed-length string
        vals = [f.b[d + i * size:d + (i + 1) * size].rstrip(b"\x00") for i in range(n)]
    elif cls == 9:                                 # variable-length string: (length, global heap address, object index)
        vals = []
        for i in range(n):
            q = d + 16 * i
            ln, gaddr, idx = f._u32(q), f._u64(q + 4), f._u32(q + 12)
            vals.append(_global_heap_object(f, gaddr, idx)[:ln])
    elif cls == 1:
        dt = {4: np.float32, 8: np.float64}[size]
        return name, np.frombuffer(f.b, dtype=dt, count=n, offset=d).reshape(shape).copy()
    else:
        raise NotImplementedError(f"attribute datatype class {cls}")
    return name, (vals if shape else vals[0])


def _global_heap_object(f: H5File, addr: int, index: int) -> bytes:
    assert f.b[addr:addr + 4] == b"GCOL"
    size = f._u64(addr + 8)
    p, end = addr + 16, addr + size
    while p + 16 <= end:
        idx, osz = f._u16(p), f._u64(p + 8)
        if idx == index:
            return f.b[p + 16:p + 16 + osz]
        if idx == 0:
            break
        p += 16 + (osz + 7) // 8 * 8
    raise ValueError(f"global heap object {index} not found")


def read_structure(path: str):
    """{'/': attrs, 'encoder': attrs, 'encoder/conv2d_1/kernel:0': (shape, dtype), ...}: every group with its attributes
    (names -> values; strings as bytes) and every dataset with its shape and dtype."""
    f = H5File(path)
    out = {}

    def walk(hdr, cached, prefix):
        msgs = f._messages(hdr)
        ch = f._children(hdr, cached)
        if ch is None:
            d = f._dataset(hdr)
            if d is not None:
                out[prefix] = (d.shape, d.dtype)
            return
        out[prefix or "/"] = dict(_attr_value(f, body) for t, body, _ in msgs if t == 0x0C)
        for name, (h2, c2) in ch.items():
            walk(h2, c2, f"{prefix}/{name}" if prefix else name)
    walk(f.root_header, (f.root_btree, f.root_heap), "")
    return out


# ---------------------------------------------------------------------------------------------------------- writer
_UNDEF = 0xFFFFFFFFFFFFFFFF
_LEAF_K, _NODE_K = 4, 16                # symbol-node and group B-tree K, as libhdf5 writes them


class _Writer:
    """Superblock 0 / object header 1 / symbol-table groups / contiguous datasets: the subset Keras 2.2.4's save_weights
    produced (h5py on libhdf5 1.10 with default settings).  Strings are stored as fixed-length, null-padded arrays."""

    def __init__(self):
        self.buf = bytearray(96)        # superblock, patched at the end

    def alloc(self, data: bytes) -> int:
        addr = len(self.buf)
        self.buf += data
        self.buf += b"\x00" * (-len(self.buf) % 8)
        return addr

    @staticmethod
    def _msg(t: int, body: bytes) -> bytes:
        body += b"\x00" * (-len(body) % 8)
        return struct.pack("<HHB3x", t, len(body), 0) + body

    def header(self, msgs) -> int:
        body = b"".join(msgs)
        return self.alloc(struct.pack("<BBHII4x", 1, 0, len(msgs), 1, len(body)) + body)

    @staticmethod
    def _space(shape) -> bytes:
        dims = b"".join(struct.pack("<Q", d) for d in shape)
        return struct.pack("<BBB5x", 1, len(shape), 1 if shape else 0) + dims + (dims if shape else b"")

    @staticmethod
    def _ftype(size: int) -> bytes:
        if size == 4:
            return bytes.fromhex("11201f00") + struct.pack("<I", 4) + bytes.fromhex("00002000170800177f000000")
        return bytes.fromhex("11203f00") + struct.pack("<I", 8) + bytes.fromhex("00004000340b0034ff030000")

    def _attr(self, name: str, value) -> bytes:
        nm = name.encode() + b"\x00"
        if isinstance(value, np.ndarray):
            a = np.ascontiguousarray(value, dtype=value.dtype.newbyteorder("<"))
            dtype, space, data = self._ftype(a.dtype.itemsize), self._space(a.shape), a.tobytes()
        else:
            vals = [value] if isinstance(value, bytes) else list(value)
            size = max([len(v) for v in vals] + [1])
            dtype = struct.pack("<BBBBI", 0x13, 0x01, 0, 0, size)
            space = self._space(() if isinstance(value, bytes) else (len(vals),))
            data = b"".join(v.ljust(size, b"\x00") for v in vals)
        pad = lambda b: b + b"\x00" * (-len(b) % 8)
        body = struct.pack("<BBHHH", 1, 0, len(nm), len(dtype), len(space)) + pad(nm) + pad(dtype) + pad(space) + data
        return self._msg(0x0C, body)

    def dataset(self, arr: np.ndarray) -> int:
        a = np.ascontiguousarray(arr, dtype=arr.dtype.newbyteorder("<"))
        addr = self.alloc(a.tobytes())
        msgs = [self._msg(0x01, self._space(a.shape)), self._msg(0x03, self._ftype(a.dtype.itemsize)),
                self._msg(0x05, bytes.fromhex("0202020100000000")),
                self._msg(0x08, struct.pack("<BBQQ", 3, 1, addr, a.nbytes))]
        return self.header(msgs)

    def group(self, children, attrs=()):
        """children: {name: (header address, (btree, heap) or None)}.  Returns (header, btree, heap)."""
        names = sorted(children)
        heap_data = bytearray(8)                   # offset 0: the empty name
        offs = {}
        for n in names:
            offs[n] = len(heap_data)
            heap_data += n.encode() + b"\x00"
            heap_data += b"\x00" * (-len(heap_data) % 8)
        data_addr = self.alloc(bytes(heap_data))
        heap = self.alloc(b"HEAP" + bytes(4) + struct.pack("<QQQ", len(heap_data), _UNDEF, data_addr))
        snods, keys = [], [0]
        for i in range(0, max(len(names), 1), 2 * _LEAF_K):
            chunk = names[i:i + 2 * _LEAF_K]
            ents = b""
            for n in chunk:
                hdr, cache = children[n]
                ents += struct.pack("<QQII", offs[n], hdr, 1 if cache else 0, 0) + (struct.pack("<QQ", *cache) if cache else bytes(16))
            ents += bytes(40 * (2 * _LEAF_K - len(chunk)))
            snods.append(self.alloc(b"SNOD" + struct.pack("<BBH", 1, 0, len(chunk)) + ents))
            keys.append(offs[chunk[-1]] if chunk else 0)
        if len(snods) > 2 * _NODE_K:
            raise NotImplementedError("group too large for one B-tree node")
        node = b"TREE" + struct.pack("<BBHQQ", 0, 0, len(snods), _UNDEF, _UNDEF)
        for i, s in enumerate(snods):
            node += struct.pack("<QQ", keys[i], s)
        node += struct.pack("<Q", keys[len(snods)])
        node += bytes(8 * (2 * _NODE_K + 1) + 8 * 2 * _NODE_K - (len(node) - 24))
        btree = self.alloc(node)
        msgs = [self._msg(0x11, struct.pack("<QQ", btree, heap))] + [self._attr(k, v) for k, v in attrs]
        return self.header(msgs), btree, heap

    def finish(self, root) -> bytes:
        hdr, btree, heap = root
        sb = b"\x89HDF\r\n\x1a\n" + bytes([0, 0, 0, 0, 0, 8, 8, 0]) + struct.pack("<HHI", _LEAF_K, _NODE_K, 0)
        sb += struct.pack("<QQQQ", 0, _UNDEF, len(self.buf), _UNDEF)
        sb += struct.pack("<QQII", 0, hdr, 1, 0) + struct.pack("<QQ", btree, heap)
        assert len(sb) == 96
        self.buf[:96] = sb
        return bytes(self.buf)


def write_keras_weights(path: str, layers) -> None:
    """Writes a Keras 2.2.4 ``save_weights`` file of a model whose top-level layers are ``layers``:
    [(layer name, [(weight name, array), ...])], e.g. ('encoder', [('conv2d_1/kernel:0', k), ...]); a layer without weights
    gets an empty ``weight_names``.  Root attributes: layer_names, backend = tensorflow, keras_version = 2.2.4."""
    w = _Writer()
    top = {}
    for lname, weights in layers:
        # nested groups for 'sub/name:0' paths
        tree = {}
        for wname, arr in weights:
            parts = wname.split("/")
            node = tree
            for p in parts[:-1]:
                node = node.setdefault(p, {})
            node[parts[-1]] = w.dataset(np.asarray(arr))

        def build(node, attrs=()):
            ch = {}
            for k, v in node.items():
                if isinstance(v, dict):
                    hdr, bt, hp = build(v)
                    ch[k] = (hdr, (bt, hp))
                else:
                    ch[k] = (v, None)
            return w.group(ch, attrs)
        names = [n.encode() for n, _ in weights]
        wn = names if names else np.zeros((0,), np.float64)
        hdr, bt, hp = build(tree, [("weight_names", wn)])
        top[lname] = (hdr, (bt, hp))
    root = w.group(top, [("layer_names", [n.encode() for n, _ in layers]), ("backend", b"tensorflow"),
                         ("keras_version", b"2.2.4")])
    data = w.finish(root)
    tmp = path + ".tmp"
    with open(tmp, "wb") as fh:
        fh.write(data)
    import os
    os.replace(tmp, path)
