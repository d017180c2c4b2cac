"""Seeded random programs over resident sets, checked against the reference — TEST INFRASTRUCTURE ONLY.

A program is a list of steps drawn from a seed: producers that make a new resident set from live ones
(uploads, batch ops, lazy folds, flip, add_offset, add / remove_many, add / remove_range, run_optimize,
or_many / xor_many / or_many_heap, and the 64-bit set's producers), consumers that read a live set and
compare what they read with the model, and frees of random live sets in any order, operands before their
pending results included.  The model keeps, for every live handle, its width, its expected portable
blobs (computed by the reference), for a lazy set its fold inputs, whether it is still unconsumed
("pending"), whether it shares containers and which handles it was derived from.  Every expected value
comes from the model alone, never from device output, so one seed gives one program on any machine.

    python tests/program_model.py --seed S [--width 64] [--upto K]

runs the program of seed S on the GPU (up to step K) and reports the first mismatch, with the seed,
the step, the failing set's ancestry and the first differing bitmap.
"""
import argparse
import ctypes as C
import functools
import hashlib
import os
import struct
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(_HERE))
sys.path.insert(0, _HERE)

import wide_cases   # noqa: E402
from cow_oracles import STATES, bind, make   # noqa: E402
from helpers import check_result_bitmap, no_run_twins, synth_blobs, synth_blobs64   # noqa: E402
from offset_oracles import ref_add_offset_bytes   # noqa: E402
from range_oracles import ref_range, ref_range64_bytes, ref_range_bytes   # noqa: E402
from run_cases import blob_containers   # noqa: E402
from update_oracles import ref_update64_bytes, ref_update_bytes   # noqa: E402

T32 = (1 << 32) - 1
PROFILES = ["full", "nearfull", "halves", "dense", "bitset", "array", "tiny", "longruns", "shortruns", "ends"]
REALDATA = ["census1881", "weather_sept_85", "wikileaks-noquotes", "census1881_srt", "uscensus2000"]
WIDE = ["top_array", "top_run_end", "top_full_run", "top_full_bitset", "top_bitset", "len_1", "len_33", "len_257",
        "len_1025", "tiles", "full_universe"]
RANGE_KINDS = ["empty", "single", "inside", "key_edges", "whole_key", "absent_keys", "many_keys", "universe", "top",
               "all_values", "no_value"]
HIGHS = (0, 1, 7, 0x10000, 0xFFFFFFFF)   # the 64-bit buckets of synth_blobs64

PRODUCERS32 = ("from_serialized", "from_serialized_keyrange", "from_frozen", "upload", "from_values_host",
               "from_values_device", "batch", "batch_inplace", "lazy", "lazy_more", "repair", "flip", "add_offset",
               "add_many", "remove_many", "add_range", "remove_range", "run_optimize", "remove_runs", "or_many",
               "or_many_keyrange", "xor_many", "or_many_heap")
PRODUCERS64 = ("from_serialized64", "from_values64_host", "from_values64_device", "op64", "add_many64",
               "remove_many64", "add_range64", "remove_range64", "run_optimize64", "remove_runs64")
CONSUMERS32 = ("serialize", "cardinalities", "container_count", "payload_bytes", "and_cardinality", "relations",
               "query", "to_uint32", "frozen", "download_all", "download_stream", "foreach_async",
               "add_cardinality_device", "refusal", "algorithmic_bytes")
CONSUMERS64 = ("serialize64", "cardinalities64", "and_cardinality64")
# producers whose results share containers with their operand (when the operand does not share itself)
SHARING = {"batch", "batch_inplace", "add_offset", "add_many", "remove_many", "add_range", "remove_range", "op64",
           "add_many64", "remove_many64", "add_range64", "remove_range64"}

DEFAULT_SEEDS32 = (1, 2, 3, 4, 5, 6)
DEFAULT_SEEDS64 = (101, 102, 103)
STEPS32, STEPS64 = 60, 40


# ------------------------------------------------------------------------------------------- reference
BIG = 1 << 20   # bitmaps above this cardinality are never spelled out value by value


def _card(R, blob):
    r = R.deserialize(blob)
    c = R.card(r)
    R.free(r)
    return c


def _vals(R, blob):
    """The values of a bitmap, or None above BIG values (the full universe holds 2^32)."""
    r = R.deserialize(blob)
    v = R.to_array(r) if R.card(r) <= BIG else None
    R.free(r)
    return v


def _ref_query(R):
    """R.L's roaring_bitmap_contains / rank / get_index / select, typed (roaring.h)."""
    L = R.L
    for name, res, args in (("contains", C.c_bool, [C.c_uint32]), ("rank", C.c_uint64, [C.c_uint32]),
                            ("get_index", C.c_int64, [C.c_uint32]),
                            ("select", C.c_bool, [C.c_uint32, C.POINTER(C.c_uint32)]),
                            ("and_cardinality", C.c_uint64, [C.c_void_p])):
        f = getattr(L, "roaring_bitmap_" + name)
        f.restype, f.argtypes = res, [C.c_void_p] + args
    return L


def _transform(R, blob, fn):
    r = R.deserialize(blob)
    fn(r)
    ok, why = R.validate(r)
    assert ok, why
    out = R.serialize(r)
    R.free(r)
    return out


def keyrange_bytes(R, blob, key_lo, key_hi):
    """The bitmap restricted to the containers of keys [key_lo, key_hi] (whole containers are dropped)."""
    rm = ref_range(R, "remove")

    def cut(r):
        if key_lo > 0:
            rm(r, 0, (key_lo << 16) - 1)
        if key_hi < 65535:
            rm(r, (key_hi + 1) << 16, T32)
    return _transform(R, blob, cut)


def payload_of(blob):
    """container_size_in_bytes summed over the containers of a portable blob."""
    return sum(2 * c if t == "array" else 8192 if t == "bitset" else 2 + 4 * nr for _, t, c, nr in blob_containers(blob))


def r64_buckets(blob):
    """[(high 32 bits, 32-bit portable blob)] of a 64-bit portable blob (roaring64 portable format)."""
    n = int.from_bytes(blob[:8], "little")
    pos, out = 8, []
    for _ in range(n):
        high = int.from_bytes(blob[pos:pos + 4], "little")
        pos += 4
        size = _portable_len(blob, pos)
        out.append((high, blob[pos:pos + size]))
        pos += size
    assert pos == len(blob), "trailing bytes"
    return out


def _portable_len(blob, pos):
    """Length of the 32-bit portable bitmap starting at blob[pos] (walked as run_cases.blob_containers walks it)."""
    b = blob[pos:]
    cookie, = struct.unpack_from("<I", b, 0)
    if cookie & 0xFFFF == 12347:
        n = (cookie >> 16) + 1
        flags = b[4:4 + (n + 7) // 8]
        pos = 4 + (n + 7) // 8
        isrun = [bool(flags[i // 8] >> (i % 8) & 1) for i in range(n)]
        data = pos + 4 * n + (4 * n if n >= 4 else 0)
    else:
        n, = struct.unpack_from("<I", b, 4)
        pos, isrun = 8, [False] * n
        data = pos + 8 * n
    for i in range(n):
        _, cm1 = struct.unpack_from("<HH", b, pos + 4 * i)
        if isrun[i]:
            nr, = struct.unpack_from("<H", b, data)
            data += 2 + 4 * nr
        elif cm1 + 1 > 4096:
            data += 8192
        else:
            data += 2 * (cm1 + 1)
    return data


def r64_remove_runs_bytes(R, blob):
    """Every bucket's roaring_bitmap_remove_run_compression, re-framed in the 64-bit portable format."""
    parts = r64_buckets(blob)
    out = [len(parts).to_bytes(8, "little")]
    for high, b in parts:
        out.append(high.to_bytes(4, "little"))
        out.append(_transform(R, b, R.L.roaring_bitmap_remove_run_compression))
    return b"".join(out)


def r64_run_optimize_bytes(R, blob):
    r = R.r64_deserialize(blob)
    R.L.roaring64_bitmap_run_optimize(r)
    out = R.r64_serialize(r)
    R.L.roaring64_bitmap_free(r)
    return out


def r64_card(R, blob):
    r = R.r64_deserialize(blob)
    c = int(R.L.roaring64_bitmap_get_cardinality(r))
    R.L.roaring64_bitmap_free(r)
    return c


class Inputs:
    """The bitmaps programs draw their sets from (built once per reference library)."""

    def __init__(self, R):
        syn = synth_blobs(R, 7001, 40, key_space=6, max_keys=6, profiles=PROFILES) + \
            synth_blobs(R, 7002, 20, key_space=10, max_keys=9)
        self.synth = syn + no_run_twins(R, syn)
        self.real = {ds: _load_realdata(ds)[:60] for ds in REALDATA}
        wide = dict(wide_cases.bitmaps(R))
        self.wide = [wide[n] for n in WIDE]
        self.empty = R.serialize(R.from_values(np.zeros(0, np.uint32), False))
        self.full = wide["full_universe"]
        self.b64 = synth_blobs64(R, 7003, 40, profiles=PROFILES) + synth_blobs64(R, 7004, 20)
        self.empty64 = R.r64_from_values(np.zeros(0, np.uint64))

    def draw32(self, rng, n):
        flavor = rng.integers(0, 4)
        out = []
        for _ in range(n):
            f = flavor if flavor < 3 else rng.integers(0, 3)
            u = rng.random()
            if u < 0.05:
                out.append(self.empty)
            elif u < 0.07:
                out.append(self.full)
            elif f == 0:
                out.append(self.synth[rng.integers(0, len(self.synth))])
            elif f == 1:
                ds = self.real[REALDATA[rng.integers(0, len(REALDATA))]]
                out.append(ds[rng.integers(0, len(ds))])
            else:
                out.append(self.wide[rng.integers(0, len(self.wide))])
        return out

    def draw64(self, rng, n):
        return [self.empty64 if rng.random() < 0.05 else self.b64[rng.integers(0, len(self.b64))] for _ in range(n)]


def _load_realdata(ds):
    import croaring_b200.datasets as dsm
    return dsm.load_realdata(ds)


@functools.lru_cache(maxsize=None)
def inputs(R):
    return Inputs(R)


# ------------------------------------------------------------------------------------------- the model
# Containers one producer call may read.  The device reserves a worst-case result slot per container (up to a
# bitset's 8 KiB), so a call over many full-universe bitmaps could reserve more than the device holds.
LIMIT = 300000


def _nc(blob):
    """The container count of a portable blob, from its cookie."""
    cookie, = struct.unpack_from("<I", blob, 0)
    return (cookie >> 16) + 1 if cookie & 0xFFFF == 12347 else struct.unpack_from("<I", blob, 4)[0]


def _cost(x, i):
    """Containers bitmap i of the set x holds (a lazy set: those of all its fold inputs)."""
    return _nc(x.blobs[i]) if x.blobs is not None else sum(_nc(b) for b in x.lazy[2][i])


def _trim(items, cost):
    """The longest prefix of items (at least one) whose summed cost stays within LIMIT."""
    tot = 0
    for k, it in enumerate(items):
        tot += cost(it)
        if tot > LIMIT and k:
            return items[:k]
    return items


def _big(x):
    """A set too large for one producer call over all its bitmaps."""
    n = len(x.blobs) if x.blobs is not None else len(x.lazy[2])
    return sum(_cost(x, i) for i in range(n)) > LIMIT


class H:
    """What the model knows of one handle."""

    def __init__(self, hid, width, blobs, step, parents, shares=False, pending=False, lazy=None):
        self.id, self.width, self.blobs, self.step = hid, width, blobs, step
        self.parents, self.shares, self.pending, self.lazy = tuple(parents), shares, pending, lazy
        self.alive = True
        self.bound = False     # bind_host(True) in force
        self.host = False      # uploaded from host bitmaps


class Program:
    """The steps of one seeded program and the coverage it reaches (computed with the reference alone)."""

    def __init__(self, R, seed, width=32, n_steps=None, stream_switch=None):
        self.R, self.seed, self.width = R, seed, width
        self.rng = np.random.default_rng(seed)
        self.inp = inputs(R)
        self.Rc = bind(R)
        self.h = {}
        self.steps = []
        self.stats = {"producers": {}, "consumers": {}, "pending_freed_operand": 0, "sharing_operand": 0,
                      "free_with_pending_dependent": 0, "max_depth": 0}
        self.depth = {}
        n_steps = n_steps or (STEPS32 if width == 32 else STEPS64)
        switch = stream_switch if stream_switch is not None else (width == 32 and seed % 2 == 0)
        self.on_stream = False
        for k in range(n_steps):
            if switch and k in (n_steps // 3, 2 * n_steps // 3):
                self.on_stream = not self.on_stream
                self._emit({"k": "set_stream", "on": self.on_stream})
            self._round(k)
        if self.on_stream:
            self.on_stream = False
            self._emit({"k": "set_stream", "on": False})
        for hid in [i for i, x in self.h.items() if x.alive]:
            self._free(hid)
        self._emit({"k": "download_wait"})

    # -- bookkeeping
    def _emit(self, st):
        st["i"] = len(self.steps)
        self.steps.append(st)
        return st

    def _live(self, width=None, lazy=None):
        return [x for x in self.h.values() if x.alive and (width is None or x.width == width) and
                (lazy is None or bool(x.lazy) == lazy)]

    def _pick(self, xs):
        return xs[self.rng.integers(0, len(xs))] if xs else None

    def _new(self, kind, width, blobs, parents, lazy=None, deferred=True):
        hid = len(self.h)
        ps = [self.h[p] for p in parents]
        shares = kind in SHARING and any(not p.shares for p in ps)
        x = H(hid, width, blobs, len(self.steps), parents, shares=shares, pending=deferred and bool(parents), lazy=lazy)
        self.h[hid] = x
        self.depth[hid] = 1 + max([self.depth[p] for p in parents], default=0)
        self.stats["max_depth"] = max(self.stats["max_depth"], self.depth[hid])
        self.stats["producers"][kind] = self.stats["producers"].get(kind, 0) + 1
        return x

    def _read(self, x, as_operand=False):
        """x is read by a consumer or as an operand: the coverage counters and its pending state."""
        if x.pending and any(not self.h[p].alive for p in x.parents) and not as_operand:
            self.stats["pending_freed_operand"] += 1
        if as_operand and x.shares:
            self.stats["sharing_operand"] += 1
        x.pending = False

    def _free(self, hid):
        x = self.h[hid]
        if any(y.alive and y.pending and hid in y.parents for y in self.h.values()):
            self.stats["free_with_pending_dependent"] += 1
        x.alive = False
        self._emit({"k": "free", "h": hid})

    # -- one round: a producer, checks of its result and of other live sets, maybe a free
    def _round(self, k):
        rng = self.rng
        if not self._live(self.width) or rng.random() < 0.08:
            x = self._upload()
        else:
            x = self._produce()
        if x is not None and x.parents and rng.random() < 0.4:
            # free an operand while x may still be pending: x must not need it any more
            ps = [p for p in x.parents if self.h[p].alive]
            if ps:
                self._free(self._pick(ps))
        if x is not None and rng.random() < 0.7:
            self._check(x, 1 + int(rng.integers(0, 2)))
        others = [y for y in self._live() if x is None or y.id != x.id]
        for _ in range(int(rng.integers(0, 3))):
            if others:
                self._check(self._pick(others), 1)
        if k % 6 == 5:
            for y in self._live():
                if not y.lazy:
                    self._consume(y, "serialize" if y.width == 32 else "serialize64")
        if self.width == 32 and rng.random() < 0.15:
            self._emit({"k": "download_wait"})
        bound = [y for y in self._live(32) if y.bound]
        if bound and rng.random() < 0.1:
            y = self._pick(bound)
            y.bound = False
            self._emit({"k": "bind_host", "h": y.id, "on": False})
        if rng.random() < 0.3 and self._live():
            self._free(self._pick(self._live()).id)

    def _upload(self):
        rng = self.rng
        if self.width == 64:
            kinds = ["from_serialized64", "from_values64_host", "from_values64_device"]
            kind = kinds[rng.integers(0, 3)]
            blobs = self.inp.draw64(rng, int(rng.integers(8, 41)))
            if kind == "from_serialized64":
                return self._emit_new({"k": kind, "blobs": blobs}, kind, 64, blobs, [], deferred=False)
            vals = [self._vals64(b) for b in blobs]
            vals = [self._jumble(v) for v in vals]
            exp = [self.R.r64_from_values(v, run_optimize=False) for v in vals]
            return self._emit_new({"k": kind, "vals": vals}, kind, 64, exp, [], deferred=False)
        kinds = ["from_serialized", "from_serialized_keyrange", "upload", "from_values_host", "from_values_device"]
        kind = kinds[rng.integers(0, len(kinds))]
        blobs = self.inp.draw32(rng, int(rng.integers(8, 41)))
        if kind == "from_serialized":
            return self._emit_new({"k": kind, "blobs": blobs}, kind, 32, blobs, [], deferred=False)
        if kind == "from_serialized_keyrange":
            lo = int(rng.integers(0, 6))
            hi = int(rng.choice([lo, lo + 2, 65535]))
            exp = [keyrange_bytes(self.R, b, lo, hi) for b in blobs]
            return self._emit_new({"k": kind, "blobs": blobs, "key_lo": lo, "key_hi": hi}, kind, 32, exp, [],
                                  deferred=False)
        if kind == "upload":
            states = [STATES[rng.integers(0, len(STATES))] for _ in blobs]
            bind_now = bool(rng.random() < 0.4)
            x = self._emit_new({"k": kind, "blobs": blobs, "states": states, "bind": bind_now}, kind, 32, blobs, [],
                               deferred=False)
            x.host, x.bound = True, bind_now
            return x
        vals = [self._jumble(v) for v in (_vals(self.R, b) for b in blobs) if v is not None]
        exp = [self._of_values(v) for v in vals]
        return self._emit_new({"k": kind, "vals": vals}, kind, 32, exp, [], deferred=False)

    def _of_values(self, v):
        r = self.R.from_values(v, run_optimize=False)
        out = self.R.serialize(r)
        self.R.free(r)
        return out

    def _jumble(self, v):
        """The values of a bitmap as a from_values input: a random subset, shuffled, some repeated."""
        rng = self.rng
        if v.size > 3000:
            v = v[rng.random(v.size) < 0.3]
        v = v.copy()
        rng.shuffle(v)
        if v.size and rng.random() < 0.5:
            v = np.concatenate([v, v[: int(rng.integers(0, min(50, v.size) + 1))]])
        return v

    def _vals64(self, blob):
        r = self.R.r64_deserialize(blob)
        n = r64_card(self.R, blob)
        out = np.empty(n, np.uint64)
        if n:
            f = self.R.L.roaring64_bitmap_to_uint64_array
            f.restype, f.argtypes = None, [C.c_void_p, C.c_void_p]
            f(r, out.ctypes.data)
        self.R.L.roaring64_bitmap_free(r)
        return out

    def _emit_new(self, st, kind, width, blobs, parents, lazy=None, deferred=True):
        x = self._new(kind, width, blobs, parents, lazy=lazy, deferred=deferred)
        st["out"] = x.id
        st["ops"] = list(parents)
        st["expect"] = blobs
        self._emit(st)
        return x

    def _sel(self, X):
        """A random selection of X's bitmaps: None (every bitmap) or an index list, repeats and the empty list
        included; a few bitmaps of a big set (whose worst-case result bounds would fill the device)."""
        rng = self.rng
        n_all = len(X.blobs)
        u = rng.random()
        if n_all == 0 or (u < 0.4 and not _big(X)):
            return None
        if u < 0.45:
            return []
        return _trim([int(i) for i in rng.integers(0, n_all, int(rng.integers(1, 41)))], lambda i: _cost(X, i))

    def _produce(self):
        rng = self.rng
        if self.width == 64:
            kind = PRODUCERS64[3 + rng.integers(0, len(PRODUCERS64) - 3)]
            return getattr(self, "_p64_" + kind)()
        lazies = self._live(32, lazy=True)
        choices = [k for k in PRODUCERS32 if k not in ("from_serialized", "from_serialized_keyrange", "upload",
                                                        "from_values_host", "from_values_device")]
        if not lazies:
            choices = [k for k in choices if k not in ("lazy_more", "repair")]
        elif rng.random() < 0.5:
            choices = ["lazy_more", "repair"]
        plain = self._live(32, lazy=False)
        if not plain:
            return self._upload()
        kind = choices[rng.integers(0, len(choices))]
        return getattr(self, "_p_" + kind)()

    def _operand(self, lazy=False):
        """A live set: often one of the latest results, so that chains grow long and results that share
        containers become operands themselves."""
        xs = self._live(self.width, lazy=lazy)
        if len(xs) > 3 and self.rng.random() < 0.6:
            xs = xs[-3:]
        return self._pick(xs)

    # -- 32-bit producers
    def _p_from_frozen(self):
        X = self._operand()
        self._read(X, as_operand=True)
        return self._emit_new({"k": "from_frozen", "src": X.id}, "from_frozen", 32, X.blobs, [X.id], deferred=False)

    def _pairs(self, A, B):
        rng = self.rng
        u = rng.random()
        na = len(A.blobs) if A.blobs is not None else len(A.lazy[2])
        if u < 0.07 or not na or not B.blobs:
            return [], []
        n = int(rng.integers(1, 41))
        ia = rng.integers(0, na, n)
        ib = rng.integers(0, len(B.blobs), n)
        if u < 0.2:
            ib = ia % len(B.blobs)
        pairs = _trim([(int(i), int(j)) for i, j in zip(ia, ib)], lambda p: _cost(A, p[0]) + _cost(B, p[1]))
        return [i for i, _ in pairs], [j for _, j in pairs]

    def _batch(self, inplace):
        rng = self.rng
        A = self._operand()
        B = A if rng.random() < 0.25 else self._operand()
        op = ("and", "or", "xor", "andnot")[rng.integers(0, 4)]
        ia, ib = self._pairs(A, B)
        f = self.R.op_inplace_bytes if inplace else self.R.op_bytes
        exp = [f(op, A.blobs[i], B.blobs[j]) for i, j in zip(ia, ib)]
        for X in {A.id: A, B.id: B}.values():
            self._read(X, as_operand=True)
        kind = "batch_inplace" if inplace else "batch"
        x = self._emit_new({"k": kind, "a": A.id, "b": B.id, "op": op, "ia": ia, "ib": ib}, kind, 32, exp,
                           sorted({A.id, B.id}))
        if op == "and":
            x.shares = False
        return x

    def _p_batch(self):
        return self._batch(False)

    def _p_batch_inplace(self):
        return self._batch(True)

    def _p_lazy(self):
        rng = self.rng
        A = self._operand()
        B = A if rng.random() < 0.25 else self._operand()
        op, conv = (("or", False), ("or", True), ("xor", False))[rng.integers(0, 3)]
        ia, ib = self._pairs(A, B)
        ins = [[A.blobs[i], B.blobs[j]] for i, j in zip(ia, ib)]
        for X in {A.id: A, B.id: B}.values():
            self._read(X, as_operand=True)
        return self._emit_new({"k": "lazy", "a": A.id, "b": B.id, "op": op, "conv": conv, "ia": ia, "ib": ib},
                              "lazy", 32, None, sorted({A.id, B.id}), lazy=(op, conv, ins))

    def _p_lazy_more(self):
        L = self._operand(lazy=True)
        S = self._operand()
        op, conv, ins = L.lazy
        ia, ib = self._pairs(L, S)
        new = [ins[i] + [S.blobs[j]] for i, j in zip(ia, ib)]
        self._read(L, as_operand=True)
        self._read(S, as_operand=True)
        return self._emit_new({"k": "lazy_more", "a": L.id, "b": S.id, "op": op, "conv": conv, "ia": ia, "ib": ib},
                              "lazy_more", 32, None, sorted({L.id, S.id}), lazy=(op, conv, new))

    def _p_repair(self):
        L = self._operand(lazy=True)
        op, conv, ins = L.lazy
        exp = [self.R.lazy_fold_bytes(op, conv, i) for i in ins]
        self._read(L, as_operand=True)
        return self._emit_new({"k": "repair", "src": L.id}, "repair", 32, exp, [L.id])

    def _single(self, kind, fn, **args):
        """A producer over one operand with a selection: fn(blob, item) gives item's expected bytes."""
        X = self._operand()
        sel = self._sel(X)
        items = list(range(len(X.blobs))) if sel is None else sel
        st = {"k": kind, "src": X.id, "idx": sel, **args}
        exp = [fn(X.blobs[i], k, st) for k, i in enumerate(items)]
        self._read(X, as_operand=True)
        return self._emit_new(st, kind, 32, exp, [X.id])

    def _p_flip(self):
        rng = self.rng
        u = rng.random()
        if u < 0.2:
            s, e = 0, 1 << 32
        elif u < 0.3:
            s = e = int(rng.integers(0, 1 << 20))
        elif u < 0.4:
            s, e = 0xFFFF0000 + int(rng.integers(0, 65536)), 1 << 32
        else:
            s = int(rng.integers(0, 7 << 16))
            e = s + int(rng.integers(1, 3 << 16))
        return self._single("flip", lambda b, k, st: self.R.flip_bytes(b, s, e), start=s, end=e)

    def _p_add_offset(self):
        rng = self.rng
        mode = int(rng.integers(0, 4))   # aligned / unaligned / negative / mixed

        def draw():
            m = mode if mode < 3 else int(rng.integers(0, 3))
            if m == 0:
                return int(rng.integers(-4, 5)) << 16
            if m == 1:
                return int(rng.integers(1, 400000))
            return -int(rng.integers(1, 1 << 33))
        X = self._operand()
        sel = self._sel(X)
        n = len(X.blobs) if sel is None else len(sel)
        offs = [draw() for _ in range(n)]
        items = list(range(len(X.blobs))) if sel is None else sel
        exp = [ref_add_offset_bytes(self.R, X.blobs[i], o) for i, o in zip(items, offs)]
        self._read(X, as_operand=True)
        return self._emit_new({"k": "add_offset", "src": X.id, "idx": sel, "offsets": offs}, "add_offset", 32, exp,
                              [X.id])

    def _update_vals(self, blob):
        rng = self.rng
        v = _vals(self.R, blob)
        parts = [rng.integers(0, 8 << 16, int(rng.integers(0, 60))).astype(np.uint32)]
        if v is not None and v.size:
            parts.append(rng.choice(v, int(rng.integers(0, 60))))
        keys = rng.integers(0, 8, 3).astype(np.uint32) << np.uint32(16)
        parts += [keys, keys + np.uint32(65535), np.array([T32], np.uint32)[: int(rng.integers(0, 2))]]
        out = np.concatenate(parts).astype(np.uint32)
        rng.shuffle(out)
        return out

    def _update(self, op):
        X = self._operand()
        sel = self._sel(X)
        items = list(range(len(X.blobs))) if sel is None else sel
        vals = [self._update_vals(X.blobs[i]) for i in items]
        exp = [ref_update_bytes(self.R, op, X.blobs[i], v) for i, v in zip(items, vals)]
        self._read(X, as_operand=True)
        kind = op + "_many"
        return self._emit_new({"k": kind, "src": X.id, "idx": sel, "vals": vals,
                               "device": bool(self.rng.random() < 0.4)}, kind, 32, exp, [X.id])

    def _p_add_many(self):
        return self._update("add")

    def _p_remove_many(self):
        return self._update("remove")

    def _range(self, blob):
        """A closed range [lo, hi] of a random kind for this bitmap (lo > hi: empty)."""
        rng = self.rng
        kind = RANGE_KINDS[rng.integers(0, len(RANGE_KINDS))]
        k = int(rng.integers(0, 6))
        if kind == "empty":
            return 10, 5
        if kind == "inside":
            a, b = sorted(rng.integers(0, 65536, 2).tolist())
            return (k << 16) + a, (k << 16) + b
        if kind == "key_edges":
            return 65535, 65536
        if kind == "whole_key":
            return k << 16, (k << 16) + 65535
        if kind == "absent_keys":
            return (40 << 16) + 5, (42 << 16) + 100
        if kind == "many_keys":
            return int(rng.integers(0, 3000)), (5 << 16) + int(rng.integers(0, 65536))
        if kind == "universe":
            return 0, T32
        if kind == "top":
            return 0xFFFF0000, T32
        v = _vals(self.R, blob)
        if v is None:   # the full universe or close: its values are everything
            v = np.array([0, T32], np.uint32)
        if kind == "single":
            x = int(rng.choice(v)) if v.size and rng.random() < 0.5 else int(rng.integers(0, 6 << 16))
            return x, x
        if kind == "all_values":
            return (int(v[0]), int(v[-1])) if v.size else (0, 0)
        gaps = np.flatnonzero(np.diff(v.astype(np.int64)) > 1) if v.size else np.zeros(0, np.int64)
        if gaps.size:
            g = int(rng.choice(gaps))
            return int(v[g]) + 1, int(v[g + 1]) - 1
        return (int(v[-1]) + 1, int(v[-1]) + 70000) if v.size and int(v[-1]) < T32 - 70000 else (7, 7)

    def _range_update(self, op):
        X = self._operand()
        sel = self._sel(X)
        items = list(range(len(X.blobs))) if sel is None else sel
        rs = [self._range(X.blobs[i]) for i in items]
        # the universe add on a full-universe bitmap is cheap; on everything else keep results small
        exp = [ref_range_bytes(self.R, op, X.blobs[i], a, z) for i, (a, z) in zip(items, rs)]
        self._read(X, as_operand=True)
        kind = op + "_range"
        return self._emit_new({"k": kind, "src": X.id, "idx": sel, "lo": [a for a, _ in rs], "hi": [z for _, z in rs]},
                              kind, 32, exp, [X.id])

    def _p_add_range(self):
        return self._range_update("add")

    def _p_remove_range(self):
        return self._range_update("remove")

    def _p_run_optimize(self):
        X = self._operand()
        exp = [_transform(self.R, b, self.R.L.roaring_bitmap_run_optimize) for b in X.blobs]
        self._read(X, as_operand=True)
        return self._emit_new({"k": "run_optimize", "src": X.id}, "run_optimize", 32, exp, [X.id])

    def _p_remove_runs(self):
        X = self._operand()
        if sum(_nc(b) for b in X.blobs) > LIMIT // 10:   # full-universe runs as bitsets: optimize instead
            return self._p_run_optimize()
        exp = [_transform(self.R, b, self.R.L.roaring_bitmap_remove_run_compression) for b in X.blobs]
        self._read(X, as_operand=True)
        return self._emit_new({"k": "remove_runs", "src": X.id}, "remove_runs", 32, exp, [X.id])

    def _many(self, kind):
        rng = self.rng
        X = self._operand()
        sel = None if (rng.random() < 0.4 and not _big(X)) or not X.blobs else \
            _trim([int(i) for i in rng.integers(0, len(X.blobs), int(rng.integers(0, 30)))], lambda i: _cost(X, i))
        items = list(range(len(X.blobs))) if sel is None else sel
        sub = [X.blobs[i] for i in items]
        st = {"k": kind, "src": X.id, "idx": sel}
        name = "or_many" if kind == "or_many_keyrange" else kind
        exp = self.R.many_bytes(name, sub)
        if kind == "or_many_keyrange":
            lo = int(rng.integers(0, 6))
            hi = int(rng.choice([lo, lo + 3, 65535]))
            st.update(key_lo=lo, key_hi=hi)
            exp = keyrange_bytes(self.R, exp, lo, hi)
        elif sel is None and kind != "or_many_heap":
            st["algo_bytes"] = sum(payload_of(b) for b in X.blobs)   # the whole set's input bytes
            self.stats["consumers"]["algorithmic_bytes"] = self.stats["consumers"].get("algorithmic_bytes", 0) + 1
        self._read(X, as_operand=True)
        return self._emit_new(st, kind, 32, [exp], [X.id], deferred=False)

    def _p_or_many(self):
        return self._many("or_many")

    def _p_or_many_keyrange(self):
        return self._many("or_many_keyrange")

    def _p_xor_many(self):
        return self._many("xor_many")

    def _p_or_many_heap(self):
        return self._many("or_many_heap")

    # -- 64-bit producers
    def _p64_op64(self):
        rng = self.rng
        A = self._operand()
        B = A if rng.random() < 0.25 else self._operand()
        op = ("and", "or", "xor", "andnot")[rng.integers(0, 4)]
        ia, ib = self._pairs(A, B)
        exp = [self.R.r64_op_bytes(op, A.blobs[i], B.blobs[j]) for i, j in zip(ia, ib)]
        for X in {A.id: A, B.id: B}.values():
            self._read(X, as_operand=True)
        x = self._emit_new({"k": "op64", "a": A.id, "b": B.id, "op": op, "ia": ia, "ib": ib}, "op64", 64, exp,
                           sorted({A.id, B.id}))
        if op == "and":
            x.shares = False
        return x

    def _update64(self, op):
        rng = self.rng
        X = self._operand()
        sel = self._sel(X)
        items = list(range(len(X.blobs))) if sel is None else sel
        vals = []
        for i in items:
            v = self._vals64(X.blobs[i])
            hs = np.array(HIGHS, np.uint64)[rng.integers(0, len(HIGHS), int(rng.integers(0, 40)))]
            new = (hs << np.uint64(32)) + rng.integers(0, 6 << 16, hs.size).astype(np.uint64)
            parts = [new, rng.choice(v, int(rng.integers(0, 30))) if v.size else np.zeros(0, np.uint64)]
            vals.append(np.concatenate(parts).astype(np.uint64))
        exp = [ref_update64_bytes(self.R, op, X.blobs[i], v) for i, v in zip(items, vals)]
        self._read(X, as_operand=True)
        kind = op + "_many64"
        return self._emit_new({"k": kind, "src": X.id, "idx": sel, "vals": vals,
                               "device": bool(rng.random() < 0.4)}, kind, 64, exp, [X.id])

    def _p64_add_many64(self):
        return self._update64("add")

    def _p64_remove_many64(self):
        return self._update64("remove")

    def _range64(self):
        rng = self.rng
        h = int(HIGHS[rng.integers(0, len(HIGHS))])
        u = rng.random()
        if u < 0.1:
            return 10, 5
        if u < 0.5:
            a, b = sorted(rng.integers(0, 6 << 16, 2).tolist())
            return (h << 32) + a, (h << 32) + b
        if u < 0.7 and h < 0xFFFFFFFF:   # across one bucket boundary
            return (h << 32) + T32 - int(rng.integers(0, 70000)), ((h + 1) << 32) + int(rng.integers(0, 70000))
        if u < 0.85:
            return (0xFFFFFFFF << 32) + 0xFFFF0000, (1 << 64) - 1
        return h << 32, (h << 32) + (3 << 16) - 1

    def _range_update64(self, op):
        X = self._operand()
        sel = self._sel(X)
        items = list(range(len(X.blobs))) if sel is None else sel
        rs = [self._range64() for _ in items]
        exp = [ref_range64_bytes(self.R, op, X.blobs[i], a, z) for i, (a, z) in zip(items, rs)]
        self._read(X, as_operand=True)
        kind = op + "_range64"
        return self._emit_new({"k": kind, "src": X.id, "idx": sel, "lo": [a for a, _ in rs], "hi": [z for _, z in rs]},
                              kind, 64, exp, [X.id])

    def _p64_add_range64(self):
        return self._range_update64("add")

    def _p64_remove_range64(self):
        return self._range_update64("remove")

    def _p64_run_optimize64(self):
        X = self._operand()
        exp = [r64_run_optimize_bytes(self.R, b) for b in X.blobs]
        self._read(X, as_operand=True)
        return self._emit_new({"k": "run_optimize64", "src": X.id}, "run_optimize64", 64, exp, [X.id])

    def _p64_remove_runs64(self):
        X = self._operand()
        exp = [r64_remove_runs_bytes(self.R, b) for b in X.blobs]
        self._read(X, as_operand=True)
        return self._emit_new({"k": "remove_runs64", "src": X.id}, "remove_runs64", 64, exp, [X.id])

    # -- consumers
    def _check(self, x, n):
        rng = self.rng
        if x.lazy:
            if rng.random() < 0.5:
                self._consume(x, "refusal")
            return
        kinds = CONSUMERS32 if x.width == 32 else CONSUMERS64
        for _ in range(n):
            kind = kinds[rng.integers(0, len(kinds))]
            if kind == "algorithmic_bytes":
                kind = "payload_bytes"
            self._consume(x, kind)

    def _consume(self, x, kind):
        rng = self.rng
        R = self.R
        if kind == "to_uint32" and sum(_card(R, b) for b in x.blobs) > BIG:
            kind = "serialize"   # too many values to spell out: read the bytes instead
        st = {"k": kind, "h": x.id}
        if kind == "refusal":
            if x.lazy:
                st["call"], st["match"] = "add_range", "add_range_closed: the set is in a lazy state"
            else:
                st["call"], st["match"] = "remove_range", r"remove_range_closed: index out of range"
        elif kind in ("serialize", "serialize64", "download_all", "download_stream", "foreach_async"):
            st["expect"] = x.blobs
            if kind == "download_all":
                n = len(x.blobs)
                st["sample"] = sorted({int(i) for i in rng.integers(0, n, min(n, 6))}) if n else []
        elif kind == "frozen":
            st["expect"] = [R.frozen_bytes(b) for b in x.blobs]
        elif kind in ("cardinalities", "add_cardinality_device"):
            st["expect"] = [_card(R, b) for b in x.blobs]
        elif kind == "cardinalities64":
            st["expect"] = [r64_card(R, b) for b in x.blobs]
        elif kind == "container_count":
            st["expect"] = sum(len(blob_containers(b)) for b in x.blobs)
        elif kind == "payload_bytes":
            st["expect"] = sum(payload_of(b) for b in x.blobs)
        elif kind == "to_uint32":
            st["expect"] = [_vals(R, b) for b in x.blobs]
        elif kind in ("and_cardinality", "relations", "and_cardinality64"):
            Y = self._pick([y for y in self._live(x.width, lazy=False)])
            self._read(Y)
            ia, ib = self._pairs(x, Y)
            st.update(other=Y.id, ia=ia, ib=ib)
            if kind == "and_cardinality64":
                st["expect"] = [R.r64_and_cardinality(x.blobs[i], Y.blobs[j]) for i, j in zip(ia, ib)]
            else:
                L = _ref_query(R)
                out = []
                for i, j in zip(ia, ib):
                    a, b = R.deserialize(x.blobs[i]), R.deserialize(Y.blobs[j])
                    if kind == "and_cardinality":
                        out.append(int(L.roaring_bitmap_and_cardinality(a, b)))
                    else:
                        out.append(int(L.roaring_bitmap_equals(a, b)) | int(L.roaring_bitmap_is_subset(a, b)) << 1 |
                                   int(L.roaring_bitmap_is_strict_subset(a, b)) << 2)
                    R.free(a)
                    R.free(b)
                st["expect"] = out
        elif kind == "query":
            self._query(x, st)
        self._read(x)
        self.stats["consumers"][kind] = self.stats["consumers"].get(kind, 0) + 1
        self._emit(st)

    def _query(self, x, st):
        """Point queries against numpy.searchsorted on the values, or against the reference's own functions for
        a bitmap too large to spell out."""
        rng = self.rng
        qk = ("contains", "rank", "get_index", "select")[rng.integers(0, 4)]
        n = len(x.blobs)
        idx = sorted(int(i) for i in rng.integers(0, n, int(rng.integers(0, 80)))) if n else []
        qs, exp = [], []
        L = _ref_query(self.R)
        for i in sorted(set(idx)):
            v = _vals(self.R, x.blobs[i])
            r = self.R.deserialize(x.blobs[i])
            card = self.R.card(r)
            for _ in range(idx.count(i)):
                if qk == "select":
                    q = int(rng.integers(0, min(card + 3, 1 << 32)))
                    if v is not None:
                        e = int(v[q]) if q < v.size else -1
                    else:
                        out = C.c_uint32()
                        e = int(out.value) if L.roaring_bitmap_select(r, q, C.byref(out)) else -1
                else:
                    u = rng.random()
                    if card and u < 0.4:   # a value and its neighbours: run and container edges
                        j = int(rng.integers(0, card))
                        q = (int(v[j]) if v is not None else j) + int(rng.integers(-1, 2))
                    elif u < 0.7:
                        q = (int(rng.integers(0, 8)) << 16) + int(rng.choice([0, 1, 65534, 65535]))
                    else:
                        q = int(rng.choice([0, T32, int(rng.integers(0, 1 << 32))]))
                    q = min(max(q, 0), T32)
                    if v is not None:
                        pos = int(np.searchsorted(v, q, "right"))
                        hit = pos > 0 and int(v[pos - 1]) == q
                        e = int(hit) if qk == "contains" else pos if qk == "rank" else (pos - 1 if hit else -1)
                    else:
                        e = int(getattr(L, "roaring_bitmap_" + qk)(r, q))
                qs.append(q)
                exp.append(e)
            self.R.free(r)
        st.update(query=qk, idx=idx, values=qs, expect=exp, device=bool(rng.random() < 0.3))

    # -- coverage
    def ancestry(self, hid):
        """The steps that produced hid and its ancestors, oldest first."""
        seen, todo = set(), [hid]
        while todo:
            h = todo.pop()
            if h in seen:
                continue
            seen.add(h)
            todo.extend(self.h[h].parents)
        return sorted(self.h[h].step for h in seen)


# ------------------------------------------------------------------------------------------- the executor
class Mismatch(AssertionError):
    pass


class Runner:
    """Runs a Program on the device (croaring_b200 as rb) and checks every consumer step."""

    def __init__(self, rb, R, prog):
        self.rb, self.R, self.p = rb, R, prog
        self.sets, self.hostbm, self.keep = {}, [], []
        self.digest = hashlib.sha256()
        self.async_got, self.async_expect = {}, []
        self.stream = None

    def _fail(self, st, what, hid=None, first=None):
        p = self.p
        lines = [f"program seed {p.seed} (width {p.width}) step {st['i']} ({st['k']}): {what}"]
        if first is not None:
            lines.append(f"first differing bitmap: {first}")
        if hid is not None:
            anc = p.ancestry(hid)
            lines.append(f"handle {hid} ancestry: " + "; ".join(f"#{i} {p.steps[i]['k']}" for i in anc))
            frees = [s["i"] for s in p.steps[:st["i"]] if s["k"] == "free"]
            lines.append(f"frees before: " + ", ".join(f"#{i}(h{p.steps[i]['h']})" for i in frees))
        lines.append(f"replay: python tests/program_model.py --seed {p.seed} --width {p.width} --upto {st['i']}")
        raise Mismatch("\n".join(lines))

    def _eq_list(self, st, got, exp, hid, what):
        self._hash(got)
        if list(got) != list(exp):
            first = next((k for k in range(min(len(got), len(exp))) if got[k] != exp[k]), min(len(got), len(exp)))
            detail = f"{got[0]} != expected {exp[0]}" if len(got) == len(exp) == 1 else \
                f"{len(got)} vs {len(exp)} entries"
            self._fail(st, f"{what} differs ({detail})", hid, first)

    def _hash(self, xs):
        for x in xs:
            self.digest.update(x if isinstance(x, bytes) else np.asarray(x).tobytes())

    def run(self, upto=None):
        for st in self.p.steps:
            if upto is not None and st["i"] > upto:
                break
            try:
                self.step(st)
            except Mismatch:
                raise
            except Exception as e:
                self._fail(st, f"{type(e).__name__}: {e}", st.get("h", st.get("out")))
        return self.digest.hexdigest()

    def _tensor(self, arrays, width):
        import torch
        flat = np.concatenate(arrays) if arrays else np.zeros(0, np.uint32 if width == 32 else np.uint64)
        flat = flat.astype(np.uint32 if width == 32 else np.uint64)
        off = np.zeros(len(arrays) + 1, np.int64)
        np.cumsum([a.size for a in arrays], out=off[1:])
        sv = flat.view(np.int32 if width == 32 else np.int64)
        t = torch.from_numpy(sv.copy()).cuda()
        o = torch.from_numpy(off).cuda()
        if self.stream is None:   # the library's own stream reads them: torch's writes first
            torch.cuda.current_stream().synchronize()
        self.keep += [t, o]
        return t, o

    def _device_ctx(self):
        import contextlib
        import torch
        return torch.cuda.stream(self.stream) if self.stream is not None else contextlib.nullcontext()

    def step(self, st):
        rb, R, k = self.rb, self.R, st["k"]
        S = self.sets
        if k == "free":
            S.pop(st["h"]).free()
            return
        if k == "download_wait":
            rb.download_wait()
            for hid, exp, st0 in self.async_expect:
                got = [self.async_got[(hid, st0["i"])].get(i) for i in range(len(exp))]
                self._eq_list(st0, got, exp, hid, "foreach_async bytes")
            self.async_expect, self.async_got = [], {}
            return
        if k == "set_stream":
            import torch
            if st["on"]:
                self.stream = torch.cuda.Stream()
                self.keep.append(self.stream)
                rb.set_stream(self.stream.cuda_stream)
            else:
                rb.set_stream(None)
                self.stream = None
            return
        if k == "bind_host":
            S[st["h"]].bind_host(st["on"])
            return
        if "out" in st:
            S[st["out"]] = self._produce(st)
            return
        self._consume(st)

    def _produce(self, st):
        rb, R, k = self.rb, self.R, st["k"]
        S = self.sets
        if k == "from_serialized":
            return rb.DeviceSet.from_serialized(st["blobs"])
        if k == "from_serialized_keyrange":
            return rb.DeviceSet.from_serialized(st["blobs"], st["key_lo"], st["key_hi"])
        if k == "from_frozen":
            return rb.DeviceSet.from_frozen(S[st["src"]].serialize_all(frozen=True))
        if k == "upload":
            import types
            Rc = bind(R)
            xs = [make(Rc, b, s) for b, s in zip(st["blobs"], st["states"])]
            self.hostbm += xs
            X = rb.DeviceSet.upload([types.SimpleNamespace(ptr=p) for p in xs])
            return X.bind_host(True) if st["bind"] else X
        if k in ("from_values_host", "from_values64_host"):
            cls = rb.DeviceSet if k == "from_values_host" else rb.DeviceSet64
            return cls.from_values(st["vals"])
        if k in ("from_values_device", "from_values64_device"):
            w = 32 if k == "from_values_device" else 64
            cls = rb.DeviceSet if w == 32 else rb.DeviceSet64
            with self._device_ctx():
                t, o = self._tensor(st["vals"], w)
            return cls.from_values(t, o)
        if k == "from_serialized64":
            return rb.DeviceSet64.from_serialized(st["blobs"])
        ia, ib = np.array(st.get("ia", []), np.uint32), np.array(st.get("ib", []), np.uint32)
        if k in ("batch", "batch_inplace"):
            return S[st["a"]].batch(st["op"], S[st["b"]], ia, ib, inplace_rules=k == "batch_inplace")
        if k == "lazy":
            return S[st["a"]].batch(st["op"], S[st["b"]], ia, ib, lazy=True, bitsetconversion=st["conv"])
        if k == "lazy_more":
            return S[st["a"]].batch(st["op"], S[st["b"]], ia, ib, lazy=True, inplace_rules=True,
                                    bitsetconversion=st["conv"])
        if k == "op64":
            return S[st["a"]].op(st["op"], S[st["b"]], ia, ib)
        X = S[st["src"]]
        idx = None if st.get("idx") is None else np.array(st["idx"], np.uint32)
        if k == "repair":
            return X.repair_after_lazy()
        if k == "flip":
            return X.flip(st["start"], st["end"], idx=idx)
        if k == "add_offset":
            return X.add_offset(st["offsets"], idx=idx)
        if k in ("add_many", "remove_many", "add_many64", "remove_many64"):
            f = getattr(X, k.replace("64", ""))
            if st["device"]:
                with self._device_ctx():
                    t, o = self._tensor(st["vals"], X._width)
                return f(t, o, idx=idx)
            return f(st["vals"], idx=idx)
        if k in ("add_range", "remove_range", "add_range64", "remove_range64"):
            f = getattr(X, k.replace("64", ""))
            end = [z + 1 if a <= z else a for a, z in zip(st["lo"], st["hi"])]
            return f(st["lo"], end, idx=idx)
        if k in ("run_optimize", "run_optimize64"):
            return X.run_optimize()
        if k == "remove_runs":
            return X.run_optimize(remove_runs=True)
        if k == "remove_runs64":
            return X.run_optimize(0)
        if k == "or_many_keyrange":
            return X.or_many(idx, key_lo=st["key_lo"], key_hi=st["key_hi"])
        out = getattr(X, k)(idx)
        if "algo_bytes" in st:
            got = rb.last_algorithmic_bytes()
            if got != st["algo_bytes"]:
                self._fail(st, f"last_algorithmic_bytes {got} != the input set's {st['algo_bytes']}", st["src"])
        return out

    def _consume(self, st):
        rb, R, k = self.rb, self.R, st["k"]
        hid = st["h"]
        X = self.sets[hid]
        if k in ("serialize", "serialize64"):
            self._eq_list(st, X.serialize_all(), st["expect"], hid, "portable bytes")
        elif k == "frozen":
            self._eq_list(st, X.serialize_all(frozen=True), st["expect"], hid, "frozen bytes")
        elif k in ("cardinalities", "cardinalities64"):
            self._eq_list(st, [int(c) for c in X.cardinalities()], st["expect"], hid, "cardinalities")
        elif k == "container_count":
            self._eq_list(st, [X.container_count], [st["expect"]], hid, "container_count")
        elif k == "payload_bytes":
            self._eq_list(st, [X.payload_bytes], [st["expect"]], hid, "payload_bytes")
        elif k == "to_uint32":
            got = X.to_uint32_arrays()
            self._hash(got)
            for j, (g, e) in enumerate(zip(got, st["expect"])):
                if not np.array_equal(g, e):
                    self._fail(st, "to_uint32_arrays differs", hid, j)
            if len(got) != len(st["expect"]):
                self._fail(st, "to_uint32_arrays count differs", hid)
        elif k in ("and_cardinality", "and_cardinality64", "relations"):
            Y = self.sets[st["other"]]
            ia, ib = np.array(st["ia"], np.uint32), np.array(st["ib"], np.uint32)
            got = X.relations(Y, ia, ib) if k == "relations" else X.and_cardinality(Y, ia, ib)
            self._eq_list(st, [int(v) for v in got], st["expect"], hid, k)
        elif k == "query":
            vals = np.array(st["values"], np.uint32)
            idx = np.array(st["idx"], np.uint32)
            if st["device"] and vals.size:
                import torch
                with self._device_ctx():
                    tv = torch.from_numpy(vals.view(np.int32).copy()).cuda()
                    ti = torch.from_numpy(idx.view(np.int32).copy()).cuda()
                got = getattr(X, st["query"])(tv, ti).cpu().numpy()
            else:
                got = getattr(X, st["query"])(vals, idx)
            self._eq_list(st, [int(v) for v in got], st["expect"], hid, st["query"])
        elif k == "download_all":
            bms = X.download_all()
            for j in st["sample"]:
                try:
                    check_result_bitmap(R, bms[j], st["expect"][j], f"bitmap {j}")
                except AssertionError as e:
                    self._fail(st, f"download_all: {e}", hid, j)
            self._hash([bms[j].serialize() for j in st["sample"]])
        elif k == "download_stream":
            got = []
            for arr, n in X.download_stream(chunk_bitmaps=7):
                got += [rb.Bitmap(arr[j], own=False).serialize() for j in range(n)]
                rb.DeviceSet.free_raw(arr, n)
            self._eq_list(st, got, st["expect"], hid, "download_stream bytes")
        elif k == "foreach_async":
            box = {}
            self.async_got[(hid, st["i"])] = box

            def visit(i, p, box=box):
                box[int(i)] = rb.Bitmap(p, own=False).serialize()
                return 0
            fn = rb.api.VISIT_FN(lambda i, p, _ctx: visit(i, p))
            self.keep.append(fn)
            X.foreach_async(None, fn)
            self.async_expect.append((hid, st["expect"], st))
        elif k == "add_cardinality_device":
            import torch
            acc = torch.full((1,), 5, dtype=torch.int64, device="cuda")
            torch.cuda.current_stream().synchronize()
            X.add_cardinality_device(acc.data_ptr())
            rb.synchronize()
            self._eq_list(st, [int(acc.item()) - 5], [sum(st["expect"])], hid, "add_cardinality_device")
        elif k == "refusal":
            try:
                if st["call"] == "add_range":
                    X.add_range(0, 5)
                else:
                    X.remove_range(0, 5, idx=[len(X) + 3])
            except rb.RB200Error as e:
                import re
                if not re.search(st["match"], str(e)):
                    self._fail(st, f"refusal says {e!r}, expected {st['match']!r}", hid)
            else:
                self._fail(st, "the documented refusal did not happen", hid)
        else:
            raise AssertionError(f"unknown consumer {k}")

    def close(self):
        """Frees what the program left (after a failure) and the host bitmaps of its uploads."""
        for X in self.sets.values():
            X.free()
        self.sets = {}
        try:
            self.rb.download_wait()
        finally:
            self.rb.set_stream(None)
            self.rb.synchronize()
            for p in self.hostbm:
                self.R.free(p)
            self.hostbm, self.keep = [], []


def seeds_from_env(default32=DEFAULT_SEEDS32, default64=DEFAULT_SEEDS64):
    """RB200_PROGRAM_SEEDS=a-b: the 32-bit seeds a..b and 64-bit seeds 1000+a..1000+b (a longer soak)."""
    e = os.environ.get("RB200_PROGRAM_SEEDS")
    if not e:
        return list(default32), list(default64)
    a, _, b = e.partition("-")
    r = range(int(a), int(b or a) + 1)
    return list(r), [1000 + s for s in r]


def run_program(rb, R, seed, width, upto=None):
    prog = Program(R, seed, width)
    run = Runner(rb, R, prog)
    try:
        return run.run(upto)
    finally:
        run.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--seed", type=int, required=True)
    ap.add_argument("--width", type=int, default=32, choices=(32, 64))
    ap.add_argument("--upto", type=int, default=None)
    a = ap.parse_args()
    import croaring_b200 as rb
    from oracle.refbind import ref
    rb.init(0)
    print(run_program(rb, ref(), a.seed, a.width, a.upto))


if __name__ == "__main__":
    main()
