#!/usr/bin/env python
"""Time of DeviceSet64.contains / rank / get_index / select (rb200_set64_batch_query: roaring64_bitmap_contains /
rank / get_index / select, one value per query, against a resident 64-bit set).

One JSON line for the card (name, power limit, max SM clock), then one per real-data set and kind:
  set            the set's bitmaps with their 32-bit values copied into the high-32 buckets 0, 1, 2^16 and
                 2^32 - 1, so every bitmap spans four buckets
  queries        10^6 seeded queries over the set's bitmaps (drawn uniformly): half present values of their
                 bitmap and half uniform below its largest value + 1; select: half ranks below the bitmap's
                 cardinality and half uniform below twice it + 1
  call_ms        median over --reps calls of the whole call, host values and indices in, answers and found
                 flags out, timed on the host around the call, which ends in a stream synchronise
  kernel_ms      median device time of k_query64 (torch.profiler, CUDA activity, in a pass of its own after the
                 timed one; the prefix cardinalities were built by the warm-up call)
  parity         every answer and found flag equals what the reference's roaring64 query returns, computed from
                 the values the reference holds for each bitmap (roaring64_bitmap_to_uint64_array)
There is no reference baseline: the reference has no bulk 64-bit rank (nor contains or select), and a ctypes loop
over single calls would time ctypes.
"""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import croaring_b200 as rb  # noqa: E402
from helpers import DATASETS  # noqa: E402
from oracle.refbind import ref  # noqa: E402

NQ = 1_000_000
HIGHS = (0, 1, 0x10000, 0xFFFFFFFF)
KINDS = ("contains", "rank", "get_index", "select")
T64 = np.uint64((1 << 64) - 1)


def spread_blobs(R, blobs):
    """(64-bit blobs, sorted uint64 values per bitmap): every bitmap's values in each bucket of HIGHS."""
    out, arrays = [], []
    for b in blobs:
        r = R.deserialize(b)
        v32 = R.to_array(r).astype(np.uint64)
        R.free(r)
        v = np.concatenate([v32 + (np.uint64(h) << np.uint64(32)) for h in HIGHS])
        out.append(R.r64_from_values(v))
        arrays.append(ref_values(R, out[-1]))
    return out, arrays


def ref_values(R, blob):
    L = R.L
    L.roaring64_bitmap_to_uint64_array.restype = None
    L.roaring64_bitmap_to_uint64_array.argtypes = [C.c_void_p, C.c_void_p]
    r = R.r64_deserialize(blob)
    a = np.empty(int(L.roaring64_bitmap_get_cardinality(r)), dtype=np.uint64)
    if a.size:
        L.roaring64_bitmap_to_uint64_array(r, a.ctypes.data)
    L.roaring64_bitmap_free(r)
    return a


def workload(arrays, kind, seed):
    """(idx, vals) of NQ queries."""
    rng = np.random.default_rng(seed)
    cards = np.array([a.size for a in arrays], dtype=np.int64)
    idx = rng.integers(0, len(arrays), NQ)
    idx[:NQ // 2] = rng.choice(np.flatnonzero(cards), NQ // 2)   # present values need a non-empty bitmap
    c = cards[idx]
    if kind == "select":
        vals = np.where(np.arange(NQ) < NQ // 2, rng.integers(0, np.maximum(c, 1)), rng.integers(0, 2 * c + 1))
        return idx.astype(np.uint32), vals.astype(np.uint64)
    top = np.array([a[-1] if a.size else np.uint64(1 << 16) for a in arrays], dtype=np.uint64)[idx]
    off = np.r_[0, np.cumsum(cards)]
    flat = np.concatenate(arrays)
    present = flat[off[idx[:NQ // 2]] + rng.integers(0, c[:NQ // 2])]
    uniform = rng.integers(0, top[NQ // 2:], dtype=np.uint64, endpoint=True)
    return idx.astype(np.uint32), np.concatenate([present, uniform])


def expected(arrays, kind, idx, vals):
    """(out, found) of every query from each bitmap's values, as the reference's roaring64 query returns them."""
    out, found = np.empty(idx.size, dtype=np.uint64), np.empty(idx.size, dtype=bool)
    for b in np.unique(idx):
        m = idx == b
        a, v = arrays[b], vals[m]
        if kind == "select":
            f = v < np.uint64(a.size)
            o = np.where(f, a[np.minimum(v, np.uint64(max(a.size - 1, 0)))] if a.size else T64, T64)
        else:
            p = np.searchsorted(a, v, side="right")   # values <= v
            hit = (p > 0) & (a[np.maximum(p - 1, 0)] == v) if a.size else np.zeros(v.size, bool)
            f = hit if kind != "rank" else np.ones(v.size, bool)
            o = {"contains": hit.astype(np.uint64), "rank": p.astype(np.uint64),
                 "get_index": np.where(hit, (p - 1).astype(np.uint64), T64)}[kind]
        out[m], found[m] = o, f
    return out, found


def kernel_ms(fn, reps):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
    ts = [e.device_time for e in prof.events() if re.search(r"k_query64(<|I)", e.name) and e.device_time > 0]
    return round(float(np.median(ts)) / 1e3, 4) if ts else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"gpu": card}), flush=True)
    rb.init(0)
    R = ref()
    for ds in DATASETS:
        blobs, arrays = spread_blobs(R, rb.load_realdata(ds))
        S = rb.DeviceSet64.from_serialized(blobs)
        for j, kind in enumerate(KINDS):
            idx, vals = workload(arrays, kind, 1000 * len(ds) + j)
            fn = lambda: rb.api._query64(S, kind, vals, idx)   # noqa: E731
            got, found = fn()   # warm: pools, modules, prefix cardinalities
            call = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                fn()
                call.append((time.perf_counter() - t0) * 1e3)
            exp, exp_found = expected(arrays, kind, idx, vals)
            line = {"workload": f"{ds} {kind}", "bitmaps": len(blobs), "buckets": len(HIGHS), "queries": NQ,
                    "call_ms": round(float(np.median(call)), 4), "kernel_ms": kernel_ms(fn, min(a.reps, 5)),
                    "parity": bool((got == exp).all() and (found == exp_found).all())}
            print(json.dumps(line), flush=True)
        S.free()


if __name__ == "__main__":
    main()
