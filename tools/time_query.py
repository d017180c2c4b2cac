#!/usr/bin/env python
"""Time of DeviceSet.contains / rank / select (rb200_batch_query: roaring_bitmap_contains / rank / select, one
value per query, against a resident set) and the reference's rank baseline.

One JSON line for the card (name, power limit, max SM clock), then one per real-data set and kind:
  queries        10^6 seeded queries over the set's bitmaps (drawn uniformly): half present values of their
                 bitmap and half uniform below its largest value + 1; select: half ranks below the bitmap's
                 cardinality and half uniform below twice it + 1
  call_ms        median over --reps calls of the whole call, host values and indices in, answers out, timed
                 on the host around the call, which ends in a stream synchronise
  kernel_ms      median device time of the query kernel (torch.profiler, CUDA activity, in a pass of its own
                 after the timed one; the prefix cardinalities were built by the warm-up call)
  ref_ms         rank only: roaring_bitmap_rank_many of every bitmap over its queries sorted, one thread.  The
                 reference has no bulk contains or select, and a ctypes loop over single calls would time
                 ctypes, so those lines carry none
  parity         every answer equals the reference's: rank against roaring_bitmap_rank_many, contains and
                 select against the values the reference holds for each bitmap (to_uint32_array)
"""
import argparse
import ctypes as C
import json
import os
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


def workload(arrays, kind, seed):
    """(idx, vals) of NQ queries."""
    rng = np.random.default_rng(seed)
    cards = np.array([a.size for a in arrays], dtype=np.int64)
    idx = rng.integers(0, len(arrays), NQ)
    idx[:NQ // 2] = rng.choice(np.flatnonzero(cards), NQ // 2)   # present values need a non-empty bitmap
    c = cards[idx]
    if kind == "select":
        vals = np.where(np.arange(NQ) < NQ // 2, rng.integers(0, np.maximum(c, 1)), rng.integers(0, 2 * c + 1))
    else:
        top = np.array([int(a[-1]) + 1 if a.size else 1 << 16 for a in arrays], dtype=np.int64)[idx]
        off = np.r_[0, np.cumsum(cards)]
        flat = np.concatenate(arrays)
        present = flat[off[idx[:NQ // 2]] + rng.integers(0, c[:NQ // 2])]
        vals = np.concatenate([present, rng.integers(0, top[NQ // 2:])])
    return idx.astype(np.uint32), vals.astype(np.uint32)


def expected(arrays, kind, idx, vals):
    """contains / select answers from each bitmap's values."""
    out = np.empty(idx.size, dtype=np.int64)
    for b in np.unique(idx):
        m = idx == b
        a, v = arrays[b].astype(np.int64), vals[m].astype(np.int64)
        if kind == "select":
            out[m] = np.where(v < a.size, a[np.minimum(v, max(a.size - 1, 0))] if a.size else -1, -1)
        else:
            p = np.searchsorted(a, v)
            out[m] = (p < a.size) & (a[np.minimum(p, max(a.size - 1, 0))] == v) if a.size else 0
    return out


def ref_rank_many(R, blobs, idx, vals):
    """(answers, ms): roaring_bitmap_rank_many per bitmap over its queries sorted, one thread."""
    L = R.L
    L.roaring_bitmap_rank_many.restype = None
    L.roaring_bitmap_rank_many.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    order = np.lexsort((vals, idx))
    si, sv = idx[order], np.ascontiguousarray(vals[order])
    ans = np.empty(NQ, dtype=np.uint64)
    bounds = np.r_[0, np.flatnonzero(np.diff(si)) + 1, NQ]
    ms = 0.0
    for lo, hi in zip(bounds[:-1].tolist(), bounds[1:].tolist()):
        r = R.deserialize(blobs[si[lo]])
        t0 = time.perf_counter()
        L.roaring_bitmap_rank_many(r, sv.ctypes.data + 4 * lo, sv.ctypes.data + 4 * hi, ans.ctypes.data + 8 * lo)
        ms += (time.perf_counter() - t0) * 1e3
        R.free(r)
    out = np.empty(NQ, dtype=np.int64)
    out[order] = ans.astype(np.int64)
    return out, ms


def kernel_ms(fn, reps):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
    ts = [e.device_time for e in prof.events() if "k_query" in e.name and e.device_time > 0]
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
        blobs = rb.load_realdata(ds)
        ptrs = [R.deserialize(b) for b in blobs]
        arrays = [R.to_array(p) for p in ptrs]
        for p in ptrs:
            R.free(p)
        S = rb.DeviceSet.from_serialized(blobs)
        for j, kind in enumerate(("contains", "rank", "select")):
            idx, vals = workload(arrays, kind, 1000 * len(ds) + j)
            fn = getattr(S, kind)
            got = fn(vals, idx=idx)   # warm: pools, modules, prefix cardinalities
            call = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                fn(vals, idx=idx)
                call.append((time.perf_counter() - t0) * 1e3)
            line = {"workload": f"{ds} {kind}", "bitmaps": len(blobs), "queries": NQ,
                    "call_ms": round(float(np.median(call)), 4),
                    "kernel_ms": kernel_ms(lambda: fn(vals, idx=idx), min(a.reps, 5))}
            if kind == "rank":
                exp, ms = ref_rank_many(R, blobs, idx, vals)
                line["ref_ms"] = round(ms, 3)
            else:
                exp = expected(arrays, kind, idx, vals)
            line["parity"] = bool((got == exp).all())
            print(json.dumps(line), flush=True)
        S.free()


if __name__ == "__main__":
    main()
