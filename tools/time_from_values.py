#!/usr/bin/env python
"""Warm call times of DeviceSet.from_values (rb200_set_from_uint32 / _device: roaring_bitmap_of_ptr of
a whole batch on the device) against the reference's single-threaded roaring_bitmap_of_ptr.

One JSON line for the card, then one per workload:
  device_ms / host_ms   median call time with device (torch CUDA tensor) / host (numpy) input; the
                        call ends in a synchronise of the library stream
  *_gbs                 input GB/s at 4 bytes per value
  sort_ran              some bitmap's values are not non-decreasing, so the library sorts them
  parity                sha256 of the serialized set == that of the reference's of_ptr results
  ref_ms                reference of_ptr time, summed over ref_bitmaps bitmaps (all of them unless
                        --ref-limit-shuffled cuts a shuffled workload short)
Workloads: the real-data suite's values, 200 Zipfian bitmaps x 10^7 values per bench.py density
(sorted and shuffled per bitmap), 10^6 bitmaps of 16 values.
"""
import argparse
import hashlib
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
import croaring_b200.workloads as wl  # noqa: E402
from helpers import DATASETS  # noqa: E402
from oracle.refbind import ref  # noqa: E402

ZIPF_DENSITIES = [0.001, 0.003, 0.01, 0.03, 0.1, 0.3]   # bench.py's


def flat_of(arrays):
    off = np.zeros(len(arrays) + 1, dtype=np.uint64)
    np.cumsum([len(a) for a in arrays], out=off[1:])
    return np.concatenate(arrays).astype(np.uint32, copy=False), off


def sort_needed(flat, off):
    if flat.size < 2:
        return False
    dec = flat[1:] < flat[:-1]
    starts = off[1:-1][(off[1:-1] > 0) & (off[1:-1] < flat.size)].astype(np.int64)
    dec[starts - 1] = False   # a decrease across a bitmap boundary does not count
    return bool(dec.any())


def ref_results(R, flat, off, limit):
    """(sha256 of the serialized results or None, ms of of_ptr summed, bitmaps timed)"""
    h, ms, n = hashlib.sha256(), 0.0, len(off) - 1
    k = n if limit is None else min(n, limit)
    for i in range(k):
        v = np.ascontiguousarray(flat[off[i]:off[i + 1]])
        t0 = time.perf_counter()
        r = R.L.roaring_bitmap_of_ptr(v.size, v.ctypes.data)
        ms += (time.perf_counter() - t0) * 1e3
        h.update(R.serialize(r))
        R.free(r)
    return (h.hexdigest() if k == n else None), ms, k


def timed(fn, reps):
    ts = []
    for rep in range(reps + 1):   # first call warms the pools and the shapes
        t0 = time.perf_counter()
        S = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
        if rep < reps:
            S.free()
    return float(np.median(ts[1:])), S


def measure(name, flat, off, R, reps, ref_limit=None, ref_sha=None):
    N = int(off[-1])
    host_ms, S = timed(lambda: rb.DeviceSet.from_values(flat, off), reps)
    blobs = S.serialize_all()
    S.free()
    got = hashlib.sha256(b"".join(blobs)).hexdigest()
    del blobs
    t_vals = torch.from_numpy(flat.view(np.int32)).cuda()
    t_off = torch.from_numpy(off.astype(np.int64)).cuda()
    torch.cuda.current_stream().synchronize()
    dev_ms, S = timed(lambda: rb.DeviceSet.from_values(t_vals, t_off), reps)
    dev_sha = hashlib.sha256(b"".join(S.serialize_all())).hexdigest()
    S.free()
    del t_vals, t_off
    sha, ref_ms, k = ref_results(R, flat, off, ref_limit)
    exp = sha or ref_sha
    rec = {"workload": name, "bitmaps": len(off) - 1, "values": N,
           "device_ms": round(dev_ms, 3), "host_ms": round(host_ms, 3),
           "device_gbs": round(4 * N / dev_ms / 1e6, 2), "host_gbs": round(4 * N / host_ms / 1e6, 2),
           "sort_ran": sort_needed(flat, off), "parity": exp is not None and got == exp and dev_sha == exp,
           "ref_ms": round(ref_ms, 1), "ref_bitmaps": k}
    if sha is None:
        rec["parity_against"] = "reference of_ptr on the sorted values of the same bitmaps"
    print(json.dumps(rec), flush=True)
    return sha


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--zipf-bitmaps", type=int, default=200)
    ap.add_argument("--zipf-values", type=int, default=10_000_000)
    ap.add_argument("--densities", default=",".join(str(d) for d in ZIPF_DENSITIES))
    ap.add_argument("--ref-limit-shuffled", type=int, default=10,
                    help="bitmaps of a shuffled Zipf workload the reference is timed on (it runs ~20x slower "
                         "on shuffled input than on sorted)")
    ap.add_argument("--small", type=int, default=1_000_000, help="bitmaps of 16 values (0: skip)")
    ap.add_argument("--no-realdata", action="store_true")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"gpu": card}), flush=True)
    rb.init(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    rb.set_stream(stream.cuda_stream)
    R = ref()
    rng = np.random.default_rng(0)

    if not a.no_realdata:
        vals = []
        for ds in DATASETS:
            for b in rb.load_realdata(ds):
                r = R.deserialize(b)
                vals.append(R.to_array(r))
                R.free(r)
        flat, off = flat_of(vals)
        measure(f"realdata: {len(DATASETS)} sets", flat, off, R, a.reps)

    for d in [float(x) for x in a.densities.split(",") if x]:
        U = wl.zipf_universe(a.zipf_values, d)
        A = wl.zipf_arena(a.zipf_bitmaps, U, a.zipf_values, run_optimize=False)
        S = rb.DeviceSet.from_serialized(A)
        A.free()
        vals = S.to_uint32_arrays()
        S.free()
        flat, off = flat_of(vals)
        del vals
        sha = measure(f"zipf d={d} sorted", flat, off, R, a.reps)
        for i in range(len(off) - 1):
            rng.shuffle(flat[off[i]:off[i + 1]])
        measure(f"zipf d={d} shuffled", flat, off, R, a.reps, ref_limit=a.ref_limit_shuffled, ref_sha=sha)
        del flat

    if a.small:
        off = np.arange(a.small + 1, dtype=np.uint64) * 16
        flat = rng.integers(0, 1 << 32, size=16 * a.small, dtype=np.uint64).astype(np.uint32)
        measure(f"{a.small} bitmaps x 16 random values", flat, off, R, a.reps)


if __name__ == "__main__":
    main()
