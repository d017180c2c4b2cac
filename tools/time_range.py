#!/usr/bin/env python
"""Time of DeviceSet.add_range / remove_range (rb200_batch_add_range_closed / remove_range_closed:
roaring_bitmap_add_range_closed / remove_range_closed of every bitmap of a resident set, one range per bitmap)
against the reference's single-threaded calls.

One JSON line for the card (name, power limit, max SM clock), then one per workload:
  call_ms        median over --reps calls of the whole call, host ranges in, resident result out, timed on
                 the host around the call and a stream synchronise; the L2 flushed before every call by
                 writing a buffer larger than it on the library stream
  op_ms          median device time of the call's kernels (rb200_set_op_stats: from the plan's start to the
                 end of the directory's compaction)
  ref_ms         the reference's add_range_closed / remove_range_closed summed over the same bitmaps and
                 ranges, one thread, on copies made outside the timed window
  parity         sha256 of the serialized results == that of the reference's
Workloads: every bitmap of each real-data set, with one range per bitmap of each width: inside one key (1000
values from just above its smallest value), one key exactly (the key of its median value), 256 keys (from
just above its smallest value) and the whole 32-bit universe.
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
from helpers import DATASETS  # noqa: E402
from oracle.refbind import ref  # noqa: E402
from range_oracles import ref_range  # noqa: E402

T32 = (1 << 32) - 1
WIDTHS = ["inside_key", "one_key", "256_keys", "universe"]


def ranges(R, blobs, width):
    """Closed (lo, hi) arrays, one range per bitmap."""
    lo, hi = [], []
    for b in blobs:
        r = R.deserialize(b)
        v = R.to_array(r)
        R.free(r)
        first = int(v[0]) if v.size else 0
        if width == "inside_key":
            a = first + 1
            z = min(a + 999, (a | 0xFFFF))
        elif width == "one_key":
            k = (int(v[v.size // 2]) >> 16) if v.size else 0
            a, z = k << 16, (k << 16) + 0xFFFF
        elif width == "256_keys":
            a = first + 1
            z = min(a + (256 << 16) - 1, T32)
        else:
            a, z = 0, T32
        lo.append(a)
        hi.append(z)
    return np.array(lo, np.uint32), np.array(hi, np.uint32)


def ref_results(R, blobs, op, lo, hi):
    h, ms, fn = hashlib.sha256(), 0.0, ref_range(R, op)
    copies = [R.deserialize(b) for b in blobs]
    for r, a, z in zip(copies, lo.tolist(), hi.tolist()):
        t0 = time.perf_counter()
        fn(r, a, z)
        ms += (time.perf_counter() - t0) * 1e3
    for r in copies:
        h.update(R.serialize(r))
        R.free(r)
    return h.hexdigest(), ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"gpu": card}), flush=True)
    rb.init(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    rb.set_stream(stream.cuda_stream)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > the 50 MB L2
    L = rb.lib()
    R = ref()
    for ds in DATASETS:
        blobs = rb.load_realdata(ds)
        S = rb.DeviceSet.from_serialized(blobs)
        n = len(blobs)
        for op in ("add", "remove"):
            fn = getattr(L, f"rb200_batch_{op}_range_closed")
            for width in WIDTHS:
                lo, hi = ranges(R, blobs, width)
                X = rb.DeviceSet(fn(S.ptr, None, n, lo.ctypes.data, hi.ctypes.data))   # warm: pools, modules
                got = hashlib.sha256(b"".join(X.serialize_all())).hexdigest()
                X.free()
                call, opm = [], []
                for _ in range(a.reps):
                    flush.zero_()
                    stream.synchronize()
                    t0 = time.perf_counter()
                    X = rb.DeviceSet(fn(S.ptr, None, n, lo.ctypes.data, hi.ctypes.data))
                    rb.synchronize()
                    call.append((time.perf_counter() - t0) * 1e3)
                    opm.append(X.op_stats()[0])
                    X.free()
                sha, ref_ms = ref_results(R, blobs, op, lo, hi)
                print(json.dumps({"workload": f"{ds} {op}_range {width}", "bitmaps": n,
                                  "call_ms": round(float(np.median(call)), 4), "op_ms": round(float(np.median(opm)), 4),
                                  "ref_ms": round(ref_ms, 3), "parity": got == sha}), flush=True)
        S.free()


if __name__ == "__main__":
    main()
