#!/usr/bin/env python
"""Time of DeviceSet.add_many / remove_many (rb200_batch_add_many / remove_many: roaring_bitmap_add_many /
remove_many of every bitmap of a resident set) against the reference's single-threaded calls.

One JSON line for the card (name, power limit, max SM clock), then one per workload:
  call_ms        median over --reps calls of the whole call, host values in, resident result out: the
                 values' upload and bitmap build, the update and the result's counters, timed on the host
                 around the call and a stream synchronise; the L2 flushed before every call by writing a
                 buffer larger than it on the library stream
  op_ms          median device time of the update's batch op alone (rb200_set_op_stats: CUDA events from
                 its first to its last enqueued work)
  algo_bytes     the batch op's algorithmic bytes (container_size_in_bytes of the containers a computed
                 cell reads and writes; shared containers move nothing)
  ref_ms         the reference's add_many / remove_many summed over the same bitmaps and values, one
                 thread (deserialisation excluded)
  parity         sha256 of the serialized results == that of the reference's
Workloads: every bitmap of each real-data set, updated with 1 % and 10 % of its cardinality (seeded):
adds drawn uniformly below its largest value, removals drawn from its values.
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
from update_oracles import ref_update  # noqa: E402

FRACTIONS = [0.01, 0.10]


def value_lists(R, blobs, op, frac, seed):
    rng = np.random.default_rng(seed)
    out = []
    for b in blobs:
        r = R.deserialize(b)
        have = R.to_array(r)
        R.free(r)
        m = max(1, int(have.size * frac))
        if op == "add":
            out.append(rng.integers(0, int(have[-1]) + 2 if have.size else 1 << 20, m).astype(np.uint32))
        else:
            out.append(rng.choice(have, size=min(m, have.size), replace=False).astype(np.uint32) if have.size
                       else np.zeros(0, np.uint32))
    return out


def ref_results(R, blobs, op, lists):
    h, ms, fn = hashlib.sha256(), 0.0, ref_update(R, op)
    for b, v in zip(blobs, lists):
        r = R.deserialize(b)
        t0 = time.perf_counter()
        fn(r, v.size, v.ctypes.data)
        ms += (time.perf_counter() - t0) * 1e3
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
    R = ref()
    for ds in DATASETS:
        blobs = rb.load_realdata(ds)
        S = rb.DeviceSet.from_serialized(blobs)
        for op in ("add", "remove"):
            for frac in FRACTIONS:
                lists = value_lists(R, blobs, op, frac, 1000 * len(ds) + int(frac * 100) + (op == "add"))
                up = S.add_many if op == "add" else S.remove_many
                X = up(lists)   # warm: pools, modules
                got = hashlib.sha256(b"".join(X.serialize_all())).hexdigest()
                X.free()
                call, opm, ab = [], [], 0
                for _ in range(a.reps):
                    flush.zero_()
                    stream.synchronize()
                    t0 = time.perf_counter()
                    X = up(lists)
                    rb.synchronize()
                    call.append((time.perf_counter() - t0) * 1e3)
                    d_ms, _, ab = X.op_stats()
                    opm.append(d_ms)
                    X.free()
                sha, ref_ms = ref_results(R, blobs, op, lists)
                print(json.dumps({"workload": f"{ds} {op}_many {int(frac * 100)}%", "bitmaps": len(blobs),
                                  "values": int(sum(v.size for v in lists)),
                                  "call_ms": round(float(np.median(call)), 4), "op_ms": round(float(np.median(opm)), 4),
                                  "algo_bytes": ab, "ref_ms": round(ref_ms, 3), "parity": got == sha}), flush=True)
        S.free()


if __name__ == "__main__":
    main()
