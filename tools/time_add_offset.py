#!/usr/bin/env python
"""Device time of DeviceSet.add_offset (rb200_batch_add_offset: roaring_bitmap_add_offset of a whole
resident set) against the reference's single-threaded roaring_bitmap_add_offset.

One JSON line for the card (name, power limit, max SM clock), then one per workload:
  device_ms      median over --reps calls of the op's device time (CUDA events on the library stream,
                 from the op's first to its last enqueued work), the L2 flushed before every call by
                 writing a buffer larger than it on the same stream
  algo_bytes     the op's algorithmic bytes (rb200_set_op_stats): container_size_in_bytes of every
                 source container that contributes a computed part, plus every computed output
  algo_gbs       algo_bytes / device_ms, and hbm_share: that rate over 3.35 TB/s
  ref_ms         the reference's add_offset summed over the same bitmaps (deserialisation excluded)
  parity         sha256 of the serialized results == that of the reference's
Workloads: every bitmap of each real-data set, shifted by a split offset (12345) and a key-aligned
one (7 x 65536).
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
from offset_oracles import ref_add_offset  # noqa: E402
from oracle.refbind import ref  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
OFFSETS = [12345, 7 * 65536]


def ref_results(R, blobs, off):
    h, ms, add_offset = hashlib.sha256(), 0.0, ref_add_offset(R)
    for b in blobs:
        r = R.deserialize(b)
        t0 = time.perf_counter()
        x = add_offset(r, off)
        ms += (time.perf_counter() - t0) * 1e3
        h.update(R.serialize(x))
        R.free(x)
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
        for off in OFFSETS:
            X = S.add_offset(off)   # warm: pools, modules
            got = hashlib.sha256(b"".join(X.serialize_all())).hexdigest()
            X.free()
            ms, ab = [], 0
            for _ in range(a.reps):
                flush.zero_()
                X = S.add_offset(off)
                d_ms, _, ab = X.op_stats()
                ms.append(d_ms)
                X.free()
            sha, ref_ms = ref_results(R, blobs, off)
            dev = float(np.median(ms))
            gbs = ab / dev / 1e6 if dev > 0 else 0.0
            print(json.dumps({"workload": f"{ds} offset {off}", "bitmaps": len(blobs),
                              "containers": S.container_count, "device_ms": round(dev, 4),
                              "algo_bytes": ab, "algo_gbs": round(gbs, 1),
                              "hbm_share": round(gbs * 1e9 / HBM_BYTES_PER_S, 4),
                              "ref_ms": round(ref_ms, 2), "parity": got == sha}), flush=True)
        S.free()


if __name__ == "__main__":
    main()
