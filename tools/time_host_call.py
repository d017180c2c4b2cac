#!/usr/bin/env python
"""Host time of the nine headline batch calls (bench.py's step: census1881, weather_sept_85,
wikileaks-noquotes x AND / OR / XOR over all pairs), split by phase of rb200_batch_op.

Needs the timing variant of the library, which records every call's phases:

    python -m croaring_b200.build -DRB200_HOST_TIMING --out=/tmp/rb200_timing.so
    RB200_LIB=/tmp/rb200_timing.so python tools/time_host_call.py --steps 30 --warmup 5

Prints one JSON line: per phase the median and p90 host us per call (over every call of the timed
steps), the same per (dataset, op), the median step time (CUDA events, L2 flushed between steps as in
bench.py) and `head_idle_us`, the host time from the start of a step until the first call has
enqueued its pair-list copy, the first device work of the step: the device is idle that long.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import croaring_b200 as rb  # noqa: E402

DATASETS = ["census1881", "weather_sept_85", "wikileaks-noquotes"]
OPS = ["and", "or", "xor"]
# the order of the phase durations in a record (rb200_host.cu, HostTiming)
PHASES = ["checks", "staging", "pair_loop", "copy_enqueue", "items_block", "set_new", "call_begin",
          "launches", "finish"]


def take(L):
    n = L.rb200_host_timing_take(None, 0)
    buf = (C.c_double * max(n, 1))()
    L.rb200_host_timing_take(buf, n)
    return np.frombuffer(buf, dtype=np.float64, count=n).reshape(-1, 2 + len(PHASES)).copy()


def stats(us):
    return {"median": round(float(np.median(us)), 2), "p90": round(float(np.percentile(us, 90)), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--tag", default=os.path.basename(os.environ.get("RB200_LIB", "product")))
    a = ap.parse_args()
    L = rb.lib()
    if not hasattr(L, "rb200_host_timing_take"):
        sys.exit("time_host_call: the library has no phase timing; build it with -DRB200_HOST_TIMING "
                 "and point RB200_LIB at it")
    L.rb200_host_timing_take.restype = C.c_size_t
    L.rb200_host_timing_take.argtypes = [C.c_void_p, C.c_size_t]
    rb.init(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    rb.set_stream(stream.cuda_stream)
    sets, pairs = {}, {}
    for ds in DATASETS:
        blobs = rb.load_realdata(ds)
        sets[ds] = rb.DeviceSet.from_serialized(blobs)
        i, j = np.triu_indices(len(blobs), 1)
        pairs[ds] = (i.astype(np.uint32), j.astype(np.uint32))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    d_chk = torch.zeros(1, dtype=torch.int64, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    recs, step_ms, head_us = [], [], []
    for it in range(a.warmup + a.steps):
        flush.zero_()
        torch.cuda.synchronize()
        take(L)
        d_chk.zero_()
        torch.cuda.synchronize()
        e0.record(stream)
        t0 = time.perf_counter()   # CLOCK_MONOTONIC, the clock of the records
        res = []
        for ds in DATASETS:
            ia, ib = pairs[ds]
            for op in OPS:
                r = sets[ds].batch(op, sets[ds], ia, ib)
                r.add_cardinality_device(d_chk.data_ptr())
                res.append(r)
        e1.record(stream)
        torch.cuda.synchronize()
        rec = take(L)
        for r in res:
            r.free()
        if len(rec) != len(DATASETS) * len(OPS):
            sys.exit(f"time_host_call: {len(rec)} batch calls recorded in a step, expected 9")
        if it >= a.warmup:
            recs.append(rec)
            step_ms.append(e0.elapsed_time(e1))
            head_us.append((rec[0, 1] - t0) * 1e6)
    R = np.stack(recs)                       # steps x 9 calls x (2 + phases)
    ph_us = R[:, :, 2:] * 1e6
    out = {"tag": a.tag, "steps": a.steps, "gpu": torch.cuda.get_device_name(0),
           "host_us_per_call": stats(ph_us.sum(axis=2).ravel()),
           "phases_us": {p: stats(ph_us[:, :, k].ravel()) for k, p in enumerate(PHASES)},
           "per_call_us": {f"{ds}/{op}": stats(ph_us[:, d * len(OPS) + o, :].sum(axis=1))
                           for d, ds in enumerate(DATASETS) for o, op in enumerate(OPS)},
           "host_us_per_step": stats(ph_us.sum(axis=(1, 2))),
           "head_idle_us": stats(np.array(head_us)),
           "step_ms": stats(np.array(step_ms))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
