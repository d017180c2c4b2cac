#!/usr/bin/env python
"""Wall time of every bulk download path for the library RB200_LIB points at (default: the product
build), on the all-pairs OR and XOR results of weather_sept_85 (19 900 bitmaps each), from an
unbound and a host-bound input set: download_all, download_begin/next/end, foreach, foreach_many
and foreach_async + download_wait.  Median of --reps after one warm-up; the paths take turns within
each repetition.  Freeing the downloaded bitmaps is not timed for download_all; the streaming
download frees each chunk as it goes, as its callers do.  One JSON line."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import croaring_b200 as rb  # noqa: E402


def paths(R):
    lib = rb.api.lib()
    n = len(R)
    visit = C.cast(lib.rb200_visit_sum_cardinality, C.c_void_p)

    def download_all():
        out = (C.c_void_p * n)()
        t0 = time.perf_counter()
        assert lib.rb200_set_download_all(R.ptr, out) == 0, rb.last_error()
        dt = time.perf_counter() - t0
        lib.rb200_bitmaps_free(out, n)
        return dt

    def download_stream():
        t0 = time.perf_counter()
        st = lib.rb200_download_begin(R.ptr, 4096)
        assert st, rb.last_error()
        out = (C.c_void_p * max(1, lib.rb200_download_chunk_capacity(st)))()
        while True:
            m = lib.rb200_download_next(st, out)
            assert m != 2 ** 64 - 1, rb.last_error()
            if m == 0:
                break
            lib.rb200_bitmaps_free(out, m)
        lib.rb200_download_end(st)
        return time.perf_counter() - t0

    def foreach():
        acc = C.c_uint64(0)
        t0 = time.perf_counter()
        assert lib.rb200_download_foreach(R.ptr, visit, C.byref(acc)) == 0, rb.last_error()
        return time.perf_counter() - t0

    def foreach_many():
        acc = C.c_uint64(0)
        sets = (C.c_void_p * 1)(R.ptr)
        t0 = time.perf_counter()
        assert lib.rb200_download_foreach_many(sets, 1, visit, C.byref(acc)) == 0, rb.last_error()
        return time.perf_counter() - t0

    def foreach_async():
        acc = rb.CardinalitySum()
        t0 = time.perf_counter()
        R.foreach_async(acc)
        rb.download_wait()
        return time.perf_counter() - t0

    return {f.__name__: f for f in (download_all, download_stream, foreach, foreach_many, foreach_async)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--tag", default=os.path.basename(os.environ.get("RB200_LIB", "product")))
    a = ap.parse_args()
    rb.init(0)
    lib = rb.api.lib()
    blobs = rb.load_realdata("weather_sept_85")
    host = [rb.Bitmap.deserialize(b) for b in blobs]
    i, j = np.triu_indices(len(blobs), 1)
    ia, ib = i.astype(np.uint32), j.astype(np.uint32)
    out = {"tag": a.tag, "reps": a.reps, "host_threads": os.environ.get("RB200_HOST_THREADS", "default"),
           "ms": {}, "d2h_bytes": {}}
    for bound in (False, True):
        S = rb.DeviceSet.upload(host).bind_host() if bound else rb.DeviceSet.from_serialized(blobs)
        for op in ("or", "xor"):
            R = S.batch(op, S, ia, ib)
            fns = paths(R)
            times = {name: [] for name in fns}
            for rep in range(a.reps + 1):
                for name, f in fns.items():
                    dt = f()
                    if rep:
                        times[name].append(dt)
                    out["d2h_bytes"][f"{op}/{'bound' if bound else 'unbound'}/{name}"] = \
                        int(lib.rb200_last_download_bytes())
            for name, ts in times.items():
                out["ms"][f"{op}/{'bound' if bound else 'unbound'}/{name}"] = round(float(np.median(ts)) * 1e3, 2)
            R.free()
        S.free()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
