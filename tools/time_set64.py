#!/usr/bin/env python
"""Warm call times of the resident 64-bit sets (rb200_set64_*, DeviceSet64).

One JSON line for the card (name, power limit), then one per measurement:
  resident  all-pairs AND / OR / XOR over a real-data set whose every bitmap is copied into 4 high-32
            buckets (0, 1, 0x10000, 0xFFFFFFFF), median of --reps warm calls, each ending in a
            synchronise of the library stream:
              resident_ms            rb200_set64_batch_op on a resident set (result stays on the device)
              resident_serialize_ms  the same + rb200_set64_serialize (the result's bytes on the host)
              per_call_ms            rb200_r64_batch_op_serialized (parse, upload, op, serialize, all in one call)
              ref_ms / ref_pairs     the reference's roaring64_bitmap_<op>, single thread, on the first
                                     ref_pairs pairs (deserialized objects in, objects out)
              parity                 resident and per-call bytes agree, and match the reference on its pairs
  builder   rb200_set64_from_uint64 (host input) / _device (CUDA tensor input) on 200 Zipfian bitmaps of
            10^7 values (bench.py's family) mapped to 64 bits as ((v >> s) << 32) | v, s = bits of the
            universe - 2, so the values of every bitmap spread over 4 buckets, sorted and shuffled per
            bitmap; parity against the
            reference's roaring64_bitmap_of_ptr on the first --ref-bitmaps bitmaps
  ab        with --ab LIB_A,LIB_B: the roaring64_bitmap_and drop-in symbol (median of 200 calls) and one
            rb200_r64_batch_op_serialized call (all-pairs AND of census1881 in 4 buckets, median of --reps)
            for two builds of the library, in fresh processes, alternating for --ab-rounds rounds
"""
import argparse
import ctypes as C
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

DATASETS = ["census1881", "weather_sept_85", "wikileaks-noquotes",
            "census1881_srt", "wikileaks-noquotes_srt", "uscensus2000"]
HIGHS = (0, 1, 0x10000, 0xFFFFFFFF)
OPS = {"and": 0, "or": 1, "xor": 2, "andnot": 3}


def spread_blobs(R, ds):
    import croaring_b200 as rb
    out = []
    for b in rb.load_realdata(ds):
        r = R.deserialize(b)
        v = R.to_array(r).astype(np.uint64)
        R.free(r)
        out.append(R.r64_from_values(np.concatenate([v + (np.uint64(h) << np.uint64(32)) for h in HIGHS])))
    return out


class SerializedCall:
    """rb200_r64_batch_op_serialized through plain ctypes on library L (any build of it)."""

    def __init__(self, L, blobs):
        n = len(blobs)
        self.L = L
        self.keep = blobs
        self.ptrs = (C.c_char_p * n)(*blobs)
        self.lens = (C.c_size_t * n)(*[len(b) for b in blobs])
        self.n = n
        f = L.rb200_r64_batch_op_serialized
        f.restype = C.c_int
        f.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                      C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rb200_serialized_free.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.rb200_serialized_free.restype = None

    def __call__(self, op, ia, ib, digest=False):
        buf, off, ln = C.c_void_p(), C.POINTER(C.c_uint64)(), C.POINTER(C.c_uint64)()
        rc = self.L.rb200_r64_batch_op_serialized(OPS[op], self.ptrs, self.lens, self.n, self.ptrs, self.lens, self.n,
                                                  ia.ctypes.data, ib.ctypes.data, ia.size, C.byref(buf),
                                                  C.byref(off), C.byref(ln))
        assert rc == 0
        h = None
        if digest:
            h = hashlib.sha256()
            for k in range(ia.size):
                h.update(C.string_at(buf.value + off[k], ln[k]))
            h = h.hexdigest()
        self.L.rb200_serialized_free(buf, off, ln)
        return h


def timed(fn, reps):
    ts = []
    for _ in range(reps + 1):   # the first call warms the pools and the shapes
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts[1:]))


def digest(blobs):
    h = hashlib.sha256()
    for b in blobs:
        h.update(b)
    return h.hexdigest()


def resident(R, a):
    import croaring_b200 as rb
    L = rb.lib()
    for ds in a.datasets.split(","):
        blobs = spread_blobs(R, ds)
        i, j = np.triu_indices(len(blobs), 1)
        ia, ib = i.astype(np.uint32), j.astype(np.uint32)
        S = rb.DeviceSet64.from_serialized(blobs)
        call = SerializedCall(L, blobs)
        objs = [R.r64_deserialize(b) for b in blobs]
        for op in ("and", "or", "xor"):
            def res_op():
                S.op(op, S, ia, ib).free()   # free waits for the op: the call ends with its work done
                rb.synchronize()
            res_ms = timed(res_op, a.reps)
            def res_serialize():
                R64 = S.op(op, S, ia, ib)
                buf, off, ln = C.c_void_p(), C.POINTER(C.c_uint64)(), C.POINTER(C.c_uint64)()
                assert L.rb200_set64_serialize(R64.ptr, C.byref(buf), C.byref(off), C.byref(ln)) == 0
                L.rb200_serialized_free(buf, off, ln)
                R64.free()
            ser_ms = timed(res_serialize, a.reps)
            per_ms = timed(lambda: call(op, ia, ib), a.reps)
            got = S.op(op, S, ia, ib).serialize_all()
            k = min(a.ref_pairs, ia.size)
            f = getattr(R.L, f"roaring64_bitmap_{op}")
            t0 = time.perf_counter()
            outs = [f(objs[ia[p]], objs[ib[p]]) for p in range(k)]
            ref_ms = (time.perf_counter() - t0) * 1e3
            ref = [R.r64_serialize(o) for o in outs]
            for o in outs:
                R.L.roaring64_bitmap_free(o)
            parity = got[:k] == ref and call(op, ia, ib, digest=True) == digest(got)
            print(json.dumps({"measure": "resident", "dataset": f"{ds} x 4 buckets", "op": op, "pairs": int(ia.size),
                              "resident_ms": round(res_ms, 3), "resident_serialize_ms": round(ser_ms, 3),
                              "per_call_ms": round(per_ms, 3), "ref_ms": round(ref_ms, 1), "ref_pairs": k,
                              "parity": parity}), flush=True)
        for o in objs:
            R.L.roaring64_bitmap_free(o)
        S.free()


def builder(R, a):
    import torch
    import croaring_b200 as rb
    import croaring_b200.workloads as wl
    rng = np.random.default_rng(0)
    for d in [float(x) for x in a.densities.split(",") if x]:
        U = wl.zipf_universe(a.zipf_values, d)
        A = wl.zipf_arena(a.zipf_bitmaps, U, a.zipf_values, run_optimize=False)
        S32 = rb.DeviceSet.from_serialized(A)
        A.free()
        vals = S32.to_uint32_arrays()
        S32.free()
        off = np.zeros(len(vals) + 1, dtype=np.uint64)
        np.cumsum([len(v) for v in vals], out=off[1:])
        flat = np.empty(int(off[-1]), dtype=np.uint64)
        shift = np.uint64(max(0, (U - 1).bit_length() - 2))
        for k, v in enumerate(vals):
            w = flat[off[k]:off[k + 1]]
            w[:] = v
            w |= (w >> shift) << np.uint64(32)
        del vals
        N = int(off[-1])
        buckets = len(np.unique(flat[::997] >> np.uint64(32)))
        for order in ("sorted", "shuffled"):
            if order == "shuffled":
                for k in range(len(off) - 1):
                    rng.shuffle(flat[off[k]:off[k + 1]])
            host_ms = timed(lambda: rb.DeviceSet64.from_values(flat, off).free(), a.reps)
            host = rb.DeviceSet64.from_values(flat, off)
            t_vals = torch.from_numpy(flat.view(np.int64)).cuda()
            t_off = torch.from_numpy(off.astype(np.int64)).cuda()
            torch.cuda.current_stream().synchronize()
            dev_ms = timed(lambda: rb.DeviceSet64.from_values(t_vals, t_off).free(), a.reps)
            dev = rb.DeviceSet64.from_values(t_vals, t_off)
            del t_vals, t_off
            hb, db = host.serialize_all(), dev.serialize_all()
            host.free()
            dev.free()
            k = min(a.ref_bitmaps, len(off) - 1)
            ref = [R.r64_from_values(flat[off[i]:off[i + 1]], run_optimize=False) for i in range(k)]
            print(json.dumps({"measure": "builder", "workload": f"zipf d={d} {order}", "bitmaps": len(off) - 1,
                              "values": N, "buckets_seen": buckets, "host_ms": round(host_ms, 2),
                              "device_ms": round(dev_ms, 2), "device_gbs": round(8 * N / dev_ms / 1e6, 1),
                              "parity": hb == db and hb[:k] == ref, "ref_bitmaps": k}), flush=True)
            del hb, db
        del flat


AB_WORKER = r'''
import ctypes as C, json, os, sys, time
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tools"))
G = C.CDLL(os.path.join(sys.argv[1], "oracle", "_ref", "libroaring_ref.so"), mode=os.RTLD_GLOBAL)
from oracle.refbind import ref
import time_set64 as T
R = ref()
L = C.CDLL(sys.argv[2], mode=os.RTLD_LOCAL)
assert L.rb200_init(0) == 0
reps = int(sys.argv[3])
blobs = T.spread_blobs(R, "census1881")
objs = [R.r64_deserialize(b) for b in blobs]
L.roaring64_bitmap_and.restype = C.c_void_p
L.roaring64_bitmap_and.argtypes = [C.c_void_p, C.c_void_p]
ts = []
for rep in range(220):
    t0 = time.perf_counter()
    o = L.roaring64_bitmap_and(objs[rep % 50], objs[(rep % 50) + 1])
    ts.append((time.perf_counter() - t0) * 1e6)
    assert o
    R.L.roaring64_bitmap_free(o)
call = T.SerializedCall(L, blobs)
i, j = np.triu_indices(len(blobs), 1)
ia, ib = i.astype(np.uint32), j.astype(np.uint32)
ser_ms = T.timed(lambda: call("and", ia, ib), reps)
print(json.dumps({"dropin_and_us": round(float(np.median(ts[20:])), 1), "serialized_and_ms": round(ser_ms, 3),
                  "sha": call("and", ia, ib, digest=True)}))
'''


def ab(a):
    libs = a.ab.split(",")
    rows = {lib: [] for lib in libs}
    for _ in range(a.ab_rounds):
        for lib in libs:
            p = subprocess.run([sys.executable, "-c", AB_WORKER, ROOT, os.path.abspath(lib), str(a.reps)],
                               capture_output=True, text=True, timeout=900)
            assert p.returncode == 0, p.stderr[-2000:]
            rows[lib].append(json.loads(p.stdout.strip().splitlines()[-1]))
    for lib in libs:
        d = [r["dropin_and_us"] for r in rows[lib]]
        s = [r["serialized_and_ms"] for r in rows[lib]]
        print(json.dumps({"measure": "ab", "lib": lib, "dropin_and_us": d, "serialized_and_ms": s,
                          "dropin_and_us_median": float(np.median(d)), "serialized_and_ms_median": float(np.median(s)),
                          "sha": sorted({r["sha"] for r in rows[lib]})}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--datasets", default=",".join(DATASETS))
    ap.add_argument("--ref-pairs", type=int, default=500)
    ap.add_argument("--zipf-bitmaps", type=int, default=200)
    ap.add_argument("--zipf-values", type=int, default=10_000_000)
    ap.add_argument("--densities", default="0.01")
    ap.add_argument("--ref-bitmaps", type=int, default=3)
    ap.add_argument("--skip", default="", help="comma list of resident,builder")
    ap.add_argument("--ab", default="", help="LIB_A,LIB_B: compare two builds of the library")
    ap.add_argument("--ab-rounds", type=int, default=4)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"gpu": card}), flush=True)
    if a.ab:
        ab(a)
    skip = set(a.skip.split(","))
    if {"resident", "builder"} <= skip:
        return
    import croaring_b200 as rb
    from oracle.refbind import ref
    rb.init(0)
    R = ref()
    if "resident" not in skip:
        resident(R, a)
    if "builder" not in skip:
        builder(R, a)


if __name__ == "__main__":
    main()
