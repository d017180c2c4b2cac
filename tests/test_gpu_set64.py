"""Resident 64-bit sets (DeviceSet64 / rb200_set64_*): upload, batched roaring64_bitmap_of_ptr,
pairwise ops, run_optimize and device-side 64-bit serialization, byte for byte against the
unmodified reference's roaring64 functions."""
import ctypes as C
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

import croaring_b200 as rb
from helpers import DATASETS, OPS, synth_blobs64

pytestmark = pytest.mark.gpu

HIGHS = (0, 1, 0x10000, 0xFFFFFFFF)


def _r64_run_optimize(R, blob):
    r = R.r64_deserialize(blob)
    R.L.roaring64_bitmap_run_optimize(r)
    out = R.r64_serialize(r)
    R.L.roaring64_bitmap_free(r)
    return out


def _r64_card(R, blob):
    r = R.r64_deserialize(blob)
    c = int(R.L.roaring64_bitmap_get_cardinality(r))
    R.L.roaring64_bitmap_free(r)
    return c


def _values32(R, blob):
    r = R.deserialize(blob)
    v = R.to_array(r)
    R.free(r)
    return v


def _spread(v32, highs=HIGHS):
    """The same 32-bit values in every bucket of `highs`."""
    return np.concatenate([v32.astype(np.uint64) + (np.uint64(h) << np.uint64(32)) for h in highs])


def _flat(arrays):
    off = np.zeros(len(arrays) + 1, dtype=np.uint64)
    np.cumsum([len(a) for a in arrays], out=off[1:])
    flat = np.concatenate(arrays).astype(np.uint64) if arrays else np.zeros(0, np.uint64)
    return flat, off


def _shuffled_with_dups(rng, vals):
    extra = rng.choice(vals, size=len(vals) // 3) if len(vals) else vals
    w = np.concatenate([vals, extra]).astype(np.uint64)
    rng.shuffle(w)
    return w


def test_round_trip_synthetic_and_realdata(R):
    for seed in (91, 92):
        blobs = synth_blobs64(R, seed, 60)
        S = rb.DeviceSet64.from_serialized(blobs)
        assert len(S) == 60
        assert S.serialize_all() == blobs
        assert [int(c) for c in S.cardinalities()] == [_r64_card(R, b) for b in blobs]
    for ds in DATASETS:
        blobs = [R.r64_from_values(_spread(_values32(R, b))) for b in rb.load_realdata(ds)[:30]]
        assert rb.DeviceSet64.from_serialized(blobs).serialize_all() == blobs, ds


def test_empty_bucket_is_dropped_like_the_reference(R):
    r = R.from_values(np.array([1, 2, 70000], np.uint32))
    b1 = R.serialize(r)
    R.free(r)
    empty32 = struct.pack("<II", 12346, 0)
    blob = struct.pack("<Q", 3) + struct.pack("<I", 1) + b1 + struct.pack("<I", 2) + empty32 + \
        struct.pack("<I", 9) + b1
    exp = R.r64_serialize(R.r64_deserialize(blob))
    S = rb.DeviceSet64.from_serialized([blob, struct.pack("<Q", 1) + struct.pack("<I", 4) + empty32])
    assert S.serialize_all() == [exp, struct.pack("<Q", 0)]
    assert [int(c) for c in S.cardinalities()] == [6, 0]
    # the empty bucket takes no part in an op either
    got = S.op("or", S, [0, 1], [1, 0]).serialize_all()
    assert got == [exp, exp]


def _op_blobs(R):
    blobs = synth_blobs64(R, 93, 30)
    empty = R.r64_from_values(np.zeros(0, np.uint64))
    lo = R.r64_from_values(np.arange(5000, dtype=np.uint64) * 7 + (np.uint64(3) << np.uint64(32)))
    hi = R.r64_from_values(np.arange(5000, dtype=np.uint64) * 7 + (np.uint64(4) << np.uint64(32)))
    # same bucket (high32 = 3) as lo, other 48-bit keys: the AND of the two keeps no container
    other_keys = R.r64_from_values(np.arange(300, dtype=np.uint64) + (np.uint64(3) << np.uint64(32))
                                   + np.uint64(1 << 20))
    return blobs + [empty, lo, hi, other_keys]


def test_ops_and_cardinality_distinct_and_same_sets(R):
    blobs = _op_blobs(R)
    A = rb.DeviceSet64.from_serialized(blobs[:20])
    B = rb.DeviceSet64.from_serialized(blobs[20:])
    rng = np.random.default_rng(4)
    ia = rng.integers(0, 20, 120).astype(np.uint32)
    ib = rng.integers(0, len(blobs) - 20, 120).astype(np.uint32)
    for op in OPS:
        got = A.op(op, B, ia, ib).serialize_all()
        for k in range(len(ia)):
            assert got[k] == R.r64_op_bytes(op, blobs[ia[k]], blobs[20 + ib[k]]), (op, k)
    cards = A.and_cardinality(B, ia, ib)
    assert [int(c) for c in cards] == [R.r64_and_cardinality(blobs[a], blobs[20 + b]) for a, b in zip(ia, ib)]
    S = rb.DeviceSet64.from_serialized(blobs)
    n = len(blobs)
    # every pair with the empty bitmap, disjoint buckets (lo, hi) and disjoint keys in one bucket
    e, lo, hi, ok_ = n - 4, n - 3, n - 2, n - 1
    sa = np.array([e, e, 0, lo, lo, hi, lo, ok_, 5, 5] + list(range(n)), dtype=np.uint32)
    sb = np.array([e, 0, e, hi, lo, lo, ok_, lo, 5, 6] + list(range(n))[::-1], dtype=np.uint32)
    for op in OPS:
        got = S.op(op, S, sa, sb).serialize_all()
        for k in range(len(sa)):
            assert got[k] == R.r64_op_bytes(op, blobs[sa[k]], blobs[sb[k]]), (op, k)
    cards = S.and_cardinality(S, sa, sb)
    assert [int(c) for c in cards] == [R.r64_and_cardinality(blobs[a], blobs[b]) for a, b in zip(sa, sb)]


def test_buckets_that_become_empty_vanish(R):
    blobs = _op_blobs(R)
    S = rb.DeviceSet64.from_serialized(blobs)
    n = len(blobs)
    idx = np.arange(n, dtype=np.uint32)
    empty = R.r64_from_values(np.zeros(0, np.uint64))
    for op in ("xor", "andnot"):
        X = S.op(op, S, idx, idx)
        assert X.serialize_all() == [empty] * n
        assert [int(c) for c in X.cardinalities()] == [0] * n
        # the all-empty buckets take no part in the next op
        Y = X.op("or", S, idx, idx[::-1].copy())
        assert Y.serialize_all() == [blobs[i] for i in idx[::-1]]
        assert [int(c) for c in X.and_cardinality(S, idx, idx)] == [0] * n
    lo, ok_ = n - 3, n - 1
    A = S.op("and", S, [lo, ok_], [ok_, lo])
    assert A.serialize_all() == [empty, empty]
    assert A.op("xor", S, [0, 1], [lo, ok_]).serialize_all() == [blobs[lo], blobs[ok_]]


def test_chained_fold_and_run_optimize(R):
    blobs = synth_blobs64(R, 94, 64)
    S = rb.DeviceSet64.from_serialized(blobs)
    folds = np.arange(64, dtype=np.uint32).reshape(8, 8)   # 8 folds of 8 operands each
    for op in OPS:
        acc = S.op(op, S, folds[:, 0], folds[:, 1])
        for k in range(2, 8):   # every step takes the resident result of the previous one
            acc = acc.op(op, S, np.arange(8, dtype=np.uint32), folds[:, k])
        exp = []
        for f in folds:
            e = R.r64_op_bytes(op, blobs[f[0]], blobs[f[1]])
            for k in range(2, 8):
                e = R.r64_op_bytes(op, e, blobs[f[k]])
            exp.append(e)
        assert acc.serialize_all() == exp, op
        assert acc.run_optimize().serialize_all() == [_r64_run_optimize(R, e) for e in exp], op
        assert [int(c) for c in acc.cardinalities()] == [_r64_card(R, e) for e in exp], op


def _builder_bitmaps():
    k = np.uint64(5 << 32) | np.uint64(3 << 16)   # one 48-bit key
    a4096 = np.arange(4096, dtype=np.uint64) * 16 + k
    a4097 = np.arange(4097, dtype=np.uint64) * 15 + k
    lows = np.array([7, 1 << 20, 0xFFFFFFFF], dtype=np.uint64)
    return [
        np.zeros(0, np.uint64),                                                       # empty at the start
        a4096,                                                                        # 4096 distinct: array
        a4097,                                                                        # 4097: bitset
        np.repeat(a4096, 5),                                                          # still an array
        np.concatenate([lows + (np.uint64(8) << np.uint64(32)), lows + (np.uint64(9) << np.uint64(32))]),   # same low32, adjacent buckets
        np.zeros(0, np.uint64),                                                       # empty in the middle
        np.array([0, 2 ** 64 - 1], dtype=np.uint64),
        (np.arange(100_000, dtype=np.uint64) << np.uint64(32)) | np.uint64(7),        # one value in each of many buckets
        np.arange(70000, dtype=np.uint64) + (np.uint64(0xFFFFFFFF) << np.uint64(32)),
        np.zeros(0, np.uint64),                                                       # empty at the end
    ]


def test_builder_edge_cases_sorted_and_shuffled(R):
    rng = np.random.default_rng(6)
    bms = _builder_bitmaps()
    exp = [R.r64_from_values(v, run_optimize=False) for v in bms]
    S = rb.DeviceSet64.from_values(bms)
    assert S.serialize_all() == exp
    assert [int(c) for c in S.cardinalities()] == [len(np.unique(v)) for v in bms]
    flat, off = _flat([_shuffled_with_dups(rng, v) for v in bms])
    S2 = rb.DeviceSet64.from_values(flat, off)
    assert S2.serialize_all() == exp
    assert S2.run_optimize().serialize_all() == [_r64_run_optimize(R, e) for e in exp]
    assert rb.DeviceSet64.from_values([]).serialize_all() == []
    assert len(rb.DeviceSet64.from_values(np.zeros(0, np.uint64), [0])) == 0
    # built sets chain into ops
    ia = np.arange(len(bms), dtype=np.uint32)
    ib = ia[::-1].copy()
    for op in OPS:
        got = S.op(op, S2, ia, ib).serialize_all()
        assert got == [R.r64_op_bytes(op, exp[a], exp[b]) for a, b in zip(ia, ib)], op


def test_builder_realdata_and_a_large_bitmap(R):
    rng = np.random.default_rng(8)
    vals = [_spread(_values32(R, b), HIGHS[:2]) for b in rb.load_realdata("census1881")[:40]]
    exp = [R.r64_from_values(v, run_optimize=False) for v in vals]
    assert rb.DeviceSet64.from_values(vals).serialize_all() == exp
    flat, off = _flat([_shuffled_with_dups(rng, v) for v in vals])
    assert rb.DeviceSet64.from_values(flat, off).serialize_all() == exp
    # >= 5 M values over a few buckets: bitsets, arrays and a key of 4096 + a few values
    big = np.concatenate([rng.integers(0, 1 << 24, 3_000_000, dtype=np.uint64),
                          rng.integers(1 << 32, 1 << 40, 2_000_000, dtype=np.uint64),
                          rng.integers(7 << 32, (7 << 32) + (300 << 16), 500_000, dtype=np.uint64)])
    e = R.r64_from_values(big, run_optimize=False)
    assert rb.DeviceSet64.from_values([big]).serialize_all() == [e]
    assert rb.DeviceSet64.from_values([np.sort(big)[::-1].copy(), np.sort(big)]).serialize_all() == [e, e]


def test_builder_device_input_matches_host_input(R):
    import torch
    rng = np.random.default_rng(10)
    bms = _builder_bitmaps() + [_spread(_values32(R, b)) for b in rb.load_realdata("weather_sept_85")[:10]]
    flat, off = _flat([_shuffled_with_dups(rng, v) for v in bms])
    host = rb.DeviceSet64.from_values(flat, off).serialize_all()
    assert host == [R.r64_from_values(v, run_optimize=False) for v in bms]
    stream = torch.cuda.Stream()
    rb.set_stream(stream.cuda_stream)
    try:
        with torch.cuda.stream(stream):
            t = torch.from_numpy(flat.view(np.int64)).cuda()
            t_off = torch.from_numpy(off.astype(np.int64)).cuda()
        assert rb.DeviceSet64.from_values(t, t_off).serialize_all() == host
        assert np.array_equal(t.cpu().numpy().view(np.uint64), flat)   # unsorted input left as it was
        assert rb.DeviceSet64.from_values(t, torch.from_numpy(off.astype(np.int64))).serialize_all() == host
    finally:
        rb.set_stream(None)


_INMEM = r'''
import ctypes as C, os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
import numpy as np
ref_so = os.path.join(sys.argv[1], "oracle", "_ref", "libroaring_ref.so")
G = C.CDLL(ref_so, mode=os.RTLD_GLOBAL)
from oracle.refbind import ref
import croaring_b200 as rb
from helpers import synth_blobs64, OPS
R = ref()
rb.init(0)
L = rb.lib()
blobs = synth_blobs64(R, 95, 24)
bms = [R.r64_deserialize(b) for b in blobs]
S = rb.DeviceSet64(L.rb200_set64_upload((C.c_void_p * len(bms))(*bms), len(bms)))
assert S.serialize_all() == blobs
rng = np.random.default_rng(2)
ia = rng.integers(0, 24, 40).astype(np.uint32); ib = rng.integers(0, 24, 40).astype(np.uint32)
for op in OPS:
    res = S.op(op, S, ia, ib)
    out = (C.c_void_p * 40)()
    assert L.rb200_set64_download_all(res.ptr, out) == 0, rb.last_error()
    for k in range(40):
        why = C.c_char_p()
        assert R.L.roaring64_bitmap_internal_validate(out[k], C.byref(why)), why.value
        assert R.r64_serialize(out[k]) == R.r64_op_bytes(op, blobs[ia[k]], blobs[ib[k]]), (op, k)
        R.L.roaring64_bitmap_free(out[k])
print("set64 in-memory ok")
'''


def test_in_memory_upload_and_download():
    """rb200_set64_upload / rb200_set64_download_all on the host application's roaring64_bitmap_t
    objects, in a process where the reference is loaded globally."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", _INMEM, root], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "set64 in-memory ok" in p.stdout, (p.stdout[-500:], p.stderr[-1500:])
