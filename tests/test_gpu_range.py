"""GPU parity of rb200_batch_add_range_closed / remove_range_closed (roaring_bitmap_add_range_closed /
remove_range_closed, roaring.c:251, 302): every result byte-identical to the reference's range update of the
same bitmap, and valid for its validator, over the synthetic container mixes, their no-run twins, the
real-data sets and the wide directories; every producer of S; chaining; batch shapes, sharing lifetimes,
copy-on-write flags, op stats, launches and refusals."""
import types

import numpy as np
import pytest

import croaring_b200.datasets as dsm
import wide_cases
from cow_oracles import bind, cow_of, make
from helpers import DATASETS, check_result_bitmap, no_run_twins, sha_concat, synth_blobs
from range_oracles import ref_range_bytes
from update_oracles import ref_update_bytes

pytestmark = pytest.mark.gpu

PROFILES = ["full", "nearfull", "halves", "dense", "bitset", "array", "tiny", "longruns", "shortruns", "ends"]
KINDS = ["empty", "single", "inside", "key_edges", "whole_key", "absent_keys", "many_keys", "universe", "top",
         "all_values", "no_value"]
T32 = (1 << 32) - 1


def _inputs(R, seed):
    blobs = synth_blobs(R, seed, 30, key_space=6, max_keys=6, profiles=PROFILES if seed % 3 else None)
    return blobs + no_run_twins(R, blobs)


def _vals(R, blob):
    r = R.deserialize(blob)
    v = R.to_array(r)
    R.free(r)
    return v


def _range(R, blob, kind, rng):
    """One closed range [lo, hi] of the given kind for this bitmap (lo > hi: empty)."""
    k = int(rng.integers(0, 6))
    if kind == "empty":
        return 10, 5
    if kind == "single":
        v = _vals(R, blob)
        x = int(rng.choice(v)) if v.size and rng.random() < 0.5 else int(rng.integers(0, 6 << 16))
        return x, x
    if kind == "inside":
        a, b = sorted(rng.integers(0, 65536, 2).tolist())
        return (k << 16) + a, (k << 16) + b
    if kind == "key_edges":
        return 65535, 65536
    if kind == "whole_key":
        return k << 16, (k << 16) + 65535
    if kind == "absent_keys":
        return (40 << 16) + 5, (42 << 16) + 100
    if kind == "many_keys":
        return int(rng.integers(0, 3000)), (5 << 16) + int(rng.integers(0, 65536))
    if kind == "universe":
        return 0, T32
    if kind == "top":
        return 0xFFFF0000, T32
    v = _vals(R, blob)
    if kind == "all_values":
        return (int(v[0]), int(v[-1])) if v.size else (0, 0)
    # no_value: a gap between two values, or past the last one
    gaps = np.flatnonzero(np.diff(v.astype(np.int64)) > 1) if v.size else np.zeros(0, np.int64)
    if gaps.size:
        g = int(rng.choice(gaps))
        return int(v[g]) + 1, int(v[g + 1]) - 1
    return (int(v[-1]) + 1, int(v[-1]) + 70000) if v.size and int(v[-1]) < T32 - 70000 else (7, 7)


def _ranges(R, blobs, kind, seed):
    rng = np.random.default_rng(seed)
    rs = [_range(R, b, kind, rng) for b in blobs]
    return np.array([a for a, _ in rs], np.uint64), np.array([b for _, b in rs], np.uint64)


def _expect(R, op, blobs, lo, hi):
    return [ref_range_bytes(R, op, b, a, z) for b, a, z in zip(blobs, lo, hi)]


def _apply(S, op, lo, hi, idx=None):
    """The update through the mirror's half-open form: [lo, hi + 1), with lo > hi as the empty [lo, lo)."""
    end = [int(z) + 1 if int(a) <= int(z) else int(a) for a, z in zip(lo, hi)]
    f = S.add_range if op == "add" else S.remove_range
    return f([int(a) for a in lo], end, idx=idx)


@pytest.mark.parametrize("op", ["add", "remove"])
@pytest.mark.parametrize("seed", [11, 12])
def test_range_vs_reference(rb, R, seed, op):
    blobs = _inputs(R, seed)
    S = rb.DeviceSet.from_serialized(blobs)
    for j, kind in enumerate(KINDS):
        lo, hi = _ranges(R, blobs, kind, seed * 100 + j)
        expect = _expect(R, op, blobs, lo, hi)
        res = _apply(S, op, lo, hi)
        assert res.serialize_all() == expect, kind
        if kind in ("inside", "key_edges", "top", "all_values", "no_value"):
            for k, bm in enumerate(res.download_all()):
                check_result_bitmap(R, bm, expect[k], f"{op} {kind} bitmap {k}")
    # one batch mixing every kind
    rng = np.random.default_rng(seed)
    rs = [_range(R, b, KINDS[i % len(KINDS)], rng) for i, b in enumerate(blobs)]
    lo, hi = np.array([a for a, _ in rs], np.uint64), np.array([b for _, b in rs], np.uint64)
    assert _apply(S, op, lo, hi).serialize_all() == _expect(R, op, blobs, lo, hi)


def test_closed_c_abi(rb, R):
    """The closed C entry points themselves, the 2^32 - 1 end included."""
    blobs = _inputs(R, 14)[:8]
    S = rb.DeviceSet.from_serialized(blobs)
    L = rb.lib()
    lo = np.array([0, 5, 65535, 0xFFFF0000, 10, 3, 0, 70000], np.uint32)
    hi = np.array([T32, 5, 65536, T32, 9, 200000, 0, 0xFFFFFFF0], np.uint32)
    for op in ("add", "remove"):
        p = getattr(L, f"rb200_batch_{op}_range_closed")(S.ptr, None, 0, lo.ctypes.data, hi.ctypes.data)
        assert rb.DeviceSet(p).serialize_all() == _expect(R, op, blobs, lo, hi), op


@pytest.mark.parametrize("ds", DATASETS)
def test_range_realdata_sha(rb, R, ds):
    blobs = dsm.load_realdata(ds)
    S = rb.DeviceSet.from_serialized(blobs)
    for op in ("add", "remove"):
        for j, kind in enumerate(("inside", "whole_key", "many_keys", "all_values", "no_value")):
            lo, hi = _ranges(R, blobs, kind, len(ds) * 10 + j)
            got = _apply(S, op, lo, hi).serialize_all()
            assert sha_concat(got) == sha_concat(_expect(R, op, blobs, lo, hi)), (ds, op, kind)


def test_wide_cases(rb, R):
    names, blobs = zip(*wide_cases.bitmaps(R))
    S = rb.DeviceSet.from_serialized(list(blobs))
    for op in ("add", "remove"):
        for j, kind in enumerate(("inside", "key_edges", "whole_key", "many_keys", "top")):
            lo, hi = _ranges(R, blobs, kind, 300 + j)
            expect = _expect(R, op, blobs, lo, hi)
            res = _apply(S, op, lo, hi)
            assert res.serialize_all() == expect, (op, kind)
            if kind in ("top", "key_edges"):
                for k, bm in enumerate(res.download_all()):
                    check_result_bitmap(R, bm, expect[k], f"{op} {kind} {names[k]}")


def _producers(rb, R, blobs):
    """(name, set holding blobs' bitmaps or their transforms, the expected bytes of its bitmaps)."""
    n = len(blobs)
    S = rb.DeviceSet.from_serialized(blobs)
    out = [("upload", S, blobs)]
    hosts = [rb.Bitmap.deserialize(b) for b in blobs]
    out.append(("host upload", rb.DeviceSet.upload(hosts), blobs))
    out.append(("frozen", rb.DeviceSet.from_frozen(S.serialize_all(frozen=True)), blobs))
    vals = [_vals(R, b) for b in blobs]
    V = rb.DeviceSet.from_values(vals)
    out.append(("from_values", V, V.serialize_all()))
    out.append(("run_optimize", V.run_optimize(), V.run_optimize().serialize_all()))
    out.append(("or_many", S.or_many(), S.or_many().serialize_all()))
    ia = np.arange(n, dtype=np.uint32)
    ib = (ia + 1) % n
    out.append(("batch", S.batch("or", S, ia, ib), S.batch("or", S, ia, ib).serialize_all()))
    out.append(("add_offset", S.add_offset(70000), S.add_offset(70000).serialize_all()))
    add = [np.array([1, 65536, 200000], np.uint32)] * n
    out.append(("add_many", S.add_many(add), S.add_many(add).serialize_all()))
    # pending results whose operands are freed before the range update reads them
    T = rb.DeviceSet.from_serialized(blobs)
    P = T.batch("andnot", T, ia, ib)
    Q = T.add_many(add)
    T.free()
    out.append(("batch, operands freed", P, [R.op_bytes("andnot", blobs[i], blobs[j]) for i, j in zip(ia, ib)]))
    out.append(("add_many, operands freed", Q, [ref_update_bytes(R, "add", b, v) for b, v in zip(blobs, add)]))
    return out


def test_every_producer(rb, R):
    blobs = _inputs(R, 15)[:20]
    for name, X, have in _producers(rb, R, blobs):
        for op in ("add", "remove"):
            for j, kind in enumerate(("inside", "many_keys", "whole_key", "no_value")):
                lo, hi = _ranges(R, have, kind, 400 + j)
                assert _apply(X, op, lo, hi).serialize_all() == _expect(R, op, have, lo, hi), (name, op, kind)


def test_chaining(rb, R):
    blobs = _inputs(R, 16)
    n = len(blobs)
    S = rb.DeviceSet.from_serialized(blobs)
    lo, hi = _ranges(R, blobs, "many_keys", 16)
    A = _apply(S, "add", lo, hi)
    added = _expect(R, "add", blobs, lo, hi)
    lo2, hi2 = _ranges(R, added, "inside", 17)
    D = _apply(A, "remove", lo2, hi2)             # a range result into another range call
    removed = _expect(R, "remove", added, lo2, hi2)
    assert D.serialize_all() == removed
    ia = np.arange(n, dtype=np.uint32)
    ib = (ia + 3) % n
    for op in ("and", "or", "xor", "andnot"):
        assert A.batch(op, D, ia, ib).serialize_all() == [R.op_bytes(op, added[i], removed[j]) for i, j in zip(ia, ib)], op
    probe = np.array([int(lo[k]) for k in range(n)], np.uint32)   # each bitmap asked about its range's start
    got = D.contains(probe)
    for k in range(n):
        assert bool(got[k]) == (int(probe[k]) in set(_vals(R, removed[k]).tolist())), k
    # ten rounds of alternating adds and removes against the reference applied round by round (no universe
    # add: the next round's ranges are drawn from the values, read on the host)
    rounds = ["inside", "many_keys", "whole_key", "no_value", "key_edges", "single", "absent_keys", "all_values",
              "top", "inside"]
    X, cur = S, blobs
    for rnd, kind in enumerate(rounds):
        op = "add" if rnd % 2 == 0 else "remove"
        l, h = _ranges(R, cur, kind, 500 + rnd)
        X = _apply(X, op, l, h)
        cur = _expect(R, op, cur, l, h)
        assert X.serialize_all() == cur, rnd


def test_batch_shapes_and_launches(rb, R):
    blobs = _inputs(R, 18)
    S = rb.DeviceSet.from_serialized(blobs)
    idx = np.array([5, 5, 0, 17, 5, len(blobs) - 1, 2, 2], dtype=np.uint32)
    rng = np.random.default_rng(18)
    rs = [_range(R, blobs[i], KINDS[k % len(KINDS)], rng) for k, i in enumerate(idx)]
    lo, hi = np.array([a for a, _ in rs], np.uint64), np.array([b for _, b in rs], np.uint64)
    for op in ("add", "remove"):
        got = _apply(S, op, lo, hi, idx=idx).serialize_all()
        assert got == [ref_range_bytes(R, op, blobs[i], a, z) for i, a, z in zip(idx, lo, hi)], op
        # scalars broadcast to every item
        f = S.add_range if op == "add" else S.remove_range
        assert f(1000, 200000).serialize_all() == [ref_range_bytes(R, op, b, 1000, 199999) for b in blobs], op
        # n == 0
        empty = f([], [], idx=np.zeros(0, np.uint32))
        assert len(empty) == 0 and empty.serialize_all() == []
    E = rb.DeviceSet.from_values([])
    assert len(E.add_range(0, 10)) == 0
    # a fixed number of launches whatever n is
    big = rb.DeviceSet.from_serialized((blobs * 17)[:1000])
    for op in ("add", "remove"):
        f = big.add_range if op == "add" else big.remove_range
        keep = [f(100, 300000, idx=[3])]   # (mirrors fetched, nothing left to launch but the call's own)
        rb.synchronize()
        k0 = rb.kernel_launches()
        keep.append(f(100, 300000, idx=[3]))
        k1 = rb.kernel_launches()
        keep.append(f(100, 300000))
        k2 = rb.kernel_launches()
        assert len(keep[-1]) == 1000 and k1 - k0 == k2 - k1 > 0, (op, k1 - k0, k2 - k1)


def test_cow_flags_follow_S(rb, R):
    Rc = bind(R)
    rng = np.random.default_rng(19)
    blobs = _inputs(R, 19)[:9]
    states = [("plain", "cow", "cow-copy")[i % 3] for i in range(len(blobs))]
    xs = [make(Rc, b, s) for b, s in zip(blobs, states)]
    S = rb.DeviceSet.upload([types.SimpleNamespace(ptr=p) for p in xs])
    rs = [_range(R, b, ("inside", "many_keys", "empty")[i % 3], rng) for i, b in enumerate(blobs)]
    lo, hi = np.array([a for a, _ in rs], np.uint64), np.array([b for _, b in rs], np.uint64)
    for op in ("add", "remove"):
        res = _apply(S, op, lo, hi)
        fn = getattr(Rc.L, f"roaring_bitmap_{op}_range_closed")
        for k, (b, s) in enumerate(zip(blobs, states)):
            x = make(Rc, b, s)
            fn(x, int(lo[k]), int(hi[k]))   # the reference unshares what it touches
            exp = (Rc.serialize(x), cow_of(Rc, x))
            Rc.free(x)
            g = res.download(k)
            assert (g.serialize(), cow_of(Rc, g.ptr)) == exp, (op, k, s)
    for x in xs:
        Rc.free(x)


def test_sharing_lifetimes_stats_and_refusals(rb, R):
    blobs = _inputs(R, 20)
    L = rb.lib()
    base = int(L.rb200_device_bytes_in_use())
    S = rb.DeviceSet.from_serialized(blobs)
    lo, hi = _ranges(R, blobs, "inside", 20)
    A = _apply(S, "add", lo, hi)                 # shares S's containers outside the range
    expect = _expect(R, "add", blobs, lo, hi)
    S.free()
    assert A.serialize_all() == expect
    A2 = _apply(A, "remove", lo, hi)            # from a result that shares: copies instead
    A.free()
    assert A2.serialize_all() == _expect(R, "remove", expect, lo, hi)
    for k, bm in enumerate(A2.download_all()):
        check_result_bitmap(R, bm, _expect(R, "remove", expect, lo, hi)[k], f"after free {k}")
    A2.free()
    assert int(L.rb200_device_bytes_in_use()) == base
    # op stats: an empty range moves nothing; one boundary key reads its input and writes its output
    S = rb.DeviceSet.from_serialized(blobs)
    assert S.add_range(10, 5).op_stats()[2] == 0
    ms, _, ab = S.add_range(3, 9, idx=[1]).op_stats()
    assert ms > 0 and ab > 0
    # refusals: a lazy set, an index out of range, NULL ranges with items
    lz = S.batch("or", S, np.array([0], np.uint32), np.array([1], np.uint32), lazy=True)
    with pytest.raises(rb.RB200Error, match="add_range_closed: the set is in a lazy state"):
        lz.add_range(0, 5)
    with pytest.raises(rb.RB200Error, match=r"remove_range_closed: index out of range: idx\[1\] = 999"):
        S.remove_range(0, 5, idx=[0, 999])
    assert not L.rb200_batch_add_range_closed(S.ptr, None, 0, None, None)
    assert rb.last_error() == "add_range_closed: min / max is NULL"
    # NULL ranges with no items are an empty call
    p = L.rb200_batch_remove_range_closed(S.ptr, np.zeros(0, np.uint32).ctypes.data, 0, None, None)
    assert p and len(rb.DeviceSet(p)) == 0
    assert S.add_range(7, 8).serialize_all() == [ref_range_bytes(R, "add", b, 7, 7) for b in blobs]
