"""GPU parity of rb200_batch_add_many / remove_many (roaring_bitmap_add_many / remove_many, roaring.c:134,
696): every result byte-identical to the reference's update of the same bitmap with the same values, and
valid for its validator, over the synthetic container mixes, their no-run twins, large runs and the
real-data sets; batch shapes, device values, chaining, sharing lifetimes, op stats and refusals."""

import numpy as np
import pytest

import croaring_b200.datasets as dsm
from helpers import DATASETS, check_result_bitmap, no_run_twins, sha_concat, synth_blobs
from offset_oracles import ref_add_offset_bytes
from test_update_host import containers
from update_oracles import ref_update_bytes

pytestmark = pytest.mark.gpu

PROFILES = ["full", "nearfull", "halves", "dense", "bitset", "array", "tiny", "longruns", "shortruns", "ends"]
KINDS = ["empty", "no_change", "new_keys", "edges", "emptying", "unsorted_dups", "extremes"]


def _inputs(R, seed):
    blobs = synth_blobs(R, seed, 30, key_space=6, max_keys=6, profiles=PROFILES if seed % 3 else None)
    return blobs + no_run_twins(R, blobs)


def _values(R, blobs, op, kind, seed):
    """One uint32 value list per bitmap of the given kind."""
    rng = np.random.default_rng(seed)
    out = []
    for k, b in enumerate(blobs):
        r = R.deserialize(b)
        have = R.to_array(r)
        R.free(r)
        if kind == "empty":
            v = np.zeros(0, np.uint32)
        elif kind == "no_change":   # add: only present values; remove: only absent ones
            if op == "add":
                v = rng.choice(have, size=min(have.size, 300), replace=False) if have.size else np.zeros(0, np.uint32)
            else:
                cand = rng.integers(0, 6 << 16, 600).astype(np.uint32)
                v = np.setdiff1d(cand, have)
        elif kind == "new_keys":    # keys no bitmap of the mix holds, dense enough for a bitset in one
            v = np.concatenate([rng.integers(40 << 16, 41 << 16, 5000), rng.integers(50 << 16, (50 << 16) + 300, 40)])
        elif kind == "edges":       # about 4096 values per touched key: arrays, bitsets and runs cross their edges
            keys = rng.choice(6, size=2, replace=False)
            if op == "add":
                v = np.concatenate([(int(kk) << 16) + rng.choice(65536, size=int(rng.integers(1, 4200)), replace=False)
                                    for kk in keys])
            else:
                v = have[rng.random(have.size) < rng.choice([0.02, 0.5, 0.95])] if have.size else have
        elif kind == "emptying":    # whole keys or the whole bitmap
            if op == "add" or not have.size:
                v = have if op == "remove" else np.arange(0, 65536)   # add: a full key
            elif k % 2:
                v = have
            else:
                v = have[(have >> 16) == (have[0] >> 16)]
        elif kind == "unsorted_dups":
            base = rng.integers(0, 6 << 16, 3000)
            if have.size and op == "remove":
                base = np.concatenate([base, rng.choice(have, size=min(have.size, 3000))])
            v = rng.permutation(np.concatenate([base, base[: base.size // 3]]))
        else:                       # extremes
            v = np.array([0, 0xFFFFFFFF, 0xFFFF, 0x10000, 0xFFFF0000, 1, 0xFFFFFFFE], dtype=np.uint64)
        out.append(np.asarray(v).astype(np.uint32))
    return out


def _expect(R, op, blobs, lists):
    return [ref_update_bytes(R, op, b, v) for b, v in zip(blobs, lists)]


def _update(S, op, *a, **kw):
    return S.add_many(*a, **kw) if op == "add" else S.remove_many(*a, **kw)


@pytest.mark.parametrize("op", ["add", "remove"])
@pytest.mark.parametrize("seed", [91, 92, 93])
def test_update_vs_reference(rb, R, seed, op):
    blobs = _inputs(R, seed)
    S = rb.DeviceSet.from_serialized(blobs)
    for j, kind in enumerate(KINDS):
        lists = _values(R, blobs, op, kind, seed * 10 + j)
        expect = _expect(R, op, blobs, lists)
        res = _update(S, op, lists)
        assert res.serialize_all() == expect, kind
        if kind in ("edges", "extremes", "emptying"):
            for k, bm in enumerate(res.download_all()):
                check_result_bitmap(R, bm, expect[k], f"{op} {kind} bitmap {k}")


def test_large_runs(rb, R):
    """A run that receives more than 4096 values, and removals that cut a run into 32768 runs: results
    past 8 KiB per container, inside the slab bound."""
    full = R.from_values(np.arange(0, 1 << 17, dtype=np.uint32))   # two full runs
    part = R.from_values(np.arange(1000, 3000, dtype=np.uint32))
    blobs = [R.serialize(full), R.serialize(part)]
    R.free(full)
    R.free(part)
    S = rb.DeviceSet.from_serialized(blobs)
    odd = np.arange(1, 1 << 17, 2, dtype=np.uint32)
    spaced = np.arange(4000, 4000 + 2 * 6000, 2, dtype=np.uint32)
    cases = [("remove", [odd, odd[:10]]), ("remove", [odd[: 1 << 15], np.arange(1001, 2999, 2, dtype=np.uint32)]),
             ("add", [spaced, spaced]), ("add", [np.zeros(0, np.uint32), np.arange(0, 65536, 2, dtype=np.uint32)])]
    for op, lists in cases:
        expect = _expect(R, op, blobs, lists)
        res = _update(S, op, lists)
        assert res.serialize_all() == expect, op
        for k, bm in enumerate(res.download_all()):
            check_result_bitmap(R, bm, expect[k], f"{op} large {k}")
    # the 32768-run containers of the first case, read from the bytes
    got = containers(_update(S, "remove", [odd, odd[:10]]).serialize_all()[0])
    assert [c[1:] for c in got] == [(3, 32768, 32768)] * 2
    # and chained: the big runs are operands of the next update
    X = S.remove_many([odd, odd[:10]])
    step1 = _expect(R, "remove", blobs, [odd, odd[:10]])
    back = [np.arange(1, 30001, 2, dtype=np.uint32), np.arange(0, 100, dtype=np.uint32)]
    assert X.add_many(back).serialize_all() == _expect(R, "add", step1, back)


def _one_percent(R, blobs, op, seed, frac=0.01):
    rng = np.random.default_rng(seed)
    out = []
    for b in blobs:
        r = R.deserialize(b)
        have = R.to_array(r)
        R.free(r)
        m = max(1, int(have.size * frac))
        if op == "add":
            hi = int(have[-1]) + 2 if have.size else 1 << 20
            out.append(rng.integers(0, hi, m).astype(np.uint32))
        else:
            out.append(rng.choice(have, size=min(m, have.size), replace=False).astype(np.uint32) if have.size
                       else np.zeros(0, np.uint32))
    return out


@pytest.mark.parametrize("ds", DATASETS)
def test_update_realdata_sha(rb, R, ds):
    blobs = dsm.load_realdata(ds)
    S = rb.DeviceSet.from_serialized(blobs)
    for op in ("add", "remove"):
        lists = _one_percent(R, blobs, op, len(ds) + (op == "add"))
        got = _update(S, op, lists).serialize_all()
        assert sha_concat(got) == sha_concat(_expect(R, op, blobs, lists)), (ds, op)


def test_batch_shapes(rb, R):
    blobs = _inputs(R, 94)
    S = rb.DeviceSet.from_serialized(blobs)
    rng = np.random.default_rng(94)
    idx = np.array([5, 5, 0, 17, 5, len(blobs) - 1, 2, 2], dtype=np.uint32)
    lists = [rng.integers(0, 6 << 16, int(rng.integers(0, 3000))).astype(np.uint32) for _ in idx]
    for op in ("add", "remove"):
        assert _update(S, op, lists, idx=idx).serialize_all() == \
            [ref_update_bytes(R, op, blobs[i], v) for i, v in zip(idx, lists)], op
        # the flat layout with offsets
        offs = np.concatenate([[0], np.cumsum([v.size for v in lists])])
        assert _update(S, op, np.concatenate(lists), offs, idx=idx).serialize_all() == \
            [ref_update_bytes(R, op, blobs[i], v) for i, v in zip(idx, lists)], op
        # n == 0
        empty = _update(S, op, [], idx=np.zeros(0, np.uint32))
        assert len(empty) == 0 and empty.serialize_all() == []
    # idx None over an empty set
    E = rb.DeviceSet.from_values([])
    assert len(E.add_many([])) == 0


def test_device_values(rb, R):
    import torch
    blobs = _inputs(R, 95)
    S = rb.DeviceSet.from_serialized(blobs)
    for op in ("add", "remove"):
        lists = _values(R, blobs, op, "unsorted_dups", 95)
        flat = np.concatenate(lists)
        offs = np.concatenate([[0], np.cumsum([v.size for v in lists])]).astype(np.int64)
        tv = torch.from_numpy(flat.view(np.int32)).cuda()
        torch.cuda.synchronize()
        host = _update(S, op, lists).serialize_all()
        assert _update(S, op, tv, torch.from_numpy(offs).cuda()).serialize_all() == host, op
        assert _update(S, op, tv, offs).serialize_all() == host, op
        assert host == _expect(R, op, blobs, lists)


def _ref_run_optimize(R, b):
    r = R.deserialize(b)
    R.L.roaring_bitmap_run_optimize(r)
    out = R.serialize(r)
    R.free(r)
    return out


def test_chaining(rb, R):
    from oracle.oraclebind import oracle
    blobs = _inputs(R, 96)
    n = len(blobs)
    S = rb.DeviceSet.from_serialized(blobs)
    la = _values(R, blobs, "add", "edges", 961)
    lr = _values(R, blobs, "remove", "edges", 962)
    A, D = S.add_many(la), S.remove_many(lr)
    added, removed = _expect(R, "add", blobs, la), _expect(R, "remove", blobs, lr)
    ia = np.arange(n, dtype=np.uint32)
    ib = (ia + 1) % n
    for op in ("and", "or", "xor", "andnot"):
        assert A.batch(op, D, ia, ib).serialize_all() == [R.op_bytes(op, added[i], removed[j]) for i, j in zip(ia, ib)], op
    assert A.or_many().serialize_all()[0] == oracle().many_bytes("or_many", added)
    assert D.add_offset(5536).serialize_all() == [ref_add_offset_bytes(R, b, 5536) for b in removed]
    assert A.run_optimize().serialize_all() == [_ref_run_optimize(R, b) for b in added]
    assert rb.DeviceSet.from_frozen(D.serialize_all(frozen=True)).serialize_all() == removed
    for k, bm in enumerate(D.download_all()):
        check_result_bitmap(R, bm, removed[k], f"download {k}")
    # ten rounds of alternating adds and removes against the reference applied round by round
    X, cur = S, blobs
    for rnd in range(10):
        op = "add" if rnd % 2 == 0 else "remove"
        lists = _values(R, cur, op, "edges" if rnd % 3 else "unsorted_dups", 970 + rnd)
        X = _update(X, op, lists)
        cur = _expect(R, op, cur, lists)
        assert X.serialize_all() == cur, rnd


def test_sharing_lifetimes_and_bound_host(rb, R):
    blobs = _inputs(R, 97)
    L = rb.lib()
    base = int(L.rb200_device_bytes_in_use())
    S = rb.DeviceSet.from_serialized(blobs)
    new = [np.arange(60 << 16, (60 << 16) + 5000 + 37 * k, dtype=np.uint32) for k in range(len(blobs))]
    A = S.add_many(new)                      # shares S's containers and the values' new keys
    D = S.remove_many(_values(R, blobs, "remove", "edges", 97))
    expect_a = _expect(R, "add", blobs, new)
    S.free()
    assert A.serialize_all() == expect_a
    A2 = A.add_many([[1, 2, 3]] * len(blobs))   # from a result that shares: copies instead
    for k, bm in enumerate(A.download_all()):
        check_result_bitmap(R, bm, expect_a[k], f"after free {k}")
    A.free()
    assert A2.serialize_all() == _expect(R, "add", expect_a, [[1, 2, 3]] * len(blobs))
    D.free()
    A2.free()
    assert int(L.rb200_device_bytes_in_use()) == base
    # an operand uploaded from host bitmaps and bound: pass-through payloads come from the host
    hosts = [rb.Bitmap.deserialize(b) for b in blobs]
    H = rb.DeviceSet.upload(hosts).bind_host()
    for op in ("add", "remove"):
        lists = _values(R, blobs, op, "edges", 98)
        outs = _update(H, op, lists).download_all()
        exp = _expect(R, op, blobs, lists)
        for k in range(len(blobs)):
            check_result_bitmap(R, outs[k], exp[k], f"bound {op} {k}")


def _portable(t, card, ln):
    return 8192 if t == 1 else (2 * card if t == 2 else 2 + 4 * ln)


def test_op_stats(rb, R):
    blobs = dsm.load_realdata("weather_sept_85")[:50]
    S = rb.DeviceSet.from_serialized(blobs)
    for op in ("add", "remove"):
        assert _update(S, op, [[]] * len(blobs)).op_stats()[2] == 0, op
    # one key of one bitmap touched: that key's input and output, nothing else
    b = blobs[3]
    key, t, card, ln = containers(b)[0]
    v = (key << 16) + 7
    X = S.add_many([[v]], idx=[3])
    out = containers(X.serialize_all()[0])[0]
    assert out[0] == key
    ab = X.op_stats()[2]
    assert 0 < ab <= _portable(t, card, ln) + 2 + _portable(*out[1:]), ab


def test_refusals(rb, R):
    blobs = _inputs(R, 99)[:6]
    S = rb.DeviceSet.from_serialized(blobs)
    L = rb.lib()
    one = lambda v: np.array([v], dtype=np.uint32)
    lz = S.batch("or", S, one(0), one(1), lazy=True)
    with pytest.raises(rb.RB200Error, match="add_many: the set is in a lazy state"):
        lz.add_many([[1]])
    with pytest.raises(rb.RB200Error, match=r"remove_many: index out of range: idx\[1\] = 6"):
        S.remove_many([[1], [2]], idx=[0, 6])
    vals = np.array([1, 2, 3], dtype=np.uint32)
    dec = np.array([0, 2, 1, 3], dtype=np.uint64)
    idx3 = np.array([0, 1, 2], dtype=np.uint32)
    assert not L.rb200_batch_add_many(S.ptr, idx3.ctypes.data, 3, vals.ctypes.data, dec.ctypes.data)
    assert "add_many: offsets decrease at bitmap 1" in rb.last_error()
    ok_off = np.array([0, 1, 2, 3], dtype=np.uint64)
    assert not L.rb200_batch_remove_many(S.ptr, idx3.ctypes.data, 3, None, ok_off.ctypes.data)
    assert rb.last_error() == "remove_many: values are NULL"
    assert not L.rb200_batch_add_many(S.ptr, idx3.ctypes.data, 3, vals.ctypes.data, None)
    assert "add_many: offsets are NULL" in rb.last_error()
    # device offsets that decrease, checked on the host before any kernel reads values through them
    import torch
    tv = torch.arange(3, dtype=torch.int32, device="cuda")
    to = torch.tensor([0, 2, 1, 3], dtype=torch.int64, device="cuda")
    assert not L.rb200_batch_remove_many_device(S.ptr, idx3.ctypes.data, 3, tv.data_ptr(), to.data_ptr())
    assert "offsets decrease at bitmap 1" in rb.last_error()
    # NULL values with a zero count are an empty update
    zero = np.zeros(len(blobs) + 1, dtype=np.uint64)
    p = L.rb200_batch_add_many(S.ptr, None, 0, None, zero.ctypes.data)
    assert p
    assert rb.DeviceSet(p).serialize_all() == blobs
    # the set is still usable
    assert S.add_many([[3]] * len(blobs)).serialize_all() == _expect(R, "add", blobs, [[3]] * len(blobs))
