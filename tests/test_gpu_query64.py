"""GPU parity of the 64-bit point queries (rb200_set64_batch_query / _device): every answer and found flag equals
what the reference's roaring64_bitmap_contains / rank / get_index / select return for the same bitmap, called
once per query, over synthetic bucket mixes with and without runs, real data spread over buckets, ranks past
2^32 inside one bitmap, the value 2^64 - 1, empty bitmaps and empty buckets and every producer of a resident
64-bit set; host / device and selection equivalences; the cached prefix cardinalities; and the refusals."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import croaring_b200 as rb_mod
from helpers import DATASETS, synth_blobs64
from range_oracles import ref_range64_bytes
from test_gpu_set64 import _spread, _values32
from test_gpu_update import PROFILES
from update_oracles import ref_update64_bytes

pytestmark = pytest.mark.gpu

KINDS = ("contains", "rank", "get_index", "select")
QK = rb_mod.api.QUERIES
HIGHS = (0, 1, 7, 0x10000, 0xFFFFFFFF)
T32, T64 = 1 << 32, (1 << 64) - 1


def _bind(R):
    """The reference's 64-bit query functions (roaring64.h), all exported by libroaring_ref.so."""
    L, V, U = R.L, C.c_void_p, C.c_uint64
    for name, res, args in (("roaring64_bitmap_contains", C.c_bool, [V, U]),                       # roaring64.c:682
                            ("roaring64_bitmap_rank", U, [V, U]),                                  # :804
                            ("roaring64_bitmap_get_index", C.c_bool, [V, U, C.POINTER(U)]),        # :827
                            ("roaring64_bitmap_select", C.c_bool, [V, U, C.POINTER(U)]),           # :779
                            ("roaring64_bitmap_to_uint64_array", None, [V, V])):
        getattr(L, name).restype = res
        getattr(L, name).argtypes = args
    return L


def ref_answers(R, ptrs, kind, idx, vals):
    """(out, found): the reference's answer to every query, one call each; a false return is 2^64 - 1."""
    L = _bind(R)
    out, found = np.empty(len(vals), dtype=np.uint64), np.empty(len(vals), dtype=bool)
    el = C.c_uint64()
    f = {"contains": L.roaring64_bitmap_contains, "rank": L.roaring64_bitmap_rank,
         "get_index": L.roaring64_bitmap_get_index, "select": L.roaring64_bitmap_select}[kind]
    for k, (i, v) in enumerate(zip(idx.tolist(), vals.tolist())):
        if kind == "contains":
            found[k] = f(ptrs[i], v)
            out[k] = int(found[k])
        elif kind == "rank":
            out[k], found[k] = f(ptrs[i], v), True
        else:
            found[k] = f(ptrs[i], v, C.byref(el))
            out[k] = el.value if found[k] else T64
    return out, found


class Ref:
    """Reference 64-bit bitmaps holding what a resident set should hold."""

    def __init__(self, R, blobs):
        self.R = R
        self.ptrs = [R.r64_deserialize(b) for b in blobs]

    def values(self, i):
        L = _bind(self.R)
        out = np.empty(int(L.roaring64_bitmap_get_cardinality(self.ptrs[i])), dtype=np.uint64)
        if out.size:
            L.roaring64_bitmap_to_uint64_array(self.ptrs[i], out.ctypes.data)
        return out

    def close(self):
        for p in self.ptrs:
            self.R.L.roaring64_bitmap_free(p)
        self.ptrs = []


def _u64(xs):
    """Python ints as a uint64 array, modulo 2^64 (card - 1 of an empty bitmap is 2^64 - 1: any u64 is a query)."""
    return np.array([int(x) % (1 << 64) for x in xs], dtype=np.uint64)


def _edge_values(a, rng, extra=24):
    """0, 2^64 - 1, every bucket's first and last value, h << 32 and its neighbours for every present bucket
    and the next one, values in absent buckets between and around the present ones, values at and next to
    every container's and run's first and last value, random present and uniform values."""
    one = np.uint64(1)
    c = [_u64([0, 1, T64, T64 - 1, T32 - 1, T32, T32 + 1]),
         rng.integers(0, T64, extra, dtype=np.uint64, endpoint=True)]
    if a.size:
        hi = a >> np.uint64(32)
        bb = np.r_[0, np.flatnonzero(np.diff(hi)) + 1]
        be = np.r_[bb[1:] - 1, a.size - 1]
        highs = hi[bb]
        kb = np.r_[0, np.flatnonzero(np.diff(a >> np.uint64(16))) + 1]
        ke = np.r_[kb[1:] - 1, a.size - 1]
        rs = np.r_[0, np.flatnonzero(np.diff(a) != one) + 1]
        re = np.r_[rs[1:] - 1, a.size - 1]
        pts = np.concatenate([a[bb], a[be], a[kb], a[ke], a[rs], a[re]])
        base = np.concatenate([highs, highs + one]) << np.uint64(32)   # (wraps past the top bucket)
        c += [pts - one, pts, pts + one, base - one, base, base + one]
        # absent buckets: next to every present one and halfway between neighbours
        near = np.concatenate([highs - one, highs + one, highs + (np.r_[np.diff(highs), 2] >> one)])
        c.append((near << np.uint64(32)) | rng.integers(0, T32, near.size, dtype=np.uint64))
        c.append(rng.choice(a, extra))
    return np.concatenate(c)


def _edge_ranks(a, rng, extra=24):
    """Ranks 0, 1, card - 1, card, card + 1, 2^32 - 1, 2^32, 2^32 + 1, 2^64 - 1, around every bucket boundary
    of the prefix and the first rank of every 48-bit key, and random ranks below the cardinality."""
    card = a.size
    c = [_u64([0, 1, card - 1, card, card + 1, T32 - 1, T32, T32 + 1, T64, T64 - 1]),
         rng.integers(0, max(card, 1), extra, dtype=np.uint64)]
    if card:
        bb = np.r_[0, np.flatnonzero(np.diff(a >> np.uint64(32))) + 1, card].astype(np.uint64)
        kb = np.r_[0, np.flatnonzero(np.diff(a >> np.uint64(16))) + 1].astype(np.uint64)
        one = np.uint64(1)
        c += [bb - one, bb, bb + one, kb - one, kb, kb + one]
    return np.concatenate(c)


def _queries(ref, rng, cap):
    """{kind: (idx, vals)}: the edge queries of every bitmap, interleaved, at most cap per kind."""
    iv, vv, ir, rr = [], [], [], []
    for i in range(len(ref.ptrs)):
        a = ref.values(i)
        v, r = _edge_values(a, rng), _edge_ranks(a, rng)
        iv.append(np.full(v.size, i))
        vv.append(v)
        ir.append(np.full(r.size, i))
        rr.append(r)
    out = {}
    for kinds, idx, vals in ((("contains", "rank", "get_index"), iv, vv), (("select",), ir, rr)):
        idx, vals = np.concatenate(idx), np.concatenate(vals)
        pick = rng.permutation(idx.size)[:cap]
        for k in kinds:
            out[k] = (idx[pick].astype(np.uint32), vals[pick])
    return out


def check(S, ref, seed, cap=20000, what=""):
    """Every kind over the edge queries of every bitmap of S, answers and found flags, against the reference."""
    rng = np.random.default_rng(seed)
    for kind, (idx, vals) in _queries(ref, rng, cap).items():
        got, gf = rb_mod.api._query64(S, kind, vals, idx)
        exp, ef = ref_answers(ref.R, ref.ptrs, kind, idx, vals)
        bad = np.flatnonzero((got != exp) | (gf != ef))
        assert not bad.size, (f"{what} {kind}: {bad.size} of {idx.size} differ, first: bitmap {idx[bad[0]]} "
                              f"value {vals[bad[0]]} -> ({got[bad[0]]}, {gf[bad[0]]}), reference "
                              f"({exp[bad[0]]}, {ef[bad[0]]})")


def _empty(R):
    return R.r64_from_values(np.zeros(0, np.uint64))


def _inputs(R, seed, n=24):
    return synth_blobs64(R, seed, n, highs=HIGHS, profiles=PROFILES if seed % 2 else None) + [_empty(R)]


def _torch(a, dtype=np.int64):
    import torch
    a = np.ascontiguousarray(a, dtype=np.uint64 if dtype == np.int64 else np.uint32)
    return torch.from_numpy(a.view(dtype)).cuda()


def _checked(R, S, blobs, seed, what, cap=20000):
    ref = Ref(R, blobs)
    check(S, ref, seed, cap=cap, what=what)
    ref.close()


# ----------------------------------------------------------------------------------------- inputs
@pytest.mark.parametrize("seed", [81, 82, 83])
def test_synthetic_mixes(rb, R, seed):
    """Buckets 0, 1, 7, 2^16 and 2^32 - 1 in random subsets, run-optimized or not, with the container
    profiles of the update tests for the odd seeds."""
    blobs = _inputs(R, seed, 40)
    _checked(R, rb.DeviceSet64.from_serialized(blobs), blobs, seed, f"mix {seed}")


@pytest.mark.parametrize("ds", DATASETS)
def test_realdata_spread(rb, R, ds):
    blobs = [R.r64_from_values(_spread(_values32(R, b))) for b in rb.load_realdata(ds)[:60]]
    _checked(R, rb.DeviceSet64.from_serialized(blobs), blobs, len(ds), ds, cap=40000)


def test_ranks_past_2_32_and_the_top_value(rb, R):
    """[0, 2^33 + 5] as full buckets (made by the range add on the device and by the reference's), and a
    bitmap ending at 2^64 - 1: rank, get_index and select around 2^32 and 2^33 and at the top are exact."""
    E = rb.DeviceSet64.from_serialized([_empty(R), _empty(R)])
    top_lo = T64 - T32 - 10
    A = E.add_range([0, top_lo], [(1 << 33) + 6, 1 << 64])
    blobs = [ref_range64_bytes(R, "add", _empty(R), 0, (1 << 33) + 5),
             ref_range64_bytes(R, "add", _empty(R), top_lo, T64)]
    assert A.serialize_all() == blobs
    around = [T32 - 2, T32 - 1, T32, T32 + 1, (1 << 33) - 1, 1 << 33, (1 << 33) + 1, (1 << 33) + 5, (1 << 33) + 6, T64]
    # bitmap 0 holds 0 .. 2^33 + 5: rank(x) = x + 1, get_index(x) = x, select(r) = r
    v = np.array(around, dtype=np.uint64)
    inside = v <= np.uint64((1 << 33) + 5)
    assert (A.rank(v, idx=0) == np.where(inside, v + np.uint64(1), np.uint64((1 << 33) + 6))).all()
    gi, gf = A.get_index(v, idx=0)
    assert (gf == inside).all() and (gi == np.where(inside, v, np.uint64(T64))).all()
    sv, sf = A.select(v, idx=0)
    assert (sf == inside).all() and (sv == np.where(inside, v, np.uint64(T64))).all()
    # bitmap 1 ends at 2^64 - 1: select of its last rank gives it, found; past the cardinality, not found
    card = T64 - top_lo + 1
    sv, sf = A.select([card - 1, card, card + 1, 0], idx=1)
    assert sv.tolist() == [T64, T64, T64, top_lo] and sf.tolist() == [True, False, False, True]
    assert A.rank([T64, top_lo - 1, top_lo], idx=1).tolist() == [card, 0, 1]
    assert A.contains([T64, T64 - 1, top_lo - 1], idx=1).tolist() == [True, True, False]
    gi, gf = A.get_index([T64, top_lo - 1], idx=1)
    assert gi.tolist() == [card - 1, T64] and gf.tolist() == [True, False]
    # and against the reference, one call per query (whole buckets of 65536 containers: few queries)
    ref = Ref(R, blobs)
    for kind in KINDS:
        for b in (0, 1):
            q = np.array(around + [top_lo - 1, top_lo, top_lo + 1, card - 1, card], dtype=np.uint64)
            idx = np.full(q.size, b, np.uint32)
            got, gf = rb.api._query64(A, kind, q, idx)
            exp, ef = ref_answers(R, ref.ptrs, kind, idx, q)
            assert (got == exp).all() and (gf == ef).all(), (kind, b, got, exp)
    ref.close()


def test_empty_bitmaps_and_empty_buckets(rb, R):
    e = _empty(R)
    S = rb.DeviceSet64.from_serialized([e, e])
    v = np.array([0, 1, T32, T64], dtype=np.uint64)
    for b in (0, 1):
        assert not S.contains(v, idx=b).any() and (S.rank(v, idx=b) == 0).all()
        for kind in ("get_index", "select"):
            out, found = getattr(S, kind)(v, idx=b)
            assert (out == np.uint64(T64)).all() and not found.any()
    # results holding empty buckets: x XOR x, an XOR emptying one bucket in the middle, removals
    blobs = _inputs(R, 84, 16)
    S = rb.DeviceSet64.from_serialized(blobs)
    n = len(blobs)
    idx = np.arange(n, dtype=np.uint32)
    X = S.op("xor", S, idx, idx)
    _checked(R, X, [e] * n, 1, "x xor x")
    mid = np.arange(3000, dtype=np.uint64) * 5 + (np.uint64(7) << np.uint64(32))
    outer = [np.arange(100, dtype=np.uint64) + (np.uint64(h) << np.uint64(32)) for h in (0, 0xFFFFFFFF)]
    ab = [R.r64_from_values(np.concatenate([outer[0], mid, outer[1]])), R.r64_from_values(mid)]
    AB = rb.DeviceSet64.from_serialized(ab)
    Y = AB.op("xor", AB, [0, 1], [1, 1])
    _checked(R, Y, [R.r64_op_bytes("xor", ab[0], ab[1]), e], 2, "xor emptying a bucket")
    lists = [mid, mid]
    Z = AB.remove_many(lists)
    _checked(R, Z, [ref_update64_bytes(R, "remove", b, v) for b, v in zip(ab, lists)], 3, "remove_many")
    W = AB.remove_range(7 << 32, 8 << 32)
    _checked(R, W, [ref_range64_bytes(R, "remove", b, 7 << 32, (8 << 32) - 1) for b in ab], 4, "remove_range")
    # every bitmap of S with its bucket 7 removed
    V = S.remove_range(7 << 32, 8 << 32)
    _checked(R, V, [ref_range64_bytes(R, "remove", b, 7 << 32, (8 << 32) - 1) for b in blobs], 5, "remove bucket 7")


# ----------------------------------------------------------------------------------------- producers
def test_every_producer(rb, R):
    import torch
    blobs = _inputs(R, 85, 30)
    ref = Ref(R, blobs)
    vals = [ref.values(i) for i in range(len(blobs))]
    S = rb.DeviceSet64.from_serialized(blobs)
    check(S, ref, 1, what="upload_serialized")
    check(rb.DeviceSet64.from_values(vals), ref, 2, what="from_values host")
    off = np.zeros(len(vals) + 1, dtype=np.int64)
    np.cumsum([v.size for v in vals], out=off[1:])
    flat = torch.from_numpy(np.concatenate(vals).view(np.int64)).cuda()
    check(rb.DeviceSet64.from_values(flat, torch.from_numpy(off).cuda()), ref, 3, what="from_values device")
    check(S.run_optimize(0), ref, 4, what="run_optimize 0")
    check(S.run_optimize(1), ref, 5, what="run_optimize 1")
    ref.close()
    rng = np.random.default_rng(85)
    highs = np.array(HIGHS, dtype=np.uint64)
    lists = [(rng.choice(highs, 400) << np.uint64(32)) | rng.integers(0, 6 << 16, 400, dtype=np.uint64) for _ in blobs]
    picks = [rng.choice(v, min(v.size, 300), replace=False) if v.size else v for v in vals]
    _checked(R, S.add_many(lists), [ref_update64_bytes(R, "add", b, v) for b, v in zip(blobs, lists)], 6, "add_many")
    _checked(R, S.remove_many(picks), [ref_update64_bytes(R, "remove", b, v) for b, v in zip(blobs, picks)], 7,
             "remove_many")
    lo, hi = (1 << 32) - 70000, (1 << 32) + 300000   # (few containers: the reference walks them per query)
    _checked(R, S.add_range(lo, hi + 1), [ref_range64_bytes(R, "add", b, lo, hi) for b in blobs], 8, "add_range")
    lo, hi = 1 << 16, (0x10000 << 32) + 300000
    _checked(R, S.remove_range(lo, hi + 1), [ref_range64_bytes(R, "remove", b, lo, hi) for b in blobs], 9,
             "remove_range")


def test_batch_results_pending_and_outliving_their_operands(rb, R):
    blobs = _inputs(R, 86, 24)
    n = len(blobs)
    ia = np.arange(n, dtype=np.uint32)
    ib = ((ia + 5) % n).astype(np.uint32)
    S, T = rb.DeviceSet64.from_serialized(blobs), rb.DeviceSet64.from_serialized(blobs[::-1])
    expect = {op: [R.r64_op_bytes(op, blobs[i], blobs[::-1][j]) for i, j in zip(ia, ib)]
              for op in ("and", "or", "xor", "andnot")}
    # queried while still pending
    first = S.op("or", T, ia, ib)
    _checked(R, first, expect["or"], 10, "or, pending")
    results = {op: S.op(op, T, ia, ib) for op in expect}
    S.free()
    T.free()
    for k, (op, X) in enumerate(results.items()):
        _checked(R, X, expect[op], 11 + k, f"{op} after its operands were freed")


_INMEM = r'''
import ctypes as C, os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
import numpy as np
G = C.CDLL(os.path.join(sys.argv[1], "oracle", "_ref", "libroaring_ref.so"), mode=os.RTLD_GLOBAL)
from oracle.refbind import ref
import croaring_b200 as rb
from helpers import synth_blobs64
from test_gpu_query64 import Ref, check
R = ref()
rb.init(0)
blobs = synth_blobs64(R, 87, 20)
r = Ref(R, blobs)
S = rb.DeviceSet64(rb.lib().rb200_set64_upload((C.c_void_p * len(blobs))(*r.ptrs), len(blobs)))
check(S, r, 87, what="rb200_set64_upload")
print("set64 in-memory queries ok")
'''


def test_in_memory_upload():
    """rb200_set64_upload of the host application's roaring64_bitmap_t objects, in a process where the
    reference is loaded globally."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", _INMEM, root], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "set64 in-memory queries ok" in p.stdout, (p.stdout[-500:], p.stderr[-1500:])


# ----------------------------------------------------------------------------------------- equivalences
def test_public_methods_and_device_variant(rb, R):
    import torch
    blobs = _inputs(R, 88, 24)
    ref = Ref(R, blobs)
    S = rb.DeviceSet64.from_serialized(blobs)
    for kind, (idx, vals) in _queries(ref, np.random.default_rng(88), 30000).items():
        out, found = rb.api._query64(S, kind, vals, idx)
        assert out.dtype == np.uint64 and found.dtype == bool
        pub = getattr(S, kind)(vals, idx=idx)
        if kind == "contains":
            assert pub.dtype == bool and (pub == found).all() and (out == found).all()
        elif kind == "rank":
            assert pub.dtype == np.uint64 and (pub == out).all() and found.all()
        else:
            assert (pub[0] == out).all() and (pub[1] == found).all()
        for dt, tdt in ((np.int64, torch.int64), (np.uint64, torch.uint64)):
            tv = torch.from_numpy(vals.view(dt)).cuda()
            for ti in (torch.from_numpy(idx.view(np.int32)).cuda(), idx):   # device idx, host idx
                d_out, d_found = rb.api._query64(S, kind, tv, ti)
                assert d_out.is_cuda and d_out.dtype == tdt and d_found.dtype == torch.bool
                assert (d_out.cpu().numpy().view(np.uint64) == out).all(), (kind, tdt)
                assert (d_found.cpu().numpy() == found).all(), (kind, tdt)
        # a scalar idx with device values
        one = idx == idx[0]
        d_out, d_found = rb.api._query64(S, kind, _torch(vals[one]), int(idx[0]))
        assert (d_out.cpu().numpy().view(np.uint64) == out[one]).all() and (d_found.cpu().numpy() == found[one]).all()
    # the public methods on device values
    v = _torch(np.arange(len(blobs), dtype=np.uint64) << np.uint64(32))
    assert S.contains(v).dtype == torch.bool and S.rank(v).dtype == torch.int64
    gi, gf = S.get_index(v)
    assert gi.dtype == torch.int64 and gf.dtype == torch.bool
    ref.close()


def test_selections_agree(rb, R):
    blobs = _inputs(R, 89, 24)
    n = len(blobs)
    S = rb.DeviceSet64.from_serialized(blobs)
    rng = np.random.default_rng(89)
    vals = (rng.choice(np.array(HIGHS, dtype=np.uint64), n) << np.uint64(32)) | rng.integers(0, 6 << 16, n, dtype=np.uint64)
    ranks = rng.integers(0, 6000, n, dtype=np.uint64)
    for kind in KINDS:
        q = ranks if kind == "select" else vals
        f = lambda *a, **k: rb.api._query64(S, kind, *a, **k)
        none = f(q, None)
        for other in (f(q, np.arange(n)), f(_torch(q), None)):
            other = [x.cpu().numpy() if hasattr(x, "cpu") else x for x in other]
            assert (other[0].view(np.uint64) == none[0]).all() and (other[1] == none[1]).all(), kind
        for b in (0, 5, n - 1):   # a scalar asks every value of one bitmap
            one, many = f(q, b), f(q, np.full(n, b))
            assert (one[0] == many[0]).all() and (one[1] == many[1]).all(), (kind, b)
            assert one[0][b] == none[0][b] and one[1][b] == none[1][b], (kind, b)


# ----------------------------------------------------------------------------------------- launches, memory
def test_zero_queries_launch_nothing(rb, R):
    S = rb.DeviceSet64.from_serialized(_inputs(R, 90, 8))
    E = rb.DeviceSet64.from_values([])
    L = rb.lib()
    before = rb.kernel_launches()
    for kind in KINDS:
        out, found = rb.api._query64(S, kind, np.zeros(0, np.uint64), np.zeros(0, np.uint32))
        assert out.dtype == np.uint64 and out.size == 0 and found.size == 0
        out, found = rb.api._query64(S, kind, _torch([]), _torch([], np.int32))
        assert out.numel() == 0 and found.numel() == 0
        assert L.rb200_set64_batch_query(1, S.ptr, None, 0, None, None, None) == -1   # idx NULL: one per bitmap
        assert "vals are NULL" in rb.last_error()
    idx = np.zeros(1, np.uint32)
    assert L.rb200_set64_batch_query(0, S.ptr, idx.ctypes.data, 0, None, None, None) == 0
    assert L.rb200_set64_batch_query(3, E.ptr, None, 0, None, None, None) == 0
    assert L.rb200_set64_batch_query_device(2, E.ptr, None, 0, None, None, None) == 0
    assert E.rank([]).size == 0 and E.select(_torch([]))[0].numel() == 0
    assert rb.kernel_launches() == before


def test_prefix_cardinalities_are_cached(rb, R):
    blobs = [R.r64_from_values(_spread(_values32(R, b))) for b in rb.load_realdata("census1881")[:100]]
    L = rb.lib()
    base = int(L.rb200_device_bytes_in_use())
    S = rb.DeviceSet64.from_serialized(blobs)
    held = int(L.rb200_device_bytes_in_use())
    rng = np.random.default_rng(91)
    q = (rng.choice(np.array([0, 1, 0x10000], dtype=np.uint64), len(blobs)) << np.uint64(32)) | \
        rng.integers(0, 1 << 20, len(blobs), dtype=np.uint64)
    for _ in range(2):   # contains builds neither prefix: one launch, nothing kept
        before = rb.kernel_launches()
        S.contains(q)
        assert rb.kernel_launches() == before + 1
        assert int(L.rb200_device_bytes_in_use()) == held
    before = rb.kernel_launches()
    first = S.rank(q)
    assert rb.kernel_launches() > before + 1
    assert int(L.rb200_device_bytes_in_use()) > held
    for kind in ("rank", "get_index", "select", "contains"):
        before = rb.kernel_launches()
        out, _ = rb.api._query64(S, kind, q, None)
        assert rb.kernel_launches() == before + 1, kind
        if kind == "rank":
            assert (out == first).all()
    S.free()
    assert int(L.rb200_device_bytes_in_use()) == base
    # a batch result, queried while pending: the same, and its memory goes back with it
    S = rb.DeviceSet64.from_serialized(blobs)
    ia = np.arange(len(blobs), dtype=np.uint32)
    X = S.op("xor", S, ia, ia[::-1].copy())
    S.free()
    X.rank(q)
    before = rb.kernel_launches()
    X.select(q)
    assert rb.kernel_launches() == before + 1
    X.free()
    assert int(L.rb200_device_bytes_in_use()) == base


# ----------------------------------------------------------------------------------------- refusals
def test_refusals(rb, R):
    import torch
    blobs = _inputs(R, 92, 6)[:6]
    S = rb.DeviceSet64.from_serialized(blobs)
    L = rb.lib()
    S.rank(np.zeros(6, np.uint64))   # (builds the prefix cardinalities)
    before = rb.kernel_launches()
    # an index out of range, on the host: before any launch
    with pytest.raises(rb.RB200Error, match=r"^set64_query: index out of range: idx\[2\] = 6, the set holds 6 bitmaps$"):
        S.rank([1, 2, 3], idx=[0, 5, 6])
    # an unknown kind
    vals, out, found = np.array([1, 2], dtype=np.uint64), np.zeros(2, np.uint64), np.zeros(2, np.uint8)
    two = np.array([0, 1], dtype=np.uint32)
    for kind in (-1, 4, 99):
        assert L.rb200_set64_batch_query(kind, S.ptr, two.ctypes.data, 2, vals.ctypes.data, out.ctypes.data, None) == -1
        assert rb.last_error() == f"set64_query: unknown query kind {kind}"
        assert L.rb200_set64_batch_query_device(kind, S.ptr, None, 0, None, None, None) == -1
        assert rb.last_error() == f"set64_query_device: unknown query kind {kind}"
    with pytest.raises(rb.RB200Error, match="unknown query kind"):
        rb.api._query64(S, "maximum", [1], 0)
    # NULL vals / out with queries
    for fn, what in ((L.rb200_set64_batch_query, "set64_query"), (L.rb200_set64_batch_query_device, "set64_query_device")):
        assert fn(1, S.ptr, None, 6, None, out.ctypes.data, None) == -1
        assert rb.last_error() == f"{what}: vals are NULL"
        assert fn(1, S.ptr, None, 6, vals.ctypes.data, None, None) == -1
        assert rb.last_error() == f"{what}: out is NULL"
    # host pointers (pageable and pinned) passed to the device variant
    dv, dout, didx = _torch([1, 2]), torch.zeros(2, dtype=torch.int64, device="cuda"), _torch([0, 1], np.int32)
    dfound = torch.zeros(2, dtype=torch.bool, device="cuda")
    pinned = torch.zeros(2, dtype=torch.int64).pin_memory()
    for args, name in (((None, 2, vals.ctypes.data, dout.data_ptr(), None), "vals"),
                       ((None, 2, dv.data_ptr(), out.ctypes.data, None), "out"),
                       ((None, 2, dv.data_ptr(), pinned.data_ptr(), None), "out"),
                       ((two.ctypes.data, 2, dv.data_ptr(), dout.data_ptr(), None), "idx"),
                       ((didx.data_ptr(), 2, dv.data_ptr(), dout.data_ptr(), found.ctypes.data), "found")):
        assert L.rb200_set64_batch_query_device(1, S.ptr, *args) == -1
        assert rb.last_error() == f"set64_query_device: {name} is not device memory of the library's device"
    assert rb.kernel_launches() == before
    # an index out of range on the device: the kernel answers the rest, 2^64 - 1 / not found in that slot, and
    # the call fails with the host check's message naming the first such position
    for kind in KINDS:
        good, good_f = rb.api._query64(S, kind, [1, 1, 1], [0, 5, 2])
        idx = _torch([0, 7, 5, 1000, 2], np.int32)
        q = _torch([1, 1, 1, 1, 1])
        d_out = torch.full((5,), 12345, dtype=torch.int64, device="cuda")
        d_found = torch.ones(5, dtype=torch.bool, device="cuda")
        torch.cuda.synchronize()
        before = rb.kernel_launches()
        assert L.rb200_set64_batch_query_device(QK[kind], S.ptr, idx.data_ptr(), 5, q.data_ptr(), d_out.data_ptr(),
                                                d_found.data_ptr()) == -1
        assert rb.last_error() == "set64_query_device: index out of range: idx[1] = 7, the set holds 6 bitmaps"
        assert rb.kernel_launches() == before + 1
        assert d_out.cpu().numpy().view(np.uint64).tolist() == [good[0], T64, good[1], T64, good[2]], kind
        assert d_found.cpu().numpy().tolist() == [good_f[0], False, good_f[1], False, good_f[2]], kind
    with pytest.raises(rb.RB200Error, match=r"^set64_query_device: index out of range: idx\[1\] = 7"):
        S.rank(q, idx=idx)
    # the set is still usable
    assert (S.contains([1, 2], idx=[0, 0]) == S.contains(_torch([1, 2]), idx=_torch([0, 0], np.int32)).cpu().numpy()).all()

