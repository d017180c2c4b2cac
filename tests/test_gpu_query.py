"""GPU parity of the point queries (rb200_batch_query / _device): every contains / rank / get_index / select
answer equals the reference's roaring_bitmap_contains / rank / get_index / select of the same bitmap, called
once per query, over the synthetic container mixes and their no-run twins, the real-data sets, the long-
directory / top-of-key-space catalogue and every producer of a resident set; the edges of containers and
runs, empty bitmaps and the full universe; host / device and selection equivalences; the cached prefix
cardinalities; and the refusals."""
import ctypes as C

import numpy as np
import pytest

import croaring_b200.datasets as dsm
import wide_cases
from cow_oracles import STATES, make
from helpers import DATASETS, no_run_twins, synth_blobs
from offset_oracles import ref_add_offset_bytes
from test_gpu_update import PROFILES
from update_oracles import ref_update_bytes

pytestmark = pytest.mark.gpu

KINDS = ("contains", "rank", "get_index", "select")
U32 = 1 << 32


def _bind(R):
    """The reference's query functions (roaring.h:478, 1023-1057), all exported by libroaring_ref.so."""
    L = R.L
    for name, res, args in (("roaring_bitmap_contains", C.c_bool, [C.c_void_p, C.c_uint32]),
                            ("roaring_bitmap_rank", C.c_uint64, [C.c_void_p, C.c_uint32]),
                            ("roaring_bitmap_get_index", C.c_int64, [C.c_void_p, C.c_uint32]),
                            ("roaring_bitmap_select", C.c_bool, [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)])):
        getattr(L, name).restype = res
        getattr(L, name).argtypes = args
    return L


def ref_answers(R, ptrs, kind, idx, vals):
    """The reference's answer to every query, one call each."""
    L = _bind(R)
    out = np.empty(len(vals), dtype=np.int64)
    if kind == "select":
        el = C.c_uint32()
        for k, (i, v) in enumerate(zip(idx.tolist(), vals.tolist())):
            out[k] = el.value if L.roaring_bitmap_select(ptrs[i], v, C.byref(el)) else -1
        return out
    f = {"contains": L.roaring_bitmap_contains, "rank": L.roaring_bitmap_rank,
         "get_index": L.roaring_bitmap_get_index}[kind]
    for k, (i, v) in enumerate(zip(idx.tolist(), vals.tolist())):
        out[k] = int(f(ptrs[i], v))
    return out


class Ref:
    """Reference bitmaps holding what a resident set should hold (deserialized blobs, or given pointers)."""

    def __init__(self, R, blobs=None, ptrs=None):
        self.R = R
        self.ptrs = ptrs if ptrs is not None else [R.deserialize(b) for b in blobs]

    def close(self):
        for p in self.ptrs:
            self.R.free(p)
        self.ptrs = []


def _edge_values(a, rng, extra=24):
    """Values at, just below and just past every container's first and last value and every run's ends
    (maximal stretches of consecutive values), values in absent keys around the present ones, the ends of
    the key space and random present and uniform values."""
    c = [np.array([0, 1, 0xFFFF, 0x10000, 0xFFFF0000, 0xFFFFFFFE, 0xFFFFFFFF], dtype=np.int64),
         rng.integers(0, U32, extra)]
    if a.size:
        a = a.astype(np.int64)
        hi = a >> 16
        kb = np.r_[0, np.flatnonzero(np.diff(hi)) + 1]
        ke = np.r_[kb[1:] - 1, a.size - 1]
        rb = np.r_[0, np.flatnonzero(np.diff(a) != 1) + 1]
        re = np.r_[rb[1:] - 1, a.size - 1]
        pts = np.concatenate([a[kb], a[ke], a[rb], a[re]])
        c += [pts - 1, pts, pts + 1]
        keys = hi[kb]
        near = np.concatenate([keys - 1, keys + 1, [keys[0] - 2, keys[-1] + 2, 0, 65535]])
        c.append((near << 16) + rng.integers(0, 65536, near.size))
        c.append(rng.choice(a, extra))
    v = np.concatenate(c)
    return v[(v >= 0) & (v < U32)]


def _edge_ranks(a, rng, extra=24):
    """Ranks 0, 1, card - 1, card, card + 1, 2^32 - 1, around the first rank of every key, and random
    ranks below the cardinality."""
    card = a.size
    c = [np.array([0, 1, card - 1, card, card + 1, U32 - 1], dtype=np.int64), rng.integers(0, max(card, 1), extra)]
    if card:
        kb = np.r_[0, np.flatnonzero(np.diff(a.astype(np.int64) >> 16)) + 1]
        c += [kb - 1, kb, kb + 1]
    r = np.concatenate(c)
    return r[(r >= 0) & (r < U32)]


def _queries(R, ptrs, rng, cap):
    """{kind: (idx, vals)}: the edge queries of every bitmap, interleaved, at most cap per kind."""
    iv, vv, ir, rr = [], [], [], []
    for i, p in enumerate(ptrs):
        a = R.to_array(p)
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
            out[k] = (idx[pick].astype(np.uint32), vals[pick].astype(np.uint32))
    return out


def check(S, ref, seed, cap=20000, what=""):
    """Every kind over the edge queries of every bitmap of S, against the reference."""
    rng = np.random.default_rng(seed)
    for kind, (idx, vals) in _queries(ref.R, ref.ptrs, rng, cap).items():
        got = getattr(S, kind)(vals, idx=idx)
        exp = ref_answers(ref.R, ref.ptrs, kind, idx, vals)
        bad = np.flatnonzero(got != exp)
        assert not bad.size, (f"{what} {kind}: {bad.size} of {idx.size} differ, first: bitmap {idx[bad[0]]} "
                              f"value {vals[bad[0]]} -> {got[bad[0]]}, reference {exp[bad[0]]}")


def _empty(R):
    r = R.from_values(np.zeros(0, np.uint32))
    b = R.serialize(r)
    R.free(r)
    return b


def _inputs(R, seed):
    blobs = synth_blobs(R, seed, 30, key_space=6, max_keys=6, profiles=PROFILES if seed % 3 else None)
    return blobs + no_run_twins(R, blobs) + [_empty(R)]


def _torch(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).cuda()


# ----------------------------------------------------------------------------------------- inputs
@pytest.mark.parametrize("seed", [61, 62, 63])
def test_synthetic_mixes(rb, R, seed):
    blobs = _inputs(R, seed)
    ref = Ref(R, blobs)
    check(rb.DeviceSet.from_serialized(blobs), ref, seed, what=f"mix {seed}")
    ref.close()


@pytest.mark.parametrize("ds", DATASETS)
def test_realdata(rb, R, ds):
    blobs = dsm.load_realdata(ds)
    ref = Ref(R, blobs)
    check(rb.DeviceSet.from_serialized(blobs), ref, len(ds), cap=100000, what=ds)
    ref.close()


def test_wide_catalogue(rb, R):
    """Long directories (up to all 65536 keys) and the top of the key space; the reference walks the
    directory linearly per query, so the long bitmaps get fewer queries."""
    cases = [(n, b) for n, b in wide_cases.bitmaps(R) if n not in ("full_universe", "half_universe")]
    blobs = [b for _, b in cases]
    ref = Ref(R, blobs)
    check(rb.DeviceSet.from_serialized(blobs), ref, 64, cap=12000, what="catalogue")
    ref.close()


def test_full_universe(rb, R):
    """All 2^32 values as 65536 full runs and as 65536 full bitsets: counts past 32 bits."""
    full, half = wide_cases.bitmap(R, "full_universe"), wide_cases.bitmap(R, "half_universe")
    runs = rb.DeviceSet.from_serialized([full, half, _empty(R)])
    bitsets = runs.run_optimize(remove_runs=True)
    ref = Ref(R, [full, half, _empty(R)])
    rng = np.random.default_rng(65)
    for S, form in ((runs, "runs"), (bitsets, "bitsets")):
        assert list(S.rank([0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF])) == [U32, U32 // 2, 0], form
        assert list(S.select([U32 - 1, U32 // 2 - 1, 0])) == [0xFFFFFFFF, 0xFFFEFFFF, -1], form
        assert list(S.select([0, U32 // 2, U32 - 1])) == [0, -1, -1], form
        assert list(S.get_index([0xFFFFFFFF, 0xFFFEFFFF, 0])) == [U32 - 1, U32 // 2 - 1, -1], form
        assert list(S.contains([0xFFFFFFFF, 0xFFFFFFFF, 0])) == [1, 0, 0], form
        # edges of every 4096th key and random values / ranks, against the reference
        keys = np.arange(0, 65536, 4096, dtype=np.int64)
        vals = np.concatenate([(keys << 16) + d for d in (0, 1, 0xFFFE, 0xFFFF)] +
                              [((keys + 1) << 16) - 1, rng.integers(0, U32, 200), [0, U32 - 1]])
        ranks = np.concatenate([vals, keys << 16, (keys << 16) - 1, [U32 - 1, U32 - 2]])
        ranks = ranks[(ranks >= 0) & (ranks < U32)]
        for b in range(3):
            for kind, q in (("contains", vals), ("rank", vals), ("get_index", vals), ("select", ranks)):
                q = q.astype(np.uint32)
                idx = np.full(q.size, b, np.uint32)
                exp = ref_answers(R, ref.ptrs, kind, idx, q)
                assert (getattr(S, kind)(q, idx=b) == exp).all(), (form, b, kind)
    ref.close()


def test_empty_bitmaps(rb, R):
    e = _empty(R)
    S = rb.DeviceSet.from_serialized([e, e])
    v = np.array([0, 1, 65535, 65536, 0xFFFFFFFF], dtype=np.uint32)
    for b in (0, 1):
        assert (S.contains(v, idx=b) == 0).all() and (S.rank(v, idx=b) == 0).all()
        assert (S.get_index(v, idx=b) == -1).all() and (S.select(v, idx=b) == -1).all()
    # a set of empty bitmaps only: no containers, no prefix cardinalities, no reads of them
    assert S.container_count == 0
    assert list(S.rank(v[:2])) == [0, 0] and list(S.select(v[:2])) == [-1, -1]


# ----------------------------------------------------------------------------------------- producers
def test_every_producer(rb, R, O):
    blobs = _inputs(R, 66)
    ref = Ref(R, blobs)
    S = rb.DeviceSet.from_serialized(blobs)
    check(S, ref, 1, what="from_serialized")
    check(rb.DeviceSet.from_frozen(S.serialize_all(frozen=True)), ref, 2, what="from_frozen")
    check(rb.DeviceSet.from_values([R.to_array(p) for p in ref.ptrs]), ref, 3, what="from_values")
    check(S.run_optimize(), ref, 4, what="run_optimize")
    check(S.run_optimize(remove_runs=True), ref, 5, what="remove_run_compression")
    # upload from host bitmaps, copy-on-write inputs included; the reference answers on the same bitmaps
    for st in STATES:
        ptrs = [make(R, b, st) for b in blobs]
        U = rb.DeviceSet.upload([rb.Bitmap(p, own=False) for p in ptrs])
        check(U, Ref(R, ptrs=ptrs), 6, what=f"upload {st}")
        U.free()
        Ref(R, ptrs=ptrs).close()
    # folds
    check(S.or_many(), Ref(R, [O.many_bytes("or_many", blobs)]), 7, what="or_many")
    check(S.xor_many(), Ref(R, [O.many_bytes("xor_many", blobs)]), 8, what="xor_many")
    ref.close()


def test_results_outliving_their_operands(rb, R):
    """Batch results, key-aligned add_offset results and add_many results point into their operands'
    payloads: query them, still pending, after the operands are freed."""
    blobs = _inputs(R, 67)
    n = len(blobs)
    ia = np.arange(n, dtype=np.uint32)
    ib = (ia + 7) % n
    S, T = rb.DeviceSet.from_serialized(blobs), rb.DeviceSet.from_serialized(blobs[::-1])
    rng = np.random.default_rng(67)
    lists = [rng.integers(0, 8 << 16, 500).astype(np.uint32) for _ in blobs]
    new = [np.arange((40 + k % 3) << 16, ((40 + k % 3) << 16) + 3000 + k, dtype=np.uint32) for k in range(n)]
    results = {
        "or": (S.batch("or", T, ia, ib), [R.op_bytes("or", blobs[i], blobs[::-1][j]) for i, j in zip(ia, ib)]),
        "andnot": (S.batch("andnot", T, ia, ib), [R.op_bytes("andnot", blobs[i], blobs[::-1][j]) for i, j in zip(ia, ib)]),
        "xor": (S.batch("xor", T, ia, ib), [R.op_bytes("xor", blobs[i], blobs[::-1][j]) for i, j in zip(ia, ib)]),
        "offset+2^16": (S.add_offset(65536), [ref_add_offset_bytes(R, b, 65536) for b in blobs]),
        "offset-3*2^16": (S.add_offset(-3 * 65536), [ref_add_offset_bytes(R, b, -3 * 65536) for b in blobs]),
        "offset+12345": (S.add_offset(12345), [ref_add_offset_bytes(R, b, 12345) for b in blobs]),
        "add_many": (S.add_many(lists), [ref_update_bytes(R, "add", b, v) for b, v in zip(blobs, lists)]),
        "add_many new keys": (S.add_many(new), [ref_update_bytes(R, "add", b, v) for b, v in zip(blobs, new)]),
        "remove_many": (S.remove_many(lists), [ref_update_bytes(R, "remove", b, v) for b, v in zip(blobs, lists)]),
    }
    S.free()
    T.free()
    for seed, (name, (X, expect)) in enumerate(results.items()):
        ref = Ref(R, expect)
        check(X, ref, 100 + seed, what=name)
        ref.close()
    # a result of a result that shares (it copies instead) and of an update's shared new keys
    A = results["add_many new keys"][0]
    B = A.batch("or", A, ia, ib)
    results["add_many new keys"] = None
    del A
    exp_a = [ref_update_bytes(R, "add", b, v) for b, v in zip(blobs, new)]
    ref = Ref(R, [R.op_bytes("or", exp_a[i], exp_a[j]) for i, j in zip(ia, ib)])
    check(B, ref, 120, what="or of add_many")
    ref.close()


# ----------------------------------------------------------------------------------------- equivalences
def test_host_and_device_variants_agree(rb, R):
    import torch
    blobs = _inputs(R, 68)
    ref = Ref(R, blobs)
    S = rb.DeviceSet.from_serialized(blobs)
    for kind, (idx, vals) in _queries(R, ref.ptrs, np.random.default_rng(68), 30000).items():
        host = getattr(S, kind)(vals, idx=idx)
        dev = getattr(S, kind)(_torch(vals), idx=_torch(idx))
        assert dev.is_cuda and dev.dtype == torch.int64
        assert (dev.cpu().numpy() == host).all(), kind
        # idx given as a host array or a scalar with device values
        assert (getattr(S, kind)(_torch(vals), idx=idx).cpu().numpy() == host).all(), kind
        one = idx == idx[0]
        assert (getattr(S, kind)(_torch(vals[one]), idx=int(idx[0])).cpu().numpy() == host[one]).all(), kind
    ref.close()


def test_selections_agree(rb, R):
    blobs = _inputs(R, 69)
    n = len(blobs)
    S = rb.DeviceSet.from_serialized(blobs)
    rng = np.random.default_rng(69)
    vals = rng.integers(0, 6 << 16, n).astype(np.uint32)
    ranks = rng.integers(0, 3000, n).astype(np.uint32)
    for kind in KINDS:
        q = ranks if kind == "select" else vals
        f = getattr(S, kind)
        none = f(q)
        assert (f(q, idx=np.arange(n)) == none).all(), kind
        assert (f(_torch(q)).cpu().numpy() == none).all(), kind
        # a scalar asks every value of one bitmap
        for b in (0, 5, n - 1):
            assert (f(q, idx=b) == f(q, idx=np.full(n, b))).all(), (kind, b)
            assert f(q, idx=b)[b] == none[b], (kind, b)


def test_zero_queries_launch_nothing(rb, R):
    S = rb.DeviceSet.from_serialized(_inputs(R, 70))
    E = rb.DeviceSet.from_values([])
    L = rb.lib()
    before = rb.kernel_launches()
    for kind in KINDS:
        out = getattr(S, kind)(np.zeros(0, np.uint32), idx=np.zeros(0, np.uint32))
        assert out.dtype == np.int64 and out.size == 0
        assert getattr(S, kind)(_torch([]), idx=_torch([])).numel() == 0
        assert L.rb200_batch_query(1, S.ptr, None, 0, None, None) == -1   # idx NULL: one query per bitmap
        assert "vals are NULL" in rb.last_error()
    idx = np.zeros(1, np.uint32)
    assert L.rb200_batch_query(0, S.ptr, idx.ctypes.data, 0, None, None) == 0
    assert E.rank([]).size == 0 and L.rb200_batch_query(3, E.ptr, None, 0, None, None) == 0
    assert E.select(_torch([])).numel() == 0
    assert rb.kernel_launches() == before


# ----------------------------------------------------------------------------------------- scan cache
def test_prefix_cardinalities_are_cached(rb, R):
    blobs = dsm.load_realdata("census1881")[:200]
    L = rb.lib()
    base = int(L.rb200_device_bytes_in_use())
    S = rb.DeviceSet.from_serialized(blobs)
    held = int(L.rb200_device_bytes_in_use())
    q = np.random.default_rng(71).integers(0, 1 << 20, len(blobs)).astype(np.uint32)
    for _ in range(2):   # contains never builds the scan: one launch, nothing kept
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
        out = getattr(S, kind)(q)
        assert rb.kernel_launches() == before + 1, kind
        if kind == "rank":
            assert (out == first).all()
    S.free()
    assert int(L.rb200_device_bytes_in_use()) == base


# ----------------------------------------------------------------------------------------- refusals
def test_refusals(rb, R):
    import torch
    blobs = _inputs(R, 72)[:6]
    S = rb.DeviceSet.from_serialized(blobs)
    L = rb.lib()
    one = lambda v: np.array([v], dtype=np.uint32)
    # a lazy set: its c_card may carry CARD_UNKNOWN
    lz = S.batch("or", S, one(0), one(1), lazy=True)
    for kind in KINDS:
        with pytest.raises(rb.RB200Error, match="query: the set is in a lazy state"):
            getattr(lz, kind)([1])
        with pytest.raises(rb.RB200Error, match="query_device: the set is in a lazy state"):
            getattr(lz, kind)(_torch([1]))
    before = rb.kernel_launches()
    # an index out of range, on the host: before any launch
    with pytest.raises(rb.RB200Error, match=r"^query: index out of range: idx\[2\] = 6, the set holds 6 bitmaps$"):
        S.rank([1, 2, 3], idx=[0, 5, 6])
    assert rb.kernel_launches() == before
    # an unknown kind
    vals, out = np.array([1, 2], dtype=np.uint32), np.zeros(2, np.int64)
    for kind in (-1, 4, 99):
        assert L.rb200_batch_query(kind, S.ptr, None, 0, vals.ctypes.data, out.ctypes.data) == -1
        assert rb.last_error() == f"query: unknown query kind {kind}"
        assert L.rb200_batch_query_device(kind, S.ptr, None, 0, None, None) == -1
        assert rb.last_error() == f"query_device: unknown query kind {kind}"
    with pytest.raises(rb.RB200Error, match="unknown query kind"):
        rb.api._query(S, "maximum", [1], 0)
    # host pointers (pageable and pinned) passed to the device variant: refused before any launch
    dv, dout, didx = _torch([1, 2]), torch.zeros(2, dtype=torch.int64, device="cuda"), _torch([0, 1])
    pinned = torch.zeros(2, dtype=torch.int64).pin_memory()
    for args, name in (((None, 2, vals.ctypes.data, dout.data_ptr()), "vals"),
                       ((None, 2, dv.data_ptr(), out.ctypes.data), "out"),
                       ((None, 2, dv.data_ptr(), pinned.data_ptr()), "out"),
                       ((vals.ctypes.data, 2, dv.data_ptr(), dout.data_ptr()), "idx")):
        assert L.rb200_batch_query_device(1, S.ptr, *args) == -1
        assert rb.last_error() == f"query_device: {name} is not device memory of the library's device"
    assert rb.kernel_launches() == before
    # an index out of range on the device: the kernel answers the rest, -1 in that slot, and the call
    # fails with the host check's message naming the first such position
    good = S.rank([1, 1, 1], idx=[0, 5, 2])   # (builds the prefix cardinalities)
    idx = _torch([0, 7, 5, 1000, 2])
    q = _torch([1, 1, 1, 1, 1])
    d_out = torch.full((5,), 12345, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    before = rb.kernel_launches()
    assert L.rb200_batch_query_device(1, S.ptr, idx.data_ptr(), 5, q.data_ptr(), d_out.data_ptr()) == -1
    assert rb.last_error() == "query_device: index out of range: idx[1] = 7, the set holds 6 bitmaps"
    assert rb.kernel_launches() == before + 1
    got = d_out.cpu().numpy()
    assert list(got) == [good[0], -1, good[1], -1, good[2]]
    with pytest.raises(rb.RB200Error, match=r"query_device: index out of range: idx\[1\] = 7"):
        S.rank(q, idx=idx)
    # the set is still usable
    assert list(S.contains([1, 2], idx=[0, 0])) == list(S.contains(_torch([1, 2]), idx=_torch([0, 0])).cpu().numpy())
