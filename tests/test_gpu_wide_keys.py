"""GPU parity on long directories and at the top of the key space (tests/wide_cases.py): directories
of 31 to 65536 containers, key 65535 in every container form, the 16 key tiles of the many-way index,
pairs on both sides of the single-launch path's 512-container limit, many-way lists on both sides of
the 512-input gather round, XOR results of more than 1024 and of 65536 keys, and cardinalities of
2^32.  Every entry point compares bytes with the reference, and its results pass the reference's
validator; every failure names its case."""
import os
import subprocess
import sys

import numpy as np
import pytest

import run_cases as rc
import wide_cases as wc
from croaring_b200 import sharding as sh
from helpers import OPS, check_result_bitmap
from offset_oracles import ref_add_offset_bytes
from update_oracles import ref_update_bytes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYM = {"and": "__and__", "or": "__or__", "xor": "__xor__", "andnot": "__sub__"}
LAZY = [("or", False), ("or", True), ("xor", False)]
U32 = 1 << 32
FLIPS = [(0, U32), (65535 << 16, U32), ((4095 << 16) + 7, (13000 << 16) + 5)]   # the last ends in tile 3
KEY_RANGES = [(4095, 4096), (61440, 65535), (65535, 65535)]
CARD_FAMILY = ("and_cardinality", "or_cardinality", "xor_cardinality", "andnot_cardinality", "jaccard_index",
               "intersect", "equals", "is_subset", "is_strict_subset")


def _u32(a):
    return np.asarray(a, dtype=np.uint32)


def _catalogue(R):
    """{name: blob} of the single bitmaps and of both operands of every fused pair."""
    out = dict(wc.bitmaps(R))
    for name, a, b in wc.fused_pairs(R):
        out[name + ".a"], out[name + ".b"] = a, b
    return out


def _validated(R, S, k, exp, what):
    """One result of a set, downloaded, byte-exact and valid for the reference."""
    check_result_bitmap(R, S.download(k), exp, what)


def _ref_scalars(R, a, b):
    """The reference's and_cardinality and relations bits (equals | subset << 1 | strict << 2)."""
    ra, rb_ = R.deserialize(a), R.deserialize(b)
    c = int(R.L.roaring_bitmap_and_cardinality(ra, rb_))
    rel = (R.L.roaring_bitmap_equals(ra, rb_) | R.L.roaring_bitmap_is_subset(ra, rb_) << 1 |
           R.L.roaring_bitmap_is_strict_subset(ra, rb_) << 2)
    R.free(ra)
    R.free(rb_)
    return c, int(rel)


def _ref_conv(R, blob, remove_runs):
    r = R.deserialize(blob)
    if remove_runs:
        R.L.roaring_bitmap_remove_run_compression(r)
    else:
        R.L.roaring_bitmap_run_optimize(r)
    out = R.serialize(r)
    R.free(r)
    return out


# ------------------------------------------------------------------------------ 1. batched pairwise ops
def small_pairs():
    """Fewer than 16384 result items in all: the batch runs without class-ordered tickets."""
    lens = [f"len_{n}" for n in wc.LENS]
    pairs = list(zip(lens[1:], lens[2:])) + [("len_1025", "len_31"), ("tiles", "len_1025"), ("len_1", "len_1"),
                                              ("tiles", "tiles"), ("top_array", "top_full_run"),
                                              ("top_full_bitset", "top_run_end"), ("top_bitset", "top_full_bitset"),
                                              ("top_full_run", "top_array"), ("top_run_end", "top_bitset")]
    return pairs + [(f"fused_{t}.a", f"fused_{t}.b") for t in wc.FUSED]


def big_pairs():
    """Far more than 16384 items: 65536-container directories next to one-container pairs in the same
    4-pair blocks of the planner and finalize."""
    return [("all_keys", "top_full_run"), ("len_1", "len_1"), ("top_full_bitset", "all_keys"), ("len_1", "len_31"),
            ("even_keys", "odd_keys"), ("len_1", "len_1"), ("odd_keys", "all_keys"), ("len_32", "len_1"),
            ("all_keys", "even_keys"), ("len_1025", "all_keys"), ("full_universe", "half_universe"),
            ("half_universe", "all_keys"), ("tiles", "full_universe"), ("len_1", "len_1"), ("top_array", "all_keys")]


def check_batched(rb, R, pairs):
    cat = _catalogue(R)
    names = sorted({x for p in pairs for x in p})
    S = rb.DeviceSet.from_serialized([cat[x] for x in names])
    ia = _u32([names.index(a) for a, _ in pairs])
    ib = _u32([names.index(b) for _, b in pairs])
    blobs = [(cat[a], cat[b]) for a, b in pairs]
    n = 0
    for op in OPS:
        for inplace in (False, True):
            res = S.batch(op, S, ia, ib, inplace_rules=inplace)
            got = res.serialize_all()
            for k, (a, b) in enumerate(blobs):
                exp = R.op_inplace_bytes(op, a, b) if inplace else R.op_bytes(op, a, b)
                assert got[k] == exp, f"{pairs[k]}: batch {op} inplace={inplace}"
                n += 1
            _validated(R, res, 0, got[0], f"{pairs[0]}: batch {op} inplace={inplace}")
            res.free()
    for op, conv in LAZY:
        res = S.batch(op, S, ia, ib, lazy=True, bitsetconversion=conv).repair_after_lazy()
        got = res.serialize_all()
        for k, (a, b) in enumerate(blobs):
            assert got[k] == R.lazy_fold_bytes(op, conv, [a, b]), f"{pairs[k]}: batch lazy {op} conv={conv}"
            n += 1
        _validated(R, res, 0, got[0], f"{pairs[0]}: batch lazy {op} conv={conv}")
        res.free()
    card = S.and_cardinality(S, ia, ib)
    rel = S.relations(S, ia, ib)
    for k, (a, b) in enumerate(blobs):
        c, r = _ref_scalars(R, a, b)
        assert int(card[k]) == c, f"{pairs[k]}: and_cardinality {int(card[k])} != {c}"
        assert int(rel[k]) == r, f"{pairs[k]}: relations {int(rel[k])} != {r}"
    return n


def test_batched_pairs_below_ticket_threshold(rb, R):
    pairs = small_pairs()
    items = sum(len(rc.blob_containers(_catalogue(R)[x])) for p in pairs for x in p)
    assert items < 16384
    assert check_batched(rb, R, pairs) == 11 * len(pairs)


def test_batched_pairs_above_ticket_threshold(rb, R):
    assert check_batched(rb, R, big_pairs()) == 11 * len(big_pairs())


# ------------------------------------------------------------------------------ 2. drop-in symbols
def _dropin_pairs(R):
    """The fused pairs both ways, each operand with itself, a subset of it (a AND b, a), and the top
    forms against each other."""
    out = []
    for name, a, b in wc.fused_pairs(R):
        out += [(name, a, b), (name + " swapped", b, a), (name + " a,a", a, a),
                (name + " a&b,a", R.op_bytes("and", a, b), a)]
    tops = [f"top_{f}" for f in wc.TOP_FORMS]
    for x, y in zip(tops, tops[1:] + tops[:1]):
        out.append((f"{x} x {y}", wc.bitmap(R, x), wc.bitmap(R, y)))
    return out


def _ref_scalar(R, fn, a, b):
    ra, rb_ = R.deserialize(a), R.deserialize(b)
    v = getattr(R.L, f"roaring_bitmap_{fn}")(ra, rb_)
    R.free(ra)
    R.free(rb_)
    return v


def test_dropin_symbols(rb, R):
    seen = {"strict": 0, "equal": 0}
    for name, a, b in _dropin_pairs(R):
        y = rb.Bitmap.deserialize(b)
        for op in OPS:
            x = rb.Bitmap.deserialize(a)
            check_result_bitmap(R, getattr(x, SYM[op])(y), R.op_bytes(op, a, b), f"{name}: {op}")
            check_result_bitmap(R, x.inplace(op, y), R.op_inplace_bytes(op, a, b), f"{name}: {op} inplace")
        x = rb.Bitmap.deserialize(a)
        for fn in CARD_FAMILY:
            got, exp = getattr(x, fn)(y), _ref_scalar(R, fn, a, b)
            assert got == exp, f"{name}: {fn} {got} != {exp}"
        seen["equal"] += x.equals(y)
        seen["strict"] += x.is_strict_subset(y)
    assert seen["equal"] >= len(wc.FUSED) and seen["strict"] >= len(wc.FUSED), seen


# ------------------------------------------------------------------------------ 3. flip
def test_flip_batched_and_dropin(rb, R):
    bitmaps = list(wc.bitmaps(R))
    S = rb.DeviceSet.from_serialized([b for _, b in bitmaps])
    for s, e in FLIPS:
        res = S.flip(s, e)
        got = res.serialize_all()
        for k, (name, b) in enumerate(bitmaps):
            assert got[k] == R.flip_bytes(b, s, e), f"{name}: batch flip [{s}, {e})"
        _validated(R, res, 5, got[5], f"{bitmaps[5][0]}: batch flip [{s}, {e})")
        res.free()
    for name in [f"top_{f}" for f in wc.TOP_FORMS] + ["tiles", "len_1025", "full_universe"]:
        b = wc.bitmap(R, name)
        for s, e in FLIPS:
            x = rb.Bitmap.deserialize(b)
            check_result_bitmap(R, x.flip(s, e), R.flip_bytes(b, s, e), f"{name}: flip [{s}, {e})")
            check_result_bitmap(R, x.flip_inplace(s, e), R.flip_bytes(b, s, e, inplace=True),
                                f"{name}: flip_inplace [{s}, {e})")


# ------------------------------------------------------------------------------ 4. many-way
def _many_inputs(R):
    cat = [b for name, b in wc.bitmaps(R) if not name.endswith("universe")]
    return list(wc.many_lists(R)) + [("catalogue", tuple(cat))]


def check_or_many(rb, R):
    """or_many of every list, whole and over the key ranges, with card_per_key."""
    n = 0
    for name, blobs in _many_inputs(R):
        S = rb.DeviceSet.from_serialized(list(blobs))
        exp = R.many_bytes("or_many", blobs)
        res = S.or_many()
        _validated(R, res, 0, exp, f"{name}: or_many")
        res.free()
        for lo, hi in KEY_RANGES:
            cpk = np.zeros(65536, dtype=np.uint32)
            res = S.or_many(key_lo=lo, key_hi=hi, card_per_key=cpk)
            part = sh.slice_blob_by_keys(exp, lo, hi)
            assert res.serialize_all()[0] == part, f"{name}: or_many keys [{lo}, {hi}]"
            keys, cards = sh.blob_key_cards(part)
            want = np.zeros(65536, dtype=np.uint32)
            want[keys.astype(np.int64)] = cards
            assert np.array_equal(cpk, want), f"{name}: card_per_key of keys [{lo}, {hi}]"
            assert len(keys), f"{name}: keys [{lo}, {hi}] hold nothing"
            res.free()
            n += 1
        S.free()
    return n


@pytest.mark.parametrize("index", ["window", "atomic"])
def test_or_many_with_forced_index(R, index):
    """The index builder is chosen once per process (RB200_OR_MANY_INDEX): each runs in a child."""
    code = (f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
            "import croaring_b200 as rb\nfrom oracle.refbind import ref\nimport test_gpu_wide_keys as t\n"
            "rb.init(0)\nprint('checked', t.check_or_many(rb, ref()))\n")
    env = dict(os.environ, RB200_OR_MANY_INDEX=index)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert f"checked {len(KEY_RANGES) * len(_many_inputs(R))}" in r.stdout, r.stdout[-2000:]


def test_or_many_heap_and_xor_many(rb, R):
    for name, blobs in _many_inputs(R):
        S = rb.DeviceSet.from_serialized(list(blobs))
        for fold in ("or_many_heap", "xor_many"):
            res = getattr(S, fold)()
            _validated(R, res, 0, R.many_bytes(fold, blobs), f"{name}: {fold}")
            res.free()
        S.free()


# ------------------------------------------------------------------------------ 5. add_offset
OFFSETS = [1, -1, 65535, 65536, -65536, U32 - 1, -(U32 - 1)]


def test_add_offset(rb, R):
    names = [f"top_{f}" for f in wc.TOP_FORMS] + ["tiles", "all_keys"]
    blobs = [wc.bitmap(R, x) for x in names]
    S = rb.DeviceSet.from_serialized(blobs)
    for off in OFFSETS:
        res = S.add_offset(off)
        got = res.serialize_all()
        for k, (name, b) in enumerate(zip(names, blobs)):
            assert got[k] == ref_add_offset_bytes(R, b, off), f"{name}: add_offset {off}"
        _validated(R, res, len(names) - 1, got[-1], f"all_keys: add_offset {off}")
        res.free()
    # one batch mixing key-aligned and split offsets, bitmaps repeated
    idx = _u32([6, 0, 5, 6, 4, 1, 3, 2, 6, 5])
    offs = [65536, 7, -(5 << 16), -65535, U32 - 65536, 1, 1 << 31, -(U32 - 1), -3, (12 << 16) + 99]
    got = S.add_offset(offs, idx=idx).serialize_all()
    for k, (i, off) in enumerate(zip(idx, offs)):
        assert got[k] == ref_add_offset_bytes(R, blobs[i], off), f"{names[i]}: add_offset {off} in a mixed batch"


# ------------------------------------------------------------------------------ 6. add_many / remove_many
def _update_values(R, blob):
    """The edge values, one value on every key, and values the bitmap holds (so removal empties keys)."""
    r = R.deserialize(blob)
    held = R.to_array(r)
    R.free(r)
    rng = np.random.default_rng(len(blob))
    every_key = (np.arange(65536, dtype=np.uint32) << np.uint32(16)) | rng.integers(0, 65536, 65536).astype(np.uint32)
    some_held = held[rng.choice(held.size, min(held.size, 40000), replace=False)]
    return np.r_[_u32([0, 0xFFFF, 0x10000, 0xFFFF0000, 0xFFFFFFFF]), every_key, some_held, held[-3:]]


def test_add_and_remove_many(rb, R):
    names = [f"top_{f}" for f in wc.TOP_FORMS] + ["all_keys"]
    blobs = [wc.bitmap(R, x) for x in names]
    vals = [_update_values(R, b) for b in blobs]
    S = rb.DeviceSet.from_serialized(blobs)
    for op in ("add", "remove"):
        res = getattr(S, f"{op}_many")(vals)
        got = res.serialize_all()
        for k, (name, b) in enumerate(zip(names, blobs)):
            assert got[k] == ref_update_bytes(R, op, b, vals[k]), f"{name}: {op}_many"
        _validated(R, res, len(names) - 1, got[-1], f"all_keys: {op}_many")
        res.free()


# ------------------------------------------------------------------------------ 7. conversions, downloads
def test_conversions_and_downloads(rb, R):
    """The catalogue after the 1025 inputs of list_1025: 1064 bitmaps, so the long directories sit in
    the second 1024-bitmap round of the download and serializer scans."""
    cat = _catalogue(R)
    x = wc.many_list(R, "list_1025")
    names = [f"list_1025[{k}]" for k in range(len(x))] + list(cat)
    blobs = list(x) + [cat[n] for n in cat]
    S = rb.DeviceSet.from_serialized(blobs)
    for remove in (False, True):
        got = S.run_optimize(remove_runs=remove).serialize_all()
        for k, name in enumerate(names):
            assert got[k] == _ref_conv(R, blobs[k], remove), f"{name}: run_optimize(remove_runs={remove})"
    portable = S.serialize_all()
    for k, name in enumerate(names):
        assert portable[k] == blobs[k], f"{name}: serialize_all"
    frozen = S.serialize_all(frozen=True)
    for k, name in enumerate(names):
        assert frozen[k] == R.frozen_bytes(blobs[k]), f"{name}: serialize_all(frozen=True)"
    assert rb.DeviceSet.from_serialized(portable).serialize_all() == blobs
    assert rb.DeviceSet.from_frozen(frozen).serialize_all() == blobs
    for chunk in (1, 97):
        k = 0
        for arr, n in S.download_stream(chunk):
            for i in range(n):
                ok, why = R.validate(arr[i])
                assert ok, f"{names[k]}: download_stream({chunk}): {why}"
                assert R.serialize(arr[i]) == blobs[k], f"{names[k]}: download_stream({chunk})"
                k += 1
            rb.DeviceSet.free_raw(arr, n)
        assert k == len(names)
    # to_uint32_arrays: not on the universes, whose 2^32 and 2^31 values would take 16 and 8 GiB
    small = [k for k, name in enumerate(names) if not name.endswith("universe")]
    T = rb.DeviceSet.from_serialized([blobs[k] for k in small])
    for k, arr in zip(small, T.to_uint32_arrays()):
        r = R.deserialize(blobs[k])
        assert np.array_equal(arr, R.to_array(r)), f"{names[k]}: to_uint32_arrays"
        R.free(r)


# ------------------------------------------------------------------------------ 8. the full universe
def test_full_universe(rb, R):
    full, half = wc.bitmap(R, "full_universe"), wc.bitmap(R, "half_universe")
    empty = wc.assemble(R, [], [])
    S = rb.DeviceSet.from_serialized([full, half, empty])
    assert S.cardinalities().tolist() == [U32, U32 // 2, 0]
    assert S.serialize_all() == [full, half, empty]
    ia, ib = _u32([0, 0, 1, 1]), _u32([0, 1, 0, 1])
    assert S.and_cardinality(S, ia, ib).tolist() == [U32, U32 // 2, U32 // 2, U32 // 2]
    rel = S.relations(S, ia, ib).tolist()
    assert rel == [_ref_scalars(R, [full, half][i], [full, half][j])[1] for i, j in zip(ia, ib)]
    assert rel[0] == 3 and rel[2] == 6
    for op in ("or", "xor", "andnot"):
        res = S.batch(op, S, _u32([0, 1]), _u32([1, 0]))
        exp = [R.op_bytes(op, full, half), R.op_bytes(op, half, full)]
        assert res.serialize_all() == exp, f"full x half: {op}"
        assert res.cardinalities().tolist() == [{"or": U32, "xor": U32 // 2, "andnot": U32 // 2}[op],
                                                {"or": U32, "xor": U32 // 2, "andnot": 0}[op]], op
        _validated(R, res, 0, exp[0], f"full x half: {op}")
        res.free()
    # xor_many: full ^ full is empty; full ^ empty keeps every key and 2^32 values
    for sel, card in (([0, 0], 0), ([0, 2], U32), ([2, 0, 1], U32 // 2)):
        res = S.xor_many(_u32(sel))
        _validated(R, res, 0, R.many_bytes("xor_many", [[full, half, empty][i] for i in sel]), f"xor_many {sel}")
        assert res.cardinalities().tolist() == [card], sel
        res.free()
    cpk = np.zeros(65536, dtype=np.uint32)
    res = S.or_many(_u32([0, 1]), card_per_key=cpk)
    _validated(R, res, 0, full, "or_many(full, half)")
    assert np.all(cpk == 65536)
    assert res.cardinalities().tolist() == [U32]
    x, y = rb.Bitmap.deserialize(full), rb.Bitmap.deserialize(half)
    assert x.or_cardinality(y) == _ref_scalar(R, "or_cardinality", full, half) == U32
    assert x.jaccard_index(y) == _ref_scalar(R, "jaccard_index", full, half) == 0.5
    assert x.and_cardinality(x) == U32
    res = S.add_offset(1, idx=_u32([0, 1]))
    for k, b in enumerate([full, half]):
        _validated(R, res, k, ref_add_offset_bytes(R, b, 1), f"universe #{k}: add_offset 1")


# ------------------------------------------------------------------------------ 9. 64-bit
def test_set64_buckets_0_and_top(rb, R):
    """Catalogue bitmaps as buckets 0 and 0xFFFFFFFF of 64-bit bitmaps."""
    parts = [("top_full_bitset", "all_keys"), ("all_keys", "top_array"), ("tiles", "len_1025"),
             ("even_keys", "odd_keys"), ("len_1", "top_run_end"), ("odd_keys", "even_keys")]
    blobs = []
    for i, (lo, hi) in enumerate(parts):
        v = []
        for bucket, name in ((0, lo), (0xFFFFFFFF, hi)):
            r = R.deserialize(wc.bitmap(R, name))
            v.append(R.to_array(r).astype(np.uint64) | np.uint64(bucket << 32))
            R.free(r)
        blobs.append(R.r64_from_values(np.concatenate(v), run_optimize=bool(i % 2)))
    S = rb.DeviceSet64.from_serialized(blobs)
    assert S.serialize_all() == blobs
    ia, ib = _u32([0, 1, 2, 3, 4, 5, 1]), _u32([1, 0, 2, 5, 3, 3, 4])
    for op in OPS:
        got = S.op(op, S, ia, ib).serialize_all()
        for k, (i, j) in enumerate(zip(ia, ib)):
            assert got[k] == R.r64_op_bytes(op, blobs[i], blobs[j]), f"64-bit {op} {parts[i]} x {parts[j]}"
    card = S.and_cardinality(S, ia, ib)
    for k, (i, j) in enumerate(zip(ia, ib)):
        assert int(card[k]) == R.r64_and_cardinality(blobs[i], blobs[j]), f"64-bit and_cardinality {parts[i]} x {parts[j]}"


def test_set64_more_than_1024_bitmaps(rb, R):
    """list_1025's inputs in bucket 0xFFFFFFFF, then the long 64-bit bitmaps: the serializer's size
    scan runs a second 1024-bitmap round."""
    blobs = []
    for k, b in enumerate(wc.many_list(R, "list_1025")):
        r = R.deserialize(b)
        blobs.append(R.r64_from_values(R.to_array(r).astype(np.uint64) | np.uint64(0xFFFFFFFF << 32),
                                       run_optimize=bool(k % 2)))
        R.free(r)
    for name in ("all_keys", "len_1025"):
        r = R.deserialize(wc.bitmap(R, name))
        v = R.to_array(r).astype(np.uint64)
        R.free(r)
        blobs.append(R.r64_from_values(np.r_[v, v | np.uint64(0xFFFFFFFF << 32)]))
    S = rb.DeviceSet64.from_serialized(blobs)
    assert S.serialize_all() == blobs
    n = len(blobs)
    ia, ib = _u32(np.arange(n - 1)), _u32(np.arange(1, n))
    for op in ("or", "xor"):
        got = S.op(op, S, ia, ib).serialize_all()
        for k in range(n - 1):
            assert got[k] == R.r64_op_bytes(op, blobs[k], blobs[k + 1]), f"64-bit {op} #{k} x #{k + 1}"
