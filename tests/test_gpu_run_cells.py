"""GPU parity of run containers at the edges of the code that handles them (tests/run_cases.py):
the interval sweep's 512 cutoff and its ties across lane splits, the rasteriser's word edges and
gap clearing, 2047 / 2048 / 8192 / 8193 / 32768-run containers, run x bitset for every op, and
non-optimal run containers.  Every pair runs in both orders through the batched path (functional,
in place, lazy + repair, cardinality, relations) and the single-pair drop-in symbols; flip, the
many-way unions / xor and the producers (run_optimize, repair_after_lazy, serialize) run on the same
containers.  The class-ordered cell list and both staging paths of the many-way union are forced in
child processes (their switches are read once per process).  Every expectation is the reference's;
every failure names its case."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import run_cases as rc
from helpers import OPS, check_result_bitmap

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAZY = [("or", False), ("or", True), ("xor", False)]
SYM = {"and": "__and__", "or": "__or__", "xor": "__xor__", "andnot": "__sub__"}


def _u32(a):
    return np.asarray(a, dtype=np.uint32)


def _ref_pair_scalars(R, a, b):
    ra, rb_ = R.deserialize(a), R.deserialize(b)
    c = int(R.L.roaring_bitmap_and_cardinality(ra, rb_))
    rel = (R.L.roaring_bitmap_equals(ra, rb_) | R.L.roaring_bitmap_is_subset(ra, rb_) << 1 |
           R.L.roaring_bitmap_is_strict_subset(ra, rb_) << 2)
    R.free(ra)
    R.free(rb_)
    return c, int(rel)


def _batched(rb, S, ia, ib, names, what, run):
    """run(S, ia, ib) -> list of bytes.  A batch the library refuses as a whole is retried one pair
    at a time, so that the failure names its case."""
    try:
        return run(S, ia, ib)
    except rb.RB200Error as e:
        for k, name in enumerate(names):
            try:
                run(S, ia[k:k + 1], ib[k:k + 1])
            except rb.RB200Error as e1:
                raise AssertionError(f"{name}: {what}: {e1}") from None
        raise AssertionError(f"{what}: {e}") from None


# ------------------------------------------------------------------------------ checks
# (plain functions: the child processes call them too; each returns how many results it compared)
def check_batched(rb, R):
    """Every catalogue pair as one DeviceSet: the four ops functional and in place, the lazy OR /
    XOR followed by a lazy in-place step and repair_after_lazy, and_cardinality, relations."""
    pairs, _ = rc.catalogue()
    names = [p[0] for p in pairs]
    blobs = [x for _, a, b in pairs for x in (a, b)]
    S = rb.DeviceSet.from_serialized(blobs)
    ia = np.arange(0, len(blobs), 2, dtype=np.uint32)
    ib = ia + 1
    n = 0
    for op in OPS:
        for inplace in (False, True):
            what = f"batch {op} inplace={inplace}"
            got = _batched(rb, S, ia, ib, names, what,
                           lambda S, x, y: S.batch(op, S, x, y, inplace_rules=inplace).serialize_all())
            for k, (name, a, b) in enumerate(pairs):
                exp = R.op_inplace_bytes(op, a, b) if inplace else R.op_bytes(op, a, b)
                assert got[k] == exp, f"{name}: {what}"
                n += 1
    for op, conv in LAZY:
        what = f"batch lazy {op} conv={conv}"
        got1 = _batched(rb, S, ia, ib, names, what, lambda S, x, y: S.batch(
            op, S, x, y, lazy=True, bitsetconversion=conv).repair_after_lazy().serialize_all())
        got2 = _batched(rb, S, ia, ib, names, what + " then in place", lambda S, x, y: S.batch(
            op, S, x, y, lazy=True, bitsetconversion=conv).batch(
            op, S, np.arange(len(x), dtype=np.uint32), x, lazy=True, inplace_rules=True,
            bitsetconversion=conv).repair_after_lazy().serialize_all())
        for k, (name, a, b) in enumerate(pairs):
            assert got1[k] == R.lazy_fold_bytes(op, conv, [a, b]), f"{name}: batch lazy {op} conv={conv}"
            assert got2[k] == R.lazy_fold_bytes(op, conv, [a, b, a]), f"{name}: batch lazy {op} conv={conv} then in place"
            n += 2
    card = S.and_cardinality(S, ia, ib)
    rel = S.relations(S, ia, ib)
    for k, (name, a, b) in enumerate(pairs):
        c, r = _ref_pair_scalars(R, a, b)
        assert int(card[k]) == c, f"{name}: and_cardinality {int(card[k])} != {c}"
        assert int(rel[k]) == r, f"{name}: relations {int(rel[k])} != {r}"
        n += 2
    return n


def check_dropin(rb, R):
    """Every catalogue pair through the drop-in symbols, one pair per call."""
    pairs, _ = rc.catalogue()
    n = 0
    for name, a, b in pairs:
        y = rb.Bitmap.deserialize(b)
        for op in OPS:
            x = rb.Bitmap.deserialize(a)
            check_result_bitmap(R, getattr(x, SYM[op])(y), R.op_bytes(op, a, b), f"{name}: {op}")
            check_result_bitmap(R, x.inplace(op, y), R.op_inplace_bytes(op, a, b), f"{name}: {op} inplace")
            n += 2
        for op, conv in LAZY:
            x = rb.Bitmap.deserialize(a)
            if op == "or":
                r = x.lazy_or(y, conv).lazy_or_inplace(x, conv).repair_after_lazy()
            else:
                r = x.lazy_xor(y).lazy_xor_inplace(x).repair_after_lazy()
            check_result_bitmap(R, r, R.lazy_fold_bytes(op, conv, [a, b, a]), f"{name}: lazy {op} conv={conv}")
            n += 1
    return n


def flip_ranges():
    """Range ends on a run's start (325), on its end + 1 (612), strictly inside runs, on 65535 /
    65536 of a key, across keys, a whole absent key and one value of an absent key (key 9)."""
    k9 = 9 << 16
    return [(325, 612), (325, 400), (400, 612), (612, 1000), (330, 65535), (0, 65536), (65535, 65536),
            (65535, 65537), (60000, (3 << 16) + 17), (65536, 2 << 16), (k9 + 5, k9 + 6), (k9, k9 + 65536),
            (3, (6 << 16) + 1)]


def check_flip(rb, R):
    _, bitmaps = rc.catalogue()
    blobs = [b for _, b in bitmaps]
    S = rb.DeviceSet.from_serialized(blobs)
    n = 0
    for s, e in flip_ranges():
        got = S.flip(s, e).serialize_all()
        for k, (name, b) in enumerate(bitmaps):
            assert got[k] == R.flip_bytes(b, s, e), f"{name}: flip [{s}, {e})"
            n += 1
    return n


def check_many(rb, R):
    """or_many (whole list and idx subsets with repeats), or_many_heap and xor_many on the sweep lists."""
    n = 0
    for name, blobs in rc.sweep_lists():
        S = rb.DeviceSet.from_serialized(blobs)
        rng = np.random.default_rng(len(blobs))
        subsets = [None] + [rng.integers(0, len(blobs), int(rng.integers(2, len(blobs) + 1))) for _ in range(2)]
        for idx in subsets:
            sub = blobs if idx is None else [blobs[i] for i in idx]
            what = f"{name} idx={'all' if idx is None else idx.tolist()}"
            i = None if idx is None else _u32(idx)
            assert S.or_many(i).serialize_all()[0] == R.many_bytes("or_many", sub), f"{what}: or_many"
            assert S.or_many_heap(i).serialize_all()[0] == R.many_bytes("or_many_heap", sub), f"{what}: or_many_heap"
            assert S.xor_many(i).serialize_all()[0] == R.many_bytes("xor_many", sub), f"{what}: xor_many"
            n += 3
    return n


CHILD = r'''
import json, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import croaring_b200 as rb
from oracle.refbind import ref
import test_gpu_run_cells as T
rb.init(0)
checked = {}
try:
    for fn in sys.argv[2:]:
        checked[fn] = getattr(T, fn)(rb, ref())
except AssertionError as e:
    print(json.dumps({"ok": False, "case": str(e)}))
else:
    print(json.dumps({"ok": True, "checked": checked}))
'''


def _child(env, *checks):
    out = subprocess.run([sys.executable, "-c", CHILD, ROOT, *checks], env=dict(os.environ, **env),
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    verdict = json.loads(out.stdout.strip().splitlines()[-1])
    assert verdict["ok"], f"{env}: {verdict['case']}"
    assert all(v > 0 for v in verdict["checked"].values())


# ------------------------------------------------------------------------------ tests
def test_pairs_batched(rb, R):
    check_batched(rb, R)


def test_pairs_dropin(rb, R):
    check_dropin(rb, R)


def test_flip(rb, R):
    check_flip(rb, R)


def test_class_ordered_tickets():
    """The pairwise sweep and the flips with the class-ordered cell list and pass-through tickets
    (by default only batches of at least 16384 item slots take them)."""
    _child({"RB200_ORDER_MIN": "0"}, "check_batched", "check_flip")


def test_many_way(rb, R):
    check_many(rb, R)


@pytest.mark.parametrize("tma", ["1", "0"], ids=["bulk_copy", "direct"])
def test_many_way_forced_staging(tma):
    _child({"RB200_OR_MANY_TMA": tma}, "check_many")


def _tie_bodies():
    """Run lists whose optimal encoding sits on a tie of the size rule: n runs with card 2n, 2n + 1
    and 2n + 2 (the array rule 2 + 4n against 2c), and 2047 / 2048 runs of more than 4096 values
    (the bitset rule 2 + 4n against 8192)."""
    out = []
    for n in (100, 2047):
        for extra in (0, 1, 2):
            out.append((f"n{n}_c2n+{extra}", [(8 * i, 2 if i < extra else 1) for i in range(n)]))
    for n in (2047, 2048):
        out.append((f"n{n}_3each", [(32 * i, 2) for i in range(n)]))
    return out


def test_run_optimize_at_size_ties(rb, R):
    """Each tie written as a run container and as an array or bitset of the same values."""
    cases = []
    for name, body in _tie_bodies():
        vals = rc.values_of(rc.run(body))
        kind = "array" if vals.size <= rc.MAX_ARRAY else "bitset"
        cases.append((name + "_as_run", rc.run_blob([rc.run(body)])))
        cases.append((name + "_as_" + kind, rc.run_blob([(rc.KEY, kind, vals.tolist())])))
    S = rb.DeviceSet.from_serialized([b for _, b in cases])
    for remove in (False, True):
        got = S.run_optimize(remove_runs=remove).serialize_all()
        for k, (name, b) in enumerate(cases):
            r = R.deserialize(b)
            (R.L.roaring_bitmap_remove_run_compression if remove else R.L.roaring_bitmap_run_optimize)(r)
            exp = R.serialize(r)
            R.free(r)
            assert got[k] == exp, f"{name}: run_optimize(remove_runs={remove})"


def test_repair_after_lazy_at_size_ties(rb, R):
    """A lazy array | run leaves the union a run container; repair_after_lazy picks its encoding.
    The array holds values of the run container, so the unions land on the ties of the size rule."""
    pairs = []
    for name, body in _tie_bodies():
        vals = rc.values_of(rc.run(body))
        pairs.append((name, rc.run_blob([rc.array(vals[::97])]), rc.run_blob([rc.run(body)])))
    blobs = [x for _, a, b in pairs for x in (a, b)]
    S = rb.DeviceSet.from_serialized(blobs)
    ia = np.arange(0, len(blobs), 2, dtype=np.uint32)
    for conv in (False, True):
        for left, right, tag in ((ia, ia + 1, ""), (ia + 1, ia, "_swapped")):
            got = S.batch("or", S, left, right, lazy=True, bitsetconversion=conv).repair_after_lazy().serialize_all()
            for k, (name, a, b) in enumerate(pairs):
                x, y = (a, b) if not tag else (b, a)
                exp = R.lazy_fold_bytes("or", conv, [x, y])
                assert got[k] == exp, f"{name}{tag}: lazy or conv={conv} + repair"
                bx, by = rb.Bitmap.deserialize(x), rb.Bitmap.deserialize(y)
                check_result_bitmap(R, bx.lazy_or(by, conv).repair_after_lazy(), exp,
                                    f"{name}{tag}: drop-in lazy or conv={conv} + repair")


def test_serialize_round_trip_of_32768_runs(rb, R):
    """The device parse and the run-cardinality recount of the largest run container, alone and in
    a multi-key bitmap, through serialize_all, the download and an identity op."""
    multi = dict((n, rc.run_blob(c)) for n, c in rc.multi_key_bitmaps())
    blobs = [rc.run_blob([rc.alternating(0)]), rc.run_blob([rc.run([(1, 0)])]), multi["multi_b"]]
    names = ["runs32768", "one_run_of_one", "multi_b"]
    S = rb.DeviceSet.from_serialized(blobs)
    ia = np.arange(len(blobs), dtype=np.uint32)
    ident = S.batch("or", S, ia, ia).serialize_all()
    cards = S.cardinalities().tolist()
    back = S.serialize_all()
    for k, (name, b) in enumerate(zip(names, blobs)):
        assert back[k] == b, f"{name}: serialize_all"
        assert cards[k] == sum(c for _, _, c, _ in rc.blob_containers(b)), f"{name}: cardinality {cards[k]}"
        check_result_bitmap(R, S.download(k), b, f"{name}: download")
        assert ident[k] == R.op_bytes("or", b, b), f"{name}: x | x"
