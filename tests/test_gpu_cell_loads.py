"""GPU parity of the array cell paths at the edges of their batched operand loads: the vectorised
filter (AND / ANDNOT / and_cardinality with an array side: 8 values per lane, 2 vectors per lane
per trip, survivors through the window buffer; one value per lane up to 32 values), the bitset
staged by cp.async next to the array's loads, the batched array rasterise (A x A AND, A x B OR /
XOR) and the cp.async staging of the A x A merge path.  Array sizes sit at the vector (8), scalar
cutoff (32), warp (256) and trip (512, 1024) boundaries and on both sides of the global-probe threshold;
survivors are all, none or alternating.  Every result is checked byte for byte against the
reference, through the batched kernel, its in-place and lazy twins and the single-pair drop-in path."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIZES = [1, 7, 8, 9, 31, 32, 33, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 4095, 4096]
OPS = ["and", "or", "xor", "andnot"]


def _blob(R, vals, run_optimize=False):
    r = R.from_values(np.asarray(sorted(set(int(v) for v in vals)), dtype=np.uint32), run_optimize=run_optimize)
    b = R.serialize(r)
    R.free(r)
    return b


def _pairs(R):
    """(left, right) blobs of one container each.  The array side takes even values below 32768, so odd
    values and the upper half are free for the other side to hold or avoid."""
    rng = np.random.default_rng(2024)
    evens = np.arange(0, 32768, 2)
    odds = np.arange(1, 65536, 2)
    pairs = []
    for n in SIZES:
        a = np.sort(rng.choice(evens, n, replace=False))
        fill = lambda k: rng.choice(odds, k, replace=False)   # values the array never holds
        A = _blob(R, a)
        # array x bitset: all / none / alternating survivors; all = a plus 4097 - n others, so that
        # the XOR is those others and stays an array
        for keep in (a, a[:0], a[::2]):
            pairs.append((A, _blob(R, np.concatenate([keep, fill(4097 - len(keep))]))))
        # array x array: all, none, alternating (the other side larger, equal and smaller)
        pairs.append((A, _blob(R, np.concatenate([a, fill(min(n, 3000))]))))
        pairs.append((A, _blob(R, fill(max(1, n // 2)))))
        pairs.append((A, _blob(R, np.concatenate([a[::2], fill(n // 4 + 1)]))))
        # array x run: all, none, blocks of 32 values in and out
        pairs.append((A, _blob(R, np.arange(0, 32768), True)))
        pairs.append((A, _blob(R, np.arange(32768, 65536), True)))
        blocks = [np.arange(a[i], a[min(i + 31, n - 1)] + 1) for i in range(0, n, 64)]
        pairs.append((A, _blob(R, np.concatenate(blocks + [np.arange(40000, 41000)]), True)))
    return pairs


@pytest.fixture(scope="module")
def cells(R):
    pairs = _pairs(R)
    # both orders: the array on the left and on the right
    blobs = [b for p in pairs for b in p]
    ia = np.arange(0, len(blobs), 2, dtype=np.uint32)
    ib = ia + 1
    return blobs, np.concatenate([ia, ib]), np.concatenate([ib, ia])


def test_batched_cells(rb, R, cells):
    blobs, ia, ib = cells
    S = rb.DeviceSet.from_serialized(blobs)
    for op in OPS:
        res = S.batch(op, S, ia, ib)
        got = res.serialize_all()
        for k in range(len(ia)):
            assert got[k] == R.op_bytes(op, blobs[ia[k]], blobs[ib[k]]), (op, k, ia[k], ib[k])
        res.free()
    cards = S.and_cardinality(S, ia, ib)
    for k in range(len(ia)):
        r = R.deserialize(R.op_bytes("and", blobs[ia[k]], blobs[ib[k]]))
        assert int(cards[k]) == R.card(r), ("and_cardinality", k)
        R.free(r)
    S.free()


def test_inplace_and_lazy_cells(rb, R, cells):
    blobs, ia, ib = cells
    S = rb.DeviceSet.from_serialized(blobs)
    for op in OPS:
        got = S.batch(op, S, ia, ib, inplace_rules=True).serialize_all()
        for k in range(len(ia)):
            assert got[k] == R.op_inplace_bytes(op, blobs[ia[k]], blobs[ib[k]]), (op, "inplace", k)
    for op, conv in (("or", False), ("or", True), ("xor", False)):
        got = S.batch(op, S, ia, ib, lazy=True, bitsetconversion=conv).repair_after_lazy().serialize_all()
        for k in range(len(ia)):
            exp = R.lazy_fold_bytes(op, conv, [blobs[ia[k]], blobs[ib[k]]])
            assert got[k] == exp, (op, "lazy", conv, k)
    S.free()


def test_single_pair_dropin(rb, R, cells):
    blobs, ia, ib = cells
    for k in range(0, len(ia), 3):
        a, b = blobs[ia[k]], blobs[ib[k]]
        x, y = rb.Bitmap.deserialize(a), rb.Bitmap.deserialize(b)
        for op, sym in (("and", "__and__"), ("or", "__or__"), ("xor", "__xor__"), ("andnot", "__sub__")):
            assert getattr(x, sym)(y).serialize() == R.op_bytes(op, a, b), (op, k)
        assert x.and_cardinality(y) == int(R.card(R.deserialize(R.op_bytes("and", a, b)))), k
        x.inplace("and", y)
        assert x.serialize() == R.op_inplace_bytes("and", a, b), ("and_inplace", k)
