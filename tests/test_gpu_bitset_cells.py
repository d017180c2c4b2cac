"""GPU parity of the cells whose result is a bitset or comes out of one: bitset x array unions /
xors / differences (cardinality taken from the shared-memory atomics of the apply pass) and bitset x
bitset cells (unions written straight to the result slot), at the edges of the type rules.  Every
pair runs in both orders, through the batched path and the single-pair drop-in path, functional,
in place and lazy, against the reference's bytes."""
import numpy as np
import pytest

from helpers import OPS

pytestmark = pytest.mark.gpu

U16 = np.arange(65536, dtype=np.uint32)


def _pick(rng, pool, n):
    return np.sort(rng.choice(pool, n, replace=False)).astype(np.uint32)


def _cases():
    """(name, left values, right values) of one container each; bitsets hold more than 4096 values."""
    rng = np.random.default_rng(2024)
    cs = []
    b5000 = _pick(rng, U16, 5000)
    rest = np.setdiff1d(U16, b5000)
    # bitset ^ array landing on exactly 4096 (array) and 4097 (bitset) values
    cs.append(("xor_to_4096", b5000, _pick(rng, b5000, 904)))
    cs.append(("xor_to_4097", b5000, _pick(rng, b5000, 903)))
    cs.append(("xor_mixed", b5000, np.sort(np.concatenate([_pick(rng, b5000, 700), _pick(rng, rest, 300)]))))
    # bitset - array down to 4096 / 4097 values and well below
    cs.append(("andnot_to_4000", b5000, _pick(rng, b5000, 1000)))
    cs.append(("andnot_to_4096", b5000, _pick(rng, b5000, 904)))
    cs.append(("andnot_to_4097", b5000, _pick(rng, b5000, 903)))
    # xor / andnot that empty the container
    cs.append(("same_bitset", b5000, b5000))
    # unions that saturate: bitset | array, bitset | bitset, and a full left bitset
    missing = _pick(rng, U16, 3000)
    cs.append(("or_saturate_array", np.setdiff1d(U16, missing), missing))
    cs.append(("or_saturate_bitset", U16[0::2], U16[1::2]))
    cs.append(("or_saturate_overlap", np.setdiff1d(U16, missing[:1500]), np.setdiff1d(U16, missing[1500:])))
    cs.append(("full_bitset_array", U16, _pick(rng, U16, 100)))
    cs.append(("full_bitset_bitset", U16, b5000))
    # arrays whose values share 32-bit words (same-word atomics), from 1 value to the 4096 maximum
    for n in (1, 31, 32, 33, 256, 257, 4095, 4096):
        words = rng.choice(2048, (n + 31) // 32, replace=False)
        vals = np.sort((words[:, None] * 32 + np.arange(32)[None, :]).ravel()[:n]).astype(np.uint32)
        cs.append((f"dense_words_{n}", b5000, vals))
    cs.append(("contiguous_4096", b5000, U16[8192:8192 + 4096]))
    # bitset x bitset and / xor on both sides of 4096
    b9000 = _pick(rng, U16, 9000)
    out9 = np.setdiff1d(U16, b9000)
    for k in (4096, 4097):
        shared = _pick(rng, b9000, k)
        other = np.sort(np.concatenate([shared, _pick(rng, out9, 5000)]))
        cs.append((f"and_to_{k}", b9000, other))
        drop = _pick(rng, b9000, k - 2048)
        cs.append((f"xor_bb_to_{k}", b9000, np.sort(np.concatenate([np.setdiff1d(b9000, drop), _pick(rng, out9, 2048)]))))
    return cs


@pytest.fixture(scope="module")
def pairs(R):
    """Serialized (left, right) pairs, both orders of every case, no run containers."""
    mk = lambda v: R.serialize(R.from_values(v, run_optimize=False))
    out = []
    for name, a, b in _cases():
        out.append((name, mk(a), mk(b)))
        out.append((name + "_swapped", mk(b), mk(a)))
    return out


@pytest.fixture(scope="module")
def batch_set(rb, pairs):
    blobs = [x for _, a, b in pairs for x in (a, b)]
    S = rb.DeviceSet.from_serialized(blobs)
    ia = np.arange(0, len(blobs), 2, dtype=np.uint32)
    return S, ia, ia + 1


@pytest.mark.parametrize("inplace", [False, True])
@pytest.mark.parametrize("op", OPS)
def test_bitset_cells_batched(rb, R, pairs, batch_set, op, inplace):
    S, ia, ib = batch_set
    got = S.batch(op, S, ia, ib, inplace_rules=inplace).serialize_all()
    for k, (name, a, b) in enumerate(pairs):
        exp = R.op_inplace_bytes(op, a, b) if inplace else R.op_bytes(op, a, b)
        assert got[k] == exp, (op, inplace, name)


@pytest.mark.parametrize("op", OPS)
def test_bitset_cells_dropin(rb, R, pairs, op):
    sym = {"and": "__and__", "or": "__or__", "xor": "__xor__", "andnot": "__sub__"}[op]
    for name, a, b in pairs:
        x, y = rb.Bitmap.deserialize(a), rb.Bitmap.deserialize(b)
        r = getattr(x, sym)(y)
        assert r.serialize() == R.op_bytes(op, a, b), (op, name)
        ok, why = R.validate(r.ptr)
        assert ok, (op, name, why)
        r.free()
        x.inplace(op, y)
        assert x.serialize() == R.op_inplace_bytes(op, a, b), (op, "inplace", name)
        ok, why = R.validate(x.ptr)
        assert ok, (op, "inplace", name, why)


@pytest.mark.parametrize("op,conv", [("or", False), ("or", True), ("xor", False)])
def test_bitset_cells_lazy(rb, R, pairs, batch_set, op, conv):
    S, ia, ib = batch_set
    got = S.batch(op, S, ia, ib, lazy=True, bitsetconversion=conv).repair_after_lazy().serialize_all()
    for k, (name, a, b) in enumerate(pairs):
        assert got[k] == R.lazy_fold_bytes(op, conv, [a, b]), (op, conv, name)
    # drop-in: lazy, then lazy in place on the lazy result, then repair
    for name, a, b in pairs:
        x, y = rb.Bitmap.deserialize(a), rb.Bitmap.deserialize(b)
        if op == "or":
            r = x.lazy_or(y, conv).lazy_or_inplace(x, conv).repair_after_lazy()
        else:
            r = x.lazy_xor(y).lazy_xor_inplace(x).repair_after_lazy()
        assert r.serialize() == R.lazy_fold_bytes(op, conv, [a, b, a]), (op, conv, name)
