"""GPU parity of rb200_set64_batch_add_range_closed / remove_range_closed (roaring64_bitmap_add_range_closed /
remove_range_closed, roaring64.c:651, 996): every result byte-identical to the reference's range update of the
same 64-bit bitmap, inside one bucket, across bucket boundaries, over absent buckets and the whole 64-bit
space, up to 2^64 - 1; chaining; and the size refusal."""
import numpy as np
import pytest

from helpers import synth_blobs64
from range_oracles import ref_range64_bytes
from update_oracles import ref_update64_bytes

pytestmark = pytest.mark.gpu

HIGHS = (0, 1, 7, 0x10000, 0xFFFFFFFF)
T32, T64 = 1 << 32, (1 << 64) - 1
# closed 64-bit ranges: one bucket, across 2^32 - 1 / 2^32, over absent buckets (at most a few full ones),
# the top of the space, the whole space, single values, empty
RANGES = [
    (5, 70000), ((7 << 32) + 100, (7 << 32) + 65535), (T32 - 3, T32 + 70000), (T32 - 1, T32),
    ((2 << 32) + 5, (4 << 32) + 9), ((3 << 32) - 1, (6 << 32) + 65536 * 3), (0x10000 << 32, (0x10000 << 32) + (T32 - 1)),
    (T64 - 100000, T64), (T64, T64), (0, T64), (1 << 40, 1 << 40), (9, 3),
]


def _expect(R, op, blobs, lo, hi):
    return [ref_range64_bytes(R, op, b, a, z) for b, a, z in zip(blobs, lo, hi)]


def _closed(S, op, lo, hi, idx=None):
    """The update through the mirror's half-open form, end up to 2^64."""
    end = [z + 1 if a <= z else a for a, z in zip(lo, hi)]
    f = S.add_range if op == "add" else S.remove_range
    return f(list(lo), end, idx=idx)


@pytest.mark.parametrize("op", ["add", "remove"])
@pytest.mark.parametrize("seed", [61, 62])
def test_range64_vs_reference(rb, R, seed, op):
    blobs = synth_blobs64(R, seed, 24, highs=HIGHS, key_space=5, max_keys=5)
    S = rb.DeviceSet64.from_serialized(blobs)
    for a, z in RANGES:
        if op == "add" and a <= z and (z >> 32) - (a >> 32) > 4:
            continue   # an add over the whole space is refused (see test_size_refusal)
        lo, hi = [a] * len(blobs), [z] * len(blobs)
        assert _closed(S, op, lo, hi).serialize_all() == _expect(R, op, blobs, lo, hi), (op, hex(a), hex(z))
    # one range per item, mixed
    rng = np.random.default_rng(seed)
    pick = [RANGES[int(rng.integers(0, len(RANGES)))] for _ in blobs]
    pick = [(a, z) if op == "remove" or a > z or (z >> 32) - (a >> 32) <= 4 else (a, a + 1000) for a, z in pick]
    lo, hi = [a for a, _ in pick], [z for _, z in pick]
    assert _closed(S, op, lo, hi).serialize_all() == _expect(R, op, blobs, lo, hi)


def test_range64_closed_abi_and_chaining(rb, R):
    blobs = synth_blobs64(R, 63, 12, highs=HIGHS)
    S = rb.DeviceSet64.from_serialized(blobs)
    L = rb.lib()
    lo = np.array([0, T32 - 1, 5, T64, (7 << 32), 3] * 2, np.uint64)
    hi = np.array([T64, T32 + 1, 4, T64, (9 << 32) + 17, 3] * 2, np.uint64)
    p = L.rb200_set64_batch_remove_range_closed(S.ptr, None, 0, lo.ctypes.data, hi.ctypes.data)
    removed = _expect(R, "remove", blobs, lo.tolist(), hi.tolist())
    D = rb.DeviceSet64(p)
    assert D.serialize_all() == removed   # (the whole-space removals leave empty bitmaps)
    lo_a = np.array([5, T32 - 2, (1 << 40), T64 - 3, 0, 77] * 2, np.uint64)
    hi_a = np.array([100, T32 + 2, (1 << 40) + 65536 * 2, T64, 65535, 7 << 32] * 2, np.uint64)
    A = rb.DeviceSet64(L.rb200_set64_batch_add_range_closed(D.ptr, None, 0, lo_a.ctypes.data, hi_a.ctypes.data))
    added = _expect(R, "add", removed, lo_a.tolist(), hi_a.tolist())
    assert A.serialize_all() == added
    n = len(blobs)
    ia = np.arange(n, dtype=np.uint32)
    ib = (ia + 1) % n
    for op in ("and", "or", "xor", "andnot"):
        assert A.op(op, S, ia, ib).serialize_all() == [R.r64_op_bytes(op, added[i], blobs[j]) for i, j in zip(ia, ib)], op
    vals = [np.array([1, T32, T64 - 1], np.uint64)] * n
    assert A.add_many(vals).serialize_all() == [ref_update64_bytes(R, "add", b, v) for b, v in zip(added, vals)]
    # idx with repeats
    idx = np.array([3, 3, 0, n - 1], np.uint32)
    got = S.add_range(T32 - 5, T32 + 5, idx=idx).serialize_all()
    assert got == [ref_range64_bytes(R, "add", blobs[i], T32 - 5, T32 + 4) for i in idx]


def test_size_refusal(rb, R):
    """An add over many full buckets is refused before any device work and leaves nothing in use."""
    blobs = synth_blobs64(R, 64, 4, highs=HIGHS)
    S = rb.DeviceSet64.from_serialized(blobs)
    L = rb.lib()
    S.cardinalities()
    base = int(L.rb200_device_bytes_in_use())
    k0 = rb.kernel_launches()
    with pytest.raises(rb.RB200Error, match="set64_add_range_closed: batch too large"):
        S.add_range(0, 1 << 64)
    with pytest.raises(rb.RB200Error, match="set64_add_range_closed: batch too large"):
        S.add_range(0, (1 << 32) * 70000, idx=[0])   # 70000 full buckets
    assert rb.kernel_launches() == k0
    assert int(L.rb200_device_bytes_in_use()) == base
    assert S.remove_range(0, 1 << 64).cardinalities().tolist() == [0] * len(blobs)
