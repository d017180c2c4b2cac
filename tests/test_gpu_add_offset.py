"""GPU parity of rb200_batch_add_offset (roaring_bitmap_add_offset, roaring.c:2426-2507): every result
byte-identical to the reference's and valid for its validator, over the synthetic container mixes,
their no-run twins and the real-data sets; batch shapes, chaining, sharing and refusals."""
import numpy as np
import pytest

import croaring_b200.datasets as dsm
from helpers import DATASETS, check_result_bitmap, no_run_twins, sha_concat, synth_blobs
from offset_oracles import ref_add_offset_bytes
from test_offset_host import OFFSETS, PROFILES, random_offsets

pytestmark = pytest.mark.gpu


def _inputs(R, seed):
    blobs = synth_blobs(R, seed, 30, key_space=6, max_keys=6, profiles=PROFILES if seed != 73 else None)
    return blobs + no_run_twins(R, blobs)


@pytest.mark.parametrize("seed", [71, 72, 73])
def test_add_offset_vs_reference(rb, R, seed):
    blobs = _inputs(R, seed)
    S = rb.DeviceSet.from_serialized(blobs)
    for off in OFFSETS + random_offsets(seed):
        res = S.add_offset(off)
        got = res.serialize_all()
        for k, b in enumerate(blobs):
            assert got[k] == ref_add_offset_bytes(R, b, off), (off, k)
    for off in (5536, -65537, 7 * 65536):
        outs = S.add_offset(off).download_all()
        for k, b in enumerate(blobs):
            check_result_bitmap(R, outs[k], ref_add_offset_bytes(R, b, off), f"offset {off} bitmap {k}")


@pytest.mark.parametrize("ds", DATASETS)
def test_add_offset_realdata_sha(rb, R, ds):
    blobs = dsm.load_realdata(ds)
    S = rb.DeviceSet.from_serialized(blobs)
    for off in (12345, 65535, 7 * 65536, -65537, 1 << 31):
        got = S.add_offset(off).serialize_all()
        assert sha_concat(got) == sha_concat([ref_add_offset_bytes(R, b, off) for b in blobs]), (ds, off)


def test_batch_shapes(rb, R):
    blobs = _inputs(R, 74)
    S = rb.DeviceSet.from_serialized(blobs)
    rng = np.random.default_rng(74)
    # idx with repeats, a different offset per item, key-aligned and split items in one batch
    idx = np.array([5, 5, 0, 17, 5, len(blobs) - 1, 2, 2], dtype=np.uint32)
    offs = [0, 65536 * 3, 12345, -65536, -1, 1 << 32, int(rng.integers(-(1 << 20), 1 << 20)), 65535]
    got = S.add_offset(offs, idx).serialize_all()
    assert got == [ref_add_offset_bytes(R, blobs[i], o) for i, o in zip(idx, offs)]
    # n == 0
    empty = S.add_offset([], np.zeros(0, np.uint32))
    assert len(empty) == 0 and empty.serialize_all() == []
    # empty inputs, and results emptied by the shift (every value pushed out of [0, 2^32))
    E = rb.DeviceSet.from_values([np.zeros(0, np.uint32), np.array([5, 70000], np.uint32)])
    e_blobs = E.serialize_all()
    for off in (0, 77, -(1 << 20), 1 << 40, -(1 << 40), 65536):
        assert E.add_offset(off).serialize_all() == [ref_add_offset_bytes(R, b, off) for b in e_blobs], off
    gone = S.add_offset(-(1 << 32))
    assert gone.serialize_all() == [ref_add_offset_bytes(R, b, -(1 << 32)) for b in blobs]
    assert all(c == 0 for c in gone.cardinalities())


def test_chaining(rb, R):
    blobs = _inputs(R, 75)
    n = len(blobs)
    S = rb.DeviceSet.from_serialized(blobs)
    A = S.add_offset(5536)                      # computed containers
    K = S.add_offset(2 * 65536)                 # shares S's containers
    shifted = [ref_add_offset_bytes(R, b, 5536) for b in blobs]
    aligned = [ref_add_offset_bytes(R, b, 2 * 65536) for b in blobs]
    ia = np.arange(n, dtype=np.uint32)
    ib = (ia + 1) % n
    for op in ("and", "or", "xor", "andnot"):
        got = A.batch(op, K, ia, ib).serialize_all()
        assert got == [R.op_bytes(op, shifted[i], aligned[j]) for i, j in zip(ia, ib)], op
    from oracle.oraclebind import oracle
    assert A.or_many().serialize_all()[0] == oracle().many_bytes("or_many", shifted)
    # add_offset of add_offset results, sharing ones included
    for X, base in ((A, shifted), (K, aligned)):
        for off in (-5536, 65536, 777):
            assert X.add_offset(off).serialize_all() == [ref_add_offset_bytes(R, b, off) for b in base], off
    # frozen round trip of a result
    assert rb.DeviceSet.from_frozen(K.serialize_all(frozen=True)).serialize_all() == aligned
    assert rb.DeviceSet.from_frozen(A.serialize_all(frozen=True)).serialize_all() == shifted


def test_segment_pipeline(rb, R):
    """Per-segment local ids rebased by the segment's base id, then unioned in the global id space."""
    from oracle.oraclebind import oracle
    blobs = [b for b in dsm.load_realdata("census1881")[:40]]
    S = rb.DeviceSet.from_serialized(blobs)
    bases = [int(x) for x in np.cumsum([0] + [1_000_003] * (len(blobs) - 1))]
    G = S.add_offset(bases)
    rebased = [ref_add_offset_bytes(R, b, o) for b, o in zip(blobs, bases)]
    assert G.serialize_all() == rebased
    assert G.or_many().serialize_all()[0] == oracle().many_bytes("or_many", rebased)
    assert G.or_many().serialize_all()[0] == R.many_bytes("or_many", rebased)


def test_sharing_lifetimes_and_bound_host(rb, R):
    blobs = _inputs(R, 76)
    L = rb.lib()
    base = int(L.rb200_device_bytes_in_use())
    S = rb.DeviceSet.from_serialized(blobs)
    K = S.add_offset(-3 * 65536)
    M = S.add_offset([65536 * (i % 3) + (i % 2) * 99 for i in range(len(blobs))])
    expect_k = [ref_add_offset_bytes(R, b, -3 * 65536) for b in blobs]
    S.free()                                     # the results keep the operand's slab alive
    assert K.serialize_all() == expect_k
    for k, bm in enumerate(K.download_all()):
        check_result_bitmap(R, bm, expect_k[k], f"after free {k}")
    assert M.serialize_all() == [ref_add_offset_bytes(R, b, 65536 * (i % 3) + (i % 2) * 99) for i, b in enumerate(blobs)]
    K.free()
    M.free()
    assert int(L.rb200_device_bytes_in_use()) == base
    # an operand uploaded from host bitmaps and bound: pass-through payloads come from the host
    hosts = [rb.Bitmap.deserialize(b) for b in blobs]
    H = rb.DeviceSet.upload(hosts).bind_host()
    for off in (0, 65536, 12345):
        outs = H.add_offset(off).download_all()
        for k, b in enumerate(blobs):
            check_result_bitmap(R, outs[k], ref_add_offset_bytes(R, b, off), f"bound {off} {k}")


def test_refusals(rb, R):
    blobs = _inputs(R, 77)[:6]
    S = rb.DeviceSet.from_serialized(blobs)
    one = lambda v: np.array([v], dtype=np.uint32)
    lz = S.batch("or", S, one(0), one(1), lazy=True)
    with pytest.raises(rb.RB200Error, match="lazy"):
        lz.add_offset(5)
    with pytest.raises(rb.RB200Error, match=r"add_offset: index out of range: idx\[1\] = 6"):
        S.add_offset([1, 2], np.array([0, 6], np.uint32))
    L = rb.lib()
    assert not L.rb200_batch_add_offset(S.ptr, None, 0, None)
    assert "offsets" in rb.last_error()
    # the set is still usable
    assert S.add_offset(3).serialize_all() == [ref_add_offset_bytes(R, b, 3) for b in blobs]


def test_op_stats(rb, R):
    blobs = dsm.load_realdata("weather_sept_85")[:50]
    S = rb.DeviceSet.from_serialized(blobs)
    X = S.add_offset(12345)
    ms, cms, ab = X.op_stats()
    assert ms > 0 and cms > 0
    srcs = sum(len(b) for b in blobs)   # every source is read once, every output written once
    assert ab > srcs // 2
    Kx = S.add_offset(65536)
    assert Kx.op_stats()[2] == 0          # shared containers move nothing
