"""DeviceSet.from_values / rb200_set_from_uint32*: roaring_bitmap_of_ptr of a whole batch built on the
device, byte for byte against the unmodified reference's of_ptr (no run_optimize)."""
import numpy as np
import pytest

import croaring_b200 as rb
from helpers import DATASETS, OPS, synth_blobs

gpu = pytest.mark.gpu


def _ref_bytes(R, vals, run_optimize=False):
    r = R.from_values(vals, run_optimize=run_optimize)
    b = R.serialize(r)
    R.free(r)
    return b


def _decode(R, blobs):
    out = []
    for b in blobs:
        r = R.deserialize(b)
        out.append(R.to_array(r))
        R.free(r)
    return out


def _shuffled_with_dups(rng, vals):
    extra = rng.choice(vals, size=len(vals) // 3) if len(vals) else vals
    w = np.concatenate([vals, extra]).astype(np.uint32)
    rng.shuffle(w)
    return w


def _flat(arrays):
    off = np.zeros(len(arrays) + 1, dtype=np.uint64)
    np.cumsum([len(a) for a in arrays], out=off[1:])
    flat = np.concatenate(arrays).astype(np.uint32) if arrays else np.zeros(0, np.uint32)
    return flat, off


def test_malformed_offsets_refused_before_any_cuda_call():
    """Checked on the host before the library touches CUDA: passes without a device."""
    vals = np.arange(10, dtype=np.uint32)
    for off in ([0, 5, 3, 10], [1, 5, 10], [2, 1, 10]):
        with pytest.raises(rb.RB200Error, match="offsets"):
            rb.DeviceSet.from_values(vals, off)
    with pytest.raises(rb.RB200Error, match="offsets"):
        rb.DeviceSet.from_values(vals, [0, 5, 11])   # past the end of the values


@gpu
def test_realdata_sorted_shuffled_and_with_duplicates(rb, R):
    rng = np.random.default_rng(11)
    for ds in DATASETS:
        vals = _decode(R, rb.load_realdata(ds))
        exp = [_ref_bytes(R, v) for v in vals]
        S = rb.DeviceSet.from_values(vals)
        assert S.serialize_all() == exp, ds
        back = S.to_uint32_arrays()
        assert all(np.array_equal(a, b) for a, b in zip(back, vals)), ds
        flat, off = _flat([_shuffled_with_dups(rng, v) for v in vals])
        assert rb.DeviceSet.from_values(flat, off).serialize_all() == exp, f"{ds} shuffled"
    for bm in S.download_all()[:40]:
        ok, why = R.validate(bm.ptr)
        assert ok, why


def _edge_bitmaps():
    k3 = np.uint32(3 << 16)
    a4096 = (np.arange(4096, dtype=np.uint32) * 16) | k3
    a4097 = (np.arange(4097, dtype=np.uint32) * 15) | k3
    return [
        np.zeros(0, np.uint32),                                   # empty at the start
        a4096,                                                    # exactly 4096 distinct: array
        a4097,                                                    # 4097: bitset
        np.repeat(a4096, 7),                                      # 4096 distinct, 28672 values: still an array
        np.zeros(0, np.uint32),                                   # empty in the middle
        np.arange(65536, dtype=np.uint32) | np.uint32(9 << 16),   # a full key
        np.array([0, 0xFFFFFFFF], dtype=np.uint32),
        (np.arange(65536, dtype=np.uint32) << np.uint32(16)) | np.uint32(7),   # one value in each of 65536 keys
        np.array([5, 5, 5], dtype=np.uint32),
        np.concatenate([a4097, (np.arange(100, dtype=np.uint32) * 3) | np.uint32(4 << 16)]),
        np.zeros(0, np.uint32),                                   # empty at the end
    ]


@gpu
def test_edge_containers_and_empty_bitmaps(rb, R):
    rng = np.random.default_rng(5)
    bms = _edge_bitmaps()
    exp = [_ref_bytes(R, v) for v in bms]
    assert rb.DeviceSet.from_values(bms).serialize_all() == exp
    shuffled = [_shuffled_with_dups(rng, v) for v in bms]
    S = rb.DeviceSet.from_values(shuffled)
    assert S.serialize_all() == exp
    assert S.container_count == sum(len(np.unique(v >> np.uint32(16))) for v in bms)
    assert [int(c) for c in S.cardinalities()] == [len(np.unique(v)) for v in bms]
    # payload = container_size_in_bytes summed (an of_ptr result has no run containers)
    assert S.payload_bytes == sum(min(8192, 2 * len(np.unique(v[(v >> np.uint32(16)) == k])))
                                  for v in bms for k in np.unique(v >> np.uint32(16)))


@gpu
def test_empty_batch_and_all_empty(rb, R):
    S = rb.DeviceSet.from_values([])
    assert len(S) == 0 and S.serialize_all() == []
    S = rb.DeviceSet.from_values([np.zeros(0, np.uint32)] * 3)
    assert S.serialize_all() == [_ref_bytes(R, np.zeros(0, np.uint32))] * 3
    assert S.container_count == 0


@gpu
def test_many_tiny_bitmaps(rb, R):
    rng = np.random.default_rng(7)
    n = 100_000
    cnt = rng.integers(0, 4, size=n)
    off = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum(cnt, out=off[1:])
    flat = rng.integers(0, 1 << 32, size=int(off[-1]), dtype=np.uint64).astype(np.uint32)
    dup = rng.random(len(flat) - 1) < 0.3
    flat[1:][dup] = flat[:-1][dup]   # duplicates, within a bitmap or across the boundary
    got = rb.DeviceSet.from_values(flat, off).serialize_all()
    for i in range(n):
        assert got[i] == _ref_bytes(R, flat[off[i]:off[i + 1]]), i


@gpu
def test_one_large_bitmap_across_tiles(rb, R):
    rng = np.random.default_rng(3)
    dense = rng.integers(0, 1 << 24, size=3_000_000, dtype=np.uint64)            # ~256 keys, bitsets
    sparse = rng.integers(1 << 24, 1 << 32, size=2_000_000, dtype=np.uint64)    # arrays of a few values
    mid = rng.integers(1 << 31, (1 << 31) + (300 << 16), size=900_000, dtype=np.uint64)   # ~3000 per key
    v = np.concatenate([dense, sparse, mid]).astype(np.uint32)
    exp = _ref_bytes(R, v)
    srt = np.sort(v)
    assert rb.DeviceSet.from_values([srt]).serialize_all() == [exp]
    assert rb.DeviceSet.from_values([v]).serialize_all() == [exp]
    # the same bitmap between others: its containers start at arbitrary tile positions
    bms = [srt[:1234], srt, v[:77777], srt[5:]]
    assert rb.DeviceSet.from_values(bms).serialize_all() == [_ref_bytes(R, b) for b in bms]


@gpu
def test_chaining_run_optimize_and_batch_ops(rb, R):
    vals = _decode(R, rb.load_realdata("weather_sept_85")[:20] + rb.load_realdata("census1881")[:20]
                   + synth_blobs(R, 4, 30))
    S = rb.DeviceSet.from_values(vals)
    assert S.run_optimize().serialize_all() == [_ref_bytes(R, v, run_optimize=True) for v in vals]
    exp = [_ref_bytes(R, v) for v in vals]
    rng = np.random.default_rng(1)
    ia = rng.integers(0, len(vals), size=200).astype(np.uint32)
    ib = rng.integers(0, len(vals), size=200).astype(np.uint32)
    for op in OPS:
        got = S.batch(op, S, ia, ib).serialize_all()
        for k in range(len(ia)):
            assert got[k] == R.op_bytes(op, exp[ia[k]], exp[ib[k]]), (op, k)


@gpu
def test_device_input_matches_host_input(rb, R):
    import torch
    rng = np.random.default_rng(9)
    vals = _decode(R, rb.load_realdata("wikileaks-noquotes")[:50]) + _edge_bitmaps()
    flat, off = _flat([_shuffled_with_dups(rng, v) for v in vals])
    host = rb.DeviceSet.from_values(flat, off).serialize_all()
    assert host == [_ref_bytes(R, v) for v in vals]
    stream = torch.cuda.Stream()
    rb.set_stream(stream.cuda_stream)
    try:
        with torch.cuda.stream(stream):
            t = torch.from_numpy(flat.view(np.int32)).cuda()
            t_off = torch.from_numpy(off.astype(np.int64)).cuda()
        S = rb.DeviceSet.from_values(t, t_off)
        assert S.serialize_all() == host
        assert np.array_equal(t.cpu().numpy().view(np.uint32), flat)   # unsorted input left as it was
        S2 = rb.DeviceSet.from_values(t, torch.from_numpy(off.astype(np.int64)))   # offsets on the host
        assert S2.serialize_all() == host
    finally:
        rb.set_stream(None)


@gpu
def test_host_addresses_refused_as_device_input(rb):
    """The _device entry points read device memory of the library's device only: a host address as
    the values or as the offsets is refused before anything reads through it, and takes no memory."""
    import torch
    L = rb.api.lib()
    d_vals = torch.arange(10, dtype=torch.int32, device="cuda")
    d_off = torch.tensor([0, 4, 10], dtype=torch.int64, device="cuda")
    h_vals = np.arange(10, dtype=np.uint32)
    h_off = np.array([0, 4, 10], dtype=np.uint64)
    S = rb.DeviceSet.from_values([[1, 2], [3]])
    torch.cuda.synchronize()
    calls = {"set_from_uint32_device": lambda v, o: L.rb200_set_from_uint32_device(v, o, 2),
             "add_many_device": lambda v, o: L.rb200_batch_add_many_device(S.ptr, None, 2, v, o)}
    for entry, call in calls.items():
        for name, v, o in (("vals", h_vals.ctypes.data, d_off.data_ptr()), ("off", d_vals.data_ptr(), h_off.ctypes.data)):
            rb.synchronize()
            before = L.rb200_device_bytes_in_use()
            assert not call(v, o)
            assert rb.last_error() == f"{entry}: {name} is not device memory of the library's device"
            rb.synchronize()
            assert L.rb200_device_bytes_in_use() == before, (entry, name)
    S.free()
