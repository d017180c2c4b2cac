"""GPU parity of rb200_set64_batch_add_many / remove_many (roaring64_bitmap_add_many / remove_many,
roaring64.c:606, 950): every result byte-identical to the reference's update of the same 64-bit bitmap
with the same values, across high-32 bucket boundaries, into new buckets and emptying buckets."""
import numpy as np
import pytest

from helpers import synth_blobs64
from update_oracles import ref_update64_bytes

pytestmark = pytest.mark.gpu

HIGHS = (0, 1, 7, 0x10000, 0xFFFFFFFF)


def _present(R, blob):
    r = R.r64_deserialize(blob)
    n = int(R.L.roaring64_bitmap_get_cardinality(r))
    R.L.roaring64_bitmap_free(r)
    return n


def _lists(R, blobs, op, seed):
    rng = np.random.default_rng(seed)
    out = []
    for k, b in enumerate(blobs):
        parts = [np.array([0, (1 << 32) - 1, 1 << 32, (1 << 64) - 1, (7 << 32) + 65535, (7 << 32) + 65536],
                          dtype=np.uint64)]
        for h in HIGHS + (3, 0xABCDEF):   # existing and new buckets
            if rng.random() < 0.5:
                m = int(rng.choice([1, 50, 3000, 5000]))
                parts.append((np.uint64(h) << np.uint64(32)) + rng.integers(0, 6 << 16, m).astype(np.uint64))
        v = np.concatenate(parts)
        out.append(rng.permutation(np.concatenate([v, v[: v.size // 4]])))
    return out


def _expect(R, op, blobs, lists):
    return [ref_update64_bytes(R, op, b, v) for b, v in zip(blobs, lists)]


def _all_values(R, blob):
    """Every value of a 64-bit blob, through the reference's 32-bit buckets."""
    n = int(np.frombuffer(blob[:8], np.uint64)[0])
    pos, out = 8, []
    for _ in range(n):
        high = int(np.frombuffer(blob[pos:pos + 4], np.uint32)[0])
        pos += 4
        r = R.L.roaring_bitmap_portable_deserialize_safe(blob[pos:], len(blob) - pos)
        pos += int(R.L.roaring_bitmap_portable_size_in_bytes(r))
        out.append((np.uint64(high) << np.uint64(32)) + R.to_array(r).astype(np.uint64))
        R.free(r)
    return np.concatenate(out) if out else np.zeros(0, np.uint64)


@pytest.mark.parametrize("seed", [81, 82])
def test_update64_vs_reference(rb, R, seed):
    blobs = synth_blobs64(R, seed, 24, highs=HIGHS, key_space=5, max_keys=5)
    S = rb.DeviceSet64.from_serialized(blobs)
    for op in ("add", "remove"):
        lists = _lists(R, blobs, op, seed + (op == "add"))
        res = S.add_many(lists) if op == "add" else S.remove_many(lists)
        assert res.serialize_all() == _expect(R, op, blobs, lists), op
    # emptied buckets and bitmaps are left out of the serialized and counted results
    everything = [_all_values(R, b) for b in blobs]
    E = S.remove_many(everything)
    assert E.serialize_all() == _expect(R, "remove", blobs, everything)
    assert all(c == 0 for c in E.cardinalities())
    half = [v[(v >> np.uint64(32)) == v[0] >> np.uint64(32)] if v.size else v for v in everything]
    H = S.remove_many(half)
    exp = _expect(R, "remove", blobs, half)
    assert H.serialize_all() == exp
    assert H.cardinalities().tolist() == [_present(R, b) for b in exp]
    # chained: the emptied result updated again, and an op on it
    back = _lists(R, blobs, "add", seed + 7)
    assert H.add_many(back).serialize_all() == _expect(R, "add", exp, back)
    ia = np.arange(len(blobs), dtype=np.uint32)
    assert H.op("or", S, ia, ia).serialize_all() == [R.r64_op_bytes("or", a, b) for a, b in zip(exp, blobs)]


def test_update64_shapes_and_device_values(rb, R):
    import torch
    blobs = synth_blobs64(R, 83, 12, highs=HIGHS)
    S = rb.DeviceSet64.from_serialized(blobs)
    idx = np.array([3, 3, 0, 11, 3], dtype=np.uint32)
    lists = _lists(R, [blobs[i] for i in idx], "add", 83)
    for op in ("add", "remove"):
        up = S.add_many if op == "add" else S.remove_many
        host = up(lists, idx=idx).serialize_all()
        assert host == [ref_update64_bytes(R, op, blobs[i], v) for i, v in zip(idx, lists)], op
        flat = np.concatenate(lists)
        offs = np.concatenate([[0], np.cumsum([v.size for v in lists])]).astype(np.int64)
        tv = torch.from_numpy(flat.view(np.int64)).cuda()
        torch.cuda.synchronize()
        assert up(tv, torch.from_numpy(offs).cuda(), idx=idx).serialize_all() == host, op
        assert len(up([], idx=np.zeros(0, np.uint32))) == 0
    with pytest.raises(rb.RB200Error, match=r"set64_add_many: index out of range: idx\[0\] = 12"):
        S.add_many([[1]], idx=[12])
    with pytest.raises(rb.RB200Error, match="set64_remove_many: offsets decrease"):
        S.remove_many(np.arange(3, dtype=np.uint64), [0, 2, 1, 3], idx=[0, 1, 2])
