"""GPU test: a refused call gives back everything it took.  Each call below is refused after it has
taken device or pinned memory (a staged pair list, a slab for the result, a device parse that ran);
it must raise with its usual message and leave the device blocks handed out exactly where they
were."""
import struct

import numpy as np
import pytest

from helpers import synth_blobs, synth_blobs64

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sets(rb, R):
    blobs = synth_blobs(R, 2025, 8)
    S = rb.DeviceSet.from_serialized(blobs)
    lazy = S.batch("or", S, [0, 1], [2, 3], lazy=True)
    S64 = rb.DeviceSet64.from_serialized(synth_blobs64(R, 2025, 4))
    yield blobs, S, lazy, S64
    for s in (S, lazy, S64):
        s.free()


def _bad_run_count(R, blobs):
    """blobs with the one at index 2 replaced by a run bitmap whose first run count overflows the
    blob: the header is well formed, so only the device parse refuses it."""
    r = R.from_values(np.arange(0, 300000, 7, dtype=np.uint32), run_optimize=True)
    runblob = R.serialize(r)
    R.free(r)
    n = (struct.unpack_from("<I", runblob, 0)[0] >> 16) + 1
    hdr = 4 + (n + 7) // 8 + 4 * n + (4 * n if n >= 4 else 0)
    return blobs[:2] + [runblob[:hdr] + b"\xff\xff" + runblob[hdr + 2:]] + blobs[3:]


def _bad_bucket_contents():
    """A 64-bit blob whose one bucket is a 32-bit bitmap with an array of decreasing values: its
    headers walk cleanly, the device parse refuses the contents."""
    inner = struct.pack("<IIHHI", 12346, 1, 0, 1, 16) + struct.pack("<HH", 5, 3)
    return struct.pack("<QI", 1, 7) + inner


def _cases(rb, R, blobs, S, lazy, S64):
    import torch
    vals = torch.arange(10, dtype=torch.int32, device="cuda")
    offs = torch.tensor([0, 6, 3, 10], dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    lib = rb.api.lib()
    two = np.array([0, 1], dtype=np.uint32)   # n = 2^32 with two entries: refused before idx is read
    return [
        ("batch_op", lambda: S.batch("or", S, [0, 1, 2], [1, 99, 3]), "pair index out of range"),
        ("batch_and_cardinality", lambda: S.and_cardinality(S, [0, 99], [1, 2]), "pair index out of range"),
        ("set64_batch_op", lambda: S64.op("xor", S64, [0, 1], [1, 99]), "pair index out of range"),
        ("or_many", lambda: S.or_many(idx=[0, 99]), "or_many: index out of range"),
        ("xor_many", lambda: S.xor_many(idx=[0, 99]), "xor_many: index out of range"),
        ("or_many_heap", lambda: S.or_many_heap(idx=[0, 99]), "or_many_heap: index out of range"),
        ("flip", lambda: S.flip(0, 1 << 20, idx=[0, 99]), "flip: index out of range: idx[1] = 99"),
        ("add_offset", lambda: S.add_offset(5, idx=[0, 99]), "add_offset: index out of range: idx[1] = 99"),
        ("xor_many n = 2^32", lambda: rb.DeviceSet(lib.rb200_xor_many(S.ptr, two.ctypes.data, 1 << 32)),
         "xor_many: more than 2^32 - 1 bitmaps selected"),
        ("or_many_heap n = 2^32", lambda: rb.DeviceSet(lib.rb200_or_many_heap(S.ptr, two.ctypes.data, 1 << 32)),
         "or_many_heap: more than 2^32 - 1 bitmaps selected"),
        ("lazy batch_op", lambda: lazy.batch("and", lazy, [0], [1]), "batch op: the set is in a lazy state"),
        ("lazy serialize", lambda: lazy.serialize_all(), "serialize: the set is in a lazy state"),
        ("lazy flip", lambda: lazy.flip(0, 1 << 20), "flip: the set is in a lazy state"),
        ("device parse", lambda: rb.DeviceSet.from_serialized(_bad_run_count(R, blobs)),
         "malformed portable bitmap at index 2"),
        ("64-bit bucket contents", lambda: rb.DeviceSet64.from_serialized([_bad_bucket_contents()]),
         "invalid container contents"),
        ("set_from_uint32_device", lambda: rb.DeviceSet.from_values(vals, offs),
         "set_from_uint32: offsets decrease at bitmap 1"),
    ]


def test_refused_calls_release_what_they_took(rb, R, sets):
    lib = rb.api.lib()
    cases = _cases(rb, R, *sets)
    for _, call, _ in cases:   # warm pass: scratch the library keeps for later calls is not a leak
        with pytest.raises(rb.RB200Error):
            call()
    for name, call, msg in cases:
        rb.synchronize()
        before = lib.rb200_device_bytes_in_use()
        with pytest.raises(rb.RB200Error) as ei:
            call()
        assert msg in str(ei.value), (name, str(ei.value))
        rb.synchronize()
        assert lib.rb200_device_bytes_in_use() == before, name
