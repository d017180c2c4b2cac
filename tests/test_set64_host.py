"""CPU checks of the 64-bit resident sets (rb200_set64_*): malformed input is refused on the host,
before the library touches CUDA, so these pass without a device."""
import struct

import numpy as np
import pytest

import croaring_b200 as rb


def _blob32(vals16, key=0):
    """A 32-bit portable blob (no run containers) holding one array container."""
    n = len(vals16)
    return struct.pack("<IIHHI", 12346, 1, key, n - 1, 16) + struct.pack(f"<{n}H", *vals16)


def _blob32_keys(keys):
    """A 32-bit portable blob (no run containers) of one-value array containers, keys as given."""
    n = len(keys)
    return (struct.pack("<II", 12346, n) + b"".join(struct.pack("<HH", k, 0) for k in keys)
            + b"".join(struct.pack("<I", 8 + 8 * n + 2 * i) for i in range(n)) + struct.pack(f"<{n}H", *range(n)))


def _blob64(buckets, count=None):
    """A 64-bit portable blob: u64 bucket count, then per bucket u32 high32 + 32-bit blob."""
    body = b"".join(struct.pack("<I", h) + b for h, b in buckets)
    return struct.pack("<Q", len(buckets) if count is None else count) + body


def test_malformed_blobs_refused_before_any_cuda_call():
    good = _blob64([(1, _blob32([3, 5])), (7, _blob32([9]))])
    cases = [
        (good[:5], "shorter than its 8-byte bucket count"),
        (_blob64([], count=1 << 32), "above 2\\^32 - 1"),
        (_blob64([(7, _blob32([1])), (7, _blob32([2]))]), "not strictly increasing"),
        (_blob64([(9, _blob32([1])), (3, _blob32([2]))]), "not strictly increasing"),
        (_blob64([(1, _blob32([3, 5]))], count=2), "bucket header runs past the end"),
        (good[:-1], "runs past the end of the blob"),
        (good[:14], "runs past the end of the blob"),
        (_blob64([(1, b"\x00" * 12)]), "not a 32-bit portable bitmap"),
        (_blob64([(1, _blob32_keys([4, 4]))]), "not a 32-bit portable bitmap"),
        (_blob64([(1, _blob32_keys([2, 6, 5]))]), "not a 32-bit portable bitmap"),
    ]
    for blob, why in cases:
        with pytest.raises(rb.RB200Error, match=why):
            rb.DeviceSet64.from_serialized([good, blob])
    with pytest.raises(rb.RB200Error, match="at index 1"):
        rb.DeviceSet64.from_serialized([good, good[:-1]])


def test_malformed_offsets_and_values_refused_before_any_cuda_call():
    vals = np.arange(10, dtype=np.uint64) << np.uint64(33)
    for off in ([0, 5, 3, 10], [1, 5, 10], [2, 1, 10]):
        with pytest.raises(rb.RB200Error, match="set64_from_uint64: offsets"):
            rb.DeviceSet64.from_values(vals, off)
    with pytest.raises(rb.RB200Error, match="offsets"):
        rb.DeviceSet64.from_values(vals, [0, 5, 11])   # past the end of the values
    with pytest.raises(rb.RB200Error, match=r"\[0, 2\^64\)"):
        rb.DeviceSet64.from_values([np.array([1, -1], dtype=np.int64)])
    with pytest.raises(rb.RB200Error, match="integer"):
        rb.DeviceSet64.from_values([np.array([1.5])])
