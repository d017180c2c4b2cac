"""GPU tests of the device-side portable serialization (SURVEY.md §8(f) row 2): bytes produced on
the device equal the reference's roaring_bitmap_portable_serialize of the same results."""
import numpy as np
import pytest

from helpers import OPS, synth_blobs

pytestmark = pytest.mark.gpu


def test_serialize_inputs_roundtrip(rb, R):
    blobs = rb.load_realdata("wikileaks-noquotes")[:50] + rb.load_realdata("weather_sept_85")[:20] \
        + synth_blobs(R, 61, 60)
    empty = R.serialize(R.L.roaring_bitmap_create_with_capacity(0))
    blobs.append(empty)
    S = rb.DeviceSet.from_serialized(blobs)
    assert S.serialize_all() == blobs


@pytest.mark.parametrize("ds", ["census1881", "wikileaks-noquotes"])
def test_serialize_batch_results(rb, R, ds):
    blobs = rb.load_realdata(ds)[:80]
    S = rb.DeviceSet.from_serialized(blobs)
    i, j = np.triu_indices(len(blobs), 1)
    for op in OPS:
        res = S.batch(op, S, i.astype(np.uint32), j.astype(np.uint32))
        got = res.serialize_all()
        for k in range(0, len(got), 97):
            assert got[k] == R.op_bytes(op, blobs[i[k]], blobs[j[k]]), (ds, op, k)
        assert got == [b.serialize() for b in res.download_all()]


def test_device_deserialize_shapes(rb, R):
    """Device-side parse (k_deser_dir / k_deser_copy): odd payload alignment (run cookie with
    1-3 containers: no offset header, 5/6/7-byte preamble), > 32 containers per bitmap (chunked
    walk), empty bitmaps, and the values decode to what the reference holds."""
    vals = []
    rng = np.random.default_rng(3)
    for nkeys in (1, 2, 3, 4, 5, 33, 64, 100):
        v = []
        for k in range(nkeys):
            base = (k * 3 + 1) << 16
            if k % 3 == 0:
                v.append(base + np.arange(100, 100 + 700 * (k % 5 + 1)))          # run
            elif k % 3 == 1:
                v.append(base + np.sort(rng.choice(65536, 300 + 11 * k, replace=False)))   # array
            else:
                v.append(base + np.sort(rng.choice(65536, 20000, replace=False)))  # bitset
        vals.append(np.concatenate(v).astype(np.uint32))
    vals.append(np.zeros(0, np.uint32))
    blobs = []
    for v in vals:
        for ro in (True, False):
            r = R.from_values(v, run_optimize=ro)
            blobs.append(R.serialize(r))
            R.free(r)
    S = rb.DeviceSet.from_serialized(blobs)
    assert S.serialize_all() == blobs
    arrs = S.to_uint32_arrays()
    for k, v in enumerate(vals):
        assert np.array_equal(arrs[2 * k], v) and np.array_equal(arrs[2 * k + 1], v)
    assert S.cardinalities().tolist() == [len(v) for v in vals for _ in (0, 1)]


def test_device_deserialize_rejects_malformed(rb, R):
    good = rb.load_realdata("wikileaks-noquotes")[:6]
    r = R.from_values(np.arange(0, 300000, 7, dtype=np.uint32), run_optimize=True)
    runblob = R.serialize(r)
    R.free(r)
    bad_cases = {
        "truncated payload": good[2][: len(good[2]) - 5],
        "truncated header": good[1][:10],
        "bad cookie": b"\x01\x02\x03\x04" + good[0][4:],
        "run count overflows": None,
        "keys not increasing": None,
    }
    # corrupt the first run container's n_runs field to something huge
    import struct
    n = (struct.unpack_from("<I", runblob, 0)[0] >> 16) + 1
    hdr = 4 + (n + 7) // 8 + 4 * n + (4 * n if n >= 4 else 0)
    bad_cases["run count overflows"] = runblob[:hdr] + b"\xff\xff" + runblob[hdr + 2:]
    # swap two keys of a no-run blob
    g = bytearray(good[3])
    if struct.unpack_from("<I", g, 0)[0] == 12346 and struct.unpack_from("<I", g, 4)[0] >= 2:
        g[8:10], g[12:14] = g[12:14], g[8:10]
        bad_cases["keys not increasing"] = bytes(g)
    else:
        del bad_cases["keys not increasing"]
    for name, blob in bad_cases.items():
        with pytest.raises(rb.RB200Error) as ei:
            rb.DeviceSet.from_serialized(good[:2] + [blob] + good[4:])
        assert "malformed portable bitmap at index 2" in str(ei.value), (name, str(ei.value))
    # container CONTENTS are checked too (ADVICE r1: a run ending past 65535 would be rasterised
    # outside the warp's accumulator): run overflow, overlapping runs, unsorted array values
    content_cases = {}
    vals = np.concatenate([np.arange(0, 100), np.arange(200, 300), np.arange(70000, 80000)]).astype(np.uint32)
    r = R.from_values(vals, run_optimize=True)
    rblob = R.serialize(r)                                         # 2 run containers: {2 runs}, {1 run}
    R.free(r)
    assert struct.unpack_from("<I", rblob, 0)[0] == (12347 | (1 << 16))
    rhdr = 4 + 1 + 4 * 2                                           # cookie, run flags, key-card pairs (no offsets: n < 4)
    assert struct.unpack_from("<HHHHH", rblob, rhdr) == (2, 0, 99, 200, 99)
    rb_ = bytearray(rblob)
    struct.pack_into("<HH", rb_, rhdr + 6, 65000, 1000)            # second run: 65000 + 1000 > 65535
    content_cases["run ends past 65535"] = bytes(rb_)
    rb_ = bytearray(rblob)
    struct.pack_into("<HH", rb_, rhdr + 6, 99, 50)                 # second run starts inside the first
    content_cases["runs overlap"] = bytes(rb_)
    r = R.from_values(np.array([5, 9, 13, 70000, 70001], dtype=np.uint32), run_optimize=False)
    ab = bytearray(R.serialize(r))
    R.free(r)
    ab[8 + 8 * 2 + 8 * 0:8 + 16 + 2] = struct.pack("<H", 9)      # values 9, 9, 13: not strictly increasing
    content_cases["array values not increasing"] = bytes(ab)
    for name, blob in content_cases.items():
        with pytest.raises(rb.RB200Error) as ei:
            rb.DeviceSet.from_serialized(good[:2] + [blob] + good[4:])
        assert "malformed portable bitmap at index 2: invalid container contents" in str(ei.value), (name, str(ei.value))
    # the library keeps working afterwards
    assert rb.DeviceSet.from_serialized(good).serialize_all() == good


def test_frozen_format_both_ways(rb, R):
    """Device-side frozen format (roaring.c:3180-3456): emitted bytes equal
    roaring_bitmap_frozen_serialize; the reference's frozen_view accepts our 32-byte aligned blobs
    IN PLACE; frozen blobs parse on the device back to the same bitmaps; malformed ones are refused."""
    blobs = rb.load_realdata("weather_sept_85")[:25] + rb.load_realdata("census1881")[:25] + synth_blobs(R, 91, 50)
    r0 = R.from_values(np.zeros(0, np.uint32), False)
    blobs.append(R.serialize(r0))
    R.free(r0)
    exp = [R.frozen_bytes(b) for b in blobs]
    S = rb.DeviceSet.from_serialized(blobs)
    assert S.serialize_all(frozen=True) == exp
    # in place: hand the pinned buffer to the reference's zero-copy view
    buf, off, ln, release = S.serialize_all(copy=False, frozen=True)
    for i in range(0, len(blobs), 7):
        assert (buf.value + off[i]) % 32 == 0
        view = R.L.roaring_bitmap_frozen_view(buf.value + off[i], ln[i])
        assert view, i
        assert R.serialize(view) == blobs[i]
        R.free(view)
    release()
    # results of an op, frozen
    i, j = np.triu_indices(40, 1)
    res = S.batch("xor", S, i.astype(np.uint32), j.astype(np.uint32))
    fz = res.serialize_all(frozen=True)
    for k in range(0, len(fz), 53):
        assert fz[k] == R.frozen_bytes(R.op_bytes("xor", blobs[i[k]], blobs[j[k]])), k
    # parse
    F = rb.DeviceSet.from_frozen(exp)
    assert F.serialize_all() == blobs
    assert F.cardinalities().tolist() == S.cardinalities().tolist()
    for name, bad in {"truncated": exp[3][:-9], "cookie": exp[3][:-4] + b"\x00\x00\x00\x00",
                      "cookie bit": exp[3][:-4] + bytes([exp[3][-4] ^ 0x01]) + exp[3][-3:],
                      "length": exp[3][:100] + b"\x00\x00" + exp[3][100:]}.items():
        with pytest.raises(rb.RB200Error) as ei:
            rb.DeviceSet.from_frozen(exp[:2] + [bad] + exp[4:6])
        assert "malformed frozen bitmap at index 2" in str(ei.value), (name, str(ei.value))
