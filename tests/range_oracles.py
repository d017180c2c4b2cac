"""Checkers of roaring_bitmap_add_range_closed / remove_range_closed and their 64-bit twins for the tests
and tools/time_range.py — TEST INFRASTRUCTURE ONLY: the reference's own functions, bound from the reference
library the other checkers load (R.L), applied to portable blobs."""
import ctypes as C


def ref_range(R, op):
    """R.L's roaring_bitmap_add_range_closed / remove_range_closed(roaring_bitmap_t *, uint32_t, uint32_t),
    typed (roaring.h).  op: "add" or "remove"."""
    f = getattr(R.L, f"roaring_bitmap_{op}_range_closed")
    f.restype = None
    f.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    return f


def ref_range64(R, op):
    """R.L's roaring64_bitmap_add_range_closed / remove_range_closed(roaring64_bitmap_t *, uint64_t,
    uint64_t), typed."""
    f = getattr(R.L, f"roaring64_bitmap_{op}_range_closed")
    f.restype = None
    f.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
    return f


def ref_range_bytes(R, op, blob: bytes, lo, hi) -> bytes:
    """The reference's add_range_closed / remove_range_closed of a portable blob over [lo, hi], validated,
    as portable bytes."""
    r = R.deserialize(blob)
    ref_range(R, op)(r, int(lo), int(hi))
    ok, why = R.validate(r)
    assert ok, why
    out = R.serialize(r)
    R.free(r)
    return out


def ref_range64_bytes(R, op, blob: bytes, lo, hi) -> bytes:
    """The same for a 64-bit portable blob."""
    r = R.r64_deserialize(blob)
    ref_range64(R, op)(r, int(lo), int(hi))
    why = C.c_char_p()
    assert R.L.roaring64_bitmap_internal_validate(r, C.byref(why)), why.value
    out = R.r64_serialize(r)
    R.L.roaring64_bitmap_free(r)
    return out
