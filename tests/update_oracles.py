"""Checkers of roaring_bitmap_add_many / remove_many and their 64-bit twins for the tests and
tools/time_update.py — TEST INFRASTRUCTURE ONLY: the reference's own functions, bound from the reference
library the other checkers load (R.L), applied to portable blobs."""
import ctypes as C

import numpy as np


def _typed(R, name):
    f = getattr(R.L, name)
    f.restype = None
    f.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    return f


def ref_update(R, op):
    """R.L's roaring_bitmap_add_many / remove_many(roaring_bitmap_t *, size_t, const uint32_t *), typed
    (roaring.h:106, :420).  op: "add" or "remove"."""
    return _typed(R, f"roaring_bitmap_{op}_many")


def ref_update64(R, op):
    """R.L's roaring64_bitmap_add_many / remove_many(roaring64_bitmap_t *, size_t, const uint64_t *), typed."""
    return _typed(R, f"roaring64_bitmap_{op}_many")


def ref_update_bytes(R, op, blob: bytes, vals) -> bytes:
    """The reference's add_many / remove_many of a portable blob with vals (as given), validated, as
    portable bytes."""
    v = np.ascontiguousarray(vals, dtype=np.uint32)
    r = R.deserialize(blob)
    ref_update(R, op)(r, v.size, v.ctypes.data)
    ok, why = R.validate(r)
    assert ok, why
    out = R.serialize(r)
    R.free(r)
    return out


def ref_update64_bytes(R, op, blob: bytes, vals) -> bytes:
    """The same for a 64-bit portable blob."""
    v = np.ascontiguousarray(vals, dtype=np.uint64)
    r = R.r64_deserialize(blob)
    ref_update64(R, op)(r, v.size, v.ctypes.data)
    why = C.c_char_p()
    assert R.L.roaring64_bitmap_internal_validate(r, C.byref(why)), why.value
    out = R.r64_serialize(r)
    R.L.roaring64_bitmap_free(r)
    return out
