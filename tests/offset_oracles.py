"""Checkers of roaring_bitmap_add_offset for the tests and tools/time_add_offset.py — TEST
INFRASTRUCTURE ONLY: the reference's own function, bound from the reference library the other
checkers load, and the plain-C restatement of tests/c/add_offset_oracle.c, compiled on first use
into a temporary directory."""
import ctypes as C
import os
import subprocess
import tempfile

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "c", "add_offset_oracle.c")


def ref_add_offset(R):
    """R.L's roaring_bitmap_add_offset(const roaring_bitmap_t *, int64_t) (roaring.h:133), typed."""
    f = R.L.roaring_bitmap_add_offset
    if f.restype is not C.c_void_p:
        f.restype = C.c_void_p
        f.argtypes = [C.c_void_p, C.c_int64]
    return f


def ref_add_offset_bytes(R, blob: bytes, offset: int) -> bytes:
    """The reference's roaring_bitmap_add_offset of a portable blob, validated, as portable bytes."""
    r = R.deserialize(blob)
    out = ref_add_offset(R)(r, offset)
    ok, why = R.validate(out)
    assert ok, why
    b = R.serialize(out)
    R.free(out)
    R.free(r)
    return b


class OffsetOracle:
    def __init__(self):
        self._dir = tempfile.TemporaryDirectory(prefix="add_offset_oracle_")
        so = os.path.join(self._dir.name, "liboffset_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-std=c11", "-shared", "-o", so, _SRC])
        self.L = C.CDLL(so, mode=os.RTLD_LOCAL)
        self.L.oracle_add_offset.restype = C.c_size_t
        self.L.oracle_add_offset.argtypes = [C.c_char_p, C.c_size_t, C.c_int64, C.c_char_p, C.c_size_t]

    def add_offset_bytes(self, a: bytes, offset: int) -> bytes:
        need = self.L.oracle_add_offset(a, len(a), offset, None, 0)
        if need == C.c_size_t(-1).value:
            raise ValueError("oracle: malformed input")
        buf = C.create_string_buffer(need)
        assert self.L.oracle_add_offset(a, len(a), offset, buf, need) == need
        return buf.raw


_oracle = None


def offset_oracle():
    global _oracle
    if _oracle is None:
        _oracle = OffsetOracle()
    return _oracle
