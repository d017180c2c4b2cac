"""Python mirror of the C ABI in include/roaring_b200.h (ctypes; no torch types cross the boundary).

The names follow the reference's C API (roaring_bitmap_and / or / xor / andnot / or_many /
and_cardinality ..., /root/reference/include/roaring/roaring.h:225-348) so parity tests read
like the reference's own tests.  Everything here runs on the GPU through
libroaring_b200.so; there is no CPU fallback — if the library or a CUDA device is missing,
calls raise.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# RB200_LIB: load an experimental build instead (tuning runs, tools/time_ops.py); the product is
# always the in-tree libroaring_b200.so
LIB_PATH = os.environ.get("RB200_LIB") or os.path.join(_HERE, "libroaring_b200.so")

AND, OR, XOR, ANDNOT = 0, 1, 2, 3
OPS = {"and": AND, "or": OR, "xor": XOR, "andnot": ANDNOT}

_P = C.c_void_p
_lib = None


class RB200Error(RuntimeError):
    pass


def lib():
    """Load libroaring_b200.so (build it first with `python -m croaring_b200.build`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RB200Error(
            f"{LIB_PATH} is missing: the CUDA extension is not built "
            "(run `python -m croaring_b200.build`); there is no CPU fallback")
    L = C.CDLL(LIB_PATH, mode=os.RTLD_LOCAL)

    def sig(name, res, *args):
        f = getattr(L, name)
        f.restype = res
        f.argtypes = list(args)

    for op in ("and", "or", "xor", "andnot"):
        sig(f"roaring_bitmap_{op}_inplace", None, _P, _P)
        sig(f"roaring_bitmap_{op}", _P, _P, _P)
        sig(f"roaring_bitmap_{op}_cardinality", C.c_uint64, _P, _P)
    sig("roaring_bitmap_or_many", _P, C.c_size_t, C.POINTER(_P))
    sig("roaring_bitmap_xor_many", _P, C.c_size_t, C.POINTER(_P))
    sig("rb200_xor_many", _P, _P, _P, C.c_size_t)
    sig("roaring_bitmap_or_many_heap", _P, C.c_uint32, C.POINTER(_P))
    sig("rb200_or_many_heap", _P, _P, _P, C.c_size_t)
    sig("rb200_set_repair_after_lazy", _P, _P)
    sig("roaring_bitmap_lazy_or", _P, _P, _P, C.c_bool)
    sig("roaring_bitmap_lazy_or_inplace", None, _P, _P, C.c_bool)
    sig("roaring_bitmap_lazy_xor", _P, _P, _P)
    sig("roaring_bitmap_lazy_xor_inplace", None, _P, _P)
    sig("roaring_bitmap_repair_after_lazy", None, _P)
    sig("roaring_bitmap_jaccard_index", C.c_double, _P, _P)
    sig("roaring_bitmap_intersect", C.c_bool, _P, _P)
    sig("rb200_bitmap_portable_deserialize_safe", _P, C.c_char_p, C.c_size_t)
    sig("rb200_bitmap_portable_size_in_bytes", C.c_size_t, _P)
    sig("rb200_bitmap_portable_serialize", C.c_size_t, _P, C.c_char_p)
    sig("rb200_bitmap_free", None, _P)
    sig("rb200_bitmap_get_cardinality", C.c_uint64, _P)
    sig("rb200_bitmap_validate", C.c_bool, _P, C.POINTER(C.c_char_p))
    sig("rb200_init", C.c_int, C.c_int)
    sig("rb200_set_stream", None, _P)
    sig("rb200_synchronize", None)
    sig("rb200_last_error", C.c_char_p)
    sig("rb200_kernel_launches", C.c_uint64)
    sig("rb200_device_bytes_in_use", C.c_uint64)
    sig("rb200_last_algorithmic_bytes", C.c_uint64)
    sig("rb200_last_device_ms", C.c_float)
    sig("rb200_last_compute_ms", C.c_float)
    sig("rb200_last_download_bytes", C.c_uint64)
    sig("rb200_set_upload", _P, C.POINTER(_P), C.c_size_t)
    sig("rb200_set_upload_serialized", _P, _P, _P, C.c_size_t)
    sig("rb200_set_free", None, _P)
    sig("rb200_set_bind_host", C.c_int, _P, C.c_int)
    sig("rb200_set_count", C.c_size_t, _P)
    sig("rb200_set_container_count", C.c_uint64, _P)
    sig("rb200_set_payload_bytes", C.c_uint64, _P)
    sig("rb200_batch_op", _P, C.c_int, _P, _P, _P, _P, C.c_size_t)
    sig("rb200_batch_op_ex", _P, C.c_int, C.c_int, _P, _P, _P, _P, C.c_size_t)
    sig("rb200_batch_and_cardinality", C.c_int, _P, _P, _P, _P, C.c_size_t, _P)
    sig("rb200_or_many", _P, _P, _P, C.c_size_t)
    sig("rb200_batch_relations", C.c_int, _P, _P, _P, _P, C.c_size_t, _P)
    sig("rb200_set_op_stats", C.c_int, _P, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_uint64))
    sig("rb200_batch_flip", _P, _P, _P, C.c_size_t, C.c_uint64, C.c_uint64)
    sig("rb200_batch_add_offset", _P, _P, _P, C.c_size_t, _P)
    for name in ("rb200_batch_add_many", "rb200_batch_remove_many", "rb200_set64_batch_add_many",
                 "rb200_set64_batch_remove_many"):
        sig(name, _P, _P, _P, C.c_size_t, _P, _P)
        sig(name + "_device", _P, _P, _P, C.c_size_t, _P, _P)
    sig("rb200_batch_query", C.c_int, C.c_int, _P, _P, C.c_size_t, _P, _P)
    sig("rb200_batch_query_device", C.c_int, C.c_int, _P, _P, C.c_size_t, _P, _P)
    sig("rb200_r64_batch_op_serialized", C.c_int, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t),
        C.c_size_t, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_size_t, _P, _P, C.c_size_t,
        C.POINTER(C.c_void_p), C.POINTER(C.POINTER(C.c_uint64)), C.POINTER(C.POINTER(C.c_uint64)))
    sig("rb200_r64_batch_and_cardinality_serialized", C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t),
        C.c_size_t, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_size_t, _P, _P, C.c_size_t, _P)
    sig("roaring_bitmap_flip", _P, _P, C.c_uint64, C.c_uint64)
    sig("roaring_bitmap_flip_inplace", None, _P, C.c_uint64, C.c_uint64)
    for rel in ("equals", "is_subset", "is_strict_subset"):
        sig(f"roaring_bitmap_{rel}", C.c_bool, _P, _P)
    sig("rb200_or_many_keyrange", _P, _P, _P, C.c_size_t, C.c_uint32, C.c_uint32, _P)
    sig("rb200_set_cardinalities", C.c_int, _P, _P)
    sig("rb200_set_download", _P, _P, C.c_size_t)
    sig("rb200_set_download_all", C.c_int, _P, C.POINTER(_P))
    sig("rb200_bitmaps_free", None, C.POINTER(_P), C.c_size_t)
    sig("rb200_set_run_optimize", _P, _P, C.c_int)
    sig("rb200_set_to_uint32", C.c_int, _P, C.POINTER(C.POINTER(C.c_uint32)), C.POINTER(C.POINTER(C.c_uint64)))
    sig("rb200_values_free", None, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64))
    sig("rb200_set_from_uint32", _P, _P, _P, C.c_size_t)
    sig("rb200_set_from_uint32_device", _P, _P, _P, C.c_size_t)
    sig("rb200_set_serialize", C.c_int, _P, C.POINTER(C.c_void_p), C.POINTER(C.POINTER(C.c_uint64)),
        C.POINTER(C.POINTER(C.c_uint64)))
    sig("rb200_serialized_free", None, C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64))
    sig("rb200_set_serialize_frozen", C.c_int, _P, C.POINTER(C.c_void_p), C.POINTER(C.POINTER(C.c_uint64)),
        C.POINTER(C.POINTER(C.c_uint64)))
    sig("rb200_set_upload_frozen", _P, _P, _P, C.c_size_t)
    sig("rb200_download_begin", _P, _P, C.c_size_t)
    sig("rb200_download_chunk_capacity", C.c_size_t, _P)
    sig("rb200_download_next", C.c_size_t, _P, C.POINTER(_P))
    sig("rb200_download_end", None, _P)
    sig("rb200_download_foreach", C.c_int, _P, _P, _P)
    sig("rb200_download_foreach_many", C.c_int, C.POINTER(_P), C.c_size_t, _P, _P)
    sig("rb200_download_foreach_async", C.c_int, _P, _P, _P)
    sig("rb200_download_wait", C.c_int)
    sig("rb200_batch_op_host", C.c_int, C.c_int, C.POINTER(_P), C.POINTER(_P), C.c_size_t,
        C.POINTER(_P))
    sig("rb200_r64_batch_op", C.c_int, C.c_int, _P, _P, C.c_size_t, _P)
    sig("rb200_r64_batch_and_cardinality", C.c_int, _P, _P, C.c_size_t, _P)
    for op in ("and", "or", "xor", "andnot"):
        sig(f"roaring64_bitmap_{op}", _P, _P, _P)
        sig(f"roaring64_bitmap_{op}_cardinality", C.c_uint64, _P, _P)
    sig("roaring64_bitmap_jaccard_index", C.c_double, _P, _P)
    sig("roaring64_bitmap_intersect", C.c_bool, _P, _P)
    sig("rb200_comm_unique_id", C.c_int, C.c_char_p)
    sig("rb200_comm_init_rank", _P, C.c_char_p, C.c_int, C.c_int)
    sig("rb200_comm_adopt", _P, _P, C.c_int, C.c_int)
    sig("rb200_comm_size", C.c_int, _P)
    sig("rb200_comm_rank", C.c_int, _P)
    sig("rb200_comm_destroy", None, _P)
    sig("rb200_comm_allreduce_u64", C.c_int, _P, _P, C.c_size_t)
    sig("rb200_set_add_cardinality_device", C.c_int, _P, _P)
    sig("rb200_plan_key_ranges", C.c_int, _P, _P, C.c_size_t, C.c_int, _P, _P, _P)
    sig("rb200_blob_slice_keys", C.c_int, C.c_char_p, C.c_size_t, C.c_uint32, C.c_uint32,
        C.POINTER(C.c_void_p), C.POINTER(C.c_size_t))
    sig("rb200_blobs_concat", C.c_int, _P, _P, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t))
    sig("rb200_blob_free", None, C.c_void_p)
    sig("rb200_set_upload_serialized_keyrange", _P, _P, _P, C.c_size_t, C.c_uint32, C.c_uint32)
    sig("rb200_or_many_sharded", _P, _P, _P, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, _P,
        _P, C.POINTER(C.c_uint64))
    sig("rb200_last_collective_ms", C.c_float)
    sig("rb200_set64_upload_serialized", _P, _P, _P, C.c_size_t)
    sig("rb200_set64_upload", _P, _P, C.c_size_t)
    sig("rb200_set64_from_uint64", _P, _P, _P, C.c_size_t)
    sig("rb200_set64_from_uint64_device", _P, _P, _P, C.c_size_t)
    sig("rb200_set64_free", None, _P)
    sig("rb200_set64_count", C.c_size_t, _P)
    sig("rb200_set64_cardinalities", C.c_int, _P, _P)
    sig("rb200_set64_batch_op", _P, C.c_int, _P, _P, _P, _P, C.c_size_t)
    sig("rb200_set64_batch_and_cardinality", C.c_int, _P, _P, _P, _P, C.c_size_t, _P)
    sig("rb200_set64_run_optimize", _P, _P, C.c_int)
    sig("rb200_set64_serialize", C.c_int, _P, C.POINTER(C.c_void_p), C.POINTER(C.POINTER(C.c_uint64)),
        C.POINTER(C.POINTER(C.c_uint64)))
    sig("rb200_set64_download_all", C.c_int, _P, _P)
    _lib = L
    return L


def last_error():
    return lib().rb200_last_error().decode()


def init(device=0):
    if lib().rb200_init(int(device)) != 0:
        raise RB200Error(last_error())


def set_stream(cuda_stream_ptr):
    """Run all library work on this cudaStream_t (e.g. torch.cuda.current_stream().cuda_stream)."""
    lib().rb200_set_stream(_P(cuda_stream_ptr) if cuda_stream_ptr else None)


def synchronize():
    lib().rb200_synchronize()


def kernel_launches():
    return int(lib().rb200_kernel_launches())


def last_algorithmic_bytes():
    return int(lib().rb200_last_algorithmic_bytes())


def last_device_ms():
    return float(lib().rb200_last_device_ms())


def _u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)


def _selection(idx, n_all):
    """(array, pointer, count) of a selection of bitmaps; idx None selects all n_all of them.  The
    array is what the pointer points into: keep it alive until the call returns."""
    if idx is None:
        return None, None, n_all
    idx = _u32(idx)
    return idx, idx.ctypes.data, idx.size


class Bitmap:
    """A host roaring_bitmap_t* (reference memory layout) owned by this object."""

    def __init__(self, ptr, own=True):
        if not ptr:
            raise RB200Error(last_error() or "null bitmap")
        self.ptr = ptr
        self.own = own

    # -- construction / destruction
    @classmethod
    def deserialize(cls, blob: bytes):
        p = lib().rb200_bitmap_portable_deserialize_safe(blob, len(blob))
        if not p:
            raise RB200Error("malformed portable bitmap")
        return cls(p)

    def free(self):
        if self.ptr and self.own:
            lib().rb200_bitmap_free(self.ptr)
        self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    # -- inspection
    def serialize(self) -> bytes:
        n = lib().rb200_bitmap_portable_size_in_bytes(self.ptr)
        buf = C.create_string_buffer(n)
        m = lib().rb200_bitmap_portable_serialize(self.ptr, buf)
        assert m == n, (m, n)
        return buf.raw

    def cardinality(self) -> int:
        return int(lib().rb200_bitmap_get_cardinality(self.ptr))

    def validate(self):
        why = C.c_char_p()
        ok = lib().rb200_bitmap_validate(self.ptr, C.byref(why))
        return bool(ok), (why.value.decode() if why.value else "")

    # -- the drop-in entry points (one pair per call: upload -> kernels -> download)
    def _pair(self, name, other):
        p = getattr(lib(), f"roaring_bitmap_{name}")(self.ptr, other.ptr)
        if not p:
            raise RB200Error(last_error())
        return Bitmap(p)

    def __and__(self, o): return self._pair("and", o)
    def __or__(self, o): return self._pair("or", o)
    def __xor__(self, o): return self._pair("xor", o)
    def __sub__(self, o): return self._pair("andnot", o)

    def inplace(self, name, other):
        """roaring_bitmap_{and,or,xor,andnot}_inplace(self, other)."""
        getattr(lib(), f"roaring_bitmap_{name}_inplace")(self.ptr, other.ptr)
        return self

    # -- public lazy API (roaring.h:932-977)
    def lazy_or(self, o, bitsetconversion=False):
        p = lib().roaring_bitmap_lazy_or(self.ptr, o.ptr, bool(bitsetconversion))
        if not p:
            raise RB200Error(last_error())
        return Bitmap(p)

    def lazy_or_inplace(self, o, bitsetconversion=False):
        lib().roaring_bitmap_lazy_or_inplace(self.ptr, o.ptr, bool(bitsetconversion))
        return self

    def lazy_xor(self, o):
        p = lib().roaring_bitmap_lazy_xor(self.ptr, o.ptr)
        if not p:
            raise RB200Error(last_error())
        return Bitmap(p)

    def lazy_xor_inplace(self, o):
        lib().roaring_bitmap_lazy_xor_inplace(self.ptr, o.ptr)
        return self

    def repair_after_lazy(self):
        lib().roaring_bitmap_repair_after_lazy(self.ptr)
        return self

    def and_cardinality(self, o) -> int:
        v = int(lib().roaring_bitmap_and_cardinality(self.ptr, o.ptr))
        if v == 2 ** 64 - 1:
            raise RB200Error(last_error())
        return v

    def or_cardinality(self, o): return int(lib().roaring_bitmap_or_cardinality(self.ptr, o.ptr))
    def xor_cardinality(self, o): return int(lib().roaring_bitmap_xor_cardinality(self.ptr, o.ptr))
    def andnot_cardinality(self, o): return int(lib().roaring_bitmap_andnot_cardinality(self.ptr, o.ptr))
    def jaccard_index(self, o): return float(lib().roaring_bitmap_jaccard_index(self.ptr, o.ptr))
    def intersect(self, o): return bool(lib().roaring_bitmap_intersect(self.ptr, o.ptr))
    def flip(self, start, end):
        p = lib().roaring_bitmap_flip(self.ptr, int(start), int(end))
        if not p:
            raise RB200Error(last_error())
        return Bitmap(p)

    def flip_inplace(self, start, end):
        lib().roaring_bitmap_flip_inplace(self.ptr, int(start), int(end))
        return self

    def equals(self, o): return bool(lib().roaring_bitmap_equals(self.ptr, o.ptr))
    def is_subset(self, o): return bool(lib().roaring_bitmap_is_subset(self.ptr, o.ptr))
    def is_strict_subset(self, o): return bool(lib().roaring_bitmap_is_strict_subset(self.ptr, o.ptr))


def or_many(bitmaps):
    """roaring_bitmap_or_many on host bitmaps (drop-in symbol)."""
    arr = (_P * len(bitmaps))(*[b.ptr for b in bitmaps])
    p = lib().roaring_bitmap_or_many(len(bitmaps), arr)
    if not p:
        raise RB200Error(last_error())
    return Bitmap(p)


def or_many_heap(bitmaps):
    """roaring_bitmap_or_many_heap on host bitmaps (drop-in symbol)."""
    arr = (_P * len(bitmaps))(*[b.ptr for b in bitmaps])
    p = lib().roaring_bitmap_or_many_heap(len(bitmaps), arr)
    if not p:
        raise RB200Error(last_error())
    return Bitmap(p)


def xor_many(bitmaps):
    """roaring_bitmap_xor_many on host bitmaps (drop-in symbol)."""
    arr = (_P * len(bitmaps))(*[b.ptr for b in bitmaps])
    p = lib().roaring_bitmap_xor_many(len(bitmaps), arr)
    if not p:
        raise RB200Error(last_error())
    return Bitmap(p)


VISIT_FN = C.CFUNCTYPE(C.c_int, C.c_size_t, _P, _P)


def foreach_many(sets, fn=None):
    """rb200_download_foreach_many: several result sets as one pipelined D2H stream.  fn=None:
    the built-in visitor (sum of host-side cardinalities, every bitmap freed) — returns the sum;
    otherwise fn(index, bitmap_ptr) is called on worker threads (return non-zero to keep the bitmap)."""
    arr = (_P * len(sets))(*[s.ptr for s in sets])
    if fn is None:
        acc = C.c_uint64(0)
        cb = C.cast(lib().rb200_visit_sum_cardinality, _P)
        if lib().rb200_download_foreach_many(arr, len(sets), cb, C.byref(acc)) != 0:
            raise RB200Error(last_error())
        return int(acc.value)
    cb = VISIT_FN(lambda i, p, _ctx: int(fn(i, p) or 0))
    if lib().rb200_download_foreach_many(arr, len(sets), C.cast(cb, _P), None) != 0:
        raise RB200Error(last_error())
    return None


class CardinalitySum:
    """Accumulator for the built-in visitor (sum of host-side cardinalities); must outlive the
    downloads it is passed to."""

    def __init__(self):
        self.acc = C.c_uint64(0)

    @property
    def value(self):
        return int(self.acc.value)


def download_wait():
    """rb200_download_wait: drain every download queued with DeviceSet.foreach_async."""
    if lib().rb200_download_wait() != 0:
        raise RB200Error(last_error())


def _blob_args(blobs):
    """(char* array, size_t array, n) of a list of bytes or of a workloads.BlobArena (no copy)."""
    if hasattr(blobs, "ptrs"):
        return blobs.ptrs, blobs.lens, len(blobs)
    n = len(blobs)
    return (C.c_char_p * n)(*blobs), (C.c_size_t * n)(*[len(b) for b in blobs]), n


class Comm:
    """rb200_comm_t: the NCCL communicator of a multi-GPU job (one process per GPU), plain C ABI.
    Comm.create(rank, world, bcast) bootstraps it: rank 0 draws the NCCL unique id and
    `bcast(bytes_or_None) -> bytes` carries it to the other ranks (any out-of-band channel, e.g.
    torch.distributed.broadcast_object_list)."""

    def __init__(self, ptr):
        if not ptr:
            raise RB200Error(last_error() or "null communicator")
        self.ptr = ptr

    @classmethod
    def create(cls, rank, world, bcast=None):
        if world == 1:
            return cls(lib().rb200_comm_init_rank(b"\0" * 128, 1, 0))
        buf = C.create_string_buffer(128)
        ident = None
        if rank == 0:
            if lib().rb200_comm_unique_id(buf) != 0:
                raise RB200Error(last_error())
            ident = buf.raw
        ident = bcast(ident)
        return cls(lib().rb200_comm_init_rank(ident, world, rank))

    @property
    def size(self):
        return int(lib().rb200_comm_size(self.ptr))

    @property
    def rank(self):
        return int(lib().rb200_comm_rank(self.ptr))

    def allreduce_u64(self, device_ptr, count=1):
        if lib().rb200_comm_allreduce_u64(self.ptr, _P(device_ptr), count) != 0:
            raise RB200Error(last_error())

    def destroy(self):
        if self.ptr:
            lib().rb200_comm_destroy(self.ptr)
        self.ptr = None


def plan_key_ranges(blobs, world):
    """rb200_plan_key_ranges: ([(lo, hi)] * world balanced by container bytes, (first, last) live key)."""
    pa, la, n = _blob_args(blobs)
    lo = (C.c_uint32 * world)()
    hi = (C.c_uint32 * world)()
    span = (C.c_uint32 * 2)()
    if lib().rb200_plan_key_ranges(pa, la, n, world, lo, hi, span) != 0:
        raise RB200Error(last_error())
    return [(int(lo[g]), int(hi[g])) for g in range(world)], (int(span[0]), int(span[1]))


def blob_slice_keys(blob: bytes, key_lo, key_hi) -> bytes:
    out, ln = C.c_void_p(), C.c_size_t()
    if lib().rb200_blob_slice_keys(blob, len(blob), key_lo, key_hi, C.byref(out), C.byref(ln)) != 0:
        raise RB200Error(last_error())
    b = C.string_at(out.value, ln.value)
    lib().rb200_blob_free(out)
    return b


def blobs_concat(blobs) -> bytes:
    pa, la, n = _blob_args(blobs)
    out, ln = C.c_void_p(), C.c_size_t()
    if lib().rb200_blobs_concat(pa, la, n, C.byref(out), C.byref(ln)) != 0:
        raise RB200Error(last_error())
    b = C.string_at(out.value, ln.value)
    lib().rb200_blob_free(out)
    return b


def r64_batch_op(op, a_blobs, b_blobs, ia, ib):
    """roaring64 and/or/xor/andnot on 64-bit portable blobs: list of result blobs (bytes)."""
    ia, ib = _u32(ia), _u32(ib)
    pa, la, na = _blob_args(a_blobs)
    pb, lb, nb = _blob_args(b_blobs)
    buf, off, ln = C.c_void_p(), C.POINTER(C.c_uint64)(), C.POINTER(C.c_uint64)()
    code = OPS[op] if isinstance(op, str) else op
    if lib().rb200_r64_batch_op_serialized(code, pa, la, na, pb, lb, nb, ia.ctypes.data, ib.ctypes.data, ia.size,
                                           C.byref(buf), C.byref(off), C.byref(ln)) != 0:
        raise RB200Error(last_error())
    out = [C.string_at(buf.value + off[k], ln[k]) for k in range(ia.size)]
    lib().rb200_serialized_free(buf, off, ln)
    return out


def r64_and_cardinality(a_blobs, b_blobs, ia, ib):
    ia, ib = _u32(ia), _u32(ib)
    pa, la, na = _blob_args(a_blobs)
    pb, lb, nb = _blob_args(b_blobs)
    out = np.zeros(ia.size, dtype=np.uint64)
    if lib().rb200_r64_batch_and_cardinality_serialized(pa, la, na, pb, lb, nb, ia.ctypes.data, ib.ctypes.data,
                                                        ia.size, out.ctypes.data) != 0:
        raise RB200Error(last_error())
    return out


def r64_batch_op_inmemory(op, a_ptrs, b_ptrs):
    """rb200_r64_batch_op on in-memory roaring64_bitmap_t* (raw pointers of the host application's
    CRoaring, which must be loaded RTLD_GLOBAL in this process): list of result pointers."""
    n = len(a_ptrs)
    pa, pb, out = (_P * n)(*a_ptrs), (_P * n)(*b_ptrs), (_P * n)()
    if lib().rb200_r64_batch_op(OPS[op] if isinstance(op, str) else op, pa, pb, n, out) != 0:
        raise RB200Error(last_error())
    return [out[i] for i in range(n)]


def batch_op_host(op, a, b):
    """out[k] = a[k] op b[k] through the device: one upload, one launch sequence, one download."""
    n = len(a)
    assert len(b) == n
    pa = (_P * n)(*[x.ptr for x in a])
    pb = (_P * n)(*[x.ptr for x in b])
    out = (_P * n)()
    if lib().rb200_batch_op_host(OPS[op] if isinstance(op, str) else op, pa, pb, n, out) != 0:
        raise RB200Error(last_error())
    return [Bitmap(out[i]) for i in range(n)]


def _values_u32(a):
    """1-D integer values as a contiguous uint32 array (refused if any lies outside [0, 2^32))."""
    a = np.asarray(a)
    if a.ndim != 1 or (a.size and a.dtype.kind not in "iu"):
        raise RB200Error(f"values must be 1-D integer arrays, got {a.dtype} with shape {a.shape}")
    if a.size and a.dtype != np.uint32 and (int(a.min()) < 0 or int(a.max()) > 0xFFFFFFFF):
        raise RB200Error("values must lie in [0, 2^32)")
    return np.ascontiguousarray(a, dtype=np.uint32)


def _offsets_i64(offsets, n):
    """add_offset's offsets as n contiguous int64 values: a scalar is broadcast; values outside the
    int64 range, non-integers and a length other than n are refused (never wrapped or rounded)."""
    if isinstance(offsets, (int, np.integer)):
        offsets = [int(offsets)] * n
    a = np.asarray(offsets)
    if a.dtype == object:   # Python ints beyond what numpy holds natively
        if not all(isinstance(x, (int, np.integer)) for x in a.reshape(-1)):
            raise RB200Error("offsets must be integers")
        if any(not -(1 << 63) <= int(x) < (1 << 63) for x in a.reshape(-1)):
            raise RB200Error("offsets must lie in the int64 range [-2^63, 2^63)")
        a = a.astype(np.int64)
    if a.ndim != 1 or (a.size and a.dtype.kind not in "iu"):
        raise RB200Error(f"offsets must be a 1-D integer array, got {a.dtype} with shape {a.shape}")
    if a.dtype.kind == "u" and a.size and int(a.max()) >= (1 << 63):
        raise RB200Error("offsets must lie in the int64 range [-2^63, 2^63)")
    if a.size != n:
        raise RB200Error(f"offsets has {a.size} entries for {n} items")
    return np.ascontiguousarray(a, dtype=np.int64)


def _value_lists(values, offsets, width):
    """One list of values per bitmap, in any form from_values takes, as (flat values, n + 1 offsets,
    entry point suffix): numpy uint{width} values and uint64 offsets for host values, suffix ""; for
    a CUDA tensor, the tensor itself and its offsets as a contiguous tensor on its device, ready for
    the library stream, suffix "_device" (the entry points that read them in place)."""
    if getattr(values, "is_cuda", False):
        import torch
        dtypes = (torch.int32, torch.uint32) if width == 32 else (torch.int64, torch.uint64)
        if values.dtype not in dtypes or values.dim() != 1 or not values.is_contiguous():
            raise RB200Error(f"device values must be a contiguous 1-D int{width} / uint{width} CUDA tensor")
        if offsets is None:
            raise RB200Error("device values need offsets")
        offs = offsets if isinstance(offsets, torch.Tensor) else torch.as_tensor(np.asarray(offsets, dtype=np.int64))
        if offs.dtype not in (torch.int64, torch.uint64) or offs.dim() != 1 or offs.numel() < 1:
            raise RB200Error("offsets must be a 1-D int64 / uint64 tensor of n + 1 entries")
        last = int(offs[-1].item())
        if last < 0 or last > values.numel():
            raise RB200Error(f"offsets end at {last}, outside the {values.numel()} values")
        offs = offs.to(values.device).contiguous()
        if offs is not offsets:   # copied here: on the stream the library reads on
            torch.cuda.current_stream(values.device).synchronize()
        return values, offs, "_device"
    conv = _values_u32 if width == 32 else _values_u64
    if offsets is None:
        arrays = [np.asarray(a).reshape(-1) for a in values]
        if width == 64:   # one by one: arrays of ints past 2^63 and below it would concatenate as float64
            arrays = [conv(a) for a in arrays]
        offs = np.zeros(len(arrays) + 1, dtype=np.uint64)
        np.cumsum([a.size for a in arrays], out=offs[1:])
        flat = conv(np.concatenate(arrays) if arrays else np.zeros(0, np.uint32))
    else:
        flat = conv(values)
        offs = np.ascontiguousarray(offsets, dtype=np.int64).astype(np.uint64)
        if offs.ndim != 1 or offs.size < 1 or int(offs[-1]) > flat.size:
            raise RB200Error(f"offsets must be n + 1 entries ending at most at len(values) = {flat.size}")
    return flat, offs, ""


def _ptr(a):
    """The address of a numpy array or a torch tensor."""
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data


def _update(s, fn, values, offsets, idx):
    """fn (an add_many / remove_many entry point; fn + "_device" for CUDA tensor values) on the
    selection idx of the set s, with one list of values per selected bitmap."""
    idx, ip, n = _selection(idx, len(s))
    flat, offs, suffix = _value_lists(values, offsets, s._width)   # held until the call returns
    if len(offs) - 1 != n:
        raise RB200Error(f"{len(offs) - 1} lists of values for {n} items")
    return getattr(lib(), fn + suffix)(s.ptr, ip, n, _ptr(flat), _ptr(offs))


QUERIES = {"contains": 0, "rank": 1, "get_index": 2, "select": 3}   # RB200_Q_*


def _query_index(idx, n, n_all):
    """The bitmap of every query: (None, n_all) for idx None (one query per bitmap), else a uint32 array of
    n entries, a scalar idx broadcast to all of them."""
    if idx is None:
        if n != n_all:
            raise RB200Error(f"{n} values for the {n_all} bitmaps of the set (idx=None asks each bitmap once)")
        return None
    if np.ndim(idx) == 0:
        if not isinstance(idx, (int, np.integer)) or isinstance(idx, bool) or not 0 <= int(idx) <= 0xFFFFFFFF:
            raise RB200Error(f"idx must be an integer in [0, 2^32), got {idx!r}")
        return int(idx)
    ia = _values_u32(idx)
    if ia.size != n:
        raise RB200Error(f"idx has {ia.size} entries for {n} values")
    return ia


def _query(s, kind, values, idx):
    """out[k] = the answer of bitmap idx[k] of the set s about values[k] (rb200_batch_query); CUDA tensor
    values go through rb200_batch_query_device and the answers stay on their device."""
    if kind not in QUERIES:
        raise RB200Error(f"unknown query kind {kind!r}: one of {sorted(QUERIES)}")
    if getattr(values, "is_cuda", False):
        return _query_device(s, QUERIES[kind], values, idx)
    vals = _values_u32(values)
    ia = _query_index(idx, vals.size, len(s))
    out = np.empty(vals.size, dtype=np.int64)
    if ia is not None and not vals.size:
        return out   # (the library reads a NULL idx as one query per bitmap)
    if isinstance(ia, int):
        ia = np.full(vals.size, ia, dtype=np.uint32)
    if lib().rb200_batch_query(QUERIES[kind], s.ptr, None if ia is None else ia.ctypes.data, vals.size,
                               vals.ctypes.data, out.ctypes.data) != 0:
        raise RB200Error(last_error())
    return out


def _device_u32(t, what):
    import torch
    if t.dtype not in (torch.int32, torch.uint32) or t.dim() != 1 or not t.is_contiguous():
        raise RB200Error(f"device {what} must be a contiguous 1-D int32 / uint32 CUDA tensor")
    return t


def _query_device(s, code, values, idx):
    import torch
    values = _device_u32(values, "values")
    dev, n = values.device, values.numel()
    if isinstance(idx, torch.Tensor):
        ia = _device_u32(idx.to(dev), "idx")
        if ia.numel() != n:
            raise RB200Error(f"idx has {ia.numel()} entries for {n} values")
    else:
        ia = _query_index(idx, n, len(s))
        if isinstance(ia, int):   # expanded on the values' device, as the int32 of the same bits
            ia = torch.full((n,), ia - (1 << 32) if ia >= 1 << 31 else ia, dtype=torch.int32, device=dev)
        elif ia is not None:
            ia = torch.from_numpy(ia.view(np.int32)).to(dev)
    out = torch.empty(n, dtype=torch.int64, device=dev)
    if ia is not None and not n:
        return out   # (an empty tensor's address is NULL, which the library reads as one query per bitmap)
    # the library stream reads and writes these: what torch's stream queued on them comes first
    torch.cuda.current_stream(dev).synchronize()
    if lib().rb200_batch_query_device(code, s.ptr, None if ia is None else ia.data_ptr(), n, values.data_ptr(),
                                      out.data_ptr()) != 0:
        raise RB200Error(last_error())
    return out


class DeviceSet:
    """An ordered collection of bitmaps resident in HBM (rb200_set_t*)."""
    _width = 32   # bits per value

    def __init__(self, ptr):
        if not ptr:
            raise RB200Error(last_error() or "null set")
        self.ptr = ptr

    @classmethod
    def upload(cls, bitmaps):
        arr = (_P * len(bitmaps))(*[b.ptr for b in bitmaps])
        return cls(lib().rb200_set_upload(arr, len(bitmaps)))

    @classmethod
    def from_serialized(cls, blobs, key_lo=None, key_hi=None):
        """blobs: list of bytes or a workloads.BlobArena.  key_lo / key_hi: keep only the containers
        of that key range (what one rank of a key-sharded union uploads)."""
        arr, lens, n = _blob_args(blobs)
        if key_lo is None and key_hi is None:
            return cls(lib().rb200_set_upload_serialized(arr, lens, n))
        return cls(lib().rb200_set_upload_serialized_keyrange(arr, lens, n, key_lo or 0,
                                                              65535 if key_hi is None else key_hi))

    @classmethod
    def from_frozen(cls, blobs):
        """Resident set from roaring_bitmap_frozen_serialize blobs (parsed on the device)."""
        n = len(blobs)
        arr = (C.c_char_p * n)(*blobs)
        lens = (C.c_size_t * n)(*[len(b) for b in blobs])
        return cls(lib().rb200_set_upload_frozen(arr, lens, n))

    @classmethod
    def from_values(cls, values, offsets=None):
        """roaring_bitmap_of_ptr of every bitmap, built on the device (no run containers: chain
        .run_optimize() for those).  values: a list of 1-D integer arrays, one per bitmap; or one flat
        uint32 array with n + 1 offsets (the layout of to_uint32_arrays); or a CUDA torch tensor of
        int32 / uint32 values with offsets as a CUDA or CPU tensor, read in place on the library stream
        (order its writes before the call, e.g. by building it on the stream given to set_stream)."""
        flat, offs, suffix = _value_lists(values, offsets, 32)
        return cls(getattr(lib(), "rb200_set_from_uint32" + suffix)(_ptr(flat), _ptr(offs), len(offs) - 1))

    def free(self):
        if self.ptr:
            lib().rb200_set_free(self.ptr)
        self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def bind_host(self, enable=True):
        """Promise that the host bitmaps this set was uploaded from outlive the downloads of its
        results (pass-through containers are then not transferred back)."""
        if lib().rb200_set_bind_host(self.ptr, 1 if enable else 0) != 0:
            raise RB200Error(last_error())
        return self

    def __len__(self):
        return int(lib().rb200_set_count(self.ptr))

    @property
    def container_count(self):
        return int(lib().rb200_set_container_count(self.ptr))

    @property
    def payload_bytes(self):
        return int(lib().rb200_set_payload_bytes(self.ptr))

    def batch(self, op, other, ia, ib, inplace_rules=False, lazy=False, bitsetconversion=False,
              from_lazy_inputs=False):
        """result[k] = self[ia[k]] op other[ib[k]] as a new DeviceSet.  lazy=True: the lazy OR/XOR
        variants (result set in a lazy state: chain further lazy ops, then repair_after_lazy())."""
        ia, ib = _u32(ia), _u32(ib)
        assert ia.shape == ib.shape
        code = OPS[op] if isinstance(op, str) else op
        flags = (1 if inplace_rules else 0) | (2 if lazy else 0) | (4 if bitsetconversion else 0) | \
                (8 if from_lazy_inputs else 0)
        p = lib().rb200_batch_op_ex(code, flags, self.ptr, other.ptr,
                                    ia.ctypes.data, ib.ctypes.data, ia.size)
        return DeviceSet(p)

    def repair_after_lazy(self):
        return DeviceSet(lib().rb200_set_repair_after_lazy(self.ptr))

    def or_many_heap(self, idx=None):
        idx, ip, n = _selection(idx, len(self))
        return DeviceSet(lib().rb200_or_many_heap(self.ptr, ip, n))

    def and_cardinality(self, other, ia, ib):
        ia, ib = _u32(ia), _u32(ib)
        out = np.zeros(ia.size, dtype=np.uint64)
        rc = lib().rb200_batch_and_cardinality(self.ptr, other.ptr, ia.ctypes.data, ib.ctypes.data,
                                               ia.size, out.ctypes.data)
        if rc != 0:
            raise RB200Error(last_error())
        return out

    def flip(self, range_start, range_end, idx=None):
        """roaring_bitmap_flip of every (or the selected) bitmap over [range_start, range_end)."""
        idx, ip, n = _selection(idx, len(self))
        return DeviceSet(lib().rb200_batch_flip(self.ptr, ip, n, int(range_start), int(range_end)))

    def add_offset(self, offsets, idx=None):
        """roaring_bitmap_add_offset of every (or the selected) bitmap: result[k] = self[idx[k]] +
        offsets[k].  offsets: one integer for every item, or one per item (int64 range)."""
        idx, ip, n = _selection(idx, len(self))
        offs = _offsets_i64(offsets, n)   # held until the call returns
        return DeviceSet(lib().rb200_batch_add_offset(self.ptr, ip, n, offs.ctypes.data))

    def add_many(self, values, offsets=None, idx=None):
        """roaring_bitmap_add_many of every (or the selected) bitmap: result[k] = self[idx[k]] with the
        values of item k added.  values: any form from_values takes, one list of values per item."""
        return DeviceSet(_update(self, "rb200_batch_add_many", values, offsets, idx))

    def remove_many(self, values, offsets=None, idx=None):
        """roaring_bitmap_remove_many of every (or the selected) bitmap, as add_many."""
        return DeviceSet(_update(self, "rb200_batch_remove_many", values, offsets, idx))

    # -- point queries.  values[k] is asked of bitmap idx[k]: idx None asks bitmap k (one value per bitmap),
    # an array gives one bitmap per value, a scalar asks every value of one bitmap.  Host values (arrays,
    # lists) give a numpy int64 array; a CUDA tensor of int32 / uint32 values (read in place on the library
    # stream, order its writes before the call as for from_values) gives an int64 tensor on its device.
    def contains(self, values, idx=None):
        """roaring_bitmap_contains per query: 1 or 0."""
        return _query(self, "contains", values, idx)

    def rank(self, values, idx=None):
        """roaring_bitmap_rank per query: the number of values <= values[k] (up to 2^32)."""
        return _query(self, "rank", values, idx)

    def get_index(self, values, idx=None):
        """roaring_bitmap_get_index per query: the index of values[k] in its bitmap, or -1."""
        return _query(self, "get_index", values, idx)

    def select(self, ranks, idx=None):
        """roaring_bitmap_select per query: the value of 0-based rank ranks[k], or -1 past the cardinality."""
        return _query(self, "select", ranks, idx)

    def op_stats(self):
        """(device_ms, compute_kernel_ms, algorithmic_bytes) of the batch op that produced this set."""
        ms, cms, ab = C.c_float(), C.c_float(), C.c_uint64()
        if lib().rb200_set_op_stats(self.ptr, C.byref(ms), C.byref(cms), C.byref(ab)) != 0:
            raise RB200Error(last_error())
        return float(ms.value), float(cms.value), int(ab.value)

    def relations(self, other, ia, ib):
        """uint8 per pair: bit 0 equals, bit 1 is_subset, bit 2 is_strict_subset."""
        ia, ib = _u32(ia), _u32(ib)
        out = np.zeros(ia.size, dtype=np.uint8)
        if lib().rb200_batch_relations(self.ptr, other.ptr, ia.ctypes.data, ib.ctypes.data, ia.size,
                                       out.ctypes.data) != 0:
            raise RB200Error(last_error())
        return out

    def or_many(self, idx=None, key_lo=0, key_hi=65535, card_per_key=None):
        idx, ip, n = _selection(idx, len(self))
        cp = card_per_key.ctypes.data if card_per_key is not None else None
        if card_per_key is not None:
            assert card_per_key.dtype == np.uint32 and card_per_key.size == 65536
        p = lib().rb200_or_many_keyrange(self.ptr, ip, n, key_lo, key_hi, cp)
        return DeviceSet(p)

    def or_many_sharded(self, comm, key_lo, key_hi, span, idx=None):
        """rb200_or_many_sharded: (this rank's part as a DeviceSet, uint32 per-key cardinalities of
        the span summed over the ranks, cardinality of the whole union)."""
        idx, ip, n = _selection(idx, len(self))
        cards = np.zeros(max(0, span[1] - span[0] + 1), dtype=np.uint32)
        tot = C.c_uint64(0)
        p = lib().rb200_or_many_sharded(self.ptr, ip, n, key_lo, key_hi, span[0], span[1], comm.ptr,
                                        cards.ctypes.data, C.byref(tot))
        return DeviceSet(p), cards, int(tot.value)

    def add_cardinality_device(self, device_ptr):
        """*device_ptr (u64 in device memory) += sum of the cardinalities of the set's bitmaps."""
        if lib().rb200_set_add_cardinality_device(self.ptr, _P(device_ptr)) != 0:
            raise RB200Error(last_error())

    def xor_many(self, idx=None):
        idx, ip, n = _selection(idx, len(self))
        return DeviceSet(lib().rb200_xor_many(self.ptr, ip, n))

    def cardinalities(self):
        out = np.zeros(len(self), dtype=np.uint64)
        if lib().rb200_set_cardinalities(self.ptr, out.ctypes.data) != 0:
            raise RB200Error(last_error())
        return out

    def download(self, i):
        return Bitmap(lib().rb200_set_download(self.ptr, i))

    def download_all_raw(self):
        """All bitmaps as a ctypes array of roaring_bitmap_t* (no Python wrappers); release with
        free_raw().  bench.py's e2e leg times the visitor form (foreach_async), which shares this
        download pipeline."""
        n = len(self)
        out = (_P * n)()
        if lib().rb200_set_download_all(self.ptr, out) != 0:
            raise RB200Error(last_error())
        return out

    @staticmethod
    def free_raw(arr, n=None):
        lib().rb200_bitmaps_free(arr, len(arr) if n is None else n)

    def foreach_sum_cardinality(self):
        """Materialise every bitmap on the host (reference layout), read its cardinality with the
        host function and free it — the reference benchmark loop body, run by the library's worker
        threads (rb200_download_foreach + rb200_visit_sum_cardinality)."""
        acc = C.c_uint64(0)
        fn = C.cast(lib().rb200_visit_sum_cardinality, _P)
        if lib().rb200_download_foreach(self.ptr, fn, C.byref(acc)) != 0:
            raise RB200Error(last_error())
        return int(acc.value)

    def foreach_async(self, acc: "CardinalitySum", fn=None):
        """rb200_download_foreach_async: queue this set for the background downloader (built-in
        visitor adding into `acc`, or a VISIT_FN kept alive by the caller) and return at once."""
        cb = C.cast(lib().rb200_visit_sum_cardinality, _P) if fn is None else C.cast(fn, _P)
        ctx = C.byref(acc.acc) if fn is None else None
        if lib().rb200_download_foreach_async(self.ptr, cb, ctx) != 0:
            raise RB200Error(last_error())

    def run_optimize(self, remove_runs=False):
        """roaring_bitmap_run_optimize (or remove_run_compression) of every bitmap, on the device."""
        return DeviceSet(lib().rb200_set_run_optimize(self.ptr, 0 if remove_runs else 1))

    def to_uint32_arrays(self):
        """roaring_bitmap_to_uint32_array of every bitmap: list of numpy uint32 arrays."""
        vals = C.POINTER(C.c_uint32)()
        off = C.POINTER(C.c_uint64)()
        if lib().rb200_set_to_uint32(self.ptr, C.byref(vals), C.byref(off)) != 0:
            raise RB200Error(last_error())
        n = len(self)
        total = off[n] if n else 0
        flat = np.ctypeslib.as_array(vals, shape=(total,)).copy() if total else np.zeros(0, np.uint32)
        out = [flat[off[i]:off[i + 1]] for i in range(n)]
        lib().rb200_values_free(vals, off)
        return out

    def serialize_all(self, copy=True, frozen=False):
        """Portable (or frozen) bytes of every bitmap, serialized ON THE DEVICE and brought back in
        one D2H.  copy=True -> list of bytes; copy=False -> (base pointer, offsets, lengths, release())"""
        buf = C.c_void_p()
        off = C.POINTER(C.c_uint64)()
        ln = C.POINTER(C.c_uint64)()
        fn = lib().rb200_set_serialize_frozen if frozen else lib().rb200_set_serialize
        if fn(self.ptr, C.byref(buf), C.byref(off), C.byref(ln)) != 0:
            raise RB200Error(last_error())
        n = len(self)

        def release():
            lib().rb200_serialized_free(buf, off, ln)
        if not copy:
            return buf, off, ln, release
        out = [C.string_at(buf.value + off[i], ln[i]) for i in range(n)]
        release()
        return out

    def download_stream(self, chunk_bitmaps=1024):
        """Generator over (ctypes array of roaring_bitmap_t*, count): streaming download.  The
        caller owns each chunk's bitmaps (free with DeviceSet.free_raw(arr, n))."""
        st = lib().rb200_download_begin(self.ptr, chunk_bitmaps)
        if not st:
            raise RB200Error(last_error())
        try:
            cap = max(1, int(lib().rb200_download_chunk_capacity(st)))
            while True:
                out = (_P * cap)()
                n = lib().rb200_download_next(st, out)
                if n == 0:
                    break
                if n == 2 ** 64 - 1:
                    raise RB200Error(last_error())
                yield out, int(n)
        finally:
            lib().rb200_download_end(st)

    def download_all(self):
        n = len(self)
        out = (_P * n)()
        if lib().rb200_set_download_all(self.ptr, out) != 0:
            raise RB200Error(last_error())
        return [Bitmap(out[i]) for i in range(n)]


def _values_u64(a):
    """1-D integer values as a contiguous uint64 array (refused if any lies outside [0, 2^64))."""
    a = np.asarray(a)
    if a.ndim != 1 or (a.size and a.dtype.kind not in "iu"):
        raise RB200Error(f"values must be 1-D integer arrays, got {a.dtype} with shape {a.shape}")
    if a.size and a.dtype.kind == "i" and int(a.min()) < 0:
        raise RB200Error("values must lie in [0, 2^64)")
    return np.ascontiguousarray(a, dtype=np.uint64)


def _serialized(fn, ptr, n):
    buf = C.c_void_p()
    off = C.POINTER(C.c_uint64)()
    ln = C.POINTER(C.c_uint64)()
    if fn(ptr, C.byref(buf), C.byref(off), C.byref(ln)) != 0:
        raise RB200Error(last_error())
    out = [C.string_at(buf.value + off[i], ln[i]) for i in range(n)]
    lib().rb200_serialized_free(buf, off, ln)
    return out


class DeviceSet64:
    """An ordered collection of 64-bit bitmaps (roaring64_bitmap_t) resident in HBM (rb200_set64_t*)."""
    _width = 64   # bits per value

    def __init__(self, ptr):
        if not ptr:
            raise RB200Error(last_error() or "null set")
        self.ptr = ptr

    @classmethod
    def from_serialized(cls, blobs):
        """blobs: list of roaring64_bitmap_portable_serialize bytes."""
        arr, lens, n = _blob_args(blobs)
        return cls(lib().rb200_set64_upload_serialized(arr, lens, n))

    @classmethod
    def from_values(cls, values, offsets=None):
        """roaring64_bitmap_of_ptr of every bitmap, built on the device (no run containers: chain
        .run_optimize() for those).  values: a list of 1-D integer arrays, one per bitmap; or one flat
        array with n + 1 offsets; or a CUDA torch tensor of int64 / uint64 values (its bits read as
        uint64) with offsets as a CUDA or CPU tensor, read in place on the library stream."""
        flat, offs, suffix = _value_lists(values, offsets, 64)
        return cls(getattr(lib(), "rb200_set64_from_uint64" + suffix)(_ptr(flat), _ptr(offs), len(offs) - 1))

    def free(self):
        if self.ptr:
            lib().rb200_set64_free(self.ptr)
        self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def __len__(self):
        return int(lib().rb200_set64_count(self.ptr))

    def op(self, op, other, ia, ib):
        """result[k] = self[ia[k]] op other[ib[k]] as a new DeviceSet64 (op: and / or / xor / andnot)."""
        ia, ib = _u32(ia), _u32(ib)
        assert ia.shape == ib.shape
        code = OPS[op] if isinstance(op, str) else op
        return DeviceSet64(lib().rb200_set64_batch_op(code, self.ptr, other.ptr, ia.ctypes.data, ib.ctypes.data,
                                                      ia.size))

    def and_cardinality(self, other, ia, ib):
        ia, ib = _u32(ia), _u32(ib)
        out = np.zeros(ia.size, dtype=np.uint64)
        if lib().rb200_set64_batch_and_cardinality(self.ptr, other.ptr, ia.ctypes.data, ib.ctypes.data, ia.size,
                                                   out.ctypes.data) != 0:
            raise RB200Error(last_error())
        return out

    def cardinalities(self):
        out = np.zeros(len(self), dtype=np.uint64)
        if lib().rb200_set64_cardinalities(self.ptr, out.ctypes.data) != 0:
            raise RB200Error(last_error())
        return out

    def add_many(self, values, offsets=None, idx=None):
        """roaring64_bitmap_add_many of every (or the selected) bitmap: result[k] = self[idx[k]] with the
        values of item k added.  values: any form from_values takes, one list of values per item."""
        return DeviceSet64(_update(self, "rb200_set64_batch_add_many", values, offsets, idx))

    def remove_many(self, values, offsets=None, idx=None):
        """roaring64_bitmap_remove_many of every (or the selected) bitmap, as add_many."""
        return DeviceSet64(_update(self, "rb200_set64_batch_remove_many", values, offsets, idx))

    def run_optimize(self, mode=1):
        """mode 1: roaring64_bitmap_run_optimize of every bitmap; mode 0: the run containers removed."""
        return DeviceSet64(lib().rb200_set64_run_optimize(self.ptr, int(mode)))

    def serialize_all(self):
        """roaring64_bitmap_portable_serialize bytes of every bitmap, written on the device, one D2H."""
        return _serialized(lib().rb200_set64_serialize, self.ptr, len(self))
