"""Copy-on-write (COW) inputs for the parity tests: bitmaps built in one of four states, a view of
their containers' typecodes, the reference's flag getter, and a plain-Python model of the COW flag
the reference gives each result (the spec the host driver follows).

States of an input, built from its portable bytes:
- plain:      deserialized, flag off;
- cow:        flag on, containers its own;
- cow-copy:   roaring_bitmap_copy of a cow bitmap: flag on, every container a SHARED wrapper;
- shared-off: a cow-copy with the flag bit cleared: SHARED containers, flag off.
The reference rewrites the containers of COW inputs into SHARED wrappers as it reads them, so every
caller builds its own inputs afresh from the same bytes and state."""
import ctypes as C

import numpy as np

STATES = ("plain", "cow", "cow-copy", "shared-off")
T_BITSET, T_ARRAY, T_RUN, T_SHARED = 1, 2, 3, 4


class _RoaringArray(C.Structure):   # roaring_types.h:61-68
    _fields_ = [("size", C.c_int32), ("allocation_size", C.c_int32), ("containers", C.POINTER(C.c_void_p)),
                ("keys", C.POINTER(C.c_uint16)), ("typecodes", C.POINTER(C.c_uint8)), ("flags", C.c_uint8)]


class _Shared(C.Structure):          # shared_container_s, containers.h
    _fields_ = [("container", C.c_void_p), ("typecode", C.c_uint8)]


def bind(R):
    """The reference symbols these tests need beyond oracle/refbind.py."""
    L = R.L
    L.roaring_bitmap_get_copy_on_write.restype = C.c_bool
    L.roaring_bitmap_get_copy_on_write.argtypes = [C.c_void_p]
    L.roaring_bitmap_add_offset.restype = C.c_void_p
    L.roaring_bitmap_add_offset.argtypes = [C.c_void_p, C.c_int64]
    L.roaring_bitmap_remove_many.restype = None
    L.roaring_bitmap_remove_many.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    return R


def cow_of(R, p):
    return bool(R.L.roaring_bitmap_get_copy_on_write(p))


def containers(p):
    """[(key, typecode, shared)] of a roaring_bitmap_t*, SHARED wrappers unwrapped."""
    ra = C.cast(C.c_void_p(p), C.POINTER(_RoaringArray)).contents
    out = []
    for i in range(ra.size):
        t = ra.typecodes[i]
        shared = t == T_SHARED
        if shared:
            t = C.cast(C.c_void_p(ra.containers[i]), C.POINTER(_Shared)).contents.typecode
        out.append((ra.keys[i], t, shared))
    return out


def make(R, blob, state):
    """A fresh reference bitmap holding `blob` in `state`."""
    x = R.deserialize(blob)
    if state == "plain":
        return x
    R.L.roaring_bitmap_set_copy_on_write(x, True)
    if state == "cow":
        return x
    y = R.L.roaring_bitmap_copy(x)   # y's containers are SHARED wrappers (roaring.c:525-543)
    R.free(x)
    if state == "shared-off":
        # roaring_bitmap_set_copy_on_write(y, false) would unshare every container (roaring.h:117-126);
        # the reference reaches this state itself when a plain accumulator takes a COW input's
        # containers (lazy_xor_inplace, roaring.c:2825-2834), so the flag bit is cleared directly
        C.cast(C.c_void_p(y), C.POINTER(_RoaringArray)).contents.flags &= ~1
    return y


def fingerprint(R, p):
    """What must not change in an input: its bytes, its containers' types and wrappers, its flag."""
    return R.serialize(p), containers(p), cow_of(R, p)


# ------------------------------------------------------------------ the COW flag of a result
# inputs: [(values, cow)], values a 1-D integer array.
PAIRWISE = ("and", "or", "xor", "andnot", "lazy_or", "lazy_xor")
INPLACE = ("and_inplace", "or_inplace", "xor_inplace", "andnot_inplace", "lazy_or_inplace", "lazy_xor_inplace")
FOLDS = ("or_many", "xor_many", "or_many_heap")


def _nonempty(v):
    return len(v) > 0


def _pair(op, a, b):
    """roaring_bitmap_<op>(x1, x2), roaring.c: a union or xor with an empty operand copies the other,
    andnot copies x1 when x2 is empty, everything else takes both flags."""
    (va, fa), (vb, fb) = a, b
    if op in ("or", "xor", "lazy_or", "lazy_xor"):
        if not _nonempty(va):
            return fb
        if not _nonempty(vb):
            return fa
    if op == "andnot" and _nonempty(va) and not _nonempty(vb):
        return fa
    return fa or fb


def _inplace(op, a, b):
    """x1's flag after roaring_bitmap_<op>(x1, x2): kept, unless a union or xor overwrites an empty x1
    with a non-empty x2 (roaring_bitmap_overwrite)."""
    (va, fa), (vb, fb) = a, b
    if op.split("_inplace")[0] in ("or", "xor", "lazy_or", "lazy_xor") and not _nonempty(va) and _nonempty(vb):
        return fb
    return fa


def _fold(op, inputs):
    """roaring_bitmap_or_many / xor_many: lazy_<op>(x0, x1), then lazy_<op>_inplace(acc, xi)."""
    if not inputs:
        return False
    if len(inputs) == 1:
        return inputs[0][1]
    f = _pair("lazy_" + op, inputs[0], inputs[1])
    acc = _combine(op, inputs[0][0], inputs[1][0])
    for v, c in inputs[2:]:
        if _nonempty(v) and not _nonempty(acc):
            f = c
        acc = _combine(op, acc, v)
    return f


def _combine(op, a, b):
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    return np.union1d(a, b) if op == "or" else np.setxor1d(a, b)


def array_portable_size(v):
    """roaring_bitmap_portable_size_in_bytes of a bitmap whose containers are all arrays."""
    v = np.unique(np.asarray(v, np.int64))
    nk = len(np.unique(v >> 16))
    return 8 + 8 * nk + 2 * len(v)


def _heap(inputs, size):
    """roaring_bitmap_or_many_heap (roaring_priority_queue.c:200-247), replayed with the same min-heap
    as rb200_host.cu (strict size comparisons, the same sift loops).  size(values): the portable size of
    a bitmap holding them, for the inputs and for every temporary union."""
    if not inputs:
        return False
    if len(inputs) == 1:
        return inputs[0][1]
    # element: [size, temporary, values, flag]
    e = [[size(v), False, v, f] for v, f in inputs]

    def down(n, i):
        cur = e[i]
        while i < n >> 1:
            ch = 2 * i + 1
            if ch + 1 < n and e[ch + 1][0] < e[ch][0]:
                ch += 1
            if not e[ch][0] < cur[0]:
                break
            e[i] = e[ch]
            i = ch
        e[i] = cur

    def pop(n):
        top = e[0]
        if n > 1:
            e[0] = e[n - 1]
            down(n - 1, 0)
        return top, n - 1

    def push(n, t):
        if n < len(e):
            e[n] = t
        else:
            e.append(t)
        i = n
        while i > 0:
            p = (i - 1) >> 1
            if not t[0] < e[p][0]:
                break
            e[i] = e[p]
            i = p
        e[i] = t
        return n + 1

    n = len(e)
    for i in range(n >> 1, -1, -1):
        down(n, i)
    while n > 1:
        a, n = pop(n)
        b, n = pop(n)
        v = _combine("or", a[2], b[2])
        if a[1] and b[1]:       # lazy_or_from_lazy_inputs: a non-empty operand next to an empty one, else new
            f = b[3] if not _nonempty(a[2]) else a[3] if not _nonempty(b[2]) else False
        elif b[1]:              # lazy_or_inplace(x2, x1)
            f = _inplace("lazy_or_inplace", (b[2], b[3]), (a[2], a[3]))
        elif a[1]:
            f = _inplace("lazy_or_inplace", (a[2], a[3]), (b[2], b[3]))
        else:
            f = _pair("lazy_or", (a[2], a[3]), (b[2], b[3]))
        n = push(n, [size(v), True, v, f])
    return e[0][3]


def expected_cow(entry, inputs, size=array_portable_size):
    """The COW flag the reference leaves on the result of `entry` (x1 for the in-place twins)."""
    if entry in PAIRWISE:
        return _pair(entry, *inputs)
    if entry in INPLACE:
        return _inplace(entry, *inputs)
    if entry == "or_many_heap":
        return _heap(inputs, size)
    return _fold(entry.split("_many")[0], inputs)
