"""CPU checks of roaring_bitmap_add_range_closed / remove_range_closed on the device path's terms (-m "not gpu"):
the type rule of rb200_device.cuh (range_type) through a host-compiled probe, each probe case pinned against
the reference's own range update of a one-container bitmap; the argument errors the C ABI reports before any
device work; and the mirror's argument checks and its open-to-closed conversion, checked against the
reference's own inline wrappers."""
import ctypes as C

import numpy as np
import pytest

from croaring_b200 import api
from helpers import run_probe
from range_oracles import ref_range_bytes
from test_update_host import containers

T_BITSET, T_ARRAY, T_RUN = 1, 2, 3

PROBE = r'''
#include "rb200_device.cuh"
#include <cstdio>
using namespace rb200;
// argv: cases "add t card nruns"; prints range_type's result per case
int main(int argc, char **argv) {
    for (int i = 1; i < argc; i++) {
        int add, t, card, nruns;
        if (sscanf(argv[i], "%d %d %d %d", &add, &t, &card, &nruns) != 4) return 2;
        printf("%d\n", range_type(add != 0, t, card, nruns));
    }
    return 0;
}
'''


def _runs_of(vals):
    """[(start, end)] of sorted distinct values."""
    v = np.unique(np.asarray(vals, dtype=np.int64))
    if not v.size:
        return []
    cut = np.flatnonzero(np.diff(v) != 1)
    starts = np.concatenate([[v[0]], v[cut + 1]])
    ends = np.concatenate([v[cut], [v[-1]]])
    return list(zip(starts.tolist(), ends.tolist()))


def _stripes(nruns, width=3, step=8):
    """nruns runs of `width` values, `step` apart: a run container when run-optimized (at most 2047 runs)."""
    return np.concatenate([np.arange(step * i, step * i + width) for i in range(nruns)])


def _blob(R, vals, run_opt):
    r = R.from_values(np.asarray(vals, np.uint32), run_optimize=run_opt)
    b = R.serialize(r)
    R.free(r)
    return b


def _values(R, blob):
    r = R.deserialize(blob)
    v = R.to_array(r)
    R.free(r)
    return v


# (name, S as portable bytes (a builder of R), op, lo, hi): one container at key 0 or none, the range
# inside key 0
def _cases(R):
    full = np.arange(65536)
    run2047 = _blob(R, _stripes(2047), True)
    run2048 = ref_range_bytes(R, "add", run2047, 60000, 60002)   # a 2048-run container: 8192 bytes
    return [
        ("array 4095 + 1 value", _blob(R, np.arange(0, 8190, 2), False), "add", 1, 1),
        ("array 4095 + 2 values", _blob(R, np.arange(0, 8190, 2), False), "add", 1, 3),
        ("array 4096 + present values", _blob(R, np.arange(0, 8192, 2), False), "add", 2, 2),
        ("array 4096 + 1 value", _blob(R, np.arange(0, 8192, 2), False), "add", 1, 1),
        ("array 4000 + a range to 65536", _blob(R, np.arange(0, 4000), False), "add", 4000, 65535),
        ("array - every value", _blob(R, np.arange(100, 200), False), "remove", 0, 300),
        ("array - some values", _blob(R, np.arange(100, 200), False), "remove", 150, 300),
        ("bitset 4097 - 1 value", _blob(R, np.arange(0, 8194, 2), False), "remove", 0, 0),
        ("bitset 4098 - 1 value", _blob(R, np.arange(0, 8196, 2), False), "remove", 0, 0),
        ("bitset 4097 - an absent value", _blob(R, np.arange(0, 8194, 2), False), "remove", 1, 1),
        ("bitset 4097 + 1 value", _blob(R, np.arange(0, 8194, 2), False), "add", 1, 1),
        ("bitset - a range to 0", _blob(R, np.arange(0, 8194, 2), False), "remove", 0, 9000),
        ("bitset + the rest of the key", _blob(R, np.arange(0, 8194, 2), False), "add", 1, 65535),
        ("run 2046 + a disjoint range", _blob(R, _stripes(2046), True), "add", 60000, 60002),
        ("run 2047 + a disjoint range", run2047, "add", 60000, 60002),
        ("run 2048 + a disjoint range", run2048, "add", 62000, 62002),
        ("run 2047 + a merging range", run2047, "add", 3, 4),
        ("run 2048 + a merging range", run2048, "add", 3, 7),
        ("run + the rest of the key", _blob(R, np.arange(10, 100), True), "add", 0, 65535),
        ("run - a range that touches no value", run2048, "remove", 60003, 60005),
        ("run - its whole span", _blob(R, np.arange(10, 100), True), "remove", 10, 99),
        ("run - a cut", _blob(R, np.arange(10, 100), True), "remove", 20, 30),
        ("full run - a value", _blob(R, full, True), "remove", 7, 7),
        ("full key from an array", _blob(R, np.arange(0, 10), False), "add", 0, 65535),
        ("full key from a bitset", _blob(R, np.arange(0, 10000), False), "add", 0, 65535),
        ("full key from a run", _blob(R, np.arange(0, 10000), True), "add", 0, 65535),
        ("full key removed from a run", _blob(R, np.arange(0, 10000), True), "remove", 0, 65535),
        ("absent key + 1 value", _blob(R, [], False), "add", 5, 5),
        ("absent key + 2 values", _blob(R, [], False), "add", 5, 6),
        ("absent key + 3 values", _blob(R, [], False), "add", 5, 7),
    ]


def _probe_arg(R, blob, op, lo, hi):
    """The probe's "add t card nruns" for this update, and the reference result's container (type, card, len)
    or None when the key is dropped."""
    have = _values(R, blob)
    cs = containers(blob)
    t = cs[0][1] if cs else 0
    s = set(have.tolist())
    rng = set(range(lo, hi + 1))
    res = sorted(s | rng if op == "add" else s - rng)
    if op == "add" and t == T_RUN:   # rle16_count_less / _greater: runs that neither meet nor touch the range
        runs = _runs_of(have)
        nruns = sum(e + 1 < lo for _, e in runs) + 1 + sum(st > hi + 1 for st, _ in runs)
    else:
        nruns = len(_runs_of(res)) if t == T_RUN else 0
    got = containers(ref_range_bytes(R, op, blob, lo, hi))
    assert len(got) == (1 if res else 0)
    return f"{int(op == 'add')} {t} {len(res)} {nruns}", (got[0][1:] if got else None)


def test_range_type_probe_pinned_to_reference(R):
    cases = _cases(R)
    args = [_probe_arg(R, *c[1:]) for c in cases]
    r = run_probe(PROBE, *[a for a, _ in args])
    assert r.returncode == 0, r.stdout + r.stderr
    lines = r.stdout.split()
    assert len(lines) == len(cases)
    by = {}
    for (name, *_), (arg, ref), line in zip(cases, args, lines):
        t = int(line)
        assert t == (ref[0] if ref else 0), (name, arg, t, ref)
        by[name] = ref
    # the edges are there: the 2048-run container stays a run, 2049 runs do not; an untouched run container
    # is converted all the same; a new key is an array for one value only (container_range_of_ones gets an
    # exclusive end and counts it)
    assert by["run 2047 + a disjoint range"] == (T_RUN, 6144, 2048)
    assert by["run 2048 + a disjoint range"][0] == T_BITSET
    assert by["run - a range that touches no value"][0] == T_BITSET
    assert by["array 4096 + 1 value"][0] == T_BITSET and by["bitset 4097 - 1 value"][0] == T_ARRAY
    assert [by[f"absent key + {k} value{'s' * (k > 1)}"][0] for k in (1, 2, 3)] == [T_ARRAY, T_RUN, T_RUN]
    assert by["full key removed from a run"] is None
    for name in ("full key from an array", "full key from a bitset", "full key from a run"):
        assert by[name] == (T_RUN, 65536, 1), name


ENTRIES = [("rb200_batch_add_range_closed", "add_range_closed", C.c_uint32),
           ("rb200_batch_remove_range_closed", "remove_range_closed", C.c_uint32),
           ("rb200_set64_batch_add_range_closed", "set64_add_range_closed", C.c_uint64),
           ("rb200_set64_batch_remove_range_closed", "set64_remove_range_closed", C.c_uint64)]


def test_argument_errors_before_any_device():
    L = api.lib()
    for name, what, ct in ENTRIES:
        f = getattr(L, name)
        lo, hi = (ct * 1)(0), (ct * 1)(5)
        assert not f(None, None, 0, C.cast(lo, C.c_void_p), C.cast(hi, C.c_void_p))
        assert api.last_error() == f"{what}: S is NULL", name
        one = (C.c_uint32 * 1)(0)
        assert not f(None, C.cast(one, C.c_void_p), 1, None, C.cast(hi, C.c_void_p))
        assert api.last_error() == f"{what}: min / max is NULL", name
        assert not f(None, C.cast(one, C.c_void_p), 1, C.cast(lo, C.c_void_p), None)
        assert api.last_error() == f"{what}: min / max is NULL", name
    # an add whose range keys alone exceed 2^32 - 1 item slots: 65537 full 32-bit ranges, or one 64-bit
    # range over the whole space (2^48 keys)
    n = 65537
    idx = np.zeros(n, np.uint32)
    lo32, hi32 = np.zeros(n, np.uint32), np.full(n, 0xFFFFFFFF, np.uint32)
    assert not L.rb200_batch_add_range_closed(None, idx.ctypes.data, n, lo32.ctypes.data, hi32.ctypes.data)
    assert api.last_error() == "add_range_closed: batch too large: more than 2^32 - 1 container slots, split it"
    lo64, hi64 = np.zeros(1, np.uint64), np.full(1, 2**64 - 1, np.uint64)
    assert not L.rb200_set64_batch_add_range_closed(None, idx.ctypes.data, 1, lo64.ctypes.data, hi64.ctypes.data)
    assert api.last_error() == "set64_add_range_closed: batch too large: more than 2^32 - 1 container slots, split it"
    # 65535 full 32-bit ranges fit (2^32 - 2^16 slots before the containers), and a removal has no range slots
    assert not L.rb200_batch_add_range_closed(None, idx.ctypes.data, n - 2, lo32.ctypes.data, hi32.ctypes.data)
    assert api.last_error() == "add_range_closed: S is NULL"
    assert not L.rb200_batch_remove_range_closed(None, idx.ctypes.data, n, lo32.ctypes.data, hi32.ctypes.data)
    assert api.last_error() == "remove_range_closed: S is NULL"


class _Stub:
    """A stand-in set for the mirror's argument checks, which run before any library call."""
    def __init__(self, cls, n):
        self.ptr, self._n = None, n
        self._width = cls._width

    def __len__(self):
        return self._n


def test_mirror_argument_errors():
    for cls in (api.DeviceSet, api.DeviceSet64):
        s = _Stub(cls, 2)
        with pytest.raises(api.RB200Error, match="start has 3 entries for 2 items"):
            api._range_update(s, "rb200_batch_add_range_closed", [1, 2, 3], 10, None)
        with pytest.raises(api.RB200Error, match="end has 2 entries for 1 items"):
            api._range_update(s, "rb200_batch_add_range_closed", 0, [5, 6], [1])
        with pytest.raises(api.RB200Error, match="start must lie in"):
            api._range_update(s, "rb200_batch_add_range_closed", -1, 10, None)
        with pytest.raises(api.RB200Error, match="end must lie in"):
            api._range_update(s, "rb200_batch_add_range_closed", 0, 2**65, None)
        with pytest.raises(api.RB200Error, match="must be integers"):
            api._range_update(s, "rb200_batch_add_range_closed", 0.5, 10, None)
        with pytest.raises(api.RB200Error, match="1-D integer sequence"):
            api._range_update(s, "rb200_batch_add_range_closed", np.zeros((2, 1), np.int64), 10, None)
    # 64-bit ends reach 2^64, 32-bit ones stop at 2^64 - 1 (the wrapper's uint64_t)
    assert api._closed_ranges(0, 2**64, 1, 64)[1][0] == 2**64 - 1
    with pytest.raises(api.RB200Error, match="end must lie in"):
        api._closed_ranges(0, 2**64, 1, 32)


def test_open_to_closed_matches_the_reference_wrappers(R):
    """_closed_ranges against roaring_bitmap_add_range / remove_range themselves (the reference's inline
    wrappers, exported by its library): the closed range it gives, applied with the closed function, leaves
    the same bytes, no-ops and 32-bit truncation included."""
    L = R.L
    for op in ("add", "remove"):
        w = getattr(L, f"roaring_bitmap_{op}_range")
        w.restype = None
        w.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
    base = _blob(R, np.concatenate([np.arange(0, 70000, 3), [0xFFFFFFF0, 0xFFFFFFFF]]), True)
    T = 1 << 32
    pairs = [(0, 0), (5, 5), (6, 5), (0, 1), (10, 100000), (65535, 65537), (0, T), (T - 1, T), (T, T + 5),
             (T + 1, T + 10), (T - 5, T + 7), (3, T + 9), (T + 3, 2 * T + 9), (2**64 - 2, 2**64 - 1), (7, 2**64 - 1)]
    mins, maxs = api._closed_ranges([a for a, _ in pairs], [b for _, b in pairs], len(pairs), 32)
    for (a, b), lo, hi in zip(pairs, mins.tolist(), maxs.tolist()):
        for op in ("add", "remove"):
            r = R.deserialize(base)
            getattr(L, f"roaring_bitmap_{op}_range")(r, a, b)
            want = R.serialize(r)
            R.free(r)
            got = ref_range_bytes(R, op, base, lo, hi) if lo <= hi else base
            assert got == want, (op, a, b, lo, hi)
    # the truncation itself: [2^32, 2^32 + 5) is the closed [0, 4], [3, 2^32 + 9) is [3, 8]
    assert (mins[8], maxs[8]) == (0, 4) and (mins[11], maxs[11]) == (3, 8)
    assert mins[9] > maxs[9] and mins[12] > maxs[12]   # start past 2^32: a no-op
    # 64-bit: a no-op when start >= end, else [start, end - 1]
    m64, x64 = api._closed_ranges([5, 5, 0, 2**64 - 1], [5, 4, 2**64, 2**64], 4, 64)
    assert m64[0] > x64[0] and m64[1] > x64[1]
    assert (int(m64[2]), int(x64[2])) == (0, 2**64 - 1) and (int(m64[3]), int(x64[3])) == (2**64 - 1, 2**64 - 1)
