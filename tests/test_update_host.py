"""CPU checks of roaring_bitmap_add_many / remove_many on the device path's terms (-m "not gpu"): the type
rule and slot bound of rb200_device.cuh (decide_type_keep_run, slot_bound_keep_run) through a
host-compiled probe, each probe case pinned against the reference's own update of the same container,
and the argument errors the C ABI and the Python mirror report before any device is needed."""
import ctypes as C
import struct

import numpy as np
import pytest

from croaring_b200 import api
from helpers import run_probe
from update_oracles import ref_update_bytes

T_BITSET, T_ARRAY, T_RUN = 1, 2, 3
OP_OR, OP_ANDNOT = 1, 3

PROBE = r'''
#include "rb200_device.cuh"
#include <cstdio>
#include <cstdlib>
using namespace rb200;
// argv: cases "op tA tB cA cB lA lB card nruns"; prints "type slot" per case, slot = the bound k_plan_pairs
// reserves under RULES_KEEP_RUN
int main(int argc, char **argv) {
    for (int i = 1; i < argc; i++) {
        int op, tA, tB, card, nruns;
        unsigned cA, cB, lA, lB;
        if (sscanf(argv[i], "%d %d %d %u %u %u %u %d %d", &op, &tA, &tB, &cA, &cB, &lA, &lB, &card, &nruns) != 9) return 2;
        const int t = decide_type_keep_run(true, op, tA, tB, cA, cB, lA, lB, card, nruns);
        const unsigned slot = tA == T_RUN ? slot_bound_keep_run(lA, cB) : slot_bound(op, tA, tB, cA, cB, lA, lB);
        printf("%d %u\n", t, slot);
    }
    // the rule is off: every cell is the op's own
    if (decide_type_keep_run(false, OP_OR, T_RUN, T_BITSET, 1000, 5000, 1, 1024, 6000, 2) != T_BITSET) return 3;
    if (decide_type_keep_run(false, OP_ANDNOT, T_RUN, T_ARRAY, 65536, 1, 1, 1, 65535, 2) != T_BITSET) return 4;
    // the bound: never below what a run result can hold, 128 KiB at most
    if (slot_bound_keep_run(32768, 65536) != 131072u || slot_bound_keep_run(1, 32767) != 131072u) return 5;
    if (slot_bound_keep_run(3, 1) != 16u || slot_bound_keep_run(1, 4097) != 16400u) return 6;
    return 0;
}
'''


def containers(blob):
    """(key, type, card, len) of every container of a portable blob, read from its bytes."""
    cookie = struct.unpack_from("<I", blob, 0)[0]
    if cookie & 0xFFFF == 12347:
        n = (cookie >> 16) + 1
        runbits = blob[4:4 + (n + 7) // 8]
        pos = 4 + (n + 7) // 8
        isrun = [(runbits[i // 8] >> (i % 8)) & 1 for i in range(n)]
        has_offsets = n >= 4
    else:
        assert cookie == 12346
        n = struct.unpack_from("<I", blob, 4)[0]
        pos, isrun, has_offsets = 8, [0] * n, True
    hdr = [struct.unpack_from("<HH", blob, pos + 4 * i) for i in range(n)]
    pos += 4 * n + (4 * n if has_offsets else 0)
    out = []
    for i, (key, c1) in enumerate(hdr):
        card = c1 + 1
        if isrun[i]:
            nr = struct.unpack_from("<H", blob, pos)[0]
            out.append((key, T_RUN, card, nr))
            pos += 2 + 4 * nr
        elif card > 4096:
            out.append((key, T_BITSET, card, 1024))
            pos += 8192
        else:
            out.append((key, T_ARRAY, card, card))
            pos += 2 * card
    assert pos == len(blob)
    return out


def _runs(vals):
    v = np.unique(np.asarray(vals, dtype=np.int64))
    return int(v.size and 1 + np.count_nonzero(np.diff(v) != 1))


FULL = np.arange(65536)
# (name, values of the one container S holds, run-optimized, op, values added / removed)
CASES = [
    ("array 4096 + a new value", np.arange(0, 8192, 2), False, "add", [1]),
    ("array 4096 + a present value", np.arange(0, 8192, 2), False, "add", [2]),
    ("array 4095 + a new value", np.arange(0, 8190, 2), False, "add", [1]),
    ("bitset 4097 - a value", np.arange(0, 8194, 2), False, "remove", [4]),
    ("bitset 4098 - a value", np.arange(0, 8196, 2), False, "remove", [4]),
    ("bitset 4097 - an absent value", np.arange(0, 8194, 2), False, "remove", [5]),
    ("bitset 4097 + 5000 values", np.arange(0, 8194, 2), False, "add", np.arange(20000, 30000, 2)),
    ("array - 5000 values", np.arange(0, 4000, 2), False, "remove", np.arange(0, 10000, 2)),
    ("full run + a present value", FULL, True, "add", [100]),
    ("full run - a value", FULL, True, "remove", [100]),
    ("full run - its first value", FULL, True, "remove", [0]),
    ("run + 4097 values", np.arange(0, 1000), True, "add", np.arange(2000, 2000 + 2 * 4097, 2)),
    ("run - 4097 values", np.arange(0, 20000), True, "remove", np.arange(1, 8195, 2)),
    ("run + a neighbour", np.arange(10, 100), True, "add", [9, 100, 500]),
    ("run - every value", np.arange(10, 100), True, "remove", np.arange(0, 200)),
    ("full run - every odd value", FULL, True, "remove", np.arange(1, 65536, 2)),
    ("run + every other value", np.array([0]), True, "add", np.arange(2, 65536, 2)),
]


def _case(R, vals, run_opt, op, upd):
    """(probe argument, reference result's (type, card, len) or None when the container is dropped)."""
    r = R.from_values(np.asarray(vals, np.uint32), run_optimize=run_opt)
    blob = R.serialize(r)
    R.free(r)
    (_, tA, cA, lA), = containers(blob)
    v = R.from_values(np.asarray(upd, np.uint32), run_optimize=False)   # V: roaring_bitmap_of_ptr
    (_, tB, cB, lB), = containers(R.serialize(v))
    R.free(v)
    got = containers(ref_update_bytes(R, op, blob, upd))
    s, u = set(np.asarray(vals).tolist()), set(np.asarray(upd).tolist())
    res = sorted(s | u if op == "add" else s - u)
    code = OP_OR if op == "add" else OP_ANDNOT
    arg = f"{code} {tA} {tB} {cA} {cB} {lA} {lB} {len(res)} {_runs(res)}"
    assert len(got) == (1 if res else 0)
    return arg, (got[0][1:] if got else None)


def test_type_rule_probe_pinned_to_reference(R):
    cases = [_case(R, *c[1:]) for c in CASES]
    r = run_probe(PROBE, *[a for a, _ in cases])
    assert r.returncode == 0, r.stdout + r.stderr
    for (name, *_), (arg, ref), line in zip(CASES, cases, r.stdout.split("\n")):
        t, slot = map(int, line.split())
        if ref is None:   # emptied: dropped whatever the rule says
            continue
        rt, rcard, rlen = ref
        assert t == rt, (name, arg, t, ref)
        stored = 8192 if rt == T_BITSET else (2 * rlen if rt == T_ARRAY else 4 * rlen)
        assert stored <= slot, (name, stored, slot)
    # the edges the issue names are there: a run past 8 KiB, the 32768-run result
    by = {c[0]: ref for c, (_, ref) in zip(CASES, cases)}
    assert by["full run - every odd value"] == (T_RUN, 32768, 32768)
    assert by["run + 4097 values"][0] == T_RUN and by["run + 4097 values"][2] == 4098
    assert by["array 4096 + a new value"][0] == T_BITSET and by["bitset 4097 - a value"][0] == T_ARRAY


class _Stub:
    """A stand-in set for the mirror's argument checks, which run before any library call."""
    def __init__(self, cls, n):
        self.ptr, self._n, self._cls = None, n, cls
        self._host_values = cls._host_values

    def __len__(self):
        return self._n


def test_argument_errors_before_any_device():
    L = api.lib()
    off = (C.c_uint64 * 2)(0, 1)
    for name in ("rb200_batch_add_many", "rb200_batch_remove_many", "rb200_batch_add_many_device",
                 "rb200_batch_remove_many_device", "rb200_set64_batch_add_many", "rb200_set64_batch_remove_many",
                 "rb200_set64_batch_add_many_device", "rb200_set64_batch_remove_many_device"):
        assert not getattr(L, name)(None, None, 1, None, C.cast(off, C.c_void_p))
        what = name.replace("rb200_batch_", "").replace("rb200_set64_batch_", "set64_")
        assert api.last_error() == f"{what}: S is NULL", name
    for cls, fn in ((api.DeviceSet, "rb200_batch_add_many"), (api.DeviceSet64, "rb200_set64_batch_remove_many")):
        s = _Stub(cls, 2)
        with pytest.raises(api.RB200Error, match="3 lists of values for 2 items"):
            api._update(s, fn, [[1], [2], [3]], None, None)
        with pytest.raises(api.RB200Error, match="2 lists of values for 1 items"):
            api._update(s, fn, [[1], [2]], None, [1])   # one selected item, two lists
        with pytest.raises(api.RB200Error, match="must lie in"):
            api._update(s, fn, [[-1], [2]], None, None)
        with pytest.raises(api.RB200Error, match="ending at most"):
            api._update(s, fn, np.arange(3), [0, 2, 9], None)
        with pytest.raises(api.RB200Error, match="integer"):
            api._update(s, fn, [np.array([0.5]), [1]], None, None)
