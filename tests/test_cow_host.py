"""CPU checks of copy-on-write (COW) inputs (-m "not gpu"), pinned against the reference: the two
cases where a SHARED container changes the reference's container types, the COW flag model of
cow_oracles.expected_cow, and the xor_many step rule of rb200_device.cuh (xor_many_step_type) through
a host-compiled probe.  The GPU parity tests of test_gpu_cow.py rely on all three."""
import itertools

import numpy as np
import pytest

from cow_oracles import (FOLDS, INPLACE, PAIRWISE, T_ARRAY, T_BITSET, T_RUN, bind, containers, cow_of,
                         expected_cow, make)
from helpers import run_probe

RUN10K = np.arange(10000, dtype=np.uint32)            # key 0: one run [0, 10000)
INSIDE = (np.arange(101) * 97 + 13).astype(np.uint32)  # key 0: 101 values inside that run
FIVE = (np.arange(5) * 3 + (1 << 16)).astype(np.uint32)


@pytest.fixture(scope="module")
def Rc(R):
    return bind(R)


def _blob(R, vals, run_optimize):
    r = R.from_values(vals, run_optimize=run_optimize)
    b = R.serialize(r)
    R.free(r)
    return b


def named_blobs(R):
    """(run [0, 10000), 101 values inside it, 5 values in key 1) as portable bytes."""
    return _blob(R, RUN10K, True), _blob(R, INSIDE, False), _blob(R, FIVE, False)


def ref_lazy_xor_inplace(R, x_blob, x_state, y_blob):
    """lazy_xor_inplace(x, y) then repair_after_lazy(x) in the reference: (bytes, containers, flag)."""
    x, y = make(R, x_blob, x_state), R.deserialize(y_blob)
    R.L.roaring_bitmap_lazy_xor_inplace(x, y)
    R.L.roaring_bitmap_repair_after_lazy(x)
    ok, why = R.validate(x)
    assert ok, why
    out = (R.serialize(x), containers(x), cow_of(R, x))
    R.free(x)
    R.free(y)
    return out


def ref_many(R, name, blobs, states):
    rs = [make(R, b, s) for b, s in zip(blobs, states)]
    r = R.many(name, rs)
    ok, why = R.validate(r)
    assert ok, why
    out = (R.serialize(r), containers(r), cow_of(R, r))
    for x in rs + [r]:
        R.free(x)
    return out


def test_named_type_cases(Rc):
    R = Rc
    run, inside, five = named_blobs(R)
    # 1. lazy_xor_inplace: a SHARED left run stays a run; an own one becomes a bitset
    for state, t in (("cow-copy", T_RUN), ("shared-off", T_RUN), ("plain", T_BITSET), ("cow", T_BITSET)):
        _, cs, _ = ref_lazy_xor_inplace(R, run, state, inside)
        assert [c[:2] for c in cs] == [(0, t)], state
    # 2. xor_many(R, O, Y): key 0 enters the accumulator SHARED from a COW R
    for state, t in (("cow", T_RUN), ("cow-copy", T_RUN), ("plain", T_BITSET), ("shared-off", T_BITSET)):
        _, cs, _ = ref_many(R, "xor_many", [run, five, inside], [state, "plain", "plain"])
        assert [c[:2] for c in cs] == [(0, t), (1, T_ARRAY)], state


# ------------------------------------------------------------------ the COW flag model
def _values(i, pattern):
    """Values of non-empty input i: its own (distinct) or the same for every input (x ^ x cancels)."""
    if pattern == "same":
        return np.arange(4, dtype=np.uint32) * 7
    k = (i * 5) % 7 + 1    # sizes in a varying order, with ties
    return (np.arange(k, dtype=np.uint32) * 11 + i * 1000 + (i % 2) * 65536).astype(np.uint32)


def _ref_flag(R, entry, inputs):
    """The reference's COW flag on the result of `entry` over inputs [(values, cow)]."""
    rs = []
    for v, c in inputs:
        r = R.from_values(v, run_optimize=False)
        R.L.roaring_bitmap_set_copy_on_write(r, c)
        rs.append(r)
    L = R.L
    if entry in FOLDS:
        out = R.many(entry, rs)
    elif entry in INPLACE:
        op = entry[:-len("_inplace")]
        if op == "lazy_or":
            L.roaring_bitmap_lazy_or_inplace(rs[0], rs[1], False)
        else:
            getattr(L, f"roaring_bitmap_{entry}")(rs[0], rs[1])
        out = rs[0]
    elif entry == "lazy_or":
        out = L.roaring_bitmap_lazy_or(rs[0], rs[1], False)
    else:
        out = getattr(L, f"roaring_bitmap_{entry}")(rs[0], rs[1])
    f = cow_of(R, out)
    if out not in rs:
        R.free(out)
    for r in rs:
        R.free(r)
    return f


def test_flag_model_pairwise(Rc):
    for entry in PAIRWISE + INPLACE:
        for pattern in ("distinct", "same"):
            for (ea, ca), (eb, cb) in itertools.product(itertools.product((0, 1), (False, True)), repeat=2):
                inputs = [(_values(0, pattern) if ea else np.zeros(0, np.uint32), ca),
                          (_values(1, pattern) if eb else np.zeros(0, np.uint32), cb)]
                assert expected_cow(entry, inputs) == _ref_flag(Rc, entry, inputs), (entry, pattern, ea, ca, eb, cb)


def test_flag_model_folds_exhaustive(Rc):
    """n <= 4 inputs, every combination of empty / non-empty and cow / plain, distinct values and
    repeated ones (x ^ x cancellations)."""
    seen = {e: set() for e in FOLDS}
    for n in range(0, 5):
        for combo in itertools.product(itertools.product((0, 1), (False, True)), repeat=n):
            for pattern in ("distinct", "same"):
                inputs = [(_values(i, pattern) if e else np.zeros(0, np.uint32), c) for i, (e, c) in enumerate(combo)]
                for entry in FOLDS:
                    exp = expected_cow(entry, inputs)
                    assert exp == _ref_flag(Rc, entry, inputs), (entry, pattern, combo)
                    seen[entry].add((exp, exp == any(c for _, c in combo)))
    # the model is not the OR of the inputs' flags, and the sweep shows it for every fold
    for entry in FOLDS:
        assert (True, True) in seen[entry] and (False, False) in seen[entry], entry


def test_flag_model_named(Rc):
    a, b = np.array([1, 2], np.uint32), np.array([70000], np.uint32)
    e = np.zeros(0, np.uint32)
    cases = [("or", [(e, True), (a, False)], False),
             ("or_many", [(a, False), (b, False), (a, True)], False),
             ("xor_many", [(a, False), (b, False), (a, True)], False),
             ("or_many_heap", [(a, False), (b, False), (np.arange(5, dtype=np.uint32), True)], False),
             ("xor_many", [(a, False), (a, False), (b, True)], True),
             ("xor_many", [(a, True), (a, True), (b, False)], False),
             ("or_inplace", [(e, False), (a, True)], True)]
    for entry, inputs, f in cases:
        assert expected_cow(entry, inputs) == f == _ref_flag(Rc, entry, inputs), entry


# ------------------------------------------------------------------ the xor_many step rule
PROBE = r'''
#include "rb200_device.cuh"
#include <cstdio>
using namespace rb200;
// argv: cases "lazy tA tB cA cB lA lB card nruns"; prints the accumulator's type after the step
int main(int argc, char **argv) {
    for (int i = 1; i < argc; i++) {
        int lazy, tA, tB, card, nruns;
        unsigned cA, cB, lA, lB;
        if (sscanf(argv[i], "%d %d %d %u %u %u %u %d %d", &lazy, &tA, &tB, &cA, &cB, &lA, &lB, &card, &nruns) != 9) return 2;
        printf("%d\n", xor_many_step_type(lazy != 0, tA, tB, cA, cB, lA, lB, card, nruns));
    }
    return 0;
}
'''


def _runs(v):
    v = np.unique(np.asarray(v, np.int64))
    return int(v.size and 1 + np.count_nonzero(np.diff(v) != 1))


def _operands(rng):
    """(values, run_optimize) of one-container operands at the edges the step rule reads: arrays
    around 32 values (array_run_container_xor's threshold), 512 / 1024 (the lazy array sum) and 4096;
    bitsets; runs short and long."""
    out = []
    for c in (1, 20, 31, 32, 33, 96, 97, 500, 512, 513, 1000, 3000, 4000, 4096):
        out.append((np.sort(rng.choice(65536, c, replace=False)), False))
    for c in (4097, 6000, 40000):
        out.append((np.sort(rng.choice(65536, c, replace=False)), False))
    out.append((np.arange(10000), True))
    out.append((np.arange(65536), True))
    out.append((np.concatenate([np.arange(s, s + 100) for s in range(0, 20000, 2000)]), True))
    out.append((np.concatenate([np.arange(s, s + 3) for s in range(0, 4000, 100)]), True))
    out.append((np.concatenate([np.arange(s, s + 2500) for s in (1000, 30000)]), True))
    return [(np.asarray(v, np.uint32), ro) for v, ro in out]


def _one(p):
    (key, t, shared), = containers(p)
    assert key == 0 and not shared
    return t


def _meta(t, v):
    card = len(v)
    return card, (1024 if t == T_BITSET else card if t == T_ARRAY else _runs(v))


def test_xor_many_step_rule_probe(Rc):
    """xor_many_step_type against the type the reference's lazy_xor (lazy), lazy_xor_inplace on an own
    accumulator (in place) and lazy_xor_inplace on a SHARED one (lazy) leave, for every pair of types."""
    R = Rc
    rng = np.random.default_rng(17)
    ops = _operands(rng)
    blobs = [_blob(R, v, ro) for v, ro in ops]
    args, ref = [], []
    for (va, _), ba in zip(ops, blobs):
        for (vb, _), bb in zip(ops, blobs):
            x, y = R.deserialize(ba), R.deserialize(bb)
            tA, tB = _one(x), _one(y)
            res = np.setxor1d(va.astype(np.int64), vb.astype(np.int64))
            R.free(x)
            R.free(y)
            if not res.size:
                continue
            cA, lA = _meta(tA, va)
            cB, lB = _meta(tB, vb)
            got = []
            for how in ("lazy_xor", "plain", "cow-copy"):
                x, y = make(R, ba, "plain" if how == "lazy_xor" else how), R.deserialize(bb)
                if how == "lazy_xor":
                    r = R.L.roaring_bitmap_lazy_xor(x, y)
                    got.append(_one(r))
                    R.free(r)
                else:
                    R.L.roaring_bitmap_lazy_xor_inplace(x, y)
                    got.append(_one(x))
                R.free(x)
                R.free(y)
            for lazy, t in ((1, got[0]), (0, got[1]), (1, got[2])):
                args.append(f"{lazy} {tA} {tB} {cA} {cB} {lA} {lB} {res.size} {_runs(res)}")
                ref.append(t)
    r = run_probe(PROBE, *args)
    assert r.returncode == 0, r.stdout + r.stderr
    out = [int(t) for t in r.stdout.split()]
    assert len(out) == len(ref)
    bad = [(a, o, t) for a, o, t in zip(args, out, ref) if o != t]
    assert not bad, bad[:10]
    # the cases reach both rules where they differ: a shared accumulator's type is not the in-place one
    assert sum(ref[i + 1] != ref[i + 2] for i in range(0, len(ref), 3)) >= 10
    # every pair of types was probed
    types = {tuple(map(int, a.split()[1:3])) for a in args}
    assert types == set(itertools.product((T_BITSET, T_ARRAY, T_RUN), repeat=2))
