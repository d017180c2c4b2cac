"""GPU parity with copy-on-write (COW) inputs: every entry point fed bitmaps in the four states of
cow_oracles (plain, cow, cow-copy, shared-off) must give the reference's bytes and COW flag, leave
results the reference validates and frees, and leave its inputs as they were (DESIGN.md §2)."""
import ctypes as C
import math
import types

import numpy as np
import pytest

import synth
from cow_oracles import STATES, bind, containers, cow_of, fingerprint, make

# The sweeps take the states the reference accepts as inputs everywhere: its own or_many faults on
# a shared-off input (SHARED containers under a cleared flag), which the named cases still cover.
SWEEP_STATES = ("plain", "cow", "cow-copy")
from test_cow_host import named_blobs

pytestmark = pytest.mark.gpu

OPS = ("and", "or", "xor", "andnot")
FLIP = (3 * 65536 + 5, 5 * 65536 + 17)


@pytest.fixture(scope="module")
def Rc(R):
    return bind(R)


def _ptrs(ps):
    return [types.SimpleNamespace(ptr=p) for p in ps]


def _result(R, p, what, check=True):
    """(bytes, flag) of a result, which the reference validates (check), then frees.  The reference's
    own results are not always checked: its in-place twins put SHARED containers of a COW x2 into a
    plain x1, which its validator refuses."""
    ok, why = R.validate(p)
    assert ok or not check, (what, why)
    out = (R.serialize(p), cow_of(R, p))
    R.free(p)
    return out


def _blob(R, vals, run_optimize=True):
    r = R.from_values(np.asarray(vals, np.uint32), run_optimize=run_optimize)
    b = R.serialize(r)
    R.free(r)
    return b


# ------------------------------------------------------------------ 1. the named cases
def test_named_lazy_xor_inplace_shared_left(rb, Rc):
    R, L = Rc, rb.lib()
    run, inside, _ = named_blobs(R)
    for state in STATES:
        outs = []
        for lib in (R.L, L):
            x, y = make(R, run, state), R.deserialize(inside)
            fy = fingerprint(R, y)
            lib.roaring_bitmap_lazy_xor_inplace(x, y)
            lib.roaring_bitmap_repair_after_lazy(x)
            assert fingerprint(R, y) == fy
            R.free(y)
            outs.append(_result(R, x, state, lib is L))
        assert outs[0] == outs[1], state
    # through the resident API: an uploaded cow-copy, a lazy in-place batch, then repair
    for state in ("cow-copy", "plain"):
        x, y = make(R, run, state), R.deserialize(inside)
        fx = fingerprint(R, x)
        S = rb.DeviceSet.upload(_ptrs([x, y]))
        one = lambda v: np.array([v], np.uint32)
        got = S.batch("xor", S, one(0), one(1), inplace_rules=True, lazy=True).repair_after_lazy().download(0)
        assert fingerprint(R, x) == fx
        R.L.roaring_bitmap_lazy_xor_inplace(x, y)
        R.L.roaring_bitmap_repair_after_lazy(x)
        ref = R.serialize(x)
        assert got.serialize() == ref, state
        assert containers(got.ptr)[0][1] == (3 if state == "cow-copy" else 1), state
        for p in (x, y):
            R.free(p)


def test_named_xor_many_cow_input(rb, Rc):
    R, L = Rc, rb.lib()
    run, inside, five = named_blobs(R)
    blobs = [run, five, inside]
    for state in STATES:
        states = [state, "plain", "plain"]
        outs = []
        for lib in (R.L, L):
            xs = [make(R, b, s) for b, s in zip(blobs, states)]
            fps = [fingerprint(R, x) for x in xs] if lib is L else None
            arr = (C.c_void_p * 3)(*xs)
            r = lib.roaring_bitmap_xor_many(3, arr)
            if fps:
                assert [fingerprint(R, x) for x in xs] == fps
            outs.append(_result(R, r, state, lib is L))
            for x in xs:
                R.free(x)
        assert outs[0] == outs[1], state
        # the resident fold over the same host objects
        xs = [make(R, b, s) for b, s in zip(blobs, states)]
        got = rb.DeviceSet.upload(_ptrs(xs)).xor_many().download(0)
        assert (got.serialize(), cow_of(R, got.ptr)) == outs[0], state
        for x in xs:
            R.free(x)


# ------------------------------------------------------------------ 2. the folds
def _pool(R, rng, n):
    run, inside, five = named_blobs(R)
    blobs = [run, inside, five, _blob(R, [])]
    for i in range(n):
        v = synth.random_bitmap(rng, n_keys=int(rng.integers(0, 6)), key_space=6)
        blobs.append(_blob(R, v, bool(i % 2)))
    return blobs


def test_fold_sweep(rb, Rc):
    R, L = Rc, rb.lib()
    rng = np.random.default_rng(2024)
    blobs = _pool(R, rng, 24)
    seen_cow_bytes = 0
    for trial in range(90):
        n = int(rng.integers(0, 10))
        pick = [int(i) for i in rng.integers(0, len(blobs), n)]
        if n >= 3 and trial % 3 == 0:        # x ^ x somewhere in the fold
            j = int(rng.integers(1, n))
            pick[j] = pick[j - 1]
        if n and trial % 4 == 0:             # the named rule: a COW run cloned, then the values inside it
            pick[0], pick[-1] = 0, 1
        states = [SWEEP_STATES[int(s)] for s in rng.integers(0, 3, n)]
        for name in ("or_many", "xor_many", "or_many_heap"):
            outs = []
            for lib in (R.L, L):
                xs = [make(R, blobs[i], s) for i, s in zip(pick, states)]
                fps = [fingerprint(R, x) for x in xs] if lib is L else None
                r = getattr(lib, f"roaring_bitmap_{name}")(n, (C.c_void_p * max(n, 1))(*xs))
                if fps:
                    assert [fingerprint(R, x) for x in xs] == fps, (name, trial)
                outs.append(_result(R, r, (name, trial), lib is L))
                for x in xs:
                    R.free(x)
            assert outs[0] == outs[1], (name, trial, pick, states)
            # the resident fold: the distinct inputs uploaded once, the fold selects them by index
            uniq = sorted(set(zip(pick, states)))
            xs = [make(R, blobs[i], s) for i, s in uniq]
            idx = [uniq.index(p) for p in zip(pick, states)]
            S = rb.DeviceSet.upload(_ptrs(xs))
            got = getattr(S, name)(np.array(idx, np.uint32)).download(0)
            assert (got.serialize(), cow_of(R, got.ptr)) == outs[0], (name, trial, "resident")
            ok, why = R.validate(got.ptr)
            assert ok, why
            del got, S
            for x in xs:
                R.free(x)
            if name == "xor_many":
                plain = R.many_bytes("xor_many", [blobs[i] for i in pick]) if n else outs[0][0]
                seen_cow_bytes += plain != outs[0][0]
    assert seen_cow_bytes >= 3    # the sweep reaches the SHARED-accumulator rule


# ------------------------------------------------------------------ 3. pairwise entry points
def _big(R, seed):
    """More than 512 containers: a pair of these takes the batched path, not the single launch."""
    rng = np.random.default_rng(seed)
    keys = np.arange(600)
    v = (keys[:, None].astype(np.uint32) << 16) | rng.integers(0, 65536, (600, 3)).astype(np.uint32)
    return _blob(R, np.unique(v), False)


def _call(R, lib, entry, x, y):
    """Run `entry` on (x, y); returns what to compare: (bytes, flag) of a result, x's after an in-place
    call, or a number.  Results of our symbols must pass the reference's validator."""
    check = lib is not R.L
    if entry in OPS or entry in ("lazy_xor",) or entry.startswith("lazy_or:"):
        if entry.startswith("lazy_or:"):
            r = lib.roaring_bitmap_lazy_or(x, y, entry.endswith("1"))
        else:
            r = getattr(lib, f"roaring_bitmap_{entry}")(x, y)
        if entry.startswith("lazy"):
            lib.roaring_bitmap_repair_after_lazy(r)
        return _result(R, r, entry, check)
    if entry == "flip_inplace":
        lib.roaring_bitmap_flip_inplace(x, *FLIP)
        return R.serialize(x), cow_of(R, x)
    if entry.endswith("_inplace") or entry.startswith("lazy_or_inplace"):
        if entry.startswith("lazy_or_inplace:"):
            lib.roaring_bitmap_lazy_or_inplace(x, y, entry.endswith("1"))
        else:
            getattr(lib, f"roaring_bitmap_{entry}")(x, y)
        if entry.startswith("lazy"):
            lib.roaring_bitmap_repair_after_lazy(x)
        ok, why = R.validate(x)
        assert ok or not check, (entry, why)
        return R.serialize(x), cow_of(R, x)
    if entry == "repair_after_lazy":
        lib.roaring_bitmap_repair_after_lazy(x)
        return R.serialize(x), cow_of(R, x)
    if entry == "flip":
        return _result(R, lib.roaring_bitmap_flip(x, *FLIP), entry, check)
    v = getattr(lib, f"roaring_bitmap_{entry}")(x, y)
    return "nan" if isinstance(v, float) and math.isnan(v) else v


ENTRIES = (OPS + tuple(f"{op}_inplace" for op in OPS) +
           ("lazy_or:0", "lazy_or:1", "lazy_xor", "lazy_or_inplace:0", "lazy_or_inplace:1", "lazy_xor_inplace",
            "repair_after_lazy", "flip", "flip_inplace") +
           tuple(f"{op}_cardinality" for op in OPS) + ("jaccard_index", "intersect", "equals", "is_subset",
                                                       "is_strict_subset"))


@pytest.mark.parametrize("size", ["small", "batched"])
def test_pairwise_states(rb, Rc, size):
    R, L = Rc, rb.lib()
    run, inside, _ = named_blobs(R)
    if size == "small":
        a, b = run, _blob(R, np.concatenate([np.arange(0, 12000, 7), np.arange(1 << 16, (1 << 16) + 300)]))
    else:
        a, b = _big(R, 1), _big(R, 2)
    empty = _blob(R, [])
    fails = []
    combos = [(sa, ea, sb, eb) for sa in SWEEP_STATES for ea in (0, 1) for sb in SWEEP_STATES for eb in (0, 1)]
    for entry in ENTRIES:
        for sa, ea, sb, eb in combos:
            outs = []
            for lib in (R.L, L):
                x, y = make(R, a if ea else empty, sa), make(R, b if eb else empty, sb)
                keep = [y] if ("inplace" in entry or entry == "repair_after_lazy") else [x, y]
                fps = [fingerprint(R, p) for p in keep] if lib is L else None
                outs.append(_call(R, lib, entry, x, y))
                if fps:
                    assert [fingerprint(R, p) for p in keep] == fps, (entry, sa, ea, sb, eb)
                R.free(x)
                R.free(y)
            if outs[0] != outs[1]:
                fails.append((entry, sa, ea, sb, eb, outs[0][1:] if isinstance(outs[0], tuple) else outs[0],
                              outs[1][1:] if isinstance(outs[1], tuple) else outs[1]))
    assert not fails, fails[:12]


def test_batch_results_per_pair(rb, Rc):
    """rb200_batch_op_host and DeviceSet.upload + batch + download: the flag of every pair."""
    R = Rc
    run, _, _ = named_blobs(R)
    b = _blob(R, np.concatenate([np.arange(0, 12000, 7), np.arange(1 << 16, (1 << 16) + 300)]))
    empty = _blob(R, [])
    combos = [(sa, ea, sb, eb) for sa in SWEEP_STATES for ea in (0, 1) for sb in SWEEP_STATES for eb in (0, 1)]
    xs = [make(R, run if ea else empty, sa) for sa, ea, _, _ in combos]
    ys = [make(R, b if eb else empty, sb) for _, _, sb, eb in combos]
    S = rb.DeviceSet.upload(_ptrs(xs + ys))
    ia = np.arange(len(combos), dtype=np.uint32)
    for op in OPS:
        exp = []
        for c in combos:
            x, y = make(R, run if c[1] else empty, c[0]), make(R, b if c[3] else empty, c[2])
            exp.append(_result(R, getattr(R.L, f"roaring_bitmap_{op}")(x, y), op, False))
            R.free(x)
            R.free(y)
        host = rb.batch_op_host(op, _ptrs(xs), _ptrs(ys))
        res = S.batch(op, S, ia, ia + len(combos))
        for k, c in enumerate(combos):
            got = res.download(k)
            assert (got.serialize(), cow_of(R, got.ptr)) == exp[k], (op, c, "resident")
            assert (host[k].serialize(), cow_of(R, host[k].ptr)) == exp[k], (op, c, "batch_op_host")
    for p in xs + ys:
        R.free(p)


# ------------------------------------------------------------------ 4. resident results that keep S's flag
def test_resident_flags_follow_S(rb, Rc):
    R = Rc
    rng = np.random.default_rng(8)
    blobs = [_blob(R, synth.random_bitmap(rng, n_keys=3, key_space=5), bool(i % 2)) for i in range(6)] + [_blob(R, [])]
    states = [SWEEP_STATES[i % 3] for i in range(len(blobs))]
    xs = [make(R, bl, s) for bl, s in zip(blobs, states)]
    fps = [fingerprint(R, x) for x in xs]
    S = rb.DeviceSet.upload(_ptrs(xs))
    vals = [np.array([7, 70000, 200000], np.uint32)] * len(blobs)
    got = {"offset": S.add_offset(12345), "offset_aligned": S.add_offset(1 << 16), "add": S.add_many(vals),
           "remove": S.remove_many(vals), "flip": S.flip(*FLIP)}
    assert [fingerprint(R, x) for x in xs] == fps
    for k, (bl, s) in enumerate(zip(blobs, states)):
        for what, res in got.items():
            x = make(R, bl, s)
            v = vals[k]
            if what.startswith("offset"):
                r = R.L.roaring_bitmap_add_offset(x, 12345 if what == "offset" else 1 << 16)
            elif what == "flip":
                r = R.L.roaring_bitmap_flip(x, *FLIP)
            else:
                # the update of a bitmap keeps its flag; it runs on own containers here, since the
                # reference's remove_many corrupts the heap on SHARED ones
                r = R.deserialize(bl)
                fn = R.L.roaring_bitmap_add_many if what == "add" else R.L.roaring_bitmap_remove_many
                fn(r, v.size, v.ctypes.data)
                R.L.roaring_bitmap_set_copy_on_write(r, cow_of(R, x))
            exp = _result(R, r, what, False)
            R.free(x)
            g = res.download(k)
            assert (g.serialize(), cow_of(R, g.ptr)) == exp, (what, k, s)
    for x in xs:
        R.free(x)
