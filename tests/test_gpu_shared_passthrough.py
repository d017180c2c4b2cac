"""GPU test: results of non-lazy batch ops share their operands' pass-through containers instead of
copying them.  A result keeps its operands' slabs alive: every operand and every link of a chain can
be freed before the result is downloaded, serialized, chained, run-optimized or used in a lazy or
in-place op, in any order, and the bytes stay those of the reference; the same for 64-bit sets.  A
fold that frees its previous accumulator runs in bounded device memory, and once everything is freed
no device memory is left outstanding."""
import ctypes as C
import hashlib
import itertools

import numpy as np
import pytest

from helpers import synth_blobs, synth_blobs64

pytestmark = pytest.mark.gpu


def _inputs(rb, R):
    # real data with many unmatched keys between neighbours (census1881), run-heavy data
    # (wikileaks) and synthetic mixes with every container type
    return (rb.load_realdata("census1881")[:10] + rb.load_realdata("wikileaks-noquotes")[:6]
            + synth_blobs(R, 2024, 8))


def _pairs(n):
    ia = np.arange(n - 1, dtype=np.uint32)
    return ia, ia + 1


def _exp_chain(R, ops, blobs):
    """expected bytes of pair k after applying ops[0] to (blobs[k], blobs[k+1]), then ops[1] with
    blobs[k+2], ... (one more operand per link)."""
    out = []
    for k in range(len(blobs) - len(ops)):
        x = blobs[k]
        for d, op in enumerate(ops):
            x = R.op_bytes(op, x, blobs[k + d + 1])
        out.append(x)
    return out


def _ser(S):
    return list(S.serialize_all())


def _run_optimize_bytes(R, blob):
    r = R.deserialize(blob)
    R.L.roaring_bitmap_run_optimize(r)
    out = R.serialize(r)
    R.free(r)
    return out


def _r64_run_optimize_bytes(R, blob):
    r = R.r64_deserialize(blob)
    R.L.roaring64_bitmap_run_optimize(r)
    out = R.r64_serialize(r)
    R.L.roaring64_bitmap_free(r)
    return out


def _scenario_free_parent_first(rb, R, blobs):
    n = len(blobs)
    ia, ib = _pairs(n)
    for op in ("or", "xor", "andnot"):
        exp = [R.op_bytes(op, blobs[k], blobs[k + 1]) for k in range(n - 1)]
        # download_all / download(i) / serialize_all of a child whose operand is gone
        for how in ("download_all", "download", "serialize"):
            S = rb.DeviceSet.from_serialized(blobs)
            res = S.batch(op, S, ia, ib)
            S.free()
            if how == "download_all":
                got = [b.serialize() for b in res.download_all()]
            elif how == "download":
                got = [res.download(k).serialize() for k in range(n - 1)]
            else:
                got = _ser(res)
            assert got == exp, (op, how)
            res.free()
        # chaining a child whose operand is gone
        S = rb.DeviceSet.from_serialized(blobs)
        T = rb.DeviceSet.from_serialized(blobs)
        res = S.batch(op, S, ia, ib)
        S.free()
        k = np.arange(n - 2, dtype=np.uint32)
        res2 = res.batch("or", T, k, k + 2)
        res.free()
        T.free()
        assert _ser(res2) == _exp_chain(R, [op, "or"], blobs), op
        res2.free()


def _scenario_chain_orders(rb, R, blobs):
    """A -> R1 = A op A' -> R2 = R1 op A'' -> R3 = R2 op A''': the operand set and the three links
    freed in every order, the survivors checked after every free."""
    n = len(blobs)
    ops = ["xor", "or", "andnot"]
    exps = [_exp_chain(R, ops[:d + 1], blobs) for d in range(3)]
    m = n - 3
    for order in itertools.permutations(range(4)):
        S = rb.DeviceSet.from_serialized(blobs)
        k = np.arange(m, dtype=np.uint32)
        sets = [S]
        for d, op in enumerate(ops):
            sets.append(sets[-1].batch(op, S, k, k + d + 1))
        for step, victim in enumerate(order):
            sets[victim].free()
            for d in range(1, 4):
                if sets[d].ptr is not None:
                    assert _ser(sets[d]) == exps[d - 1][:m], (order, step, d)


def _scenario_async_then_free(rb, R, blobs):
    n = len(blobs)
    ia, ib = _pairs(n)
    digs = {}

    def visit(i, p, _ctx):
        digs[i] = hashlib.sha256(rb.Bitmap(p, own=False).serialize()).digest()
        return 0
    fn = rb.api.VISIT_FN(visit)
    acc = rb.api.CardinalitySum()
    for op in ("or", "xor"):
        A = rb.DeviceSet.from_serialized(blobs)
        B = rb.DeviceSet.from_serialized(blobs[::-1])
        res = A.batch(op, B, ia, ib)
        res.foreach_async(acc, fn)
        res.free()
        A.free()
        B.free()
        rb.download_wait()
        exp = [R.op_bytes(op, blobs[k], blobs[::-1][k + 1]) for k in range(n - 1)]
        assert [digs[k] for k in range(n - 1)] == [hashlib.sha256(e).digest() for e in exp], op


def _scenario_inplace_lazy_run_optimize(rb, R, blobs):
    """in-place rules, a lazy op (+ repair) and run_optimize applied to a result with shared
    containers, after the result's operand was freed."""
    n = len(blobs)
    ia, ib = _pairs(n)
    S = rb.DeviceSet.from_serialized(blobs)
    T = rb.DeviceSet.from_serialized(blobs)
    res = S.batch("or", S, ia, ib)
    S.free()
    mid = [R.op_bytes("or", blobs[k], blobs[k + 1]) for k in range(n - 1)]
    k = np.arange(n - 2, dtype=np.uint32)
    for op in ("and", "or", "xor", "andnot"):
        ip = res.batch(op, T, k, k + 2, inplace_rules=True)
        assert _ser(ip) == [R.op_inplace_bytes(op, mid[j], blobs[j + 2]) for j in range(n - 2)], op
        ip.free()
    for op in ("or", "xor"):
        lz = res.batch(op, T, k, k + 2, lazy=True)
        rep = lz.repair_after_lazy()
        lz.free()
        assert _ser(rep) == [R.lazy_fold_bytes(op, False, [mid[j], blobs[j + 2]]) for j in range(n - 2)], op
        rep.free()
    ro = res.run_optimize()
    res.free()
    T.free()
    assert _ser(ro) == [_run_optimize_bytes(R, m) for m in mid]
    ro.free()


def _scenario_set64_free_operands(rb, R, _blobs):
    """64-bit sets: both operands freed before the result is serialized, run-optimized or chained."""
    b64 = synth_blobs64(R, 77, 24)
    a, b = b64[:12], b64[12:]
    ia = np.arange(12, dtype=np.uint32)
    ib = ia[::-1].copy()
    for op in ("or", "xor", "andnot"):
        exp = [R.r64_op_bytes(op, a[k], b[ib[k]]) for k in range(12)]
        A64, B64 = rb.DeviceSet64.from_serialized(a), rb.DeviceSet64.from_serialized(b)
        res = A64.op(op, B64, ia, ib)
        A64.free()
        B64.free()
        assert res.serialize_all() == exp, op
        C64 = rb.DeviceSet64.from_serialized(b)
        res2 = res.op("or", C64, ia, ia)
        C64.free()
        ro = res.run_optimize()
        res.free()
        assert res2.serialize_all() == [R.r64_op_bytes("or", exp[k], b[k]) for k in range(12)], op
        res2.free()
        assert ro.serialize_all() == [_r64_run_optimize_bytes(R, e) for e in exp], op
        ro.free()


SCENARIOS = [_scenario_free_parent_first, _scenario_chain_orders, _scenario_async_then_free,
             _scenario_inplace_lazy_run_optimize, _scenario_set64_free_operands]


@pytest.mark.parametrize("scenario", SCENARIOS, ids=lambda f: f.__name__[10:])
def test_shared_passthrough(rb, R, scenario):
    scenario(rb, R, _inputs(rb, R))


def test_nothing_outstanding_after_free(rb, R):
    """After every scenario has freed what it made, the device blocks handed out are back to where
    they were (one warm pass first: scratch the library keeps for later calls is not a leak)."""
    blobs = _inputs(rb, R)
    lib = rb.api.lib()
    for s in SCENARIOS:
        s(rb, R, blobs)
    rb.synchronize()
    before = lib.rb200_device_bytes_in_use()
    for s in SCENARIOS:
        s(rb, R, blobs)
    rb.download_wait()
    rb.synchronize()
    assert lib.rb200_device_bytes_in_use() == before


def test_fold_frees_previous_accumulator_in_bounded_memory(rb, R):
    """acc = acc op S[k]; free the previous acc — 80 steps.  A result holds only its operands' own
    slabs (never what they hold), so the device memory in use stays flat instead of growing by one
    accumulator slab per step; the final accumulator is the reference's fold."""
    blobs = rb.load_realdata("census1881")[:16]
    lib = rb.api.lib()
    S = rb.DeviceSet.from_serialized(blobs)
    one = lambda v: np.array([v], dtype=np.uint32)
    acc, exp = S.batch("or", S, one(0), one(1)), R.op_bytes("or", blobs[0], blobs[1])
    use = []
    for k in range(2, 82):
        op = ("or", "xor", "andnot")[k % 3]
        nxt = acc.batch(op, S, one(0), one(k % 16))
        acc.free()
        acc = nxt
        exp = R.op_bytes(op, exp, blobs[k % 16])
        rb.synchronize()
        use.append(lib.rb200_device_bytes_in_use())
    assert _ser(acc) == [exp]
    assert max(use[40:]) <= 1.5 * max(use[:20]), use
    acc.free()
    S.free()
