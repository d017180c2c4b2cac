"""GPU parity of array x array cells whose inputs total at most 4096 values (the windowed merge path
of rb200_device.cuh: merge_arrays) against the oracle: every op, single- and multi-key bitmaps,
through the batched path, the single-pair drop-in symbols and the in-place twins."""
import struct

import numpy as np
import pytest

from helpers import OPS

pytestmark = pytest.mark.gpu

SIZES = [1, 2040, 2048, 2049, 3000, 4088, 4089, 4095, 4096]   # cA + cB
KINDS = ["disjoint", "identical", "interleaved", "clustered", "overlap"]


def _portable(containers):
    """{key: sorted u16 array (<= 4096 values)} -> portable bytes (no run containers)."""
    keys = sorted(k for k, v in containers.items() if len(v))
    head = struct.pack("<II", 12346, len(keys))
    head += b"".join(struct.pack("<HH", k, len(containers[k]) - 1) for k in keys)
    off = len(head) + 4 * len(keys)
    offs = b""
    for k in keys:
        offs += struct.pack("<I", off)
        off += 2 * len(containers[k])
    return head + offs + b"".join(np.asarray(containers[k], "<u2").tobytes() for k in keys)


def _case(kind, total, parity, rng):
    """Two sorted u16 arrays with len(a) + len(b) == total; parity 0 reaches value 0, parity 1 65535."""
    if total == 1:
        return np.array([65535 * parity], np.uint16), np.zeros(0, np.uint16)
    if kind == "disjoint":
        vals = np.sort(np.concatenate([[0, 65535], rng.choice(np.arange(1, 65535), total - 2, replace=False)]))
        side = rng.random(total) < 0.5
        side[0], side[-1] = True, False
        return vals[side].astype(np.uint16), vals[~side].astype(np.uint16)
    if kind == "identical":   # XOR of an even total is empty
        base = np.sort(np.concatenate([[0, 65535], rng.choice(np.arange(1, 65534), total // 2 - 2, replace=False)]))
        extra = [65534] if total % 2 else []
        return base.astype(np.uint16), np.sort(np.concatenate([base, extra])).astype(np.uint16)
    if kind == "interleaved":
        s = 0 if parity == 0 else 65536 - total
        vals = np.arange(s, s + total)
        return vals[0::2].astype(np.uint16), vals[1::2].astype(np.uint16)
    if kind == "clustered":
        # b is a shifted by 1 or 2: the duplicate pairs then start on odd or even merged positions,
        # so with an odd shift every lane (8) and window (256) boundary splits a pair
        shift = 1 + parity
        ca = (total + 1) // 2
        cb = total - ca
        span = max(ca, shift + cb)
        s = 0 if parity == 0 else 65536 - span
        return np.arange(s, s + ca).astype(np.uint16), np.arange(s + shift, s + shift + cb).astype(np.uint16)
    # overlap: about half of b's values are in a, scattered
    ca = total // 2
    a = np.sort(rng.choice(65536, ca, replace=False))
    a[0], a[-1] = 0, 65535
    a = np.unique(a)
    rest = np.setdiff1d(np.arange(65536), a)
    nb = total - len(a)
    shared = rng.choice(a, nb // 2, replace=False)
    b = np.sort(np.concatenate([shared, rng.choice(rest, nb - len(shared), replace=False)]))
    return a.astype(np.uint16), b.astype(np.uint16)


def _pairs():
    rng = np.random.default_rng(4096)
    pairs = []
    multi = {}
    for kind in KINDS:
        for parity in (0, 1):
            ma, mb = {}, {}
            for t, total in enumerate(SIZES):
                a, b = _case(kind, total, parity, rng)
                key = 0xFFFF * parity
                pairs.append((_portable({key: a}), _portable({key: b})))
                k = [0, 1, 2, 9, 300, 4000, 40000, 65534, 65535][t]
                ma[k], mb[k] = a, b
            multi[(kind, parity)] = (_portable(ma), _portable(mb))
    return pairs + list(multi.values())


PAIRS = _pairs()


def test_array_merge_batched(rb, O):
    blobs = [x for p in PAIRS for x in p]
    S = rb.DeviceSet.from_serialized(blobs)
    ia = np.arange(0, len(blobs), 2, dtype=np.uint32)
    for op in OPS:
        for inplace in (False, True):
            outs = S.batch(op, S, ia, ia + 1, inplace_rules=inplace).download_all()
            name = op + ("_inplace" if inplace else "")
            for k, (a, b) in enumerate(PAIRS):
                assert outs[k].serialize() == O.op_bytes(name, a, b), (name, k)


def test_array_merge_single_pair(rb, O):
    for k, (a, b) in enumerate(PAIRS):
        for op in OPS:
            x, y = rb.Bitmap.deserialize(a), rb.Bitmap.deserialize(b)
            r = x._pair(op, y)
            assert r.serialize() == O.op_bytes(op, a, b), (op, k)
            x.inplace(op, y)
            assert x.serialize() == O.op_bytes(op + "_inplace", a, b), (op + "_inplace", k)
            assert y.serialize() == b
            for z in (x, y, r):
                z.free()


def test_array_merge_lazy_inplace_xor(rb, O):
    """container_lazy_ixor of two arrays is eager: the lazy in-place XOR takes the merge path too."""
    empty = _portable({})
    blobs = [empty] + [x for p in PAIRS for x in p]
    S = rb.DeviceSet.from_serialized(blobs)
    one = lambda v: np.array([v], dtype=np.uint32)
    for k, (a, b) in enumerate(PAIRS):
        acc = S.batch("xor", S, one(1 + 2 * k), one(0), lazy=True)
        acc = acc.batch("xor", S, one(0), one(2 + 2 * k), lazy=True, inplace_rules=True)
        got = acc.repair_after_lazy().serialize_all()[0]
        assert got == O.lazy_fold_bytes("xor", False, [a, empty, b]), k
