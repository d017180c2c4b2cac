"""GPU test: deferred ops queued back to back on the stream, none of them waited for in between.  The
batch-op kernels are chained by programmatic dependent launch and hand their counters to the result
through the last CTA of k_finalize_pairs, which also zeroes them for the next op; an empty batch and
an add_offset sit in the chain.  Every result must be the reference's bytes with its counters and
times in order, and a process with plain launches (RB200_PDL=0, read when the library loads) must
produce the same bytes."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS = ("and", "or", "xor", "andnot")

CHAIN = r'''
import hashlib, sys
import numpy as np
import croaring_b200 as rb

def blobs():
    return rb.load_realdata("census1881")[:12] + rb.load_realdata("wikileaks-noquotes")[:8]

def chain():
    rb.init(0)
    B = blobs()
    S = rb.DeviceSet.from_serialized(B)
    ia, ib = (x.astype(np.uint32) for x in np.triu_indices(len(B), 1))
    none = np.zeros(0, dtype=np.uint32)
    res = []
    for op in ("and", "or", "xor", "andnot"):
        res.append((op, S.batch(op, S, ia, ib)))
        if op == "or":
            res.append(("empty", S.batch("or", S, none, none)))
            res.append(("offset", S.add_offset(np.arange(len(B), dtype=np.int64) * 70001 - 300000)))
    return B, ia, ib, res

def digest(res):
    h = hashlib.sha256()
    for _, r in res:
        for b in r.serialize_all():
            h.update(b)
    return h.hexdigest()

if __name__ == "__main__":
    print(digest(chain()[3]))
'''


def _chain_module():
    ns = {"__name__": "chain"}
    exec(compile(CHAIN, "chain", "exec"), ns)
    return ns


def test_back_to_back_ops_match_reference_and_report_counters(rb, R):
    ns = _chain_module()
    B, ia, ib, res = ns["chain"]()
    for name, r in res:
        ms, cms, ab = r.op_stats()
        if name == "empty":
            assert r.serialize_all() == []
            assert (ms, cms, ab) == (0.0, 0.0, 0)
            continue
        assert ms > 0 and 0 < cms <= ms, (name, ms, cms)
        if name == "offset":
            continue
        assert ab > 0, name
        out = r.serialize_all()
        assert len(out) == len(ia)
        for k in range(len(ia)):
            assert out[k] == R.op_bytes(name, B[ia[k]], B[ib[k]]), f"{name} pair {k}"


def test_plain_launches_give_the_same_bytes(rb):
    ns = _chain_module()
    here = ns["digest"](ns["chain"]()[3])
    env = dict(os.environ, RB200_PDL="0", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    out = subprocess.run([sys.executable, "-s", "-c", CHAIN], cwd=ROOT, env=env, capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    assert out.stdout.strip().splitlines()[-1] == here
