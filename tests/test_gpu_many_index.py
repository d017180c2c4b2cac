"""The key-major index of the N-way union (rb200_many2.cu) against the reference.

Both index builders: the library picks key windows for long directories and per-container atomics
for short ones, so the or_many parity tests are re-run in a child process with each choice FORCED
(RB200_OR_MANY_INDEX is read once per process).  The index's limits: more than 2^24 participants
of one key, and the refusal of a call whose inputs carry more than 2^32 - 1 containers."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from croaring_b200 import sharding as sh

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("index", ["window", "atomic"])
def test_or_many_parity_with_forced_index(index):
    env = dict(os.environ, RB200_OR_MANY_INDEX=index)
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", "-k", "or_many",
           "tests/test_gpu_parity.py", "tests/test_gpu_sharded.py", "tests/test_gpu_properties.py"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout


CHILD = r"""
import sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + "/tests")
import numpy as np
import croaring_b200 as rb
from helpers import synth_blobs
from oracle.refbind import ref
R = ref()
rb.init(0)
blobs = synth_blobs(R, 123, 700, key_space=300, max_keys=80, profiles=["array", "tiny", "tiny", "tiny", "longruns", "bitset", "full", "array"])
S = rb.DeviceSet.from_serialized(blobs)
out = S.or_many().download(0)
assert out.serialize() == R.many_bytes("or_many", blobs), "700-way union differs"
idx = np.arange(0, 700, 3, dtype=np.uint32)
out = S.or_many(idx).download(0)
assert out.serialize() == R.many_bytes("or_many", [blobs[i] for i in idx]), "subset union differs"
print("child ok")
"""


def test_window_index_with_several_bitmap_chunks():
    """More than 256 inputs: the window builder splits the inputs into chunks of 256 per key window and
    the fill pass offsets every chunk by the counts of the chunks before it."""
    env = dict(os.environ, RB200_OR_MANY_INDEX="window")
    r = subprocess.run([sys.executable, "-c", CHILD.format(root=ROOT)], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "child ok" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


def _wide_key_set(R):
    """24 small bitmaps, all carrying key 0 (arrays, bitsets, runs; never full there), some carrying
    keys 1-3 too (bitsets, a full run, a full bitset)."""
    rng = np.random.default_rng(20261015)
    hs = []
    for i in range(24):
        kind = i % 4
        if kind == 0:
            vals = [rng.choice(65536, 40 + 7 * i, replace=False)]                   # array
        elif kind == 1:
            vals = [rng.choice(65536, 5000 + 100 * i, replace=False)]               # bitset
        elif kind == 2:
            vals = [np.arange(s, s + 100 + i) for s in rng.choice(np.arange(0, 65536, 512), 6, replace=False)]
        else:
            vals = [rng.choice(65536, 3, replace=False), np.arange(2 << 16, 3 << 16)]   # + full run on key 2
        if i % 5 == 0:
            vals.append((1 << 16) + rng.choice(65536, 6000, replace=False))
        full_bitset = i % 7 == 3
        if full_bitset:
            vals.append(np.arange(3 << 16, 4 << 16))
        hs.append(R.from_values(np.unique(np.concatenate(vals)), run_optimize=not full_bitset))
    return hs


def test_or_many_with_more_than_2_24_participants_of_one_key(rb, R):
    """2^24 + 1 inputs share key 0: the per-key participant count no longer fits the 24 bits the
    index once had.  The inputs repeat a small resident set through idx; the reference gets the
    same repeated handles."""
    hs = _wide_key_set(R)
    n = (1 << 24) + 1
    idx = (np.arange(n, dtype=np.uint64) % len(hs)).astype(np.uint32)
    handles = np.array(hs, dtype=np.uint64)[idx]
    r = R.L.roaring_bitmap_or_many(n, handles.ctypes.data_as(C.POINTER(C.c_void_p)))
    exp = R.serialize(r)
    R.free(r)
    S = rb.DeviceSet.from_serialized([R.serialize(h) for h in hs])
    for h in hs:
        R.free(h)
    got = rb.DeviceSet(rb.api.lib().rb200_or_many(S.ptr, idx.ctypes.data, n)).download(0).serialize()
    assert got == exp
    for lo, hi in ((0, 0), (1, 65535)):
        cpk = np.zeros(65536, dtype=np.uint32)
        got = S.or_many(idx, key_lo=lo, key_hi=hi, card_per_key=cpk).download(0).serialize()
        assert got == sh.slice_blob_by_keys(exp, lo, hi)
        keys, cards = sh.blob_key_cards(got)
        assert np.array_equal(cpk[keys.astype(np.int64)], cards)


def test_or_many_refuses_more_than_2_32_containers(rb, R):
    """One bitmap with a full run on each of the 65536 keys, 65537 times: 2^32 + 2^16 containers.
    The host refuses the call before any allocation or launch."""
    r = R.L.roaring_bitmap_create_with_capacity(0)
    R.L.roaring_bitmap_add_range_closed(r, 0, 0xFFFFFFFF)
    blob = R.serialize(r)
    R.free(r)
    S = rb.DeviceSet.from_serialized([blob])
    assert S.container_count == 65536
    idx = np.zeros(65537, dtype=np.uint32)
    launches = rb.kernel_launches()
    with pytest.raises(rb.RB200Error, match="more than 2\\^32 - 1 containers"):
        S.or_many(idx)
    assert not rb.api.lib().rb200_or_many(S.ptr, idx.ctypes.data, idx.size)
    assert "2^32 - 1 containers" in rb.last_error()
    assert rb.kernel_launches() == launches
