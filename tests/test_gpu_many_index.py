"""Both index builders of the second-generation N-way union (rb200_many2.cu) against the reference:
the library picks key windows for long directories and per-container atomics for short ones, so the
or_many parity tests are re-run in a child process with each choice FORCED (RB200_OR_MANY_INDEX is
read once per process)."""
import os
import subprocess
import sys

import pytest

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
