"""k_compute_items walks its cell descriptors either in class order (batches of at least
RB200_ORDER_MIN item slots, the default for the all-pairs workload) or in item order, skipping the
holes.  One all-pairs op that has cells of every class and pass-through copies, run once with the
class-ordered list forced on and once forced off (a subprocess each: the threshold is read once per
process), must give the reference's bytes both times."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_RUN = r'''
import ctypes as C, hashlib, json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import croaring_b200 as rb
rb.init(0)
blobs = rb.load_realdata("weather_sept_85")
S = rb.DeviceSet.from_serialized(blobs)
ia, ib = np.triu_indices(len(blobs), 1)
r = S.batch("or", S, ia.astype(np.uint32), ib.astype(np.uint32))
buf, off, ln, release = r.serialize_all(copy=False)
h = hashlib.sha256()
for k in range(len(ia)):
    h.update(C.string_at(buf.value + int(off[k]), int(ln[k])))
release()
print(json.dumps({"sum_card": int(r.cardinalities().sum()), "sha256": h.hexdigest()}))
'''


@pytest.mark.parametrize("order_min", ["0", str(1 << 40)], ids=["class_order", "item_order"])
def test_allpairs_or_with_and_without_class_order(order_min):
    with open(os.path.join(ROOT, "tests", "golden", "allpairs_golden.json")) as f:
        gold = json.load(f)["weather_sept_85"]["or"]
    env = dict(os.environ, RB200_ORDER_MIN=order_min)
    out = subprocess.run([sys.executable, "-c", _RUN, ROOT], env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    got = json.loads(out.stdout.strip().splitlines()[-1])
    assert got["sum_card"] == gold["sum_card"]
    assert got["sha256"] == gold["sha256"]
