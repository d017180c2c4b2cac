#!/usr/bin/env python
"""Small, fixed workloads for ncu captures (one launch of each hot kernel after a warm-up).

  pairs   : weather_sept_85 all-pairs OR  (k_plan_pairs, k_compute_items, k_finalize_pairs)
  card    : config[3] shape: bitset-heavy and_cardinality, 2000 pairs (k_card_items)
  many    : or_many over weather_sept_85 + a dense synthetic set (k_many2_*, k_or_many2)
"""
import sys
import os

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import croaring_b200 as rb  # noqa: E402
from croaring_b200.workloads import bitset_heavy_blobs  # noqa: E402

what = sys.argv[1] if len(sys.argv) > 1 else "pairs"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
rb.init(0)
if what == "pairs":
    blobs = rb.load_realdata("weather_sept_85")
    S = rb.DeviceSet.from_serialized(blobs)
    i, j = np.triu_indices(len(blobs), 1)
    for _ in range(reps):
        r = S.batch("or", S, i.astype(np.uint32), j.astype(np.uint32))
        print("or all-pairs: device ms", rb.last_device_ms(), "compute ms",
              rb.api.lib().rb200_last_compute_ms(), "algo GB", rb.last_algorithmic_bytes() / 1e9)
        r.free()
elif what == "card":
    blobs = bitset_heavy_blobs(4000, seed=7)
    S = rb.DeviceSet.from_serialized(blobs)
    ia = np.arange(0, 4000, 2, dtype=np.uint32)
    for _ in range(reps):
        c = S.and_cardinality(S, ia, ia + 1)
        print("and_card: device ms", rb.last_device_ms(), "compute ms",
              rb.api.lib().rb200_last_compute_ms(), "GB/s",
              2000 * 16 * 16384 / (rb.api.lib().rb200_last_compute_ms() * 1e-3) / 1e9, int(c.sum()))
elif what == "many":
    blobs = rb.load_realdata("weather_sept_85") + bitset_heavy_blobs(400, seed=9)
    S = rb.DeviceSet.from_serialized(blobs)
    for _ in range(reps):
        r = S.or_many()
        print("or_many: device ms", rb.last_device_ms(), "compute ms",
              rb.api.lib().rb200_last_compute_ms(), "in GB", S.payload_bytes / 1e9)
        r.free()
