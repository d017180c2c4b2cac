"""croaring_b200 — H100-native Roaring set-algebra engine (hot path of CRoaring on sm_90a).

The product is the C-ABI library libroaring_b200.so (include/roaring_b200.h); this package is
its Python mirror (ctypes) plus workload I/O helpers.  See DESIGN.md / INTEGRATION.md.
"""
from .api import (AND, ANDNOT, OR, XOR, Bitmap, CardinalitySum, Comm, DeviceSet, RB200Error, batch_op_host,
                  download_wait, foreach_many, init, r64_and_cardinality, r64_batch_op,  # noqa: F401
                  kernel_launches, last_algorithmic_bytes, last_device_ms, last_error, lib,
                  or_many, or_many_heap, set_stream, synchronize, xor_many)
from .datasets import load_realdata, read_rbset, write_rbset  # noqa: F401
