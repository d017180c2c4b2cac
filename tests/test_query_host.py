"""CPU checks of the point queries (-m "not gpu"): rb200_batch_query / _device refuse a NULL set before any
CUDA call, and the Python mirror refuses an unknown kind and bad values or indices before it calls the
library, so none of this needs a device."""
import ctypes as C

import numpy as np
import pytest

from croaring_b200 import api


def test_null_set_refused_before_any_device():
    L = api.lib()
    vals = (C.c_uint32 * 1)(5)
    out = (C.c_int64 * 1)()
    for kind in range(4):
        assert L.rb200_batch_query(kind, None, None, 1, vals, out) == -1
        assert api.last_error() == "query: S is NULL"
        assert L.rb200_batch_query_device(kind, None, None, 1, vals, out) == -1
        assert api.last_error() == "query_device: S is NULL"
    # the set is checked first, whatever the kind
    assert L.rb200_batch_query(9, None, None, 0, None, None) == -1
    assert api.last_error() == "query: S is NULL"


class _Stub:
    """A stand-in set of n bitmaps: the mirror's checks run before the library sees its pointer."""
    def __init__(self, n):
        self.ptr, self._n = None, n

    def __len__(self):
        return self._n


@pytest.mark.parametrize("kind", ["member", "minimum", "RANK", 1])
def test_unknown_kind_refused(kind):
    with pytest.raises(api.RB200Error, match="unknown query kind"):
        api._query(_Stub(2), kind, [1, 2], None)


@pytest.mark.parametrize("kind", sorted(api.QUERIES))
def test_argument_errors(kind):
    s = _Stub(3)
    with pytest.raises(api.RB200Error, match="integer"):
        api._query(s, kind, np.array([0.5, 1.0, 2.0]), None)
    with pytest.raises(api.RB200Error, match="must lie in"):
        api._query(s, kind, [-1, 2, 3], None)
    with pytest.raises(api.RB200Error, match="must lie in"):
        api._query(s, kind, [1 << 32, 2, 3], None)
    with pytest.raises(api.RB200Error, match="integer"):
        api._query(s, kind, np.zeros((3, 1), dtype=np.uint32), None)
    # idx None asks each bitmap once: one value per bitmap
    with pytest.raises(api.RB200Error, match="2 values for the 3 bitmaps"):
        api._query(s, kind, [1, 2], None)
    # an idx array pairs with the values one to one
    with pytest.raises(api.RB200Error, match="idx has 2 entries for 3 values"):
        api._query(s, kind, [1, 2, 3], [0, 1])
    with pytest.raises(api.RB200Error, match="idx has 4 entries for 3 values"):
        api._query(s, kind, [1, 2, 3], np.array([0, 1, 2, 2], dtype=np.uint32))
    with pytest.raises(api.RB200Error, match="must lie in"):
        api._query(s, kind, [1, 2, 3], [0, -1, 2])
    with pytest.raises(api.RB200Error, match="integer"):
        api._query(s, kind, [1, 2, 3], [0.0, 1.0, 2.0])
    # a scalar idx is broadcast, and must itself be an index
    for bad in (-1, 1 << 32, 1.5, True, "0"):
        with pytest.raises(api.RB200Error, match=r"idx must be an integer in \[0, 2\^32\)"):
            api._query(s, kind, [1, 2, 3], bad)
