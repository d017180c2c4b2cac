"""CPU checks of the 64-bit point queries (-m "not gpu"): rb200_set64_batch_query / _device refuse a NULL set
before any CUDA call, and the Python mirror refuses an unknown kind and bad values or indices before it calls
the library, so none of this needs a device."""
import ctypes as C

import numpy as np
import pytest

from croaring_b200 import api


def test_null_set_refused_before_any_device():
    L = api.lib()
    vals = (C.c_uint64 * 1)(5)
    out = (C.c_uint64 * 1)()
    found = (C.c_uint8 * 1)()
    for kind in range(4):
        assert L.rb200_set64_batch_query(kind, None, None, 1, vals, out, found) == -1
        assert api.last_error() == "set64_query: S is NULL"
        assert L.rb200_set64_batch_query_device(kind, None, None, 1, vals, out, found) == -1
        assert api.last_error() == "set64_query_device: S is NULL"
    # the set is checked first, whatever the kind and the other arguments
    for kind in (-1, 9):
        assert L.rb200_set64_batch_query(kind, None, None, 0, None, None, None) == -1
        assert api.last_error() == "set64_query: S is NULL"
        assert L.rb200_set64_batch_query_device(kind, None, None, 0, None, None, None) == -1
        assert api.last_error() == "set64_query_device: S is NULL"


class _Stub:
    """A stand-in 64-bit set of n bitmaps: the mirror's checks run before the library sees its pointer."""
    def __init__(self, n):
        self.ptr, self._n = None, n

    def __len__(self):
        return self._n


@pytest.mark.parametrize("kind", ["member", "minimum", "RANK", 1])
def test_unknown_kind_refused(kind):
    with pytest.raises(api.RB200Error, match="unknown query kind"):
        api._query64(_Stub(2), kind, [1, 2], None)


@pytest.mark.parametrize("kind", sorted(api.QUERIES))
def test_argument_errors(kind):
    s = _Stub(3)
    with pytest.raises(api.RB200Error, match="integer"):
        api._query64(s, kind, np.array([0.5, 1.0, 2.0]), None)
    with pytest.raises(api.RB200Error, match="must lie in"):
        api._query64(s, kind, [-1, 2, 3], None)
    with pytest.raises(api.RB200Error, match="must lie in"):
        api._query64(s, kind, np.array([5, -(1 << 40), 3], dtype=np.int64), None)
    with pytest.raises(api.RB200Error, match="integer"):
        api._query64(s, kind, np.zeros((3, 1), dtype=np.uint64), None)
    # idx None asks each bitmap once: one value per bitmap
    with pytest.raises(api.RB200Error, match="2 values for the 3 bitmaps"):
        api._query64(s, kind, [1, 2], None)
    # an idx array pairs with the values one to one
    with pytest.raises(api.RB200Error, match="idx has 2 entries for 3 values"):
        api._query64(s, kind, [1, 2, 3], [0, 1])
    with pytest.raises(api.RB200Error, match="idx has 4 entries for 3 values"):
        api._query64(s, kind, [1 << 40, 2, 3], np.array([0, 1, 2, 2], dtype=np.uint32))
    with pytest.raises(api.RB200Error, match="must lie in"):
        api._query64(s, kind, [1, 2, 3], [0, -1, 2])
    with pytest.raises(api.RB200Error, match="must lie in"):
        api._query64(s, kind, [1, 2, 3], [0, 1 << 32, 2])
    with pytest.raises(api.RB200Error, match="integer"):
        api._query64(s, kind, [1, 2, 3], [0.0, 1.0, 2.0])
    # a scalar idx is broadcast, and must itself be an index
    for bad in (-1, 1 << 32, 1.5, True, "0"):
        with pytest.raises(api.RB200Error, match=r"idx must be an integer in \[0, 2\^32\)"):
            api._query64(s, kind, [1, 2, 3], bad)


def test_python_int_values_past_2_63():
    """A list mixing values past 2^63 with smaller ones (numpy would read it as floats) is taken exactly."""
    assert api._values_u64([0, (1 << 64) - 1, 5]).tolist() == [0, (1 << 64) - 1, 5]
    assert api._values_u64([]).dtype == np.uint64
    with pytest.raises(api.RB200Error, match=r"must lie in \[0, 2\^64\)"):
        api._values_u64([1 << 64, 1])
    with pytest.raises(api.RB200Error, match=r"must lie in \[0, 2\^64\)"):
        api._values_u64([-1, (1 << 64) - 1])
    with pytest.raises(api.RB200Error, match="integer"):
        api._values_u64([1.5, (1 << 64) - 1])
