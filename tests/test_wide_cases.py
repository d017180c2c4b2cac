"""CPU check of the long-directory / top-of-key-space catalogue (tests/wide_cases.py): every blob is
one the reference reads, validates and writes back byte for byte; every case holds what its name
claims, read back from its bytes; and the reference's own results reach the scale the cases were
built for, so the GPU tests on them cannot quietly shrink."""
import numpy as np
import pytest

import run_cases as rc
import wide_cases as wc


def _roundtrip(R, blob, what):
    r = R.deserialize(blob)
    ok, why = R.validate(r)
    out = R.serialize(r)
    R.free(r)
    assert ok, f"{what}: reference validate failed: {why}"
    assert out == blob, f"{what}: the reference writes {len(out)} B, the builder {len(blob)} B"


def _keys(blob):
    return [c[0] for c in rc.blob_containers(blob)]


def test_blobs_are_what_the_reference_writes(R):
    for name, blob in wc.bitmaps(R):
        _roundtrip(R, blob, name)
    for name, a, b in wc.fused_pairs(R):
        _roundtrip(R, a, name + ".a")
        _roundtrip(R, b, name + ".b")
    for name, blobs in wc.many_lists(R):
        for k, b in enumerate(blobs):
            _roundtrip(R, b, f"{name}[{k}]")


def test_bitmaps_hold_what_their_names_claim(R):
    cs = {name: rc.blob_containers(b) for name, b in wc.bitmaps(R)}
    assert set(cs) == ({f"top_{f}" for f in wc.TOP_FORMS} | {"all_keys", "even_keys", "odd_keys", "tiles"} |
                       {f"len_{n}" for n in wc.LENS} | {"full_universe", "half_universe"})
    last = {f: cs[f"top_{f}"][-1] for f in wc.TOP_FORMS}
    assert last["array"][:3] == (65535, "array", 3)
    assert last["run_end"][:2] == (65535, "run") and last["run_end"][2] == 65536 - 60000
    assert last["full_run"] == (65535, "run", 65536, 1)
    assert last["full_bitset"][:3] == (65535, "bitset", 65536)
    assert last["bitset"][:3] == (65535, "bitset", 5001)
    ra = R.deserialize(wc.bitmap(R, "top_array"))
    assert int(R.to_array(ra)[-1]) == 0xFFFFFFFF
    R.free(ra)
    for f in wc.TOP_FORMS:
        assert [c[0] for c in cs[f"top_{f}"]] == list(range(65500, 65536)), f
    assert [c[0] for c in cs["all_keys"]] == list(range(65536))
    assert [c[0] for c in cs["even_keys"]] == list(range(0, 65536, 2))
    assert [c[0] for c in cs["odd_keys"]] == list(range(1, 65536, 2))
    for n in wc.LENS:
        keys = [c[0] for c in cs[f"len_{n}"]]
        assert len(keys) == n, n
        if n >= 2:
            assert keys[0] == 0 and keys[-1] == 65535, n
    assert [c[0] for c in cs["tiles"]] == sorted(wc.TILE_EDGES)
    assert len(wc.TILE_EDGES) == 32 and {k // wc.TILE for k in wc.TILE_EDGES} == set(range(16))
    assert cs["full_universe"] == [(k, "run", 65536, 1) for k in range(65536)]
    assert cs["half_universe"] == [(k, "run", 65536, 1) for k in range(0, 65536, 2)]
    # the big directories mix every kind of container, full ones included
    for name in ("all_keys", "even_keys", "odd_keys", "len_1025", "tiles"):
        kinds = {(t, card == 65536) for _, t, card, _ in cs[name]}
        assert {("array", False), ("bitset", False), ("run", False), ("run", True), ("bitset", True)} <= kinds, name


def test_fused_pairs_total_their_name(R):
    names = []
    for name, a, b in wc.fused_pairs(R):
        t = int(name.split("_")[1])
        names.append(t)
        ka, kb = set(_keys(a)), set(_keys(b))
        assert len(ka) + len(kb) == t, name
        both = ka & kb
        assert 65535 in both and ka - kb and kb - ka, name
        # some matched containers are equal (AND and XOR drop their keys), some are not
        ra, rb_ = R.deserialize(a), R.deserialize(b)
        va, vb = R.to_array(ra), R.to_array(rb_)
        R.free(ra)
        R.free(rb_)
        equal = [k for k in both if np.array_equal(va[va >> 16 == k], vb[vb >> 16 == k])]
        assert 0 < len(equal) < len(both), name
    assert names == list(wc.FUSED)


def test_many_lists_have_their_shape(R):
    lists = dict(wc.many_lists(R))
    assert set(lists) == {f"list_{n}" for n in wc.MANY} | {"list_all_keys"}
    for n in wc.MANY:
        blobs = lists[f"list_{n}"]
        assert len(blobs) == n
        keys = {k for b in blobs for k in _keys(b)}
        assert {65535, 4095, 4096, 61440} <= keys, n
        assert len({k // wc.TILE for k in keys}) == 16, n
        kinds = {c[1] for b in blobs for c in rc.blob_containers(b)}
        assert kinds == {"array", "bitset", "run"}, n
    x = lists["list_1025"]
    i, j, m = wc.REPEAT
    assert i < 512 <= j and x[i] == x[j]
    own = set(_keys(x[i])) - set(wc.POOL)
    assert len(own) == 1 and own <= set(_keys(x[m]))
    # which inputs hold x[3]'s own key: x[3], x[515] and x[700] only
    assert [k for k, b in enumerate(x) if own <= set(_keys(b))] == [i, j, m]
    assert len(lists["list_all_keys"]) == 513


def test_reference_results_reach_their_scale(R):
    even, odd = wc.bitmap(R, "even_keys"), wc.bitmap(R, "odd_keys")
    assert _keys(R.op_bytes("or", even, odd)) == list(range(65536))
    assert _keys(R.op_bytes("and", even, odd)) == []
    lists = dict(wc.many_lists(R))
    n_keys = {name: len(_keys(R.many_bytes("xor_many", blobs))) for name, blobs in lists.items()}
    assert n_keys["list_1025"] > 1024, n_keys
    assert n_keys["list_all_keys"] == 65536, n_keys
    # list_1025: x[3]'s own key cancels at x[515] and is back with x[700]
    x = lists["list_1025"]
    i, j, m = wc.REPEAT
    own = (set(_keys(x[i])) - set(wc.POOL)).pop()
    assert own not in _keys(R.many_bytes("xor_many", x[:j + 1]))
    got = [c for c in rc.blob_containers(R.many_bytes("xor_many", x)) if c[0] == own]
    exp = [c for c in rc.blob_containers(x[m]) if c[0] == own]
    assert got == exp
    full = R.deserialize(wc.bitmap(R, "full_universe"))
    assert R.card(full) == 1 << 32
    half = R.deserialize(wc.bitmap(R, "half_universe"))
    assert R.card(half) == 1 << 31
    assert int(R.L.roaring_bitmap_and_cardinality(full, full)) == 1 << 32
    R.free(full)
    R.free(half)


@pytest.mark.parametrize("name", ["all_keys", "len_1025"])
def test_builder_is_seeded(R, name):
    """The catalogue is a pure function of its seeds: rebuilt, it is the same bytes."""
    first = wc.bitmap(R, name)
    wc.bitmaps.cache_clear()
    assert wc.bitmap(R, name) == first
