"""CPU check of the run-container catalogue (tests/run_cases.py): every blob is one the reference
reads, validates and writes back byte for byte, and every case sits on the edge it is named for."""
import numpy as np
import pytest

import run_cases as rc


@pytest.fixture(scope="module")
def cat():
    return rc.catalogue()


def _roundtrip(R, blob, what):
    r = R.deserialize(blob)
    ok, why = R.validate(r)
    out = R.serialize(r)
    R.free(r)
    assert ok, f"{what}: reference validate failed: {why}"
    assert out == blob, f"{what}: the reference writes {len(out)} B, the builder {len(blob)} B"


def test_blobs_are_what_the_reference_writes(R, cat):
    pairs, bitmaps = cat
    for name, blob in bitmaps:
        _roundtrip(R, blob, name)
    for name, blobs in rc.sweep_lists():
        for k, b in enumerate(blobs):
            _roundtrip(R, b, f"{name}[{k}]")


def test_builder_layouts(R):
    """Both cookies, with and without the offset header, against the reference's own serializer."""
    vals = np.r_[np.arange(10, 20), 70000, np.arange(3 << 16, (3 << 16) + 5000, 1)]
    r = R.from_values(vals, run_optimize=False)
    assert rc.run_blob([(0, "array", list(range(10, 20))), (1, "array", [70000 - 65536]),
                        (3, "bitset", list(range(5000)))]) == R.serialize(r)
    R.L.roaring_bitmap_run_optimize(r)
    exp = R.serialize(r)
    R.free(r)
    assert rc.run_blob([(0, "run", [(10, 9)]), (1, "array", [70000 - 65536]), (3, "run", [(0, 4999)])]) == exp
    four = [(k, "run", [(k, 3)]) for k in range(4)]
    r = R.from_values(np.concatenate([np.arange(k, k + 4) + (k << 16) for k in range(4)]), run_optimize=True)
    assert rc.run_blob(four) == R.serialize(r)
    R.free(r)
    assert rc.blob_containers(rc.run_blob(four)) == [(k, "run", 4, 1) for k in range(4)]


@pytest.mark.parametrize("bad", [
    (0, "run", [(5, 3), (9, 0)]),          # adjacent runs
    (0, "run", [(9, 0), (5, 1)]),          # unsorted
    (0, "run", [(65530, 6)]),              # past 65535
    (0, "array", list(range(4097))),       # an array above 4096 values reads back as a bitset
    (0, "bitset", list(range(100))),
])
def test_builder_refuses_invalid_containers(bad):
    with pytest.raises(ValueError):
        rc.run_blob([bad])


def test_cases_sit_on_their_edges(R):
    cases = rc.pair_cases()
    names = [c[0] for c in cases]
    assert len(names) == len(set(names))
    totals = {}
    for name, a, b, meta in cases:
        if "total" in meta:
            assert rc.interval_total(a, b) == meta["total"], name
            fam = name.split("_", 1)[1]
            totals.setdefault(fam, set()).add(meta["total"])
        if "runs" in meta:
            want = meta["runs"]
            got = (len(a[2]) if a[1] == "run" else None, len(b[2]) if b[1] == "run" else None)
            assert got[0] == want[0] and (want[1] is None or got[1] == want[1]), (name, got)
        if "tie" in meta:
            ia, ib = rc.intervals(a), rc.intervals(b)
            assert meta["tie"] in ia and meta["tie"] in ib, name
        if meta.get("split_tie"):
            assert len(rc.split_ties(a, b)) >= 2, name
            assert rc.interval_total(a, b) <= 512, name
        if "expect" in meta:
            op, kind = meta["expect"]
            got = rc.blob_containers(R.op_bytes(op, rc.run_blob([a]), rc.run_blob([b])))
            assert [t for _, t, _, _ in got] == [kind], (name, op, got)
    # the cutoff: every family on 511, 512 and 513; results that stay a run, become an array, go bitset
    assert totals and all(v == {511, 512, 513} for v in totals.values()), totals
    assert {"rr_run", "rr_array", "ar_run", "ar_array", "ar_bitset"} <= set(totals)
    # the run counts the kernels branch on
    counts = {len(c[2]) for _, a, b, _ in cases for c in (a, b) if c[1] == "run"}
    assert {31, 32, 33, 2047, 2048, 8192, 8193, 32768} <= counts


def test_word_edges_case():
    """Runs on bit 0 / bit 31 of a word, inside one word, and interiors of 7, 8, 9 and > 32 words."""
    body = rc._word_edges()[2]
    lo = np.array([s for s, _ in body])
    hi = lo + np.array([l for _, l in body])
    interior = np.where(lo >> 5 == hi >> 5, -1, (hi >> 5) - (lo >> 5) - 1)
    assert {7, 8, 9} <= set(interior.tolist()) and interior.max() > 32
    assert np.any(lo % 32 == 0) and np.any(hi % 32 == 31) and np.any(interior == -1)
    assert lo[0] % 32 == 0 and hi[1] % 32 == 31 and hi[-1] == 65535


def test_split_ties_cross_lanes():
    """The lane-split tie cases: equal boundaries of A and B sit on both sides of a split, for the
    end / start, start / start and end / end coincidences."""
    for kind, n in (("end_start", 64), ("start", 72), ("end", 72)):
        a, b = rc._ties(n, kind)
        m = rc.merged_boundaries(a, b)
        per = (len(m) + 31) // 32
        splits = rc.split_ties(a, b)
        assert splits and all(d % per == 0 for d in splits), kind


def test_sweep_lists_reach_both_staging_choices(R):
    """Some lists average at least 7 KiB per container and some less (the automatic choice of
    bulk-copy staging in the many-way union); big run containers on both sides of 8192 runs; and the
    'acc2' list's key 0 has an oversized run after its last in-place bitset step."""
    lists = dict(rc.sweep_lists())
    assert all(20 <= len(v) <= 300 for v in lists.values())
    avg = {}
    kinds = set()
    for name, blobs in lists.items():
        kib = sum(len(b) // 1024 + 1 for b in blobs)
        conts = [c for b in blobs for c in rc.blob_containers(b)]
        avg[name] = kib / len(conts)
        kinds |= {(t, n) for _, t, _, n in conts if t == "run" and n in (2047, 2048, 8192, 8193, 32768)}
        kinds |= {(t, card) for _, t, card, _ in conts if card == 65536}
    assert any(v >= 7 for v in avg.values()) and any(v < 7 for v in avg.values()), avg
    assert {("run", n) for n in (2047, 2048, 8192, 8193, 32768)} <= kinds
    assert {("run", 65536), ("bitset", 65536)} <= kinds
    key0 = [[c for c in rc.blob_containers(b) if c[0] == 0] for b in lists["acc2"]]
    key0 = [c[0] for c in key0 if c]
    assert [t for _, t, _, _ in key0] == ["array", "array", "bitset", "run"]
    assert key0[3][3] > 8192
