"""CPU tests (-m "not gpu") of the host-side parsers of serialized bitmaps against the reference's parser and
validator, over the seeded corpus of tests/malformed_cases.py: the portable codec behind
rb200_bitmap_portable_deserialize_safe, the blob algebra of rb200_shard.cu, and the bucket walk that refuses
a malformed 64-bit blob before any CUDA call."""
import collections
import re

import pytest

import croaring_b200 as rb
import malformed_cases as M
from croaring_b200 import sharding as sh
from program_model import keyrange_bytes

KEY_RANGES = ((0, 65535), (0, 2), (3, 65534), (32, 40))
# what parse_r64 says of a 64-bit blob whose bucket headers are malformed
R64_STRUCTURAL = ("shorter than its 8-byte bucket count", "bucket count above 2^32 - 1",
                  "truncated: a bucket header runs past the end",
                  "the high 32 bits of the buckets are not strictly increasing",
                  "a bucket runs past the end of the blob or is not a 32-bit portable bitmap")


@pytest.fixture(scope="module")
def corpus(R):
    return {fmt: M.cases(R, fmt, rb) for fmt in M.FORMATS}


@pytest.fixture(scope="module")
def verdicts(R, corpus):
    return {fmt: [M.verdict(R, fmt, b) for _, b in cs] for fmt, cs in corpus.items()}


def verdict_class(fmt, blob, v):
    if v.kind == "valid":
        return "valid" if fmt == "frozen" or v.canon == blob else "valid, not canonical"
    return v.kind if v.kind == "refused" else v.reason


def test_corpus_is_deterministic(R, corpus):
    for fmt in M.FORMATS:
        names = [n for n, _ in corpus[fmt]]
        assert len(set(names)) == len(names), fmt
        assert M.cases(R, fmt, rb) == corpus[fmt], fmt


# Every class of verdict the device must agree with, per format, with the least number of cases that
# keeps the generator from degenerating quietly.
REQUIRED = {
    "portable": {"refused": 500, "valid": 50, "valid, not canonical": 50,
                 "run start equal to last end, should have combined": 10, "cardinality is incorrect": 20,
                 "zero run count": 5, "run start + length too large": 10, "run start less than last end": 10,
                 "array elements not strictly increasing": 20, "keys not strictly increasing": 20},
    "frozen": {"refused": 300, "valid": 50, "run start equal to last end, should have combined": 10,
               "cardinality is incorrect": 20, "cardinality is too small for a bitmap container": 2,
               "cardinality exceeds DEFAULT_MAX_SIZE": 2, "zero run count": 1, "run start + length too large": 10,
               "array elements not strictly increasing": 20, "keys not strictly increasing": 5},
    "r64": {"refused": 100, "valid": 10, "valid, not canonical": 10,
            "run start equal to last end, should have combined": 2, "cardinality is incorrect": 5,
            "run start + length too large": 2, "array elements not strictly increasing": 5},
}


def test_every_verdict_class_appears(corpus, verdicts):
    for fmt in M.FORMATS:
        seen = collections.Counter(verdict_class(fmt, b, v) for (_, b), v in zip(corpus[fmt], verdicts[fmt]))
        short = {k: (seen[k], want) for k, want in REQUIRED[fmt].items() if seen[k] < want}
        assert not short, f"{fmt}: too few cases of {short}; seen {dict(seen)}"
    named = {n: v for (n, _), v in zip(corpus["portable"], verdicts["portable"])}
    assert named["targeted/adjacent@c0"].reason == "run start equal to last end, should have combined"
    assert named["targeted/bitset-card5000-of-10000@c0"].reason == "cardinality is incorrect"
    named = {n: v for (n, _), v in zip(corpus["frozen"], verdicts["frozen"])}
    assert named["frozen/array5000"].reason == "cardinality exceeds DEFAULT_MAX_SIZE"
    assert named["frozen/bitset-count9"].reason == "cardinality is too small for a bitmap container"
    assert named["frozen/array4096"].kind == named["frozen/bitset4097"].kind == "valid"


def test_host_codec_matches_the_reference(corpus, verdicts):
    """rb.Bitmap.deserialize accepts a blob iff the reference parses it with strictly increasing keys (the
    reference's parser does not check key order, its validator does, and first); what it accepts it
    serializes as the reference serializes its parse, invalid contents and all."""
    bad = []
    for (name, blob), v in zip(corpus["portable"], verdicts["portable"]):
        try:
            x = rb.Bitmap.deserialize(blob)
        except rb.RB200Error:
            if M.keys_increase(v):
                bad.append((name, "refused", v.kind, v.reason))
            continue
        got = x.serialize()
        x.free()
        if not M.keys_increase(v):
            bad.append((name, "accepted", v.kind, v.reason))
        elif got != v.canon:
            bad.append((name, "bytes differ", v.kind, v.reason))
    assert not bad, f"{len(bad)} disagreements, first {bad[:10]}"


def test_blob_algebra_matches_the_reference(R, corpus, verdicts):
    """slice_blob_by_keys / concat_blobs / plan_key_ranges accept the blobs the codec accepts; a slice is
    the reference's parse cut to the key range, serialized; on a valid blob, that is keyrange_bytes."""
    bad = []
    for (name, blob), v in zip(corpus["portable"], verdicts["portable"]):
        try:
            parts = [sh.slice_blob_by_keys(blob, lo, hi) for lo, hi in ((0, 7), (8, 300), (301, 65535))]
            full = sh.concat_blobs(parts)
            sh.plan_key_ranges([blob, full], 3)
        except rb.RB200Error:
            if M.keys_increase(v):
                bad.append((name, "refused"))
            continue
        if not M.keys_increase(v):
            bad.append((name, "accepted"))
            continue
        if full != v.canon:
            bad.append((name, "concatenated slices differ from the reference's serialization"))
        for lo, hi in KEY_RANGES:
            got = sh.slice_blob_by_keys(blob, lo, hi)
            if got != M.verdict(R, "portable", M.cut(v.canon, lo, hi)).canon:
                bad.append((name, f"slice [{lo}, {hi}] differs"))
            elif v.kind == "valid" and got != keyrange_bytes(R, blob, lo, hi):
                bad.append((name, f"slice [{lo}, {hi}] differs from keyrange_bytes"))
    assert not bad, f"{len(bad)} disagreements, first {bad[:10]}"


def test_r64_structural_refusals_come_before_any_cuda_call(corpus, verdicts):
    """A 64-bit blob the reference cannot parse is refused by the host's bucket walk, which names the
    bitmap and says what is wrong; one it parses passes that walk (and reaches the device, where there is
    one), so on a machine without a GPU the message alone separates the two."""
    structural = re.compile(r"^malformed 64-bit portable bitmap at index 0: (" +
                            "|".join(re.escape(w) for w in R64_STRUCTURAL) + ")")
    bad = []
    for (name, blob), v in zip(corpus["r64"], verdicts["r64"]):
        try:
            s = rb.DeviceSet64.from_serialized([blob])
            s.free()
            err = None
        except rb.RB200Error as e:
            err = str(e)
        if v.kind == "refused" and not (err and structural.match(err)):
            bad.append((name, "reference refuses", err))
        elif v.kind != "refused" and err and structural.match(err):
            bad.append((name, f"reference parses ({v.kind})", err))
    assert not bad, f"{len(bad)} disagreements, first {bad[:10]}"
