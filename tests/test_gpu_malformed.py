"""GPU tests of the four device parsers of serialized bitmaps (rb200_set_upload_serialized, _frozen,
_serialized_keyrange and rb200_set64_upload_serialized) against the reference's parser and validator, over
the seeded corpus of tests/malformed_cases.py.  The device holds a blob iff the reference's validator
accepts it, and then holds what the reference parsed; a refusal names the caller's index and leaves no
device memory behind."""
import ctypes as C

import numpy as np
import pytest

import malformed_cases as M

pytestmark = pytest.mark.gpu

BATCH = 48
KEY_RANGES = ((0, 2), (3, 65534))
GOOD = ("runs5", "norun33", "array1", "bitset4097")
GOOD64 = ("r64synth[1]", "r64/empty-bucket", "r64synth[2]", "r64/wide")
REFUSED = {"portable": "malformed portable bitmap at index 2", "frozen": "malformed frozen bitmap at index 2",
           "r64": "malformed 64-bit portable bitmap at index 2", "keyrange": "malformed portable bitmap at index 2"}


def _upload(rb, fmt, blobs, key_range=None):
    if fmt == "portable":
        return rb.DeviceSet.from_serialized(blobs)
    if fmt == "keyrange":
        return rb.DeviceSet.from_serialized(blobs, *key_range)
    if fmt == "frozen":
        return rb.DeviceSet.from_frozen(blobs)
    return rb.DeviceSet64.from_serialized(blobs)


def _r64_card(R, blob):
    r = R.r64_deserialize(blob)
    n = int(R.L.roaring64_bitmap_get_cardinality(r))
    R.L.roaring64_bitmap_free(r)
    return n


def _expect(R, fmt, canon):
    """(cardinality, values or None) of the bitmap the reference holds."""
    if fmt == "r64":
        return _r64_card(R, canon), None
    r = R.deserialize(canon)
    out = R.card(r), R.to_array(r)
    R.free(r)
    return out


class Run:
    """The disagreements of one format with the reference, gathered so one run names them all."""

    def __init__(self, rb, R, fmt, good, key_range=None):
        self.rb, self.R, self.fmt, self.good, self.key_range = rb, R, fmt, good, key_range
        self.bad = []
        self.L = rb.lib()

    def refuse(self, name, blob):
        """One expected refusal per call, behind two good blobs: an earlier refusal cannot hide it."""
        before = int(self.L.rb200_device_bytes_in_use())
        try:
            S = _upload(self.rb, self.fmt, self.good[:2] + [blob] + self.good[2:4], self.key_range)
        except self.rb.RB200Error as e:
            if REFUSED[self.fmt] not in str(e):
                self.bad.append((name, f"refused, but: {e}"))
        else:
            S.free()   # never an operand: the reference calls it invalid
            self.bad.append((name, "accepted"))
        if int(self.L.rb200_device_bytes_in_use()) != before:
            self.bad.append((name, "device memory left behind"))

    def accept(self, named):
        """named: [(name, blob, canon)], uploaded BATCH at a time; each set compared whole with the reference."""
        for k in range(0, len(named), BATCH):
            chunk = named[k:k + BATCH]
            before = int(self.L.rb200_device_bytes_in_use())
            try:
                S = _upload(self.rb, self.fmt, [b for _, b, _ in chunk], self.key_range)
            except self.rb.RB200Error as e:
                culprits = []
                for name, blob, _ in chunk:   # which ones?
                    try:
                        _upload(self.rb, self.fmt, [blob], self.key_range).free()
                    except self.rb.RB200Error as e1:
                        culprits.append((name, f"refused: {e1}"))
                self.bad += culprits or [(chunk[0][0], f"the batch from here refused: {e}")]
                continue
            got = S.serialize_all()
            cards = S.cardinalities().tolist()
            vals = S.to_uint32_arrays() if self.fmt != "r64" else None
            frozen = S.serialize_all(frozen=True) if self.fmt == "frozen" else None
            for j, (name, blob, canon) in enumerate(chunk):
                card, v = _expect(self.R, self.fmt, canon)
                if got[j] != canon:
                    self.bad.append((name, "serialize_all differs"))
                if cards[j] != card:
                    self.bad.append((name, f"cardinality {cards[j]}, expected {card}"))
                if vals is not None and not np.array_equal(vals[j], v):
                    self.bad.append((name, "values differ"))
                if frozen is not None and frozen[j] != self.R.frozen_bytes(canon):
                    self.bad.append((name, "frozen bytes differ"))
            S.free()
            if int(self.L.rb200_device_bytes_in_use()) != before:
                self.bad.append((chunk[0][0], "device memory left behind"))

    def finish(self):
        # the library still works after every refusal
        S = _upload(self.rb, self.fmt, self.good, self.key_range)
        assert len(S.serialize_all()) == len(self.good)
        S.free()
        assert not self.bad, f"{self.fmt}: {len(self.bad)} disagreements with the reference: {self.bad}"


def _corpus(R, rb, fmt):
    cs = M.cases(R, fmt, rb)
    return cs, [M.verdict(R, fmt, b) for _, b in cs]


@pytest.mark.parametrize("fmt", M.FORMATS)
def test_device_upload_accepts_exactly_what_the_validator_accepts(rb, R, fmt):
    cs, vs = _corpus(R, rb, fmt)
    named = dict(cs)
    good = [named[g] for g in (GOOD64 if fmt == "r64" else GOOD)]
    if fmt == "frozen":
        good = [R.frozen_bytes(dict(M.bases(R))[g]) for g in GOOD]
    run = Run(rb, R, fmt, good)
    for (name, blob), v in zip(cs, vs):
        if v.kind != "valid":
            run.refuse(name, blob)
    run.accept([(name, blob, v.canon) for (name, blob), v in zip(cs, vs) if v.kind == "valid"])
    run.finish()


@pytest.mark.parametrize("key_range", KEY_RANGES)
def test_keyrange_upload_checks_only_the_containers_it_keeps(rb, R, key_range):
    """The key-range upload slices every blob on the host and parses the slices on the device, so its
    verdict is that of the cut: a bad container outside [lo, hi] is dropped unseen (accepted), while the
    slicer refuses a blob whose keys do not strictly increase wherever that happens."""
    cs = M.cases(R, "portable", rb)
    named = dict(cs)
    run = Run(rb, R, "keyrange", [named[g] for g in GOOD], key_range)
    accepted = []
    for name, blob in cs:
        v = M.keyrange_verdict(R, blob, *key_range)
        if v.kind == "valid":
            accepted.append((name, blob, v.canon))
        else:
            run.refuse(name, blob)
    run.accept(accepted)
    run.finish()
