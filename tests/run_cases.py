"""A catalogue of run-container cases placed on the thresholds of the code that handles them.

Bitmaps are written as portable blobs by hand (`run_blob`), so a run container can hold exactly the
runs a case names, optimal for its values or not: `R.from_values(..., run_optimize=True)` only ever
makes optimal ones.  Every container is `(key, "run", [(start, length - 1), ...])`,
`(key, "array", values)` or `(key, "bitset", values)`.

The thresholds (rb200_cells.cuh / rb200_device.cuh / rb200_many2.cu / rb200_compute.cu):
  * the interval sweep of a run cell runs when (runs or values of A) + (runs or values of B) <= 512;
    its merge path gives each lane ceil(T / 32) of the T boundaries, and a boundary of A equal to one
    of B (a tie) must be judged once, also when the two sit on either side of a lane split;
  * the rasteriser stores a range's interior words itself up to 8 words and with the whole warp above
    that, and clears the n + 1 gaps around n runs in stripes of 32;
  * the size rule of a run container: 2 + 4 n against 2 c and against 8192 bytes (2047 / 2048 runs);
  * the many-way union stages a container into a 32 KiB half when it has at most 8192 runs
    (4 bytes per run on the device) and reads a larger one from global memory;
  * a cell descriptor holds run counts in 16 bits: at most 32768 runs (alternating bits).
"""
import functools
import struct

import numpy as np

SERIAL_COOKIE = 12347
SERIAL_COOKIE_NO_RUN = 12346
NO_OFFSET_THRESHOLD = 4
MAX_ARRAY = 4096
KEY = 0   # the key of the single-container pairs


# ------------------------------------------------------------------------------ the blob writer
def _card(kind, body):
    return sum(l + 1 for _, l in body) if kind == "run" else len(body)


def _payload(kind, body):
    if kind == "run":
        return struct.pack("<H", len(body)) + b"".join(struct.pack("<HH", s, l) for s, l in body)
    vals = np.asarray(body, dtype=np.int64)
    if kind == "array":
        return vals.astype("<u2").tobytes()
    bits = np.zeros(65536, dtype=np.uint8)
    bits[vals] = 1
    return np.packbits(bits, bitorder="little").tobytes()


def check_container(c):
    """Raise ValueError unless c is a valid container: sorted values, runs sorted, non-overlapping,
    non-adjacent and inside the key, an array of 1..4096 values, a bitset of more than 4096."""
    key, kind, body = c
    if not 0 <= key <= 0xFFFF:
        raise ValueError(f"key {key}")
    if kind == "run":
        if not body:
            raise ValueError("empty run container")
        prev_end = -2
        for s, l in body:
            if s <= prev_end + 1 or l < 0 or s + l > 0xFFFF:
                raise ValueError(f"run ({s}, {l}) after end {prev_end}")
            prev_end = s + l
        return
    v = np.asarray(body, dtype=np.int64)
    if v.size == 0 or np.any(np.diff(v) <= 0) or v[0] < 0 or v[-1] > 0xFFFF:
        raise ValueError(f"{kind}: values must be sorted, distinct, in [0, 65535]")
    if (kind == "array") != (v.size <= MAX_ARRAY):
        raise ValueError(f"{kind} of {v.size} values: the portable format decides by cardinality")


def run_blob(containers):
    """Portable serialization of a bitmap given container by container, as roaring_array.c writes it:
    with a run container, cookie 12347 | (size - 1) << 16, the run-flag bitset, key / card - 1 pairs
    and an offset header only from 4 containers on; without one, cookie 12346, the count, the pairs
    and the offset header."""
    cs = sorted(containers, key=lambda c: c[0])
    for c in cs:
        check_container(c)
    if len({c[0] for c in cs}) != len(cs):
        raise ValueError("duplicate key")
    n = len(cs)
    pays = [_payload(kind, body) for _, kind, body in cs]
    pairs = b"".join(struct.pack("<HH", key, _card(kind, body) - 1) for key, kind, body in cs)
    hasrun = any(kind == "run" for _, kind, _ in cs)
    if hasrun:
        flags = bytearray((n + 7) // 8)
        for i, (_, kind, _) in enumerate(cs):
            if kind == "run":
                flags[i // 8] |= 1 << (i % 8)
        head = struct.pack("<I", SERIAL_COOKIE | ((n - 1) << 16)) + bytes(flags) + pairs
        with_offsets = n >= NO_OFFSET_THRESHOLD
    else:
        head = struct.pack("<II", SERIAL_COOKIE_NO_RUN, n) + pairs
        with_offsets = True
    if with_offsets:
        off = len(head) + 4 * n
        offs = []
        for p in pays:
            offs.append(struct.pack("<I", off))
            off += len(p)
        head += b"".join(offs)
    return head + b"".join(pays)


def blob_containers(blob):
    """(key, type, cardinality, runs or None) of every container of a portable blob (either cookie)."""
    cookie, = struct.unpack_from("<I", blob, 0)
    if cookie & 0xFFFF == SERIAL_COOKIE:
        n = (cookie >> 16) + 1
        flags = blob[4:4 + (n + 7) // 8]
        pos = 4 + (n + 7) // 8
        isrun = [bool(flags[i // 8] >> (i % 8) & 1) for i in range(n)]
        data = pos + 4 * n + (4 * n if n >= NO_OFFSET_THRESHOLD else 0)
    else:
        assert cookie == SERIAL_COOKIE_NO_RUN
        n, = struct.unpack_from("<I", blob, 4)
        pos, isrun = 8, [False] * n
        data = pos + 8 * n
    out = []
    for i in range(n):
        key, cm1 = struct.unpack_from("<HH", blob, pos + 4 * i)
        card = cm1 + 1
        if isrun[i]:
            nr, = struct.unpack_from("<H", blob, data)
            out.append((key, "run", card, nr))
            data += 2 + 4 * nr
        elif card > MAX_ARRAY:
            out.append((key, "bitset", card, None))
            data += 8192
        else:
            out.append((key, "array", card, None))
            data += 2 * card
    assert data == len(blob), "trailing bytes"
    return out


# ------------------------------------------------------------------------------ building blocks
def run(body, key=KEY):
    return (key, "run", [(int(s), int(l)) for s, l in body])


def array(vals, key=KEY):
    return (key, "array", [int(v) for v in vals])


def bitset(vals, key=KEY):
    return (key, "bitset", [int(v) for v in vals])


def values_of(c):
    """Sorted low-16 values of a container."""
    _, kind, body = c
    if kind == "run":
        return np.concatenate([np.arange(s, s + l + 1) for s, l in body]).astype(np.int64)
    return np.asarray(body, dtype=np.int64)


def runs_of(vals):
    """The maximal runs of sorted distinct values."""
    v = np.asarray(vals, dtype=np.int64)
    if v.size == 0:
        return []
    cut = np.flatnonzero(np.diff(v) != 1) + 1
    starts, ends = np.r_[v[:1], v[cut]], np.r_[v[cut - 1], v[-1:]]
    return [(int(s), int(e - s)) for s, e in zip(starts, ends)]


def intervals(c):
    """Interval boundaries {start, end + 1} the sweep builds from a run or array container."""
    if c[1] == "run":
        body = c[2]
    else:
        body = runs_of(c[2])
    return [x for s, l in body for x in (s, s + l + 1)]


def interval_total(left, right):
    """(runs or values of A) + (runs or values of B), the number the sweep's cutoff compares."""
    n = lambda c: len(c[2])
    return n(left) + n(right)


def merged_boundaries(left, right):
    """The merge of both boundary lists as the sweep orders it (A first on equal values)."""
    a = [(x, 0) for x in intervals(left)]
    b = [(x, 1) for x in intervals(right)]
    return [x for x, _ in sorted(a + b)]


def split_ties(left, right):
    """Lane splits d (multiples of per = ceil(T / 32)) with an equal boundary on both sides."""
    m = merged_boundaries(left, right)
    per = (len(m) + 31) // 32
    return [d for d in range(per, len(m), per) if m[d - 1] == m[d]]


def alternating(parity=0, n=32768):
    """n single-value runs on every other value, starting at `parity`."""
    return run([(parity + 2 * i, 0) for i in range(n)])


def singles(n, stride=4, first=0):
    return run([(first + stride * i, 0) for i in range(n)])


def full_run(key=KEY):
    return run([(0, 65535)], key)


# ------------------------------------------------------------------------------ the named pairs
def _word_edges():
    """Runs at the word edges of the rasteriser: on bit 0 / bit 31 of a word, a whole word, inside
    one word, interiors of 7 / 8 / 9 whole words, a long range from bit 0 to bit 31, and an interior
    longer than the warp."""
    return run([
        (64, 0), (127, 0), (160, 31), (230, 3),
        (32 * 10 + 5, 32 * 19 + 3 - (32 * 10 + 5)),     # interior 8 words (11 .. 18)
        (32 * 25 + 7, 32 * 35 + 2 - (32 * 25 + 7)),     # interior 9 words (26 .. 34)
        (32 * 40 + 1, 32 * 48 + 30 - (32 * 40 + 1)),    # interior 7 words
        (32 * 50, 32 * 70 + 31 - 32 * 50),               # bit 0 .. bit 31, 19 interior words
        (32 * 100 + 3, 32 * 140 + 4 - (32 * 100 + 3)),  # 39 interior words
        (65535, 0),
    ])


def _gapped(n, touch_ends):
    """n runs whose gaps are ~1000 values (31 whole words): acc_and_runs clears n + 1 gaps, the
    first and last empty when the runs touch 0 and 65535."""
    if touch_ends:
        step = 65535 // (n - 1) if n > 1 else 0
        body = [(0, 499)] + [(step * i, 499) for i in range(1, n - 1)] + [(65535 - 499, 499)]
    else:
        body = [(700 + 1900 * i, 899) for i in range(n)]
    return run(body)


def _ties(n, kind):
    """n runs on each side whose boundaries all coincide pairwise (see split_ties)."""
    if kind == "end_start":    # A's end + 1 is B's start and B's end + 1 A's next start
        return run([(10 * j, 4) for j in range(n)]), run([(10 * j + 5, 4) for j in range(n)])
    if kind == "start":
        return run([(10 * j, 4) for j in range(n)]), run([(10 * j, 2) for j in range(n)])
    return run([(10 * j, 4) for j in range(n)]), run([(10 * j + 2, 2) for j in range(n)])   # equal ends


def _rng_bitset(rng, n, exclude=None):
    pool = np.arange(65536) if exclude is None else np.setdiff1d(np.arange(65536), exclude)
    return bitset(np.sort(rng.choice(pool, n, replace=False)))


def _cutoff_cases(t):
    """Cells whose interval total is t (511 / 512 / 513), named by the type of the result the
    meta['expect'] op gives."""
    cs = []
    # run x run, result a run: overlapping runs of 10 values
    cs.append((f"cut{t}_rr_run", run([(64 * i, 9) for i in range(256)]),
               run([(64 * i + 5, 9) for i in range(t - 256)]), {"total": t, "expect": ("or", "run")}))
    # run x run, result an array: single-value runs interleaved
    cs.append((f"cut{t}_rr_array", run([(4 * i, 0) for i in range(256)]),
               run([(4 * i + 2, 0) for i in range(t - 256)]), {"total": t, "expect": ("or", "array")}))
    # array x run, result a run: 4096 values in 256 runs, array values in the gaps and inside
    av = [64 * i + (32 if i % 3 else 7) for i in range(t - 256)]
    cs.append((f"cut{t}_ar_run", array(av), run([(64 * i, 15) for i in range(256)]),
               {"total": t, "expect": ("or", "run")}))
    # array x run, result an array: a run container of 512 values
    cs.append((f"cut{t}_ar_array", array([16 * i + 8 for i in range(t - 256)]),
               run([(16 * i, 1) for i in range(256)]), {"total": t, "expect": ("or", "array")}))
    # array x run with more than 4096 run values: xor is judged a bitset, the sweep hands back
    cs.append((f"cut{t}_ar_bitset", array([200 * i + (100 if i % 2 else 10) for i in range(t - 300)]),
               run([(200 * i, 19) for i in range(300)]), {"total": t, "expect": ("xor", "bitset")}))
    return cs


def pair_cases():
    """[(name, left container, right container, meta)], every container on key 0.  meta names what
    the CPU check verifies: 'total' (interval total), 'runs' (left, right run counts), 'tie'
    (an equal boundary of A and B), 'split_tie' (an equal pair across a lane split), 'expect'
    ((op, type) of the reference's result)."""
    rng = np.random.default_rng(20261016)
    cs = []
    for t in (511, 512, 513):
        cs += _cutoff_cases(t)

    # ---- boundary ties
    cs.append(("tie_end_start", run([(100, 99), (1000, 9)]), run([(200, 99), (2000, 9)]),
               {"tie": 200, "expect": ("or", "run")}))
    cs.append(("tie_equal_start", run([(100, 99), (500, 9)]), run([(100, 49), (600, 9)]), {"tie": 100}))
    cs.append(("tie_equal_end", run([(100, 99), (500, 9)]), run([(150, 49), (700, 9)]), {"tie": 200}))
    cs.append(("tie_array_run", array(range(200, 210)), run([(100, 99), (210, 5)]), {"tie": 200}))
    for kind, n in (("end_start", 64), ("start", 72), ("end", 72)):
        a, b = _ties(n, kind)
        cs.append((f"tie_split_{kind}", a, b, {"split_tie": True}))

    # ---- container ends
    cs.append(("end_single_0", run([(0, 0), (9, 5)]), run([(1, 20)]), {"tie": 1}))
    cs.append(("end_single_65535", run([(65535, 0)]), run([(65530, 4)]), {"tie": 65535}))
    cs.append(("end_to_65535", run([(65000, 535)]), run([(100, 0), (65500, 35)]), {"tie": 65536}))
    cs.append(("end_to_65535_array", run([(65000, 535)]), array([0, 64999, 65535]), {"tie": 65536}))
    cs.append(("full_run_run", full_run(), run([(0, 0), (65535, 0)]), {}))
    cs.append(("full_run_array", full_run(), array(np.sort(rng.choice(65536, 300, replace=False))), {}))
    cs.append(("full_run_bitset", full_run(), _rng_bitset(rng, 30000), {}))
    cs.append(("full_run_full_run", full_run(), full_run(), {}))

    # ---- word edges of the rasteriser, against every partner type
    we = _word_edges()
    cs.append(("words_bitset", we, _rng_bitset(rng, 33000), {}))
    cs.append(("words_array", we, array(np.sort(rng.choice(8192, 2000, replace=False))), {}))
    cs.append(("words_run", we, run([(0, 31), (96, 96), (32 * 30, 32 * 9 + 31), (32 * 120, 4000)]), {}))
    for n in (31, 32, 33):
        for ends in (False, True):
            cs.append((f"gaps{n}_{'ends' if ends else 'inner'}_bitset", _gapped(n, ends), _rng_bitset(rng, 40000),
                       {"runs": (n, None)}))
        cs.append((f"gaps{n}_run", _gapped(n, True), run([(32 * i, 700) for i in range(0, 2040, 24)]),
                   {"runs": (n, None)}))

    # ---- large run containers
    for n in (2047, 2048):   # runs of 3 values: card > 4096, the size rule's bitset tie
        big = run([(32 * i, 2) for i in range(n)])
        cs.append((f"runs{n}_run", big, run([(32 * i + 1, 2) for i in range(0, n, 2)]), {"runs": (n, None)}))
        cs.append((f"runs{n}_bitset", big, _rng_bitset(rng, 20000), {"runs": (n, None)}))
        cs.append((f"runs{n}_array", big, array(np.arange(0, 65536, 37)[:1500]), {"runs": (n, None)}))
    for n in (8192, 8193):
        cs.append((f"runs{n}_run", singles(n), singles(n, first=2), {"runs": (n, n)}))
        cs.append((f"runs{n}_bitset", singles(n), _rng_bitset(rng, 9000), {"runs": (n, None)}))
    even, odd = alternating(0), alternating(1)
    cs.append(("runs32768_complement", even, odd, {"runs": (32768, 32768), "expect": ("or", "run")}))
    cs.append(("runs32768_self", even, even, {"runs": (32768, 32768)}))
    cs.append(("runs32768_bitset", even, _rng_bitset(rng, 50000), {"runs": (32768, None)}))
    cs.append(("runs32768_array", even, array(np.arange(0, 65536, 17)[:4000]), {"runs": (32768, None)}))
    cs.append(("runs32768_run", even, _word_edges(), {"runs": (32768, None)}))

    # ---- run x bitset, every op
    holes = run([(0, 999), (5000, 24999), (40000, 9), (65000, 535)])
    cs.append(("rb_saturate", holes, bitset(np.setdiff1d(np.arange(65536), values_of(holes))),
               {"expect": ("or", "bitset")}))
    cs.append(("rb_mixed", run([(300 * i, 149) for i in range(200)]), _rng_bitset(rng, 25000), {}))
    cs.append(("rb_small_run", run([(7, 0), (4000, 2)]), _rng_bitset(rng, 6000), {}))

    # ---- run containers that are not the optimal encoding of their values
    cs.append(("nonopt_singles_array", run([(5, 0), (90, 0), (700, 0)]), array([5, 6, 91, 699, 700, 701]), {}))
    cs.append(("nonopt_pairs_run", run([(2 * i * 2, 1) for i in range(300)]), run([(3, 0), (1000, 3000)]), {}))
    return cs


def multi_key_bitmaps():
    """Named bitmaps over keys 0 .. 5 mixing the containers above (four or more containers: the run
    cookie with an offset header), and one without runs."""
    rng = np.random.default_rng(7)
    bs = lambda k, n: (k, "bitset", np.sort(rng.choice(65536, n, replace=False)).tolist())
    return [
        ("multi_a", [(0, *_word_edges()[1:]), bs(1, 20000), full_run(2), (3, "array", list(range(0, 4000, 3))),
                     (5, "run", [(32 * i, 2) for i in range(2048)])]),
        ("multi_b", [bs(0, 30000), (1, "run", [(2 * i, 0) for i in range(32768)]), (2, "array", [7, 65535]),
                     (3, "run", [(10 * j, 4) for j in range(72)]), (4, "run", [(0, 0), (65535, 0)])]),
        ("multi_c", [(0, "run", [(10 * j + 5, 4) for j in range(64)]), (2, "run", [(4 * i, 0) for i in range(8193)]),
                     (5, "run", [(0, 65535)])]),
        ("multi_norun", [bs(0, 5000), (1, "array", [1, 2, 3]), bs(4, 60000), (5, "array", list(range(100, 4196)))]),
    ]


@functools.lru_cache(maxsize=None)
def catalogue():
    """(pairs, bitmaps): pairs = [(name, left blob, right blob)] with every named pair in both orders
    and the multi-key pairs; bitmaps = [(name, blob)], every distinct operand once."""
    pairs, seen = [], {}
    for name, a, b, _ in pair_cases():
        ba, bb = run_blob([a]), run_blob([b])
        pairs.append((name, ba, bb))
        pairs.append((name + "_swapped", bb, ba))
        seen.setdefault(ba, name + ".left")
        seen.setdefault(bb, name + ".right")
    multi = [(n, run_blob(c)) for n, c in multi_key_bitmaps()]
    for i, (na, ba) in enumerate(multi):
        for nb, bb in multi[i + 1:] + multi[:i]:
            pairs.append((f"{na}_x_{nb}", ba, bb))
        seen.setdefault(ba, na)
    return pairs, [(n, b) for b, n in seen.items()]


# ------------------------------------------------------------------------------ many-way inputs
def _sweep_container(rng, key, kind):
    if kind == "run8193":
        return (key, "run", [(4 * i + int(rng.integers(0, 3)), 0) for i in range(8193)])
    if kind == "run8192":
        return (key, "run", [(4 * i + 1, 0) for i in range(8192)])
    if kind == "run32768":
        return (key, "run", [(2 * i + 1, 0) for i in range(32768)])
    if kind == "run2048":
        off = int(rng.integers(0, 29))
        return (key, "run", [(32 * i + off, 2) for i in range(2048)])
    if kind == "run2047":
        return (key, "run", [(32 * i + 5, 2) for i in range(2047)])
    if kind == "runs":
        s = np.sort(rng.choice(np.arange(0, 65536, 64), int(rng.integers(1, 200)), replace=False))
        return (key, "run", [(int(x), int(rng.integers(0, 62))) for x in s])
    if kind == "bitset":
        return (key, "bitset", np.sort(rng.choice(65536, int(rng.integers(4097, 40000)), replace=False)).tolist())
    if kind == "array":
        return (key, "array", np.sort(rng.choice(65536, int(rng.integers(1, 4097)), replace=False)).tolist())
    if kind == "full_run":
        return full_run(key)
    return (key, "bitset", list(range(65536)))   # full bitset


HEAVY = ["bitset", "bitset", "run8193", "run32768", "run2048", "run8192", "full_bitset", "array", "run2047"]
LIGHT = ["array", "array", "array", "runs", "runs", "run8193", "bitset", "run2047", "full_run"]


@functools.lru_cache(maxsize=None)
def sweep_lists():
    """[(name, [blob, ...])]: seeded lists of 20 .. 300 bitmaps over keys 0 .. 3.  The heavy lists
    average more than 7 KiB per container (the many-way union stages them by bulk copies unless told
    otherwise), the light ones less.  'acc2' puts, on key 0, two arrays, a bitset and then a run
    container of 8193 runs: the bitset is the last in-place bitset step L of key 0, so the oversized
    run lands in the second accumulator."""
    out = []
    for li, (n, mix, keys) in enumerate([(20, HEAVY, 2), (60, HEAVY, 4), (300, HEAVY, 3),
                                         (40, LIGHT, 4), (200, LIGHT, 3)]):
        rng = np.random.default_rng(1000 + li)
        blobs = []
        for _ in range(n):
            ks = np.sort(rng.choice(keys, int(rng.integers(1, keys + 1)), replace=False))
            blobs.append(run_blob([_sweep_container(rng, int(k), str(rng.choice(mix))) for k in ks]))
        out.append((f"{'heavy' if mix is HEAVY else 'light'}{n}", blobs))
    rng = np.random.default_rng(999)
    head = [[(0, "array", [1, 2, 3, 70]), _sweep_container(rng, 1, "bitset")],
            [(0, "array", list(range(1000, 1100))), _sweep_container(rng, 2, "run8193")],
            [(0, "bitset", list(range(20000, 30000)))],
            [(0, "run", [(4 * i + 2, 0) for i in range(8193)]), _sweep_container(rng, 1, "run32768")]]
    tail = [[_sweep_container(rng, int(k), str(rng.choice(["array", "runs", "run8193"])))
             for k in (1, 2)] for _ in range(24)]
    out.append(("acc2", [run_blob(c) for c in head + tail]))
    return out
