"""A seeded corpus of serialized bitmaps, well formed and malformed, and the reference's verdict on each
— TEST INFRASTRUCTURE ONLY.

Every case is built from structure, not from random bytes alone: valid bases (both cookies, 1-3 containers
without an offset header and 4+ with one, the 32-container chunk edge, arrays and bitsets at the type
boundaries, runs at the top of a container, the largest run containers, real data), then one named
mutation each of a header field, a payload boundary or a container's contents, then a fixed number of the
random byte mutations of the host fuzz.  The names say what was changed and where, e.g.
`runs5/adjacent@c3` or `norun33/trunc@payload(c32)-1`.

    cases(R, fmt, rb=None)   -> [(name, blob)] for fmt in FORMATS, deterministic (rb adds real data)
    verdict(R, fmt, blob)    -> Verdict: refused by the parser, or parsed with validate's reason, or valid
    keyrange_verdict(R, blob, lo, hi) -> the same for the upload restricted to keys [lo, hi]

The reference is run only where it is safe: parse, validate, and serialization of what it parsed (a copy).
"""
import ctypes as C
import random
import struct
from collections import namedtuple

import numpy as np

from helpers import synth_blobs, synth_blobs64

SERIAL_COOKIE, SERIAL_COOKIE_NO_RUN, FROZEN_COOKIE = 12347, 12346, 13766
NO_OFFSET_THRESHOLD, MAX_ARRAY = 4, 4096
T_BITSET, T_ARRAY, T_RUN = 1, 2, 3          # the reference's typecodes, also those of the frozen format
FORMATS = ("portable", "frozen", "r64")
RANDOM_PER_FORMAT = 300
REALDATA = (("weather_sept_85", 3), ("census1881", 2), ("wikileaks-noquotes", 2), ("uscensus2000", 2))

Verdict = namedtuple("Verdict", "kind reason canon")   # kind: "refused" | "invalid" | "valid"
# canon: the reference's portable serialization of what it parsed ("valid" and, for 32-bit portable
# blobs, "invalid" too; None otherwise)

# A container as the corpus handles it: key, its header's cardinality - 1, whether it is flagged as a
# run container, and its payload bytes (a run container's includes its 2-byte run count).
Cont = namedtuple("Cont", "key cm1 isrun payload")


# ------------------------------------------------------------------------------ portable format
def parse(blob):
    """(run cookie?, [Cont]) of a well formed portable blob; trailing bytes are ignored."""
    cookie, = struct.unpack_from("<I", blob, 0)
    if cookie & 0xFFFF == SERIAL_COOKIE:
        n = (cookie >> 16) + 1
        flags = blob[4:4 + (n + 7) // 8]
        pos = 4 + (n + 7) // 8
        isrun = [bool(flags[i // 8] >> (i % 8) & 1) for i in range(n)]
        data = pos + 4 * n + (4 * n if n >= NO_OFFSET_THRESHOLD else 0)
        runc = True
    else:
        assert cookie == SERIAL_COOKIE_NO_RUN
        n, = struct.unpack_from("<I", blob, 4)
        pos, isrun, runc = 8, [False] * n, False
        data = pos + 8 * n
    out = []
    for i in range(n):
        key, cm1 = struct.unpack_from("<HH", blob, pos + 4 * i)
        if isrun[i]:
            nr, = struct.unpack_from("<H", blob, data)
            size = 2 + 4 * nr
        else:
            size = 8192 if cm1 + 1 > MAX_ARRAY else 2 * (cm1 + 1)
        out.append(Cont(key, cm1, isrun[i], bytes(blob[data:data + size])))
        data += size
    return runc, out


def header_bytes(runc, n):
    if runc:
        return 4 + (n + 7) // 8 + 4 * n + (4 * n if n >= NO_OFFSET_THRESHOLD else 0)
    return 8 + 8 * n


def write(runc, conts, offsets=None):
    """A portable blob of conts; with the run cookie when runc (which needs at least one container).
    offsets: bytes to put in place of the offset header (the reader must not trust it)."""
    n = len(conts)
    if runc:
        flags = bytearray((n + 7) // 8)
        for i, c in enumerate(conts):
            if c.isrun:
                flags[i // 8] |= 1 << (i % 8)
        head = struct.pack("<I", SERIAL_COOKIE | ((n - 1) << 16)) + bytes(flags)
        has_off = n >= NO_OFFSET_THRESHOLD
    else:
        head = struct.pack("<II", SERIAL_COOKIE_NO_RUN, n)
        has_off = True
    head += b"".join(struct.pack("<HH", c.key, c.cm1) for c in conts)
    if has_off:
        pos, offs = header_bytes(runc, n), []
        for c in conts:
            offs.append(struct.pack("<I", pos & 0xFFFFFFFF))
            pos += len(c.payload)
        head += offsets if offsets is not None else b"".join(offs)
    return head + b"".join(c.payload for c in conts)


def boundaries(runc, conts):
    """(label, byte offset) of every header field and container payload of write(runc, conts)."""
    n = len(conts)
    out = [("cookie", 4)]
    pos = 4
    if runc:
        pos += (n + 7) // 8
        out.append(("flags", pos))
    else:
        pos += 4
        out.append(("count", pos))
    pos += 4 * n
    out.append(("pairs", pos))
    if not runc or n >= NO_OFFSET_THRESHOLD:
        pos += 4 * n
        out.append(("offsets", pos))
    for i, c in enumerate(conts):
        if c.isrun:
            out.append((f"runcount(c{i})", pos + 2))
        pos += len(c.payload)
        out.append((f"payload(c{i})", pos))
    return out


def run_c(key, runs):
    runs = list(runs)
    return Cont(key, (sum(l + 1 for _, l in runs) - 1) & 0xFFFF, True,
                struct.pack("<H", len(runs)) + b"".join(struct.pack("<HH", s, l) for s, l in runs))


def array_c(key, vals):
    vals = list(vals)
    return Cont(key, len(vals) - 1, False, struct.pack(f"<{len(vals)}H", *vals))


def bitset_c(key, vals, cm1=None):
    words = np.zeros(1024, np.uint64)
    v = np.asarray(list(vals), dtype=np.uint64)
    np.bitwise_or.at(words, (v >> np.uint64(6)).astype(np.int64), np.uint64(1) << (v & np.uint64(63)))
    return Cont(key, len(v) - 1 if cm1 is None else cm1, False, words.tobytes())


def runs_of(c):
    nr, = struct.unpack_from("<H", c.payload, 0)
    return [struct.unpack_from("<HH", c.payload, 2 + 4 * k) for k in range(nr)]


# ------------------------------------------------------------------------------ frozen format
def frozen_write(conts, types=None):
    """roaring_bitmap_frozen_serialize's layout of conts: [bitset words | runs | array values | keys |
    counts | typecodes | header]; a container whose header cardinality exceeds 4096 is a bitset unless
    types (one typecode per container) says otherwise: only the frozen format can hold a bitset of 4096
    values or fewer."""
    kinds = types or [T_RUN if c.isrun else (T_BITSET if c.cm1 + 1 > MAX_ARRAY else T_ARRAY) for c in conts]
    zones = {T_BITSET: b"", T_RUN: b"", T_ARRAY: b""}
    counts = []
    for c, t in zip(conts, kinds):
        if t == T_RUN:
            zones[t] += c.payload[2:]
            counts.append(struct.unpack_from("<H", c.payload, 0)[0])
        else:
            zones[t] += c.payload
            counts.append(c.cm1)
    n = len(conts)
    return (zones[T_BITSET] + zones[T_RUN] + zones[T_ARRAY] + b"".join(struct.pack("<H", c.key) for c in conts)
            + struct.pack(f"<{n}H", *counts) + bytes(kinds)
            + struct.pack("<I", (n << 15) | FROZEN_COOKIE))


def frozen_tables(blob):
    """(n, offset of keys, offset of counts, offset of typecodes) of a well formed frozen blob."""
    n = struct.unpack_from("<I", blob, len(blob) - 4)[0] >> 15
    t0 = len(blob) - 4 - n
    return n, t0 - 4 * n, t0 - 2 * n, t0


# ------------------------------------------------------------------------------ bases (all valid)
def _ref_blob(R, vals, run_optimize):
    r = R.from_values(np.asarray(vals, dtype=np.uint32), run_optimize=run_optimize)
    b = R.serialize(r)
    R.free(r)
    return b


def _mixed(rng, keys):
    """One container per key, cycling run / array / bitset contents."""
    out = []
    for i, k in enumerate(keys):
        if i % 3 == 0:
            s = int(rng.integers(0, 60000))
            out.append(run_c(k, [(s, int(rng.integers(0, 3000)))]) if rng.random() < 0.5
                       else run_c(k, [(s // 2, 10), (s // 2 + 20, 5), (s // 2 + 40, 1000)]))
        elif i % 3 == 1:
            out.append(array_c(k, np.sort(rng.choice(65536, int(rng.integers(1, 300)), replace=False))))
        else:
            out.append(bitset_c(k, rng.choice(65536, int(rng.integers(4097, 30000)), replace=False)))
    return out


def bases(R, rb=None):
    """[(name, blob)] of valid portable blobs."""
    rng = np.random.default_rng(20261018)
    out = [("empty", _ref_blob(R, [], False)),
           ("array1", _ref_blob(R, [5], False)),
           ("array4096", _ref_blob(R, (3 << 16) + np.arange(0, 65536, 16), False)),
           ("bitset4097", _ref_blob(R, np.arange(0, 4097 * 3, 3), False)),
           ("bitset65536", _ref_blob(R, (2 << 16) + np.arange(65536), False)),
           ("fullrun", _ref_blob(R, (2 << 16) + np.arange(65536), True)),
           ("run1", _ref_blob(R, np.arange(100, 5100), True)),
           ("runend65535", _ref_blob(R, np.arange(60000, 65536), True)),
           ("keys0_65535", _ref_blob(R, np.concatenate([np.arange(0, 4000, 2), (65535 << 16) + np.arange(65000, 65536)]),
                                     True)),
           ("alt32768", write(True, [run_c(9, [(2 * i, 0) for i in range(32768)])])),
           ("arraymax", write(False, [array_c(0, range(65535 - 99, 65536))]))]
    for n in (1, 2, 3, 5, 33, 64):   # run cookie: 1-3 containers without an offset header, odd alignment
        out.append((f"runs{n}", write(True, _mixed(rng, sorted(rng.choice(4000, n, replace=False).tolist())))))
    for n in (2, 33, 64):
        conts = [c for c in _mixed(rng, sorted(rng.choice(65536, n, replace=False).tolist())) if not c.isrun]
        out.append((f"norun{len(conts)}", write(False, conts)))
    out.append(("norun33", write(False, [array_c(k, [k, k + 7]) for k in range(0, 66, 2)])))
    if rb is not None:
        for ds, k in REALDATA:
            for i, b in enumerate(rb.load_realdata(ds)[:k]):
                out.append((f"{ds}[{i}]", b))
    for i, b in enumerate(synth_blobs(R, 71, 4)):
        out.append((f"synth[{i}]", b))
    return out


# ------------------------------------------------------------------------------ 32-bit mutations
def _replace(conts, i, c):
    return conts[:i] + [c] + conts[i + 1:]


def _structural(name, blob):
    """Mutations of the header fields and payload boundaries of one base."""
    runc, conts = parse(blob)
    n = len(conts)
    out = []

    def put(mut, b):
        out.append((f"{name}/{mut}", bytes(b)))

    for k in range(4):
        b = bytearray(blob)
        b[k] ^= 0xA5
        put(f"cookie^b{k}", b)
    if runc:
        for cnt in sorted({n - 1, n + 1, 65536} - {n}):
            if 1 <= cnt <= 65536:
                put(f"count={cnt}", struct.pack("<I", SERIAL_COOKIE | ((cnt - 1) << 16)) + blob[4:])
        put("cookie=norun", struct.pack("<I", SERIAL_COOKIE_NO_RUN) + blob[4:])
    else:
        for cnt in sorted({0, n - 1, n + 1, 65536, 65537, 2 ** 32 - 1} - {n}):
            if cnt >= 0:
                put(f"count={cnt}", blob[:4] + struct.pack("<I", cnt) + blob[8:])
    picks = sorted({0, n - 1, 31, 32} & set(range(n)))
    for i in picks:
        c = conts[i]
        if runc:   # flag flips: an array or bitset read as runs, or runs read by the header's cardinality
            put(f"flag^@c{i}", write(True, _replace(conts, i, c._replace(isrun=not c.isrun))))
        if not c.isrun:
            for cm1 in sorted({4094, 4095, 4096, c.cm1 - 1, c.cm1 + 1} - {c.cm1}):
                if 0 <= cm1 <= 0xFFFF:
                    put(f"card={cm1 + 1}@c{i}", write(runc, _replace(conts, i, c._replace(cm1=cm1))))
        if c.isrun:
            for nr in (0, len(runs_of(c)) + 1, 0xFFFF):
                put(f"nruns={nr}@c{i}", write(runc, _replace(conts, i, c._replace(payload=struct.pack("<H", nr)
                                                                                    + c.payload[2:]))))
        if i > 0:
            put(f"key=prev@c{i}", write(runc, _replace(conts, i, c._replace(key=conts[i - 1].key))))
            sw = list(conts)
            sw[i - 1], sw[i] = sw[i], sw[i - 1]
            put(f"keys-swapped@c{i - 1}c{i}", write(runc, sw))
        if i + 1 < n and conts[i + 1].key > 0:
            put(f"key=next+1@c{i}", write(runc, _replace(conts, i, c._replace(key=min(65535, conts[i + 1].key + 1)))))
    if n and (not runc or n >= NO_OFFSET_THRESHOLD):
        rnd = random.Random(n * 7919 + len(blob))
        put("offsets=garbage", write(runc, conts, bytes(rnd.randrange(256) for _ in range(4 * n))))
    # the header fields, and the payloads of the first three and the last two containers
    ends = {0, 1, 2, n - 2, n - 1}
    cut = [(label, at) for label, at in boundaries(runc, conts)
           if "(c" not in label or int(label[label.index("(c") + 2:-1]) in ends]
    wb = write(runc, conts)
    for label, at in cut:
        for d in (-1, 0, 1):
            if 0 <= at + d < len(wb):
                put(f"trunc@{label}{d:+d}" if d else f"trunc@{label}", wb[:at + d])
    put("trailing+1", blob + b"\x00")
    put("trailing+garbage", blob + bytes(range(37, 77)))
    return out


def _content(name, blob):
    """Mutations of container contents that keep the layout well formed."""
    runc, conts = parse(blob)
    out = []

    def put(mut, i, c, rc=runc):
        out.append((f"{name}/{mut}@c{i}", write(rc, _replace(conts, i, c))))

    for i, c in enumerate(conts):
        if i not in (0, 3, len(conts) - 1, 32):
            continue
        if c.isrun:
            runs = runs_of(c)
            s, l = runs[-1]
            put("run-end=65535", i, run_c(c.key, runs[:-1] + [(s, 65535 - s)]))
            s = max(s, 1) if len(runs) == 1 else s   # a last run from 0 cannot reach 65536 in 16 bits
            put("run-end=65536", i, run_c(c.key, runs[:-1] + [(s, 65536 - s)]))
            if len(runs) >= 2:
                (s0, l0), (s1, l1) = runs[0], runs[1]
                put("adjacent", i, run_c(c.key, [(s0, l0), (s0 + l0 + 1, l1)] + runs[2:]))
                put("overlap", i, run_c(c.key, [(s0, l0), (s0 + l0, l1)] + runs[2:]))
                put("out-of-order", i, run_c(c.key, [runs[1], runs[0]] + runs[2:]))
            else:
                e = s + l
                if e + 2 <= 65535:
                    put("adjacent", i, run_c(c.key, [(s, l), (e + 1, min(5, 65535 - e - 1))]))
                if s > 3:
                    put("overlap", i, run_c(c.key, [(s, l), (s + l // 2, 0)] if l > 1 else [(s - 3, 5), (s, l)]))
        elif c.cm1 + 1 <= MAX_ARRAY:
            vals = list(struct.unpack(f"<{c.cm1 + 1}H", c.payload))
            if len(vals) >= 2:
                put("array-equal", i, array_c(c.key, vals[:1] + vals[:1] + vals[2:]))
                put("array-decreasing", i, array_c(c.key, vals[1:2] + vals[:1] + vals[2:]))
            if vals[-1] != 65535:
                put("array-last=65535", i, array_c(c.key, vals[:-1] + [65535]))
        else:
            words = bytearray(c.payload)
            bit = (c.key * 977 + 12345) % 65536
            words[bit >> 3] ^= 1 << (bit & 7)
            put("bit-flip", i, c._replace(payload=bytes(words)))
            for d in (-1, 1):
                if MAX_ARRAY <= c.cm1 + d <= 0xFFFF:
                    put(f"card{d:+d}", i, c._replace(cm1=c.cm1 + d))
    return out


def _targeted():
    """Content cases the bases do not reach by themselves: the issue's adjacent runs, a bitset whose header
    cardinality is half its popcount, runs adjacent across the 32-container chunk edge."""
    rng = np.random.default_rng(7)
    out = [("targeted/adjacent@c0", write(True, [run_c(0, [(0, 99), (100, 99)])])),
           ("targeted/adjacent-after-0@c0", write(True, [run_c(0, [(0, 0), (1, 0)])])),
           ("targeted/bitset-card5000-of-10000@c0", write(False, [bitset_c(1, range(0, 20000, 2), cm1=4999)])),
           ("targeted/zero-runs@c0", write(True, [Cont(4, 0, True, struct.pack("<H", 0))]))]
    conts = _mixed(rng, list(range(40)))
    out.append(("targeted/adjacent@c32", write(True, _replace(conts, 32, run_c(32, [(10, 9), (20, 4)])))))
    out.append(("targeted/bitset-card-1@c31", write(True, _replace(conts, 31, bitset_c(31, range(5000), cm1=4998)))))
    return out


def _random(blobs, seed, count, fmt):
    """The host fuzz's byte mutations: flips near the head or anywhere, truncations, garbage tails, splices."""
    rng = random.Random(seed)
    out = []
    for k in range(count):
        b = bytearray(rng.choice(blobs))
        mode = rng.randrange(5)
        if mode == 0:
            for _ in range(rng.randrange(1, 4)):
                b[rng.randrange(min(len(b), 64))] = rng.randrange(256)
        elif mode == 1:
            for _ in range(rng.randrange(1, 6)):
                b[rng.randrange(len(b))] = rng.randrange(256)
        elif mode == 2:
            b = b[:rng.randrange(len(b))]
        elif mode == 3:
            b += bytes(rng.randrange(256) for _ in range(rng.randrange(1, 40)))
        else:
            c = rng.choice(blobs)
            j = rng.randrange(len(b))
            b = b[:j] + c[rng.randrange(len(c)):]
        out.append((f"random/{fmt}#{k}-mode{mode}", bytes(b)))
    return out


def portable_cases(R, rb=None):
    base = bases(R, rb)
    out = list(base)
    for name, blob in base:
        out += _structural(name, blob) + _content(name, blob)
    out += _targeted()
    out += _random([b for _, b in base if 0 < len(b) < 40000], 20261018, RANDOM_PER_FORMAT, "portable")
    return out


# ------------------------------------------------------------------------------ frozen
def frozen_cases(R, rb=None):
    base = bases(R, rb)
    out = [(name, R.frozen_bytes(b)) for name, b in base]
    for name, blob in base:
        runc, conts = parse(blob)
        fz = R.frozen_bytes(blob)
        n = len(conts)
        assert frozen_write(conts) == fz, name   # the writer below lays blobs out as the reference does

        def put(mut, b):
            out.append((f"{name}/frozen/{mut}", bytes(b)))

        hdr, = struct.unpack_from("<I", fz, len(fz) - 4)
        put("cookie^", fz[:-4] + struct.pack("<I", hdr ^ 0x0101))
        put("cookie=0", fz[:-4] + b"\x00\x00\x00\x00")
        for d in (-1, 1):
            if n + d >= 0:
                put(f"nc{d:+d}", fz[:-4] + struct.pack("<I", ((n + d) << 15) | FROZEN_COOKIE))
        put("length+1", b"\x00" + fz)
        if len(fz) > 4:
            put("length-1", fz[1:])
        put("trunc@header", fz[:-4])
        _, k0, n0, t0 = frozen_tables(fz)
        for i in sorted({0, n - 1, 32} & set(range(n))):
            for t in (0, 4, 255):
                b = bytearray(fz)
                b[t0 + i] = t
                put(f"type={t}@c{i}", b)
            for d in (-1, 1):
                b = bytearray(fz)
                cnt, = struct.unpack_from("<H", b, n0 + 2 * i)
                struct.pack_into("<H", b, n0 + 2 * i, (cnt + d) & 0xFFFF)
                put(f"count{d:+d}@c{i}", b)
            if i > 0:
                b = bytearray(fz)
                b[k0 + 2 * i:k0 + 2 * i + 2] = b[k0 + 2 * i - 2:k0 + 2 * i]
                put(f"key=prev@c{i}", b)
        for cname, cblob in _content(name, blob):   # the same content mutations, frozen
            out.append((cname.replace("/", "/frozen/", 1), frozen_write(parse(cblob)[1])))
    # what only the frozen format can say: an array above 4096 values, a bitset at or below 4096
    out += [("frozen/array4096", frozen_write([array_c(2, range(0, 65536, 16))])),
            ("frozen/array4097", frozen_write([array_c(2, range(4097))], [T_ARRAY])),
            ("frozen/array5000", frozen_write([array_c(2, range(5000))], [T_ARRAY])),
            ("frozen/bitset4097", frozen_write([bitset_c(1, range(4097))])),
            ("frozen/bitset4096", frozen_write([bitset_c(1, range(4096))], [T_BITSET])),
            ("frozen/bitset-count9", frozen_write([bitset_c(1, range(10))], [T_BITSET])),
            ("frozen/bitset-count9-of-11", frozen_write([bitset_c(1, range(11), cm1=9)], [T_BITSET])),
            ("frozen/zero-runs", frozen_write([Cont(4, 0, True, struct.pack("<H", 0))]))]
    out += _random([b for _, b in out[:len(base)] if 0 < len(b) < 40000], 20261019, RANDOM_PER_FORMAT, "frozen")
    return out



# ------------------------------------------------------------------------------ 64-bit
EMPTY32 = struct.pack("<II", SERIAL_COOKIE_NO_RUN, 0)


def r64_write(buckets, count=None):
    """A 64-bit portable blob: u64 bucket count, then per bucket its high 32 bits and a 32-bit blob."""
    return struct.pack("<Q", len(buckets) if count is None else count) + b"".join(
        struct.pack("<I", h) + b for h, b in buckets)


def r64_parse(blob):
    n, = struct.unpack_from("<Q", blob, 0)
    pos, out = 8, []
    for _ in range(n):
        h, = struct.unpack_from("<I", blob, pos)
        runc, conts = parse(blob[pos + 4:])
        size = header_bytes(runc, len(conts)) + sum(len(c.payload) for c in conts)
        out.append((h, blob[pos + 4:pos + 4 + size]))
        pos += 4 + size
    return out


def r64_cases(R, rb=None):
    p32 = dict(bases(R, None))
    base = [(f"r64synth[{i}]", b) for i, b in enumerate(synth_blobs64(R, 47, 8))]
    base += [("r64/none", r64_write([])),
             ("r64/empty-bucket", r64_write([(0, p32["array1"]), (5, EMPTY32), (0xFFFFFFFF, p32["runs3"])])),
             ("r64/top", r64_write([(0xFFFFFFFF, p32["keys0_65535"])])),
             ("r64/wide", r64_write([(1, p32["runs33"]), (2, p32["norun33"]), (0x10000, p32["bitset65536"])]))]
    out = list(base)
    for name, blob in base:
        bk = r64_parse(blob)
        n = len(bk)

        def put(mut, b):
            out.append((f"{name}/{mut}", bytes(b)))

        for cnt in (0, n + 1, 2 ** 32):
            if cnt != n:
                put(f"count={cnt}", r64_write(bk, cnt))
        put("trailing+1", blob + b"\x00")
        put("trailing+garbage", blob + bytes(range(90, 110)))
        for i in sorted({0, n - 1} & set(range(n))):
            h, b32 = bk[i]
            put(f"trunc@bucket{i}-1", r64_write(bk[:i] + [(h, b32[:-1])]))
            put(f"trunc@high{i}", r64_write(bk[:i], n)[:8 + sum(4 + len(x) for _, x in bk[:i]) + 2])
            if i > 0:
                put(f"high=prev@b{i}", r64_write(_replace(bk, i, (bk[i - 1][0], b32))))
                put(f"high-decreasing@b{i}", r64_write(bk[:i - 1] + [(h, bk[i - 1][1]), (bk[i - 1][0], b32)]
                                                       + bk[i + 1:]))
    # a bucket whose contents only the device checks, at every position: the refusal names the 64-bit
    # bitmap, not the bucket
    bad32 = dict(_targeted())
    for what in ("targeted/adjacent@c0", "targeted/bitset-card5000-of-10000@c0", "targeted/adjacent@c32"):
        for i in (0, 2):
            bk = r64_parse(dict(base)["r64/empty-bucket"])
            out.append((f"r64/empty-bucket/{what.split('/')[1]}@b{i}", r64_write(_replace(bk, i, (bk[i][0], bad32[what])))))
    swapped = [c for c in _structural("norun33", p32["norun33"]) if "keys-swapped@c31c32" in c[0]][0][1]
    out.append(("r64/wide/keys-swapped@b1c31c32", r64_write([(1, p32["runs33"]), (2, swapped)])))
    out += _random([b for _, b in base if 8 < len(b) < 40000], 20261020, RANDOM_PER_FORMAT, "r64")
    return out


def cases(R, fmt, rb=None):
    """[(name, blob)] of one format; rb (the product package) adds the real-data bases."""
    return {"portable": portable_cases, "frozen": frozen_cases, "r64": r64_cases}[fmt](R, rb)


# ------------------------------------------------------------------------------ verdicts
def _aligned(blob):
    """A 32-byte aligned copy of blob (frozen_view reads in place): (keep-alive buffer, address)."""
    buf = C.create_string_buffer(len(blob) + 32)
    addr = (C.addressof(buf) + 31) & ~31
    C.memmove(addr, blob, len(blob))
    return buf, addr


def verdict(R, fmt, blob):
    """The reference's verdict on one blob: Verdict("refused", None, None) when its parser returns NULL,
    Verdict("invalid", reason, canon) when roaring_bitmap_internal_validate (roaring64_...) says why not,
    Verdict("valid", "", canon) otherwise.  canon: roaring_bitmap_portable_serialize of the parse (for
    frozen blobs, of the view) — also for invalid 32-bit bitmaps, where it is a copy of what was parsed."""
    L = R.L
    if fmt == "r64":
        r = L.roaring64_bitmap_portable_deserialize_safe(blob, len(blob))
        if not r:
            return Verdict("refused", None, None)
        why = C.c_char_p()
        ok = L.roaring64_bitmap_internal_validate(r, C.byref(why))
        out = Verdict("valid", "", R.r64_serialize(r)) if ok else Verdict("invalid", why.value.decode(), None)
        L.roaring64_bitmap_free(r)
        return out
    if fmt == "frozen":
        keep, addr = _aligned(blob)
        r = L.roaring_bitmap_frozen_view(addr, len(blob))
    else:
        r = L.roaring_bitmap_portable_deserialize_safe(blob, len(blob))
    if not r:
        return Verdict("refused", None, None)
    ok, why = R.validate(r)
    out = Verdict("valid" if ok else "invalid", why, R.serialize(r))
    R.free(r)
    return out


def keys_increase(v):
    """Did the parse keep its keys strictly increasing?  (validate checks keys before any container)"""
    return v.kind == "valid" or (v.kind == "invalid" and v.reason != "keys not strictly increasing")


def cut(canon, lo, hi):
    """The portable blob of the containers of keys [lo, hi] of a parsed bitmap's serialization."""
    runc, conts = parse(canon)
    keep = [c for c in conts if lo <= c.key <= hi]
    return write(runc and any(c.isrun for c in keep), keep)


def keyrange_verdict(R, blob, lo, hi):
    """The verdict of the upload of blob restricted to keys [lo, hi].  Unlike verdict(), it is that of the
    cut, not of the whole blob: the upload slices the blob on the host, which drops the containers outside
    the range unseen, so a bad container there does not matter.  The host slicer still needs the whole
    blob to parse with strictly increasing keys."""
    v = verdict(R, "portable", blob)
    if not keys_increase(v):
        return Verdict("refused", None, None)
    return verdict(R, "portable", cut(v.canon, lo, hi))
