"""A catalogue of bitmaps with long directories and keys at the top of the key space.

The device code walks directories and key spaces in chunks: plans of 256 items in the single-pair
fused kernel (up to 512 containers, then the batched path), 32 containers per warp round in the
planner, finalize, pack and serializers, 1024 keys per round in the xor_many directory compaction,
512 inputs per gather round in the xor_many fold, 4096-key tiles in the many-way union's index, and
16-bit keys whose last value is 65535.  Every case here sits on one of those edges, under a name
that says which.

All blobs are written by the reference (`R`, oracle/refbind.py), seeded.  Most containers hold 1-3
values to keep payloads small; every few keys one holds an array, a bitset, a run, a full run or a
full bitset instead.  A bitmap is the union of a run-optimized part and a plain part on disjoint
keys, so it can hold runs and full bitsets side by side."""
import functools

import numpy as np

TILE = 4096
LENS = (1, 31, 32, 33, 63, 64, 65, 255, 256, 257, 1023, 1024, 1025)
FUSED = (256, 257, 511, 512, 513)
MANY = (511, 512, 513, 1025)
TOP_FORMS = ("array", "run_end", "full_run", "full_bitset", "bitset")
HEAVY = ("array", "bitset", "run", "full_run", "full_bitset")
# the keys every many-way list shares: the first and last key of every tile, and a few more
TILE_EDGES = tuple(k for t in range(16) for k in (t * TILE, t * TILE + TILE - 1))
POOL = tuple(sorted(set(TILE_EDGES) | {1, 4094, 30000, 32767, 32768, 61441, 65534}))
REPEAT = (3, 515, 700)   # list_1025: x[515] is x[3]; x[700] re-inserts the key the two cancel


# ------------------------------------------------------------------------------ building blocks
def _heavy(rng, kind):
    """(run-optimized?, low values) of a container of one of the HEAVY kinds."""
    if kind == "array":
        return False, rng.choice(65536, 200, replace=False)
    if kind == "bitset":
        return False, rng.choice(65536, 5000, replace=False)
    if kind == "run":
        s = int(rng.integers(0, 50000))
        return True, np.r_[np.arange(s, s + 3000), np.arange(s + 4000, s + 4500)]
    return kind == "full_run", np.arange(65536)


def _tiny(rng, keys):
    """1-3 random values in each of keys (as uint32 values)."""
    keys = np.asarray(keys, dtype=np.uint32)
    lows = rng.integers(0, 65536, (keys.size, 3)).astype(np.uint32)
    keep = np.arange(3)[None, :] < rng.integers(1, 4, keys.size)[:, None]
    return ((keys[:, None] << np.uint32(16)) | lows)[keep]


def assemble(R, runs, plain):
    """Portable bytes of the union of roaring_bitmap_of_ptr(runs) run-optimized and
    roaring_bitmap_of_ptr(plain) as built; the two must not share a key."""
    a = R.from_values(np.asarray(runs, np.uint32), run_optimize=True)
    b = R.from_values(np.asarray(plain, np.uint32), run_optimize=False)
    R.L.roaring_bitmap_or_inplace(a, b)
    out = R.serialize(a)
    R.free(a)
    R.free(b)
    return out


def mixed(R, rng, keys, every=16, fixed=None):
    """A bitmap with one container on each of keys: 1-3 values in most, one of HEAVY in turn on every
    `every`-th key (from a seeded start), and fixed = {key: (run-optimized?, low values)} as given."""
    keys = np.unique(np.asarray(keys, dtype=np.int64))
    fixed = dict(fixed or {})
    if every:
        start = int(rng.integers(0, every))
        for i, k in enumerate(keys[start::every]):
            fixed.setdefault(int(k), _heavy(rng, HEAVY[i % len(HEAVY)]))
    runs, plain = [], [_tiny(rng, [k for k in keys if int(k) not in fixed])]
    for k, (opt, lows) in fixed.items():
        (runs if opt else plain).append((np.uint32(k) << np.uint32(16)) | np.asarray(lows, np.uint32))
    cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.uint32)
    return assemble(R, cat(runs), cat(plain))


def _spread(rng, n):
    """n distinct keys spread over the whole key space, 0 and 65535 among them when n >= 2."""
    if n == 1:
        return np.array([int(rng.integers(0, 65536))])
    return np.r_[0, 65535, rng.choice(np.arange(1, 65535), n - 2, replace=False)]


def universe(R, keys):
    """Portable bytes of a bitmap holding every value of the given keys: full run containers
    (roaring_bitmap_add_range_closed), cardinality 65536 per key."""
    r = R.L.roaring_bitmap_create_with_capacity(0)
    keys = list(keys)
    if keys == list(range(65536)):
        R.L.roaring_bitmap_add_range_closed(r, 0, 0xFFFFFFFF)
    else:
        for k in keys:
            R.L.roaring_bitmap_add_range_closed(r, k << 16, (k << 16) | 0xFFFF)
    out = R.serialize(r)
    R.free(r)
    return out


# ------------------------------------------------------------------------------ the cases
def _top(R, rng, form):
    """Keys 65500-65535; key 65535 holds an array with 0xFFFFFFFF, a run ending at 65535, a full run,
    a full bitset (not run-optimized) or an ordinary bitset with 0xFFFF."""
    last = {"array": (False, [0, 7, 0xFFFF]),
            "run_end": (True, np.arange(60000, 65536)),
            "full_run": (True, np.arange(65536)),
            "full_bitset": (False, np.arange(65536)),
            "bitset": (False, np.r_[rng.choice(65535, 5000, replace=False), 0xFFFF])}[form]
    return mixed(R, rng, np.arange(65500, 65536), every=5, fixed={65535: last})


@functools.lru_cache(maxsize=None)
def bitmaps(R):
    """[(name, blob)]: top_<form>, all_keys, even_keys, odd_keys, len_<N>, tiles, full_universe,
    half_universe."""
    rng = np.random.default_rng(20261017)
    out = [(f"top_{f}", _top(R, rng, f)) for f in TOP_FORMS]
    out.append(("all_keys", mixed(R, rng, np.arange(65536), every=2048)))
    out.append(("even_keys", mixed(R, rng, np.arange(0, 65536, 2), every=2048)))
    out.append(("odd_keys", mixed(R, rng, np.arange(1, 65536, 2), every=2048)))
    for n in LENS:
        out.append((f"len_{n}", mixed(R, rng, _spread(rng, n), every=8)))
    out.append(("tiles", mixed(R, rng, TILE_EDGES, every=3)))
    out.append(("full_universe", universe(R, range(65536))))
    out.append(("half_universe", universe(R, range(0, 65536, 2))))
    return tuple(out)


def bitmap(R, name):
    return dict(bitmaps(R))[name]


@functools.lru_cache(maxsize=None)
def fused_pairs(R):
    """[(name, a, b)]: fused_<T>, two operands holding T containers together (5/8 of them in a),
    with matched keys (a quarter of them equal containers, so AND and XOR drop keys) and one-sided
    keys; key 65535 is matched."""
    rng = np.random.default_rng(512)
    out = []
    for t in FUSED:
        na = (5 * t) // 8
        nb = t - na
        m = nb // 2
        pool = np.r_[65535, rng.choice(65535, na + nb - m - 1, replace=False)]
        a_keys, b_keys = pool[:na], np.r_[pool[:m], pool[na:]]
        a = mixed(R, rng, a_keys, every=16)
        same = {int(k) for k in pool[:m:4]}
        # b: its own containers, except the equal ones copied from a's values
        ra = R.deserialize(a)
        va = R.to_array(ra)
        R.free(ra)
        keep = np.isin(va >> np.uint32(16), np.array(sorted(same), dtype=np.uint32))
        b_own = mixed(R, rng, [k for k in b_keys if int(k) not in same], every=16)
        rb_ = R.deserialize(b_own)
        vb = np.r_[R.to_array(rb_), va[keep]]
        R.free(rb_)
        b = R.from_values(np.sort(vb), run_optimize=True)
        out.append((f"fused_{t}", a, R.serialize(b)))
        R.free(b)
    return tuple(out)


def _small(rng, keys):
    """Values of a small many-way input: 1-3 values drawn from 0..15 in each of keys (inputs collide
    and cancel under XOR)."""
    keys = np.asarray(keys, dtype=np.uint32)
    lows = rng.integers(0, 16, (keys.size, 3)).astype(np.uint32)
    keep = np.arange(3)[None, :] < rng.integers(1, 4, keys.size)[:, None]
    return ((keys[:, None] << np.uint32(16)) | lows)[keep]


@functools.lru_cache(maxsize=None)
def many_lists(R):
    """[(name, blobs)]: list_<n> for n in MANY, small inputs on 2-6 keys of POOL (which holds key
    65535 and the first and last key of every tile), every 64th input with a bitset, a run or a full
    container on one of them.  list_1025 also gives each input a key of its own, so its XOR has more
    than 1024 keys; its x[515] is x[3], and x[700] holds x[3]'s own key again.  list_all_keys: 513
    inputs, input i on the keys k = i (mod 513) and on key 65535, so every key reaches the XOR."""
    rng = np.random.default_rng(65535)
    pool = np.array(POOL)
    own = rng.permutation(np.setdiff1d(np.arange(65536), pool))[:1025]
    out = []
    for n in MANY:
        blobs = []
        for i in range(n):
            keys = rng.choice(pool, int(rng.integers(2, 7)), replace=False)
            fixed = {}
            if i % 64 == 5:
                fixed[int(keys[0])] = _heavy(rng, HEAVY[(i // 64) % len(HEAVY)])
            if n == 1025:
                keys = np.r_[keys, own[i]]
                if i == REPEAT[2]:
                    keys = np.r_[keys, own[REPEAT[0]]]
            rest = [k for k in keys if int(k) not in fixed]
            runs = [(np.uint32(k) << np.uint32(16)) | np.asarray(l, np.uint32) for k, (o, l) in fixed.items() if o]
            plain = [_small(rng, rest)] + [(np.uint32(k) << np.uint32(16)) | np.asarray(l, np.uint32)
                                           for k, (o, l) in fixed.items() if not o]
            blobs.append(assemble(R, np.concatenate(runs) if runs else [], np.concatenate(plain)))
        if n == 1025:
            blobs[REPEAT[1]] = blobs[REPEAT[0]]
        out.append((f"list_{n}", tuple(blobs)))
    blobs = []
    for i in range(513):
        keys = np.arange(i, 65535, 513)
        v = np.r_[_tiny(rng, keys), np.uint32(0xFFFF0000) | np.uint32(i)]
        blobs.append(assemble(R, [], np.unique(v)))
    out.append(("list_all_keys", tuple(blobs)))
    return tuple(out)


def many_list(R, name):
    return dict(many_lists(R))[name]
