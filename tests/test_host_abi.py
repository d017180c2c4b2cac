"""CPU tests (-m "not gpu"): the C-ABI library loads, exports every symbol declared in
include/roaring_b200.h, its host-side logic (layout, portable format, validation) agrees with
the reference — and compute entry points fail loudly without a GPU (no CPU fallback)."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import croaring_b200 as rb
from helpers import synth_blobs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exports_match_header():
    hdr = open(os.path.join(ROOT, "include", "roaring_b200.h")).read()
    declared = set(re.findall(r"\b((?:roaring_bitmap|roaring64_bitmap|rb200)_[a-z0-9_]+)\s*\(", hdr))
    out = subprocess.check_output(["nm", "-D", "--defined-only", rb.api.LIB_PATH], text=True)
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    missing = declared - exported
    assert not missing, f"declared in roaring_b200.h but not exported: {sorted(missing)}"
    extra = exported - declared      # nothing else may leak (an undeclared reference name would shadow libroaring's)
    assert not extra, f"exported but not declared in roaring_b200.h: {sorted(extra)}"
    L = rb.lib()
    for name in declared:
        assert getattr(L, name) is not None


def test_portable_roundtrip_and_layout(R):
    blobs = rb.load_realdata("wikileaks-noquotes")[:40] + rb.load_realdata("weather_sept_85")[:10] \
        + synth_blobs(R, 5, 40)
    for b in blobs:
        x = rb.Bitmap.deserialize(b)
        assert x.serialize() == b
        assert x.validate()[0]
        ok, why = R.validate(x.ptr)          # reference validates OUR object
        assert ok, why
        assert R.serialize(x.ptr) == b       # reference serializes OUR object
        r = R.deserialize(b)
        assert rb.Bitmap(r, own=False).serialize() == b   # we serialize THEIR object
        assert x.cardinality() == R.card(r)
        R.free(r)
        x.own = False
        R.free(x.ptr)                        # reference frees OUR object (ownership contract)


def test_malformed_input_rejected():
    good = rb.load_realdata("census1881")[0]
    for bad in (b"", b"\x00\x01", good[:20], b"\xff" * 64, good[:-3]):
        with pytest.raises(rb.RB200Error):
            rb.Bitmap.deserialize(bad)


def test_type_rules_match_oracle_table():
    """decide_type()/slot_bound() are host+device functions; exercise them on the host through a
    tiny compiled probe so the rule table is checked even without a GPU."""
    src = r'''
#include "rb200_device.cuh"
#include <cstdio>
using namespace rb200;
int main() {
    // (op, tA, tB, cA, cB, lA, lB, card, nruns) -> type
    struct C { int op,tA,tB; unsigned cA,cB,lA,lB; int card,nruns, expect; };
    C cases[] = {
        {OP_AND, T_BITSET, T_BITSET, 9000, 9000, 1024, 1024, 4096, 0, T_ARRAY},
        {OP_AND, T_BITSET, T_BITSET, 9000, 9000, 1024, 1024, 4097, 0, T_BITSET},
        {OP_AND, T_RUN, T_BITSET, 65536, 9000, 1, 1024, 9000, 0, T_BITSET},
        {OP_AND, T_RUN, T_BITSET, 4000, 9000, 3, 1024, 10, 0, T_ARRAY},
        {OP_OR, T_BITSET, T_BITSET, 40000, 40000, 1024, 1024, 65536, 1, T_BITSET},
        {OP_OR, T_BITSET, T_RUN, 40000, 65536, 1024, 1, 65536, 1, T_RUN},
        {OP_OR, T_ARRAY, T_ARRAY, 2000, 2096, 2000, 2096, 3000, 0, T_ARRAY},
        {OP_OR, T_ARRAY, T_ARRAY, 2000, 2097, 2000, 2097, 4097, 0, T_BITSET},
        {OP_OR, T_ARRAY, T_ARRAY, 2000, 2097, 2000, 2097, 4096, 0, T_ARRAY},
        {OP_OR, T_RUN, T_RUN, 100, 100, 2, 2, 200, 3, T_RUN},
        {OP_OR, T_RUN, T_ARRAY, 10, 10, 5, 10, 20, 15, T_ARRAY},
        {OP_XOR, T_ARRAY, T_RUN, 31, 5000, 31, 3, 5031, 34, T_RUN},
        {OP_XOR, T_ARRAY, T_RUN, 40, 5000, 40, 3, 4960, 43, T_BITSET},
        {OP_XOR, T_ARRAY, T_RUN, 40, 4000, 40, 3, 4040, 43, T_ARRAY},
        {OP_XOR, T_ARRAY, T_RUN, 100, 4000, 100, 3, 4090, 90, T_ARRAY},
        {OP_ANDNOT, T_RUN, T_ARRAY, 32, 5, 1, 5, 27, 6, T_RUN},
        {OP_ANDNOT, T_RUN, T_ARRAY, 33, 5, 1, 5, 28, 6, T_ARRAY},
        {OP_ANDNOT, T_RUN, T_BITSET, 5000, 9000, 2, 1024, 4500, 0, T_BITSET},
        {OP_ANDNOT, T_RUN, T_RUN, 5000, 100, 2, 1, 4900, 3, T_RUN},
    };
    int bad = 0;
    for (auto &c : cases) {
        int t = decide_type(c.op,c.tA,c.tB,c.cA,c.cB,c.lA,c.lB,c.card,c.nruns);
        if (t != c.expect) { printf("MISMATCH op=%d tA=%d tB=%d card=%d -> %d expect %d\n", c.op,c.tA,c.tB,c.card,t,c.expect); bad++; }
        unsigned sb = slot_bound(c.op,c.tA,c.tB,c.cA,c.cB,c.lA,c.lB);
        unsigned len = t==T_BITSET?1024u:(t==T_ARRAY?(unsigned)c.card:(unsigned)c.nruns);
        if (stored_bytes(t,len) > sb) { printf("SLOT too small\n"); bad++; }
    }
    printf("bad=%d\n", bad);
    return bad;
}
'''
    out = _run_probe(src)
    assert out.returncode == 0, out.stdout


def _run_probe(src):
    """Compile a host-side probe against the library's headers with nvcc and run it."""
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        cu = os.path.join(td, "probe.cu")
        open(cu, "w").write(src)
        exe = os.path.join(td, "probe")
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-std=c++17", "--expt-relaxed-constexpr",
                               "-gencode", "arch=compute_90a,code=sm_90a",
                               "-I", os.path.join(ROOT, "croaring_b200", "csrc"), cu, "-o", exe])
        return subprocess.run([exe], capture_output=True, text=True)


def test_many2_index_formats_round_trip():
    """The N-way union's index entry (m2_entry) and per-key counter (m2_cu) are host+device helpers:
    payload offsets of 64 GiB and more, every type / flag combination, participant counts above 2^24
    and weights at every w_shift boundary survive packing and unpacking."""
    src = r'''
#include "rb200_common.h"
#include <cstdio>
using namespace rb200;
int bad = 0;
#define CHECK(c) do { if (!(c)) { printf("FAIL line %d: %s\n", __LINE__, #c); bad++; } } while (0)
int main() {
    const uint64_t offs[] = {0, (1ull << 36) - 16, 1ull << 36, (1ull << 40) + 16, (1ull << 60) - 16};
    const uint32_t poss[] = {0, 1, (1u << 24) + 1, 0xffffffffu};
    for (uint64_t off : offs)
        for (uint32_t pos : poss)
            for (uint32_t t = T_BITSET; t <= T_RUN; t++)
                for (uint32_t fl = 0; fl < 4; fl++) {
                    const uint32_t tf = t | (fl & 1 ? TF_FULL_RUN : 0) | (fl & 2 ? TF_FULL_BITSET : 0);
                    const uint4 e = m2_entry(off, pos, 4096, tf);
                    CHECK(m2_entry_off(e) == off);
                    CHECK(m2_entry_tf(e) == tf);
                    CHECK(e.y == pos && e.z == 4096);
                    const unsigned long long v = ((unsigned long long)e.y << 8) | m2_entry_tf(e);   // k_many2_fold's order key
                    CHECK((uint32_t)(v >> 8) == pos && (uint32_t)(v & 0xff) == tf);
                }
    CHECK(m2_tf(T_RUN, 1, 65536) == (T_RUN | TF_FULL_RUN));
    CHECK(m2_tf(T_BITSET, 1024, 65536) == (T_BITSET | TF_FULL_BITSET));
    CHECK(m2_tf(T_RUN, 2, 65535) == T_RUN && m2_tf(T_BITSET, 1024, 65535) == T_BITSET);
    CHECK(m2_tf(T_ARRAY, 4096, 4096) == T_ARRAY);

    const uint32_t counts[] = {0, 1, (1u << 24) - 1, 1u << 24, (1u << 24) + 1, 0xffffffffu};
    for (uint32_t c : counts)
        for (uint32_t w : {0u, 1u, 0x12345678u, 0xffffffffu}) {
            const unsigned long long cu = m2_cu(c, w);
            CHECK(m2_cu_count(cu) == c && (uint32_t)cu == w);
        }
    // w_shift: the smallest shift that keeps n * 2^13 >> w_shift below 2^32; 0 below 2^19 inputs
    const uint64_t ns[] = {1, (1u << 19) - 1, 1u << 19, (1u << 19) + 1, 1u << 20, (1u << 24) + 1, (1u << 25) - 1,
                           1u << 25, 0xffffffffu};
    for (uint64_t n : ns) {
        const uint32_t s = m2_weight_shift(n);
        CHECK(((n << 13) >> s) < (1ull << 32));
        CHECK(s == 0 || ((n << 13) >> (s - 1)) >= (1ull << 32));
        CHECK((s == 0) == (n < (1u << 19)));
        // n inputs each bringing the largest container (2^13 x 16 bytes) to one key, one atomic each:
        // the weights never carry into the count
        CHECK(m2_weight(1u << 13, s) == (1u << 13) >> s);
        const unsigned long long tot = n * m2_cu(1, m2_weight(1u << 13, s));
        CHECK(m2_cu_count(tot) == n);
        CHECK((uint32_t)tot == (uint32_t)(n * ((1u << 13) >> s)));
        if (n < (1u << 25)) CHECK(m2_cu_weight_kib(tot, s) == n * 128);   // 128 KiB each
        // n inputs of one 16-byte unit each (arrays of <= 8 values) still weigh something, so such a
        // key is split over work units as it was with exact weights
        const unsigned long long small = n * m2_cu(1, m2_weight(1, s));
        CHECK(m2_cu_count(small) == n && (uint32_t)small == n);
    }
    for (uint32_t s = 0; s <= 13; s++) {   // every w_shift an n < 2^32 can need
        CHECK(m2_weight(0, s) == 0);
        CHECK(m2_weight(1, s) == 1);   // rounded up: a small container keeps a nonzero weight
        CHECK(m2_weight((1u << s) + 1, s) == 2);
        CHECK(m2_weight(1u << 21, s) == (1u << 21) >> s);   // a window's sum: 256 of the largest containers
    }
    CHECK(m2_weight_shift((1u << 24) + 1) == 6);
    CHECK(m2_cu_weight_kib(m2_cu(3, 64 * 5), 0) == 5);   // w_shift 0: the weight is stored bytes / 16
    printf("bad=%d\n", bad);
    return bad;
}
'''
    out = _run_probe(src)
    assert out.returncode == 0, out.stdout


def test_compute_fails_loudly_without_gpu():
    """No CPU fallback: on a box without a CUDA device every compute entry point errors."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    a = rb.Bitmap.deserialize(rb.load_realdata("census1881")[0])
    with pytest.raises(rb.RB200Error):
        _ = a & a
    with pytest.raises(rb.RB200Error):
        rb.DeviceSet.upload([a])


def test_mutated_blobs_never_crash_the_host_parsers(R):
    """Seeded mutation fuzz of the two host-side portable-format readers (rb200_host.cu parse_portable
    behind rb200_bitmap_portable_deserialize_safe; rb200_shard.cu index_blob behind the blob algebra):
    byte flips, truncations, garbage tails and splices must be either refused or handled
    consistently — what one reader accepts the other slices, and accepted bytes re-serialize stably."""
    import random
    from croaring_b200 import sharding as sh
    rng = random.Random(20260923)
    base = rb.load_realdata("wikileaks-noquotes")[:10] + rb.load_realdata("census1881")[:4] + synth_blobs(R, 11, 24)
    base = [b for b in base if len(b) < 40000]
    accepted = sliceable = 0
    for _ in range(3000):
        b = bytearray(rng.choice(base))
        mode = rng.randrange(5)
        if mode == 0:
            for _k in range(rng.randrange(1, 4)):
                b[rng.randrange(min(len(b), 64))] = rng.randrange(256)
        elif mode == 1:
            for _k in range(rng.randrange(1, 6)):
                b[rng.randrange(len(b))] = rng.randrange(256)
        elif mode == 2:
            b = b[:rng.randrange(len(b))]
        elif mode == 3:
            b += bytes(rng.randrange(256) for _k in range(rng.randrange(1, 40)))
        else:
            c = rng.choice(base)
            k = rng.randrange(len(b))
            b = b[:k] + c[rng.randrange(len(c)):]
        b = bytes(b)
        try:
            x = rb.Bitmap.deserialize(b)
            s = x.serialize()
            y = rb.Bitmap.deserialize(s)
            assert y.serialize() == s
            x.free()
            y.free()
            accepted += 1
        except rb.RB200Error:
            pass
        try:
            parts = [sh.slice_blob_by_keys(b, lo, hi) for lo, hi in ((0, 7), (8, 300), (301, 65535))]
            full = sh.concat_blobs(parts)
            assert sh.slice_blob_by_keys(full, 0, 65535) == full
            sh.plan_key_ranges([b, full], 3)
            sliceable += 1
        except rb.RB200Error:
            pass
    assert accepted == sliceable and 0 < accepted < 3000
