"""CPU checks of roaring_bitmap_add_offset on the device path's terms (-m "not gpu"): the per-key type
rule of rb200_device.cuh (offset_type) through a host-compiled probe, the plain-C restatement of
tests/c/add_offset_oracle.c byte for byte against the reference, and the argument errors the C ABI and the Python mirror report before
any device is needed."""
import ctypes as C

import numpy as np
import pytest

import croaring_b200.datasets as dsm
from croaring_b200 import api
from helpers import DATASETS, no_run_twins, run_probe, synth_blobs
from offset_oracles import offset_oracle, ref_add_offset_bytes

PROFILES = ["full", "nearfull", "halves", "dense", "bitset", "array", "tiny", "longruns", "shortruns", "ends"]
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
OFFSETS = [0, 1, -1, 536, 4096, 5536, 61440, 65535, 65536, -65536, 65537, -65537, 7 * 65536, 1 << 31,
           -((1 << 32) - 1), 1 << 32, -(1 << 32), INT64_MIN, INT64_MAX,
           (65530 << 16) + 5536, (0xFFFF << 16) + 1000]


def random_offsets(seed, n=6):
    rng = np.random.default_rng(seed)
    return [int(x) for x in rng.integers(-(1 << 33), 1 << 33, n)] + [int(x) for x in rng.integers(-70000, 70000, n)]


def test_type_rule_probe():
    """offset_type() (host + device) against the table of the reference's split + container_ior +
    repair, at cardinality 4096 / 4097 / 65536, including three cases checked on the reference."""
    src = r'''
#include "rb200_device.cuh"
#include <cstdio>
using namespace rb200;
int main() {
    const int A = T_ARRAY, B = T_BITSET, R = T_RUN;
    struct Cs { int tA, tB, card, nruns, expect; };
    Cs cases[] = {
        {A, 0, 100, 100, A}, {A, 0, 4096, 4096, A},
        {B, 0, 4096, 1, A}, {B, 0, 4097, 1, B}, {B, 0, 4097, 3000, B},
        {R, 0, 4096, 1, R}, {R, 0, 4096, 1024, R}, {R, 0, 4096, 2048, A}, {R, 0, 4097, 2047, R},
        {R, 0, 4097, 2048, B}, {R, 0, 10, 6, A},
        {A, A, 4096, 9, A}, {A, A, 4097, 9, B},
        {B, B, 4096, 1, A}, {B, B, 4097, 1, B}, {B, B, 65535, 2, B},
        {B, B, 65536, 1, R},                                   // reference: [60000,65535] + [0,59999] by 5536
        {B, A, 4096, 1, A}, {B, A, 4097, 1, B}, {A, B, 4096, 1, A}, {A, B, 4097, 1, B},
        {B, A, 65536, 1, B},                                   // reference: [4096,65535] + [0,4095] by 61440
        {A, B, 65536, 1, B}, {B, R, 65536, 1, B}, {R, B, 65536, 1, B}, {B, R, 4096, 1, A}, {R, B, 4097, 1, B},
        {R, R, 637, 1, R},                                     // reference: [65000,65535] + [0,100] by 536
        {R, R, 65536, 1, R}, {R, R, 4096, 2048, A}, {R, R, 4097, 2048, B}, {R, R, 4097, 10, R},
        {A, R, 4096, 2048, A}, {A, R, 4097, 5, R}, {R, A, 4097, 2048, B}, {R, A, 65536, 1, R},
    };
    int bad = 0;
    for (auto &c : cases) {
        const int t = offset_type(c.tA, c.tB, c.card, c.nruns);
        if (t != c.expect) { printf("MISMATCH tA=%d tB=%d card=%d nruns=%d -> %d, expect %d\n", c.tA, c.tB, c.card, c.nruns, t, c.expect); bad++; }
        // every outcome fits the slot the plan reserves: min(8192, 2 x card)
        const unsigned len = t == T_BITSET ? 1024u : (t == T_ARRAY ? (unsigned)c.card : (unsigned)c.nruns);
        const unsigned cap = 2u * c.card < 8192u ? 2u * c.card : 8192u;
        if (stored_bytes(t, len) > cap) { printf("SLOT tA=%d tB=%d card=%d\n", c.tA, c.tB, c.card); bad++; }
    }
    printf("bad=%d\n", bad);
    return bad;
}
'''
    r = run_probe(src)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.parametrize("seed", [61, 62, 63])
def test_oracle_add_offset_vs_reference_synthetic(R, seed):
    blobs = synth_blobs(R, seed, 24, key_space=6, max_keys=6, profiles=PROFILES if seed != 63 else None)
    blobs += no_run_twins(R, blobs)
    for off in OFFSETS + random_offsets(seed):
        for k, b in enumerate(blobs):
            assert offset_oracle().add_offset_bytes(b, off) == ref_add_offset_bytes(R, b, off), (off, k)


@pytest.mark.parametrize("ds", DATASETS)
def test_oracle_add_offset_vs_reference_realdata(R, ds):
    blobs = dsm.load_realdata(ds)
    rng = np.random.default_rng(7)
    sample = [blobs[i] for i in sorted(rng.choice(len(blobs), size=min(12, len(blobs)), replace=False))]
    for off in [12345, 65535, 7 * 65536, -65537, 1 << 31, 5536, -1] + random_offsets(len(ds), 2):
        for k, b in enumerate(sample):
            assert offset_oracle().add_offset_bytes(b, off) == ref_add_offset_bytes(R, b, off), (ds, off, k)


def test_argument_errors_before_any_device():
    L = api.lib()
    offs = (C.c_int64 * 1)(5)
    assert not L.rb200_batch_add_offset(None, None, 0, None)
    assert "offsets" in api.last_error()
    assert not L.rb200_batch_add_offset(None, None, 1, C.cast(offs, C.c_void_p))
    assert "S is NULL" in api.last_error()
    with pytest.raises(api.RB200Error, match="3 entries for 2 items"):
        api._offsets_i64([1, 2, 3], 2)
    with pytest.raises(api.RB200Error, match="int64 range"):
        api._offsets_i64([1 << 63], 1)
    with pytest.raises(api.RB200Error, match="int64 range"):
        api._offsets_i64([INT64_MIN - 1, 0], 2)
    with pytest.raises(api.RB200Error, match="integer"):
        api._offsets_i64(np.array([0.5]), 1)
    got = api._offsets_i64([INT64_MIN, INT64_MAX, -1], 3)
    assert got.dtype == np.int64 and got.tolist() == [INT64_MIN, INT64_MAX, -1]
    assert api._offsets_i64(-65537, 3).tolist() == [-65537] * 3
