"""Shared helpers for the parity tests."""
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import synth

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "croaring_b200", "csrc")

DATASETS = ["census1881", "weather_sept_85", "wikileaks-noquotes",
            "census1881_srt", "wikileaks-noquotes_srt", "uscensus2000"]
OPS = ["and", "or", "xor", "andnot"]


def synth_blobs(R, seed, n, key_space=10, max_keys=9, profiles=None):
    """n seeded synthetic bitmaps, serialized by the reference (mixed run-optimized or not)."""
    rng = np.random.default_rng(seed)
    blobs = []
    for i in range(n):
        vals = synth.random_bitmap(rng, n_keys=int(rng.integers(0, max_keys)), key_space=key_space,
                                   profiles=profiles)
        r = R.from_values(vals, run_optimize=bool(i % 3))
        blobs.append(R.serialize(r))
        R.free(r)
    return blobs


def run_probe(src, *args):
    """Compile a host-side probe against the library's headers with nvcc and run it with args.
    nvcc runs without LD_PRELOAD (it crashes with a preloaded sanitizer runtime); the probe keeps it."""
    with tempfile.TemporaryDirectory() as td:
        cu = os.path.join(td, "probe.cu")
        open(cu, "w").write(src)
        exe = os.path.join(td, "probe")
        env = {k: v for k, v in os.environ.items() if k != "LD_PRELOAD"}
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-std=c++17", "--expt-relaxed-constexpr",
                               "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC, cu, "-o", exe], env=env)
        return subprocess.run([exe, *args], capture_output=True, text=True)


def no_run_twins(R, blobs):
    out = []
    for b in blobs:
        r = R.deserialize(b)
        R.L.roaring_bitmap_remove_run_compression(r)
        out.append(R.serialize(r))
        R.free(r)
    return out


def sha_concat(blobs):
    h = hashlib.sha256()
    for b in blobs:
        h.update(b)
    return h.hexdigest()


def check_result_bitmap(R, bm, expect_bytes, what=""):
    """bm: croaring_b200.Bitmap produced by the CUDA path. Byte-exact + valid for the reference."""
    got = bm.serialize()
    assert got == expect_bytes, f"{what}: portable bytes differ (ours {len(got)} B, ref {len(expect_bytes)} B)"
    ok, why = R.validate(bm.ptr)           # the reference's own validator on OUR object
    assert ok, f"{what}: reference validate failed: {why}"
    assert R.serialize(bm.ptr) == expect_bytes, f"{what}: reference serializer disagrees on our object"


def synth_blobs64(R, seed, n, highs=(0, 1, 7, 0x10000, 0xFFFFFFFF), key_space=5, max_keys=5, profiles=None):
    """n seeded 64-bit bitmaps (portable format, serialized by the reference): every bitmap owns a
    random subset of the high-32 buckets, each filled like a synthetic 32-bit bitmap."""
    rng = np.random.default_rng(seed)
    blobs = []
    for i in range(n):
        parts = []
        for h in highs:
            if rng.random() < 0.6:
                v = synth.random_bitmap(rng, n_keys=int(rng.integers(0, max_keys)), key_space=key_space,
                                        profiles=profiles)
                parts.append(v.astype(np.uint64) + (np.uint64(h) << np.uint64(32)))
        vals = np.concatenate(parts) if parts else np.zeros(0, np.uint64)
        blobs.append(R.r64_from_values(vals, run_optimize=bool(i % 3)))
    return blobs
