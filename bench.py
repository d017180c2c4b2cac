#!/usr/bin/env python
"""bench.py — set-ops/sec of the Roaring hot path on H100 (BASELINE.json metric).

    python bench.py --gpus N --steps K --warmup W            # our CUDA path (C ABI, sm_90a kernels)
    python bench.py --impl reference --gpus N --steps K ...   # unmodified CRoaring on host cores

Headline workload (config.workload = realdata_allpairs, SURVEY.md §8(d) config 2b): the
reference's real-data suite census1881 + weather_sept_85 + wikileaks-noquotes (200 run-optimized
bitmaps each, committed as portable-serialized fixtures), ops AND / OR / XOR on ALL 19 900
unordered bitmap pairs of each set, one batched call per (dataset, op): 179 100 set-ops per step.
At N > 1 the pair lists are SHARDED over the ranks (strong scaling: total work fixed, no data-path
collective) and the step ends with ONE NCCL all-reduce of the device-resident checksum (sum of
result cardinalities) inside the timed region; the checksum is compared with the value the
unmodified reference produced for this workload (tests/golden/allpairs_golden.json).

The same JSON line carries the other BASELINE.json configs as sub-records, each with `roofline`,
`cpu_baseline` (the unmodified reference on the host cores, same inputs) and a `parity` flag
(bytes / values identical to the reference's):
    successive      configs[1] literal: 199 successive pairs x 3 ops x 3 datasets
    card_10k        configs[3]: and_cardinality / jaccard over 10^4 bitset-heavy pairs
    or_many_zipf    configs[2]: roaring_bitmap_or_many over 200 Zipfian bitmaps x 10^7 values,
                    six densities (N = 1 only)
    or_many_sharded configs[4]: 1000 bitmaps over a 10^8 universe, key ranges over the run's N
                    GPUs + one ncclAllReduce(uint32[K]) per call, timed
See DESIGN.md §6 for the contract and the definitions of every number.

--dump-outputs DIR writes, after the timed steps, what the headline path returned in its last
step (rank 0's results): per (dataset, op) the cardinality of every result bitmap and the values of
a fixed, seeded sample of the non-empty result bitmaps, as float64 .npy files (64 MB at most in all).  The inputs
are the committed fixtures, so two builds run with the same arguments can be compared file by file.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

DATASETS = ["census1881", "weather_sept_85", "wikileaks-noquotes"]
OPS = ["and", "or", "xor"]
METRIC = "set-ops/sec (AND/OR/XOR over realdata suite)"
ZIPF_DENSITIES = [0.001, 0.003, 0.01, 0.03, 0.1, 0.3]   # 0.001 is clamped by the 32-bit universe (0.00233)

_REAL_STDOUT = None


def capture_stdout():
    """Only the JSON line may reach stdout: libraries (NCCL prints its version banner there) are
    sent to stderr for the rest of the run."""
    global _REAL_STDOUT
    if _REAL_STDOUT is None:
        sys.stdout.flush()
        _REAL_STDOUT = os.dup(1)
        os.dup2(2, 1)


def emit(line):
    data = (json.dumps(line) + "\n").encode()
    if _REAL_STDOUT is None:
        sys.stdout.write(data.decode())
        sys.stdout.flush()
    else:
        os.write(_REAL_STDOUT, data)


def log(*a):
    print("[bench]", *a, file=sys.stderr, flush=True)


def headline_config(pairs_per_dataset, set_ops_per_step):
    """`config` of the headline workload: ONE definition, printed verbatim by both arms (the reference
    arm runs on our arm's config).  `l2`, `batching` and `sharding` say how the CUDA arm executes it;
    the reference arm runs the same pairs with every result created, measured and freed on the host."""
    return {"workload": "realdata_allpairs", "datasets": DATASETS, "ops": OPS,
            "pairs_per_dataset": int(pairs_per_dataset), "set_ops_per_step": int(set_ops_per_step),
            "l2": "flushed between timed steps (256 MB memset)",
            "batching": "one rb200_batch_op call per (dataset, op); the 9 calls of a step queue back to back",
            "sharding": "pairs r, r+N, ... of every list on rank r; one NCCL all-reduce of the device "
                        "checksum closes the step (inside the timed region)"}


def all_pairs(n):
    i, j = np.triu_indices(n, 1)
    return i.astype(np.uint32), j.astype(np.uint32)


def successive_pairs(n):
    return np.arange(n - 1, dtype=np.uint32), np.arange(1, n, dtype=np.uint32)


def host_threads():
    try:
        return len(os.sched_getaffinity(0))
    except Exception:
        return os.cpu_count() or 1


def golden_allpairs():
    try:
        with open(os.path.join(ROOT, "tests", "golden", "allpairs_golden.json")) as f:
            return json.load(f)
    except Exception:
        return None


def peak_gbs():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            return float(json.load(f)["hbm_gbs"]), "MEASURED_PEAKS.json hbm_gbs"
    except Exception:
        return 3350.0, "fallback 3350 GB/s (H100 SXM data sheet HBM3 bandwidth)"


# ------------------------------------------------------------------------------- --dump-outputs
DUMP_SAMPLE = 8                      # result bitmaps per (dataset, op) whose values are written
DUMP_BUDGET = 64 << 20               # bytes of .npy payload in all


def portable_values(blob):
    """Values of one bitmap in the portable serialization (the format of the reference's
    roaring_bitmap_portable_serialize), as a sorted uint32 array."""
    cookie = int.from_bytes(blob[:4], "little")
    if cookie & 0xFFFF == 12347:                       # with run containers: run flags, no offsets below 4
        n = (cookie >> 16) + 1
        runs = np.unpackbits(np.frombuffer(blob, np.uint8, (n + 7) // 8, 4), bitorder="little")[:n]
        pos = 4 + (n + 7) // 8
        offsets = n >= 4
    elif cookie == 12346:
        n = int.from_bytes(blob[4:8], "little")
        runs, pos, offsets = np.zeros(n, np.uint8), 8, True
    else:
        raise ValueError("not a portable roaring bitmap")
    desc = np.frombuffer(blob, "<u2", 2 * n, pos).astype(np.uint32)
    pos += 4 * n + (4 * n if offsets else 0)
    out = []
    for k in range(n):
        hi, card = desc[2 * k] << 16, int(desc[2 * k + 1]) + 1
        if runs[k]:
            nr = int.from_bytes(blob[pos:pos + 2], "little")
            rl = np.frombuffer(blob, "<u2", 2 * nr, pos + 2).astype(np.uint32)
            pos += 2 + 4 * nr
            lo = np.concatenate([np.arange(a, a + l + 1, dtype=np.uint32) for a, l in zip(rl[0::2], rl[1::2])])
        elif card <= 4096:
            lo = np.frombuffer(blob, "<u2", card, pos).astype(np.uint32)
            pos += 2 * card
        else:
            bits = np.unpackbits(np.frombuffer(blob, np.uint8, 8192, pos), bitorder="little")
            lo = np.flatnonzero(bits).astype(np.uint32)
            pos += 8192
        out.append(hi | lo)
    return np.concatenate(out) if out else np.zeros(0, np.uint32)


def dump_record(res):
    """What a caller of the timed path receives from one batch call: every result's cardinality, and
    the values of DUMP_SAMPLE non-empty result bitmaps drawn with a fixed seed (the same ones on every
    run that computes the same cardinalities; empty results would sample nothing)."""
    cards = res.cardinalities()
    live = np.flatnonzero(cards)
    pick = np.sort(np.random.default_rng(len(res)).choice(live, size=min(DUMP_SAMPLE, len(live)), replace=False))
    vals = []
    for i in pick:
        bm = res.download(int(i))
        vals.append(portable_values(bm.serialize()))
        bm.free()
    return cards, pick, vals


def write_dump(out_dir, records):
    """DIR/<dataset>_<op>_{cardinality,sample_pairs,sample_offsets,sample_values}.npy, float64 (exact
    for 32-bit values and the cardinalities).  A sampled bitmap with more values than its even share
    of the budget keeps that many of them, evenly spaced: the same ones on every run."""
    os.makedirs(out_dir, exist_ok=True)
    fixed = sum(8 * (len(c) + 2 * len(p) + 1) + 4 * 128 for c, p, _ in records)   # + .npy headers
    cap = (DUMP_BUDGET - fixed) // (8 * len(records) * DUMP_SAMPLE)
    for k, (cards, pick, vals) in enumerate(records):
        if not len(pick):
            raise RuntimeError("--dump-outputs: every result of a batch call is empty, nothing to sample")
        vals = [v if len(v) <= cap else v[np.linspace(0, len(v) - 1, cap).astype(np.int64)] for v in vals]
        name = f"{DATASETS[k // len(OPS)]}_{OPS[k % len(OPS)]}"
        offs = np.concatenate([[0], np.cumsum([len(v) for v in vals])])
        flat = np.concatenate(vals) if vals else np.zeros(0)
        for suffix, arr in (("cardinality", cards), ("sample_pairs", pick),
                            ("sample_offsets", offs), ("sample_values", flat)):
            np.save(os.path.join(out_dir, f"{name}_{suffix}.npy"), np.asarray(arr, dtype=np.float64))
    log(f"dump: {len(records)} results written to {out_dir}")


# ------------------------------------------------------------------------------- clocks
class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.idx = gpu_index
        self.proc = None
        self.lines = []

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                 "-lms", "100", "-i", str(self.idx)],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for ln in self.proc.stdout:
            self.lines.append(ln.strip())

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1]))
                mx.append(float(f[2]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown",
                                "sw_power_cap"), f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": float(np.median(sm)) if sm else None,
                "sm_max_mhz": max(mx) if mx else None, "samples": len(sm),
                "reasons": sorted(reasons)}


# ------------------------------------------------------------------------------- CPU arm
def reference_allpairs(steps, warmup, threads, one_thread_pass=True):
    """The unmodified reference (oracle/_ref) on the host cores over the headline workload: warm,
    FULL workload per step, persistent thread pool with dynamic chunks (oracle/ref_bench.c).
    Used identically by `--impl reference` and by the `cpu_baseline` leg of our own line."""
    from oracle.refbench import RefBench
    import croaring_b200.datasets as dsm
    rbn = RefBench()
    sets = {ds: rbn.load(dsm.load_realdata(ds), threads) for ds in DATASETS}
    pairs = {ds: all_pairs(sets[ds][1]) for ds in DATASETS}
    ops_per_step = sum(len(pairs[ds][0]) for ds in DATASETS) * len(OPS)
    rbn.warm_pool(threads)

    def step(T, pairset):
        t, chk = 0.0, 0
        for ds in DATASETS:
            for op in OPS:
                dt, s = rbn.pairs(sets[ds], op, pairset[ds][0], pairset[ds][1], T)
                t += dt
                chk += s
        return t, chk

    for _ in range(max(1, warmup)):
        step(threads, pairs)
    tot, chk = 0.0, 0
    for _ in range(steps):
        dt, chk = step(threads, pairs)
        tot += dt
    out = {"value": ops_per_step * steps / tot, "ms_per_step": 1e3 * tot / steps, "checksum": chk,
           "threads": threads, "isa": rbn.isa(), "ops_per_step": ops_per_step}
    if one_thread_pass:
        step(1, pairs)
        dt1, chk1 = step(1, pairs)
        out["value_1thread"] = ops_per_step / dt1
        assert chk1 == chk
    succ = {ds: successive_pairs(sets[ds][1]) for ds in DATASETS}
    best = 1e9
    for _ in range(7):                      # the literal configs[1] sweep: 1 thread, best of 7
        best = min(best, step(1, succ)[0])
    out["successive_1thread"] = 3 * 3 * 199 / best
    for ds in DATASETS:
        rbn.unload(sets[ds])
    return out


def run_reference(args, rank, world):
    """`--impl reference`: rank 0 alone times the reference; the other ranks exit."""
    if rank != 0:
        return
    T = host_threads()
    r = reference_allpairs(args.steps, args.warmup, T)
    gold = golden_allpairs()
    line = {
        "impl": "reference", "metric": METRIC, "value": r["value"], "unit": "set-ops/s",
        "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": r["ms_per_step"], "higher_is_better": True, "scaling": "strong",
        "vs_baseline": None, "dtype": "u16/u64 bitwise", "data": "reference realdata fixtures",
        "config": headline_config(19900, r["ops_per_step"]),
        "checksum_sum_card": r["checksum"],
        "parity": (gold is not None and r["checksum"] == gold["bench_checksum_and_or_xor"]),
        "cpu_baseline": {"value": r["value"], "unit": "set-ops/s", "cores": T, "kind": "reference",
                         "isa": r["isa"], "value_1thread": r.get("value_1thread"),
                         "sample": "full workload per step (all 19 900 pairs x 3 ops x 3 datasets), warm, "
                                   "persistent pthread pool, pairs handed out in dynamic chunks of 16"},
        "e2e": {"value": r["value"], "unit": "set-ops/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "successive": {"workload": "realdata_successive (199 pairs x 3 ops x 3 datasets)",
                       "value": r["successive_1thread"], "unit": "set-ops/s", "threads": 1},
    }
    emit(line)


# ------------------------------------------------------------------------------- our arm
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--e2e-steps", type=int, default=5)
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--no-extras", action="store_true", help="skip the card_10k / or_many sub-records")
    ap.add_argument("--extras", default="card_10k,or_many_zipf,or_many_sharded")
    ap.add_argument("--zipf-values", type=int, default=10 ** 7)
    ap.add_argument("--zipf-bitmaps", type=int, default=200)
    ap.add_argument("--sharded-bitmaps", type=int, default=1000)
    ap.add_argument("--card-pairs", type=int, default=10 ** 4)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the headline path's last-step results to DIR/<name>.npy")
    args = ap.parse_args()
    capture_stdout()

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))

    if args.impl == "reference":
        run_reference(args, rank, world)
        return

    import torch
    import torch.distributed as dist
    import croaring_b200 as rb
    from croaring_b200 import workloads as wl

    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device — the CUDA path has no CPU fallback")
    torch.cuda.set_device(local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    rb.init(local_rank)
    # ONE explicit stream for everything that is timed: torch's current stream, the library's stream
    # (rb200_set_stream) and the CUDA events that bracket the steps.  (The legacy default stream
    # would not do: its handle is 0, which rb200_set_stream reads as "use the library's own stream".)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    rb.set_stream(stream.cuda_stream)
    assert stream.cuda_stream != 0

    def bcast(obj):
        box = [obj]
        dist.broadcast_object_list(box, src=0)
        return box[0]

    # the library's own communicator (plain C ABI over NCCL), bootstrapped through torch.distributed
    comm = rb.Comm.create(rank, world, bcast if world > 1 else None)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(x):
        t = torch.tensor([x], dtype=torch.float64, device="cuda")
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def sum_over_ranks(x):
        t = torch.tensor([x], dtype=torch.float64, device="cuda")
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.SUM)
        return float(t.item())

    peak, peak_src = peak_gbs()
    T_host = host_threads()
    gen_threads = max(2, wl._threads() // world)   # workload generator threads of this rank

    # ---- inputs: portable-serialized fixtures -> device-resident sets (outside the timed region)
    blobs = {ds: rb.load_realdata(ds) for ds in DATASETS}
    sets = {ds: rb.DeviceSet.from_serialized(blobs[ds]) for ds in DATASETS}
    full_pairs = {ds: all_pairs(len(blobs[ds])) for ds in DATASETS}
    # strong scaling: rank r owns pairs r, r + N, r + 2N, ... of every list (interleaved: balanced)
    pairs = {ds: (full_pairs[ds][0][rank::world].copy(), full_pairs[ds][1][rank::world].copy()) for ds in DATASETS}
    succ_full = {ds: successive_pairs(len(blobs[ds])) for ds in DATASETS}
    succ = {ds: (succ_full[ds][0][rank::world].copy(), succ_full[ds][1][rank::world].copy()) for ds in DATASETS}
    ops_per_step = sum(len(full_pairs[ds][0]) for ds in DATASETS) * len(OPS)
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")  # > 50 MB L2
    d_chk = torch.zeros(1, dtype=torch.int64, device="cuda")              # device-resident checksum (u64)

    stats = {"algo_bytes": 0, "kernel_ms": 0.0, "launches": 0, "checksum": 0, "device_ms": 0.0}

    def step(pairset):
        # the nine batch calls queue back to back on the stream (a call returns once its kernels are
        # enqueued); every result adds its cardinalities into the device checksum; ONE all-reduce
        # of that checksum closes the step (the only collective; a no-op at N = 1)
        d_chk.zero_()
        res = []
        for ds in DATASETS:
            ia, ib = pairset[ds]
            for op in OPS:
                r = sets[ds].batch(op, sets[ds], ia, ib)
                r.add_cardinality_device(d_chk.data_ptr())
                res.append(r)
        comm.allreduce_u64(d_chk.data_ptr(), 1)
        return res

    def timed(pairset, steps, warmup, collect, last=None):
        for _ in range(warmup):
            for r in step(pairset):
                r.free()
        barrier()
        tot_ms = 0.0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for it in range(steps):
            flush_buf.zero_()            # flush L2 between timed iterations (not timed)
            barrier()
            e0.record(stream)
            res = step(pairset)
            e1.record(stream)
            torch.cuda.synchronize()
            tot_ms += e0.elapsed_time(e1)
            keep = last is not None and it == steps - 1      # the last step's results, for --dump-outputs
            for k, r in enumerate(res):
                if collect:
                    ms, cms, ab = r.op_stats()
                    stats["algo_bytes"] += ab
                    stats["kernel_ms"] += cms
                    stats["device_ms"] += ms
                    stats["launches"] += 1
                    name = f"{DATASETS[k // len(OPS)]}/{OPS[k % len(OPS)]}"
                    pl = stats.setdefault("per_launch", {}).setdefault(name, [0.0, 0.0, 0])
                    pl[0] += cms
                    pl[1] += ms
                    pl[2] += ab
                if not keep:
                    r.free()
            if keep:
                last[:] = res
            if collect:
                stats["checksum"] = int(d_chk.item())
        barrier()
        return max_over_ranks(tot_ms)

    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    l0 = rb.kernel_launches()
    last = [] if args.dump_outputs and rank == 0 else None
    tot_ms = timed(pairs, args.steps, args.warmup, True, last)
    gpu_launches = rb.kernel_launches() - l0
    clocks = sampler.stop() if rank == 0 else None
    if last is not None:
        write_dump(args.dump_outputs, [dump_record(r) for r in last])
        for r in last:
            r.free()
    value = ops_per_step * args.steps / (tot_ms * 1e-3)
    gold = golden_allpairs()
    headline_parity = gold is not None and stats["checksum"] == gold["bench_checksum_and_or_xor"]
    log(f"headline: {value / 1e6:.2f} M set-ops/s, {tot_ms / args.steps:.3f} ms/step, checksum {stats['checksum']} "
        f"parity={headline_parity}")

    # ---- the literal configs[1] sweep: 199 successive pairs (latency-bound, reported beside)
    succ_steps = args.steps
    succ_ops = sum(len(succ_full[ds][0]) for ds in DATASETS) * len(OPS)
    succ_ms = timed(succ, succ_steps, args.warmup, False)
    succ_val = succ_ops * succ_steps / (succ_ms * 1e-3)

    # ---- drop-in call latency: census1881 csv0 AND csv1 through roaring_bitmap_and (configs[0])
    dropin = None
    if rank == 0:
        a, b = rb.Bitmap.deserialize(blobs["census1881"][0]), rb.Bitmap.deserialize(blobs["census1881"][1])
        ts = []
        for it in range(220):
            t0 = time.perf_counter()
            r = a & b
            ts.append(time.perf_counter() - t0)
            r.free()
        dropin = {"call": "roaring_bitmap_and(census1881 csv0, csv1): host roaring_bitmap_t in -> out, one pair",
                  "median_us": float(np.median(ts[20:]) * 1e6), "p90_us": float(np.percentile(ts[20:], 90) * 1e6)}

    # ---- e2e: host roaring_bitmap_t in -> host roaring_bitmap_t out through the C ABI ----------
    e2e = None
    if not args.no_e2e:
        host = {ds: [rb.Bitmap.deserialize(b) for b in blobs[ds]] for ds in DATASETS}
        h2d = d2h = 0
        e2e_chk = [0]

        def e2e_step():
            nonlocal h2d, d2h
            h2d = d2h = 0
            acc = rb.CardinalitySum()
            for ds in DATASETS:
                S = rb.DeviceSet.upload(host[ds]).bind_host()     # H2D inside the timed region; the
                # host inputs stay alive, so pass-through containers are not sent back over PCIe
                h2d += S.payload_bytes
                ia, ib = pairs[ds]
                for op in OPS:
                    r = S.batch(op, S, ia, ib)
                    # queued for the library's background downloader: D2H on its own stream +
                    # host materialisation — every result bitmap is built in the reference layout,
                    # its cardinality read with the host function, then freed (the body of the
                    # reference's benchmark loop, microbenchmarks/bench.cpp:85-96) — while this
                    # thread goes on with the next upload / op
                    r.foreach_async(acc)
                    r.free()
                S.free()
            rb.download_wait()                                    # every result has been consumed
            e2e_chk[0] = acc.value
            d2h = int(rb.api.lib().rb200_last_download_bytes())

        e2e_step()
        barrier()
        t0 = time.perf_counter()
        for _ in range(args.e2e_steps):
            e2e_step()
        torch.cuda.synchronize()
        dt = max_over_ranks(time.perf_counter() - t0)
        chk_all = int(sum_over_ranks(float(e2e_chk[0])))
        e2e = {"value": ops_per_step * args.e2e_steps / dt, "unit": "set-ops/s",
               "h2d_bytes_per_step": int(sum_over_ranks(h2d)), "d2h_bytes_per_step": int(sum_over_ranks(d2h)),
               "steps": args.e2e_steps, "host_threads": T_host,
               "checksum_sum_card": chk_all, "parity": gold is not None and chk_all == gold["bench_checksum_and_or_xor"],
               "api": "rb200_set_upload(host roaring_bitmap_t[]) + rb200_set_bind_host -> per (dataset, op): "
                      "rb200_batch_op + rb200_download_foreach_async -> rb200_download_wait (every result "
                      "materialised as a host roaring_bitmap_t in the reference layout, cardinality read "
                      "on the host, freed; downloads overlap the following uploads and ops); at N > 1 every rank "
                      "uploads the inputs and owns every N-th pair"}
        for ds in DATASETS:
            for b in host[ds]:
                b.free()

    # ---- e2e, bytes flavour: portable-serialized bitmaps in -> portable-serialized results out
    e2e_ser = None
    if not args.no_e2e:
        ser_bytes = 0

        def e2e_ser_step():
            nonlocal ser_bytes
            ser_bytes = 0
            for ds in DATASETS:
                S = rb.DeviceSet.from_serialized(blobs[ds])        # host cookie read + H2D + device parse
                ia, ib = pairs[ds]
                for op in OPS:
                    r = S.batch(op, S, ia, ib)
                    _buf, _off, _len, release = r.serialize_all(copy=False)
                    ser_bytes += int(rb.api.lib().rb200_last_download_bytes())
                    release()
                    r.free()
                S.free()

        e2e_ser_step()
        barrier()
        t0 = time.perf_counter()
        for _ in range(max(2, args.e2e_steps // 2)):
            e2e_ser_step()
        torch.cuda.synchronize()
        dt = max_over_ranks(time.perf_counter() - t0)
        e2e_ser = {"value": ops_per_step * max(2, args.e2e_steps // 2) / dt, "unit": "set-ops/s",
                   "h2d_bytes_per_step": int(world * sum(sum(map(len, blobs[ds])) for ds in DATASETS)),
                   "d2h_bytes_per_step": int(sum_over_ranks(ser_bytes)),
                   "api": "rb200_set_upload_serialized(portable bytes) -> rb200_batch_op -> "
                          "rb200_set_serialize (portable bytes of every result in pinned host memory)"}

    for ds in DATASETS:
        sets[ds].free()
    del flush_buf

    # ------------------------------------------------------------------------------ sub-records
    extras = {} if args.no_extras else {k: None for k in args.extras.split(",") if k}
    tmpdir = f"/dev/shm/rb200_bench_{os.environ.get('MASTER_PORT', 'single')}_{os.getppid() if world > 1 else os.getpid()}"

    def cpu_ref():
        from oracle.refbench import RefBench
        return RefBench()

    # ---- configs[3]: cardinality-only sweep, 10^4 pairs, bitset-heavy (density 0.5, universe 2^20)
    if "card_10k" in extras:
        P = args.card_pairs
        lo, hi = P * rank // world, P * (rank + 1) // world      # this rank's block of pairs
        t0 = time.perf_counter()
        A = wl.dense_arena(2 * (hi - lo), n_keys=16, i0=2 * lo, threads=gen_threads)
        t_gen = time.perf_counter() - t0
        S = rb.DeviceSet.from_serialized(A)
        ia = np.arange(0, 2 * (hi - lo), 2, dtype=np.uint32)
        ib = ia + 1
        algo = (hi - lo) * 16 * 16384
        kms, dms = [], []
        for it in range(args.warmup + args.steps):
            c = S.and_cardinality(S, ia, ib)
            if it >= args.warmup:
                kms.append(float(rb.api.lib().rb200_last_compute_ms()))
                dms.append(rb.last_device_ms())
        cards = S.cardinalities()
        jacc = c / (cards[ia] + cards[ib] - c)
        k_ms, d_ms = max_over_ranks(float(np.median(kms))), max_over_ranks(float(np.median(dms)))
        chk = int(sum_over_ranks(float(int(c.sum()))))
        rec = {"workload": "configs[3]: and_cardinality + jaccard, %d pairs, universe 2^20, density 0.5 "
                           "(PCG32 global stream, SURVEY 8(d) row 4)" % P,
               "pairs": P, "value": P / (d_ms * 1e-3), "unit": "set-ops/s", "device_ms_per_sweep": d_ms,
               "kernel": "k_card_items", "kernel_ms": k_ms, "algorithmic_bytes": P * 16 * 16384,
               "roofline": {"bound": "hbm", "achieved": algo / (float(np.median(kms)) * 1e-3) / 1e9, "peak": peak,
                            "unit": "GB/s", "frac": algo / (float(np.median(kms)) * 1e-3) / 1e9 / peak,
                            "peak_source": peak_src, "note": "per GPU: this rank's pairs / its kernel time"},
               "sum_and_card": chk, "mean_jaccard": float(jacc.mean()), "generate_s": t_gen,
               "sharding": "pairs split in contiguous blocks over the ranks, no collective in the timed region"}
        if not args.no_cpu:
            rbn = cpu_ref()
            h = rbn.load(A, gen_threads)
            rbn.warm_pool(gen_threads)
            dt1, s1 = rbn.pairs(h, "and_cardinality", ia[:len(ia) // 8 + 1], ib[:len(ib) // 8 + 1], 1)
            rbn.pairs(h, "and_cardinality", ia, ib, gen_threads)
            dtT, sT = rbn.pairs(h, "and_cardinality", ia, ib, gen_threads)
            rbn.unload(h)
            ok = sT == int(c.sum())
            ok = sum_over_ranks(0.0 if ok else 1.0) == 0.0
            rec["parity"] = bool(ok)
            rec["cpu_baseline"] = {"kind": "reference", "isa": rbn.isa(), "unit": "set-ops/s",
                                   "value": (hi - lo) / dtT, "cores": gen_threads,
                                   "value_1thread": (len(ia) // 8 + 1) / dt1,
                                   "gbs_1thread": (len(ia) // 8 + 1) * 16 * 16384 / dt1 / 1e9,
                                   "sample": "this rank's pairs, warm, all its host threads; 1 thread on 1/8 of them"}
        extras["card_10k"] = rec
        S.free()
        A.free()
        log("card_10k:", json.dumps({k: rec[k] for k in ("value", "kernel_ms", "sum_and_card") if k in rec}),
            "parity", rec.get("parity"))

    # ---- configs[2]: roaring_bitmap_or_many over 200 Zipfian bitmaps x 10^7 values, density sweep
    if "or_many_zipf" in extras and world == 1:
        sweep = []
        for d in ZIPF_DENSITIES:
            U = wl.zipf_universe(args.zipf_values, d)
            t0 = time.perf_counter()
            A = wl.cached_arena(f"zipf_{args.zipf_bitmaps}x{args.zipf_values}_U{U}",
                                lambda: wl.zipf_arena(args.zipf_bitmaps, U, args.zipf_values, threads=gen_threads))
            t_gen = time.perf_counter() - t0
            t0 = time.perf_counter()
            S = rb.DeviceSet.from_serialized(A)
            t_up = time.perf_counter() - t0
            in_bytes = S.payload_bytes
            kms, dms = [], []
            r = None
            for it in range(args.warmup + args.steps):
                if r is not None:
                    r.free()
                r = S.or_many()
                if it >= args.warmup:
                    kms.append(float(rb.api.lib().rb200_last_compute_ms()))
                    dms.append(rb.last_device_ms())
            out_blob = r.serialize_all()[0]
            card = int(r.cardinalities()[0])
            out_bytes = len(out_blob)
            r.free()
            S.free()
            k_ms, d_ms = float(np.median(kms)), float(np.median(dms))
            algo = in_bytes + out_bytes
            rec = {"density": d, "effective_density": args.zipf_values / U, "universe": U,
                   "bitmaps": args.zipf_bitmaps, "values_per_bitmap": args.zipf_values,
                   "input_bytes": in_bytes, "output_bytes": out_bytes, "cardinality": card,
                   "value": 1.0 / (d_ms * 1e-3), "unit": "set-ops/s (one op = one 200-way or_many)",
                   "input_bitmaps_per_s": args.zipf_bitmaps / (d_ms * 1e-3),
                   "device_ms": d_ms, "kernel": "k_or_many2", "kernel_ms": k_ms,
                   "roofline": {"bound": "hbm", "achieved": algo / (k_ms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s",
                                "frac": algo / (k_ms * 1e-3) / 1e9 / peak, "peak_source": peak_src},
                   "generate_s": t_gen, "upload_s": t_up, "sha256": hashlib.sha256(out_blob).hexdigest()}
            if not args.no_cpu:
                rbn = cpu_ref()
                h = rbn.load(A, gen_threads)
                rbn.or_many_bytes(h)
                dt, ref_blob, ref_card = rbn.or_many_bytes(h)
                rbn.unload(h)
                rec["parity"] = bool(ref_blob == out_blob and ref_card == card)
                rec["cpu_baseline"] = {"kind": "reference", "isa": rbn.isa(), "cores": 1, "value": 1.0 / dt,
                                       "unit": "set-ops/s", "seconds": dt,
                                       "gbs": algo / dt / 1e9, "sample": "the whole call, second of two runs (1 thread: "
                                       "roaring_bitmap_or_many is a single-threaded API)"}
            A.free()
            sweep.append(rec)
            log(f"or_many_zipf d={d}: {k_ms:.3f} ms kernel, {rec['roofline']['frac']:.3f} of peak, parity {rec.get('parity')}")
        extras["or_many_zipf"] = {"workload": "configs[2]: roaring_bitmap_or_many over %d Zipfian bitmaps x %d values "
                                              "(PCG32 streams, SURVEY 8(d) row 3); d = 0.001 is clamped by the 32-bit "
                                              "universe to 0.00233" % (args.zipf_bitmaps, args.zipf_values),
                                  "sweep": sweep, "parity": all(x.get("parity", False) for x in sweep) if not args.no_cpu else None}
    elif "or_many_zipf" in extras:
        extras["or_many_zipf"] = {"skipped": "single-GPU config (BASELINE.json configs[2]); run with --gpus 1"}

    # ---- configs[4]: 10^8-universe, 1000-bitmap OR, key ranges over the run's N GPUs + NCCL all-reduce
    if "or_many_sharded" in extras:
        NB, U = args.sharded_bitmaps, 10 ** 8
        # the 1000 bitmaps are generated in 8 fixed blocks shared through /dev/shm: rank r builds (or
        # finds, from an earlier run on this box) blocks r, r + N, ...; every rank then maps all of
        # them, because it needs its key range of EVERY bitmap
        NBLK = 8 if NB % 8 == 0 else 1
        per = NB // NBLK
        cdir = os.environ.get("RB200_WL_CACHE", "/dev/shm/rb200_wl_cache") or tmpdir
        t0 = time.perf_counter()
        for blk in range(rank, NBLK, world):
            wl.cached_arena(f"zipf5_U{U}_b{blk * per}_n{per}",
                            lambda blk=blk: wl.zipf_arena(per, U, None, b0=blk * per, density_draw=True,
                                                          threads=gen_threads), cache_dir=cdir).free()
        barrier()
        parts = []
        for blk in range(NBLK):
            with open(os.path.join(cdir, f"zipf5_U{U}_b{blk * per}_n{per}.json")) as f:
                parts.append((os.path.join(cdir, f"zipf5_U{U}_b{blk * per}_n{per}.bin"), json.load(f)["lens"]))
        allb = wl.MappedArena(parts)
        t_gen = time.perf_counter() - t0
        ranges, span = rb.api.plan_key_ranges(allb, world)
        klo, khi = ranges[rank]
        t0 = time.perf_counter()
        S = rb.DeviceSet.from_serialized(allb, klo, khi)   # host slicing (C) + streamed H2D of this range only
        t_up = time.perf_counter() - t0
        in_bytes = S.payload_bytes
        kms, dms, cms, wall = [], [], [], []
        part = None
        for it in range(args.warmup + args.steps):
            if part is not None:
                part.free()
            barrier()
            t0 = time.perf_counter()
            part, cards, total = S.or_many_sharded(comm, klo, khi, span)
            w = time.perf_counter() - t0
            if it >= args.warmup:
                kms.append(float(rb.api.lib().rb200_last_compute_ms()))
                dms.append(rb.last_device_ms())
                cms.append(float(rb.api.lib().rb200_last_collective_ms()))
                wall.append(w)
        part_blob = part.serialize_all()[0]
        part.free()
        S.free()
        k_ms, d_ms = max_over_ranks(float(np.median(kms))), max_over_ranks(float(np.median(dms)))
        c_ms, w_ms = max_over_ranks(float(np.median(cms))), max_over_ranks(float(np.median(wall)) * 1e3)
        in_all = sum_over_ranks(float(in_bytes))
        out_all = sum_over_ranks(float(len(part_blob)))
        rec = {"workload": "configs[4]: roaring_bitmap_or_many over %d Zipfian bitmaps, universe 10^8 (%d keys), "
                           "per-bitmap density log-uniform in [0.001, 0.3] (SURVEY 8(d) row 5)" % (NB, span[1] - span[0] + 1),
               "bitmaps": NB, "n_gpus": world, "key_ranges": ranges, "key_span": list(span),
               "input_bytes": int(in_all), "output_bytes": int(out_all), "cardinality": int(total),
               "value": 1.0 / (d_ms * 1e-3), "unit": "set-ops/s (one op = one %d-way or_many)" % NB,
               "input_bitmaps_per_s": NB / (d_ms * 1e-3),
               "device_ms_per_call": d_ms, "kernel": "k_or_many2", "kernel_ms": k_ms, "nccl_allreduce_ms": c_ms,
               "wall_ms_per_call": w_ms, "allreduce_words": span[1] - span[0] + 1,
               "roofline": {"bound": "hbm", "achieved": (in_all + out_all) / (k_ms * 1e-3) / 1e9, "peak": peak * world,
                            "unit": "GB/s", "frac": (in_all + out_all) / (k_ms * 1e-3) / 1e9 / (peak * world),
                            "peak_source": peak_src + " x n_gpus",
                            "note": "all ranks' input + output container bytes / slowest rank's kernel time"},
               "generate_s": t_gen, "upload_s": t_up,
               "collective": "one ncclAllReduce(sum) of uint32[%d] per call, on the device, inside the timed region"
                             % (span[1] - span[0] + 1)}
        parts = [None] * world
        if world > 1:
            dist.all_gather_object(parts, part_blob)
        else:
            parts = [part_blob]
        if rank == 0:
            full = rb.api.blobs_concat(parts)
            rec["sha256"] = hashlib.sha256(full).hexdigest()
            if not args.no_cpu:
                rbn = cpu_ref()
                h = rbn.load(allb, T_host)
                dt, ref_blob, ref_card = rbn.or_many_bytes(h)
                rbn.unload(h)
                rec["parity"] = bool(ref_blob == full and ref_card == total)
                rec["cpu_baseline"] = {"kind": "reference", "isa": rbn.isa(), "cores": 1, "value": 1.0 / dt,
                                       "unit": "set-ops/s", "seconds": dt, "gbs": (in_all + out_all) / dt / 1e9,
                                       "sample": "the whole 1000-way call once (1 thread: single-threaded API)"}
        extras["or_many_sharded"] = rec
        barrier()
        del allb
        log(f"or_many_sharded: {d_ms:.3f} ms/call ({k_ms:.3f} kernel, {c_ms:.3f} nccl), parity {rec.get('parity')}")

    if rank != 0:
        comm.destroy()
        if world > 1:
            dist.destroy_process_group()
        return

    # ---- roofline of the dominant kernel (k_compute_items) ------------------------------------
    achieved = stats["algo_bytes"] / (stats["kernel_ms"] * 1e-3) / 1e9 if stats["kernel_ms"] else 0.0
    traffic = None
    try:
        with open(os.path.join(ROOT, "profiles", "roofline_traffic.json")) as f:
            traffic = json.load(f).get("realdata_allpairs", {}).get("dram_bytes_per_launch")
    except Exception:
        pass
    roofline = {"bound": "hbm", "kernel": "k_compute_items", "achieved": achieved, "peak": peak,
                "unit": "GB/s", "frac": achieved / peak if peak else None, "traffic": traffic,
                "peak_source": peak_src,
                "algorithmic_bytes_per_launch": stats["algo_bytes"] / max(stats["launches"], 1),
                "kernel_ms_per_launch": stats["kernel_ms"] / max(stats["launches"], 1),
                "launches_timed": stats["launches"],
                "step_ms_in_batch_ops": stats["device_ms"] / max(args.steps, 1),
                "per_launch": {k: {"kernel_ms": v[0] / args.steps, "op_ms": v[1] / args.steps,
                                   "gbs": v[2] / max(v[0], 1e-9) / 1e6}
                               for k, v in stats.get("per_launch", {}).items()},
                "note": "rank 0's launches; inputs (0.2-8.7 MB per dataset) are L2-resident within a step by "
                        "reuse, results stream to HBM; traffic = ncu dram bytes per launch at N = 1"}

    cpu = None
    if not args.no_cpu:
        r = reference_allpairs(3, 2, T_host)
        cpu = {"value": r["value"], "unit": "set-ops/s", "cores": T_host, "kind": "reference", "isa": r["isa"],
               "value_1thread": r.get("value_1thread"), "successive_1thread": r["successive_1thread"],
               "checksum_sum_card": r["checksum"], "parity_with_gpu": r["checksum"] == stats["checksum"],
               "sample": "the FULL workload (all 19 900 pairs x 3 ops x 3 datasets), 2 warm-up + 3 timed passes, "
                         "persistent pthread pool, dynamic chunks of 16 pairs — the same routine as --impl reference"}
        headline_parity = headline_parity and cpu["parity_with_gpu"]

    line = {
        "metric": METRIC, "value": value, "unit": "set-ops/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": tot_ms / args.steps, "higher_is_better": True,
        "scaling": "strong", "vs_baseline": None, "dtype": "u16/u64 bitwise",
        "data": "reference realdata fixtures (portable-serialized, run-optimized)",
        "config": headline_config(len(full_pairs[DATASETS[0]][0]), ops_per_step),
        "checksum_sum_card": stats["checksum"],
        "parity": bool(headline_parity),
        "roofline": roofline,
        "cpu_baseline": cpu,
        "e2e": e2e,
        "e2e_serialized": e2e_ser,
        "gpu_launches": int(gpu_launches),
        "clocks": clocks,
        "dropin_call_us": dropin,
        "successive": {"workload": "realdata_successive (configs[1] literal: 199 pairs x 3 ops x 3 datasets)",
                       "value": succ_val, "unit": "set-ops/s", "set_ops_per_step": succ_ops,
                       "ms_per_step": succ_ms / succ_steps, "us_per_call": 1e3 * succ_ms / succ_steps / 9},
    }
    for k, v in extras.items():
        line[k] = v
    emit(line)
    comm.destroy()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
