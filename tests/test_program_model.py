"""The seeded random programs of tests/program_model.py, generated with the reference alone (no device):
the default seeds must reach every producer and consumer, read pending sets whose operands are gone,
feed sharing sets to further ops, free sets under pending dependents and build long chains, or the GPU
test that runs them (test_gpu_programs.py) would pass without testing those paths."""
import pytest

import program_model as pm


@pytest.fixture(scope="module")
def programs(R):
    s32, s64 = pm.DEFAULT_SEEDS32, pm.DEFAULT_SEEDS64
    return [pm.Program(R, s, 32) for s in s32] + [pm.Program(R, s, 64) for s in s64]


def _total(programs):
    tot = {"producers": {}, "consumers": {}}
    for p in programs:
        for key, v in p.stats.items():
            if isinstance(v, dict):
                for k, n in v.items():
                    tot[key][k] = tot[key].get(k, 0) + n
            elif key == "max_depth":
                tot[key] = max(tot.get(key, 0), v)
            else:
                tot[key] = tot.get(key, 0) + v
    return tot


def test_default_programs_are_not_vacuous(programs):
    tot = _total(programs)
    print("\nprogram coverage over the default seeds:")
    for key in ("producers", "consumers"):
        print(f"  {key}: " + ", ".join(f"{k} {v}" for k, v in sorted(tot[key].items())))
    for key in ("pending_freed_operand", "sharing_operand", "free_with_pending_dependent", "max_depth"):
        print(f"  {key}: {tot[key]}")
    print(f"  steps: {sum(len(p.steps) for p in programs)}")
    for k in pm.PRODUCERS32 + pm.PRODUCERS64:
        assert tot["producers"].get(k, 0) >= 3, f"producer {k} occurs {tot['producers'].get(k, 0)} times"
    for k in pm.CONSUMERS32 + pm.CONSUMERS64:
        assert tot["consumers"].get(k, 0) >= 3, f"consumer {k} occurs {tot['consumers'].get(k, 0)} times"
    assert tot["pending_freed_operand"] >= 20
    assert tot["sharing_operand"] >= 20
    assert tot["free_with_pending_dependent"] >= 10
    assert tot["max_depth"] >= 6
    # the programs switch the library stream and bind / unbind host bitmaps
    kinds = {st["k"] for p in programs for st in p.steps}
    assert {"set_stream", "bind_host", "download_wait", "free"} <= kinds
    # every program ends with nothing live
    for p in programs:
        assert not [h for h in p.h.values() if h.alive], p.seed


def test_same_seed_same_program(R, programs):
    for p in (programs[0], programs[-1]):
        q = pm.Program(R, p.seed, p.width)
        assert _fingerprint(q) == _fingerprint(p), p.seed


def _fingerprint(p):
    import hashlib
    h = hashlib.sha256()
    for st in p.steps:
        h.update(repr(sorted((k, _plain(v)) for k, v in st.items())).encode())
    return h.hexdigest()


def _plain(v):
    import numpy as np
    if isinstance(v, np.ndarray):
        return (str(v.dtype), v.tobytes())
    if isinstance(v, (list, tuple)):
        return tuple(_plain(x) for x in v)
    if isinstance(v, bytes):
        import hashlib
        return hashlib.sha256(v).hexdigest()
    return v


def test_mode0_reframing_keeps_bucket_layout(R):
    """The 64-bit remove-runs expectation re-frames each bucket's 32-bit remove_run_compression: without runs
    to remove, it gives back the blob itself."""
    import numpy as np
    blob = R.r64_from_values(np.array([5, 70000, (1 << 32) + 9, (0xFFFFFFFF << 32) + 3], np.uint64), run_optimize=False)
    assert pm.r64_remove_runs_bytes(R, blob) == blob
    runs = R.r64_from_values(np.arange(1000, 5000, dtype=np.uint64) + (7 << 32))
    flat = R.r64_from_values(np.arange(1000, 5000, dtype=np.uint64) + (7 << 32), run_optimize=False)
    assert runs != flat and pm.r64_remove_runs_bytes(R, runs) == flat
