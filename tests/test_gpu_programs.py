"""GPU test: the seeded random programs of tests/program_model.py — chains of producers over live resident
sets, frees in arbitrary order, every survivor read back — byte for byte against the reference, in this
process and again in a child process whose pools zero every block they take back (RB200_POISON_POOL=1,
read when the library loads), so that a read of a released block gives wrong bytes instead of the old
ones.  Both runs must pass every check and digest the same checked bytes, and a program must give back
every device block it took.  RB200_PROGRAM_SEEDS=a-b runs a longer list of seeds."""
import os
import subprocess
import sys

import pytest

import program_model as pm

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEEDS32, SEEDS64 = pm.seeds_from_env()
PROGRAMS = [(s, 32) for s in SEEDS32] + [(s, 64) for s in SEEDS64]

CHILD = r'''
import sys
sys.path.insert(0, "tests")
import croaring_b200 as rb
from oracle.refbind import ref
import program_model as pm
rb.init(0)
R = ref()
for arg in sys.argv[1:]:
    s, w = (int(x) for x in arg.split(":"))
    print(f"{s}:{w} {pm.run_program(rb, R, s, w)}", flush=True)
'''


@pytest.fixture(scope="module")
def digests(rb, R):
    """{(seed, width): digest} of every program run in this process; the device memory in use after each
    equals its value after the first (warm) program."""
    L = rb.lib()
    out, base = {}, None
    for s, w in PROGRAMS:
        out[(s, w)] = pm.run_program(rb, R, s, w)
        rb.download_wait()
        rb.synchronize()
        used = int(L.rb200_device_bytes_in_use())
        if base is None:
            base = used
        assert used == base, f"seed {s} width {w}: {used - base} device bytes still in use after the program"
    return out


def test_programs_match_reference(digests):
    assert len(digests) == len(PROGRAMS)


def test_programs_with_poisoned_pools(digests):
    env = dict(os.environ, RB200_POISON_POOL="1", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    args = [f"{s}:{w}" for s, w in PROGRAMS]
    out = subprocess.run([sys.executable, "-s", "-c", CHILD, *args], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1800)
    assert "libroaring_b200: pool poisoning on" in out.stderr, out.stderr[-2000:]
    assert out.returncode == 0, out.stderr[-4000:]
    got = dict(line.split(" ", 1) for line in out.stdout.strip().splitlines())
    for s, w in PROGRAMS:
        assert got.get(f"{s}:{w}") == digests[(s, w)], f"seed {s} width {w}: poisoned run digests differ"
