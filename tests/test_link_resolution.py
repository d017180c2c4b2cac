"""CPU check (-m "not gpu") of the drop-in boundary at LINK level, for the reference's C++ wrapper:
a program written against cpp/roaring/roaring.hh and linked with -lroaring_b200 ahead of
-lroaring_ref must have every hot-path symbol (roaring_bitmap_and / _or / _xor / _andnot, the
in-place twins, or_many, the cardinality family, intersect, is_subset ...) bound to
libroaring_b200.so by the dynamic linker and everything else (create, add, free, cardinality ...)
to the reference — "the header-only wrapper needs no change" (INTEGRATION.md section 3).  Nothing
is executed: LD_BIND_NOW + LD_DEBUG=bindings list the bindings at load time.  The executed form of
the same claim (C caller, results compared) is tests/test_gpu_dropin_c.py."""
import os
import re
import subprocess

import pytest

import croaring_b200 as rb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFDIR = os.path.join(ROOT, "oracle", "_ref")


@pytest.mark.skipif(not os.path.exists(os.path.join(REFDIR, "cpp_caller")), reason="needs oracle/_ref (make -C oracle)")
def test_cpp_wrapper_binds_hot_path_to_our_library():
    """tests/c/cpp_caller.cpp, compiled against the reference's headers by oracle/Makefile."""
    rb.lib()   # (built)
    exe = os.path.join(REFDIR, "cpp_caller")
    env = dict(os.environ, LD_BIND_NOW="1", LD_DEBUG="bindings")
    p = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stderr[-2000:]
    bound = {}
    for m in re.finditer(r"binding file (\S+) \[\d+\] to (\S+) \[\d+\]: normal symbol `(roaring_bitmap_\w+)'", p.stderr):
        if m.group(1) == exe:
            bound[m.group(3)] = os.path.basename(m.group(2))
    ours = ["roaring_bitmap_and", "roaring_bitmap_or", "roaring_bitmap_xor", "roaring_bitmap_andnot",
            "roaring_bitmap_and_inplace", "roaring_bitmap_or_inplace", "roaring_bitmap_xor_inplace",
            "roaring_bitmap_andnot_inplace", "roaring_bitmap_or_many", "roaring_bitmap_and_cardinality",
            "roaring_bitmap_or_cardinality", "roaring_bitmap_xor_cardinality", "roaring_bitmap_andnot_cardinality",
            "roaring_bitmap_jaccard_index", "roaring_bitmap_intersect", "roaring_bitmap_is_subset"]
    for name in ours:
        assert bound.get(name) == "libroaring_b200.so", (name, bound.get(name))
    theirs = [n for n, lib in bound.items() if lib == "libroaring_ref.so"]
    assert "roaring_bitmap_add" in theirs and "roaring_bitmap_get_cardinality" in theirs and len(theirs) >= 4
    # nothing outside the header's list leaks out of our library under a reference name
    hdr = open(os.path.join(ROOT, "include", "roaring_b200.h")).read()
    declared = set(re.findall(r"\b(roaring_bitmap_[a-z0-9_]+)\s*\(", hdr))
    assert all(n in declared for n, lib in bound.items() if lib == "libroaring_b200.so")


@pytest.mark.skipif(not os.path.exists(os.path.join(REFDIR, "dropin_caller_ref")), reason="needs oracle/_ref (make -C oracle)")
def test_ld_preload_rebinds_an_existing_binary():
    """The other deployment of INTEGRATION.md section 1: a binary linked against the reference ALONE
    (oracle/_ref/dropin_caller_ref), started under LD_PRELOAD=libroaring_b200.so — every symbol our
    header declares under a reference name is taken from our library, the rest stays the reference's."""
    exe = os.path.join(REFDIR, "dropin_caller_ref")
    env = dict(os.environ, LD_BIND_NOW="1", LD_DEBUG="bindings", LD_PRELOAD=rb.api.LIB_PATH)
    p = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=120)   # no arguments: usage, exit 2
    bound = {}
    for m in re.finditer(r"binding file (\S+) \[\d+\] to (\S+) \[\d+\]: normal symbol `(roaring\w*_bitmap_\w+)'", p.stderr):
        if m.group(1) == exe:
            bound[m.group(3)] = os.path.basename(m.group(2))
    hdr = open(os.path.join(ROOT, "include", "roaring_b200.h")).read()
    declared = set(re.findall(r"\b(roaring(?:64)?_bitmap_[a-z0-9_]+)\s*\(", hdr))
    used_ours = {n for n in bound if n in declared}
    assert len(used_ours) >= 15, sorted(bound)
    for n, lib in bound.items():
        assert lib == ("libroaring_b200.so" if n in declared else "libroaring_ref.so"), (n, lib)
