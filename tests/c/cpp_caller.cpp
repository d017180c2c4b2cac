// A C++ caller written against the REFERENCE's header-only wrapper (cpp/roaring/roaring.hh:
// operator&, operator|, operator^, operator-, the compound assignments, and_cardinality,
// fastunion).  oracle/Makefile links it with -lroaring_b200 ahead of -lroaring_ref and
// tests/test_link_resolution.py checks which library the dynamic linker binds every roaring_bitmap_* symbol to; the calls
// sit behind an argument check so the symbols are referenced without anything being executed.
#include <cstdio>

#include "roaring.hh"

int main(int argc, char **argv) {
    (void)argv;
    if (argc < 1000) return 0;
    roaring::Roaring a, b;
    a.add(1);
    b.addRange(5, 500000);
    roaring::Roaring c = a & b, d = a | b, e = a ^ b, f = a - b;
    c |= a;
    d &= b;
    e ^= a;
    f -= b;
    const roaring::Roaring *both[2] = {&a, &b};
    roaring::Roaring u = roaring::Roaring::fastunion(2, both);
    unsigned long long s = a.and_cardinality(b) + a.or_cardinality(b) + a.xor_cardinality(b) + a.andnot_cardinality(b);
    std::printf("%llu %llu %d %d %f\n", (unsigned long long)(c.cardinality() + d.cardinality() + e.cardinality() +
                                                              f.cardinality() + u.cardinality()),
                s, (int)a.intersect(b), (int)a.isSubset(b), a.jaccard_index(b));
    return 0;
}
