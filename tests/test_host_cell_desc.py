"""CPU test: the 32-byte cell descriptor of the pairwise kernel (cd_pack / cd_unpack in rb200_common.h)
is a host+device helper; every field survives packing and unpacking at its limits, compiled for the
host with nvcc."""

from helpers import run_probe


def test_cell_descriptor_round_trip():
    src = r'''
#include "rb200_common.h"
#include <cstdio>
using namespace rb200;
int bad = 0;
#define CHECK(c) do { if (!(c)) { printf("FAIL line %d: %s\n", __LINE__, #c); bad++; } } while (0)
int main() {
    // offsets: 16-byte aligned, up to the largest the descriptor holds (2^44 - 16)
    const uint64_t offs[] = {0, 16, (1ull << 36) - 16, 1ull << 36, (1ull << 40) + 16, (1ull << 44) - 16};
    const uint32_t cards[] = {0, 1, 4096, 4097, 65535, 65536};
    const uint32_t lens[] = {0, 1, 1024, 4096, 32767, 32768};
    const uint32_t caps[] = {0, 16, 8192, 131072, 262144};
    const uint32_t items[] = {0, 1, 0xfffffffeu};
    long n = 0;
    for (uint32_t kind = K_HOLE; kind <= K_COPY_B; kind++)
        for (uint32_t tA = T_BITSET; tA <= T_RUN; tA++)
            for (uint32_t tB = T_BITSET; tB <= T_RUN; tB++)
                for (int oi = 0; oi < 6; oi++)
                    for (int ci = 0; ci < 6; ci++)
                        for (int li = 0; li < 6; li++)
                            for (int unk = 0; unk < 2; unk++) {
                                CellDesc d = {};
                                d.offA = offs[oi];
                                d.offB = offs[(oi + 2) % 6];
                                d.off = offs[(oi + 4) % 6];
                                d.item = items[(oi + ci) % 3];
                                d.cA = cards[ci] | (unk ? CARD_UNKNOWN : 0u);
                                d.cB = cards[(ci + li) % 6];
                                d.lA = lens[li];
                                d.lB = lens[(li + 3) % 6];
                                d.cap = caps[(ci + oi) % 5];
                                d.tA = tA;
                                d.tB = tB;
                                d.kind = kind;
                                d.shared = ((oi + li + unk) & 1) != 0;
                                uint4 a, b;
                                cd_pack(d, a, b);
                                const CellDesc e = cd_unpack(a, b);
                                CHECK(e.offA == d.offA && e.offB == d.offB && e.off == d.off);
                                CHECK(e.item == d.item && e.cA == d.cA && e.cB == d.cB);
                                CHECK(e.lA == d.lA && e.lB == d.lB && e.cap == d.cap);
                                CHECK(e.tA == d.tA && e.tB == d.tB && e.kind == d.kind && e.shared == d.shared);
                                n++;
                            }
    // a hole is all zero
    CellDesc z = {};
    uint4 a, b;
    cd_pack(z, a, b);
    CHECK(a.x == 0 && a.y == 0 && a.z == 0 && a.w == 0 && b.x == 0 && b.y == 0 && b.z == 0 && b.w == 0);
    CHECK(cd_unpack(a, b).kind == K_HOLE);
    CHECK(sizeof(a) + sizeof(b) == 32);
    printf("cases=%ld bad=%d\n", n, bad);
    return bad;
}
'''
    out = run_probe(src)
    assert out.returncode == 0, out.stdout
