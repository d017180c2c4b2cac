"""CPU test of the host portable codec (croaring_b200/csrc/rb200_portable.h), compiled into a probe:
walking a blob and writing its containers back reproduces it byte for byte, the cookie-only count
agrees with the walk, and truncated blobs or blobs whose keys do not strictly increase are refused."""
import struct

import croaring_b200 as rb
from helpers import DATASETS, run_probe, synth_blobs

PROBE = r'''
#include "rb200_portable.h"
#include <cstdio>
#include <vector>
using namespace rb200;
int bad = 0;
size_t cur = 0;
#define CHECK(c) do { if (!(c)) { if (bad++ < 20) printf("FAIL blob %zu line %d: %s\n", cur, __LINE__, #c); } } while (0)

size_t walk_len(const uint8_t *p, size_t len) { return walk_portable(p, len, [](const PortableEntry &) {}); }

int main(int argc, char **argv) {
    const uint32_t norun[6] = {8, 16, 24, 32, 40, 48}, run[6] = {4, 9, 13, 17, 37, 45};
    for (uint32_t n = 0; n < 6; n++) {
        CHECK(portable_header_bytes(n, false) == norun[n]);
        CHECK(portable_header_bytes(n, true) == run[n]);
    }
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    std::vector<uint8_t> all;
    for (int ch; (ch = fgetc(f)) != EOF;) all.push_back((uint8_t)ch);
    fclose(f);
    for (size_t at = 0; at + 4 <= all.size(); cur++) {
        uint32_t len;
        memcpy(&len, &all[at], 4);
        const std::vector<uint8_t> buf(all.begin() + at + 4, all.begin() + at + 4 + len);   // its own allocation
        at += 4 + len;
        std::vector<PortableEntry> c;
        CHECK(walk_portable(buf.data(), len, [&c](const PortableEntry &e) { c.push_back(e); }) == len);
        uint32_t n = 0;
        bool hasrun = false, anyrun = false;
        CHECK(portable_count(buf.data(), len, n, hasrun) && n == c.size());
        for (const PortableEntry &e : c) anyrun |= e.type == T_RUN;
        CHECK(hasrun == anyrun);
        const auto entry = [&c](uint32_t i) { return c[i]; };
        CHECK(portable_size(n, entry) == len);
        std::vector<uint8_t> out(len + 16, 0xA5);
        CHECK(write_portable(out.data(), n, entry) == len);
        CHECK(memcmp(out.data(), buf.data(), len) == 0);
        CHECK(out[len] == 0xA5);
        for (size_t k = 0; k < len; k += k < 64 ? 1 : 1 + len / 64) CHECK(walk_len(buf.data(), k) == 0);
        CHECK(walk_len(buf.data(), len - 1) == 0);
        if (n >= 2) {   // key 1 equal to key 0, then the two swapped
            const size_t kc = hasrun ? 4 + (n + 7) / 8 : 8;
            std::vector<uint8_t> m = buf;
            memcpy(&m[kc + 4], &buf[kc], 2);
            CHECK(walk_len(m.data(), len) == 0);
            memcpy(&m[kc], &buf[kc + 4], 2);
            CHECK(walk_len(m.data(), len) == 0);
        }
    }
    printf("blobs=%zu bad=%d\n", cur, bad);
    return bad != 0;
}
'''


def test_walk_then_write_reproduces_every_blob(R, tmp_path):
    blobs = [b for ds in DATASETS for b in rb.load_realdata(ds)] + synth_blobs(R, 3, 60)
    path = tmp_path / "blobs.bin"
    path.write_bytes(b"".join(struct.pack("<I", len(b)) + b for b in blobs))
    out = run_probe(PROBE, str(path))
    assert out.returncode == 0, out.stdout + out.stderr
    assert f"blobs={len(blobs)} bad=0" in out.stdout
