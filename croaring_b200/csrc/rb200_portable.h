// rb200_portable.h — the portable byte format (src/roaring_array.c:469-531, :633-813 of the
// reference) on the host: one reader and one writer for every host path that handles portable bytes
// (rb200_host.cu: host bitmaps, 64-bit bucket headers, flip ranges; rb200_shard.cu: key-range slicing
// and concatenation).  Header-only, no allocation.  The device has its own warp-parallel walkers
// (k_deser_dir, k_ser_*) over the same constants.
#pragma once
#include <stddef.h>
#include <string.h>

#include "rb200_common.h"
#include "rb200_device.cuh"

namespace rb200 {

// One container, read from or written to a portable bitmap.  The payload is in the slab's stored
// layout: `len` array values, `len` runs without their n_runs prefix, or 1024 bitset words.
struct PortableEntry {
    uint16_t key;
    uint8_t type;
    uint32_t card;   // cardinality (written as card - 1; CARD_UNKNOWN is ignored).  Read: as the header
                     // states it, except a run container's: the reference ignores that field and
                     // writes the count of its runs, so the walk counts them too
    uint32_t len;
    const uint8_t *payload;
};

// Container count of a portable bitmap from its cookie alone (O(1)); false: not a portable bitmap.
inline bool portable_count(const uint8_t *buf, size_t len, uint32_t &n, bool &hasrun) {
    if (len < 4) return false;
    uint32_t cookie;
    memcpy(&cookie, buf, 4);
    if ((cookie & 0xFFFF) == SERIAL_COOKIE) {
        n = (cookie >> 16) + 1;
        hasrun = true;
    } else if (cookie == SERIAL_COOKIE_NO_RUN && len >= 8) {
        memcpy(&n, buf + 4, 4);
        hasrun = false;
    } else {
        return false;
    }
    return n <= 65536 && 4ull * n <= len;
}

// Walk the portable bitmap at buf, calling fn(const PortableEntry &) for each container in order.
// Returns its length in bytes (at most len), or 0 if it is malformed: bad cookie or count, key /
// cardinality pairs or a payload past len, keys not strictly increasing.  The offset header is
// skipped, not trusted; container contents are not checked.  fn may have seen a prefix of the
// containers of a blob that turns out malformed.
template <class F>
size_t walk_portable(const uint8_t *buf, size_t len, F &&fn) {
    uint32_t n;
    bool hasrun;
    if (!portable_count(buf, len, n, hasrun)) return 0;
    size_t pos = hasrun ? 4 + (n + 7) / 8 : 8;
    if (pos + 4ull * n > len) return 0;
    const uint8_t *flags = buf + 4, *kc = buf + pos;
    pos += 4ull * n;
    if (!hasrun || n >= NO_OFFSET_THRESHOLD) pos += 4ull * n;
    uint16_t prev = 0;
    for (uint32_t i = 0; i < n; i++) {
        PortableEntry e;
        uint16_t cm1;
        memcpy(&e.key, kc + 4 * i, 2);
        memcpy(&cm1, kc + 4 * i + 2, 2);
        if (i && e.key <= prev) return 0;
        prev = e.key;
        e.card = (uint32_t)cm1 + 1;
        if (hasrun && ((flags[i >> 3] >> (i & 7)) & 1)) {
            if (pos + 2 > len) return 0;
            uint16_t nr;
            memcpy(&nr, buf + pos, 2);
            pos += 2;
            e.type = T_RUN;
            e.len = nr;
        } else if (e.card > (uint32_t)MAX_ARRAY) {
            e.type = T_BITSET;
            e.len = 1024;
        } else {
            e.type = T_ARRAY;
            e.len = e.card;
        }
        const uint32_t sb = stored_bytes(e.type, e.len);
        if (pos + sb > len) return 0;
        e.payload = buf + pos;
        pos += sb;
        if (e.type == T_RUN) {
            e.card = 0;
            for (uint32_t k = 0; k < e.len; k++)
                e.card += ((uint32_t)e.payload[4 * k + 2] | ((uint32_t)e.payload[4 * k + 3] << 8)) + 1u;
        }
        fn(e);
    }
    return pos;
}

// Size and bytes of the portable bitmap of containers entry(0) .. entry(n - 1) (n <= 65536, keys
// increasing).  write_portable returns the bytes written, portable_size(n, entry) of them.
template <class F>
size_t portable_size(uint32_t n, F &&entry) {
    bool hasrun = false;
    size_t bytes = 0;
    for (uint32_t i = 0; i < n; i++) {
        const PortableEntry e = entry(i);
        hasrun |= e.type == T_RUN;
        bytes += portable_bytes(e.type, e.len);
    }
    return portable_header_bytes(n, hasrun) + bytes;
}

template <class F>
size_t write_portable(uint8_t *out, uint32_t n, F &&entry) {
    bool hasrun = false;
    for (uint32_t i = 0; i < n && !hasrun; i++) hasrun = entry(i).type == T_RUN;
    uint8_t *kc, *offs = nullptr;
    if (hasrun) {
        const uint32_t cookie = SERIAL_COOKIE | ((n - 1) << 16);
        memcpy(out, &cookie, 4);
        memset(out + 4, 0, (n + 7) / 8);   // run flags
        kc = out + 4 + (n + 7) / 8;
        if (n >= NO_OFFSET_THRESHOLD) offs = kc + 4ull * n;
    } else {
        memcpy(out, &SERIAL_COOKIE_NO_RUN, 4);
        memcpy(out + 4, &n, 4);
        kc = out + 8;
        offs = kc + 4ull * n;
    }
    size_t pos = portable_header_bytes(n, hasrun);
    for (uint32_t i = 0; i < n; i++) {
        const PortableEntry e = entry(i);
        const uint16_t cm1 = (uint16_t)((e.card & CARD_MASK) - 1);
        memcpy(kc + 4ull * i, &e.key, 2);
        memcpy(kc + 4ull * i + 2, &cm1, 2);
        if (offs) {
            const uint32_t o = (uint32_t)pos;
            memcpy(offs + 4ull * i, &o, 4);
        }
        if (e.type == T_RUN) {
            out[4 + i / 8] |= (uint8_t)(1u << (i % 8));
            const uint16_t nr = (uint16_t)e.len;
            memcpy(out + pos, &nr, 2);
            pos += 2;
        }
        const uint32_t sb = stored_bytes(e.type, e.len);
        memcpy(out + pos, e.payload, sb);
        pos += sb;
    }
    return pos;
}

}  // namespace rb200
