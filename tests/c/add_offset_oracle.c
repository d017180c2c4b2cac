/* tests/c/add_offset_oracle.c — TEST INFRASTRUCTURE ONLY (the checker, never the product).
 *
 * A plain-C, scalar restatement of roaring_bitmap_add_offset (CRoaring 5.1.0, src/roaring.c:2426-2507)
 * on portable-serialized bitmaps, built on the container helpers of oracle/roaring_oracle.c, which
 * it includes as it is (one translation unit, so that its static helpers are in reach).
 * tests/offset_oracles.py compiles it into a temporary directory and pins it against the reference
 * (tests/test_offset_host.py).  All file:line citations are relative to the reference's tree.
 */
#include "../../oracle/roaring_oracle.c"

/* One part of container_add_offset (containers.h:1536): the values of c that land below 65536
 * after the shift by in_off (hi == false: bitset.c:191-207, array.c:107-116, run.c:139-158) or at
 * 65536 and above, minus 65536 (hi == true: bitset.c:215-235, array.c:118-126, run.c:160-186; the
 * run across the split is cut in two, run.c:178-189).  The part keeps c's type; an empty part is
 * not made (card 0 returned, nothing allocated). */
static int offset_part(const oc_t *c, uint16_t in_off, bool hi, oc_t *part) {
    uint64_t src[WORDS], w[WORDS];
    to_words(c, src);
    memset(w, 0, sizeof(w));
    for (int i = 0; i < WORDS; i++) {
        for (uint64_t m = src[i]; m; m &= m - 1) {
            const uint32_t y = (uint32_t)(i * 64 + __builtin_ctzll(m)) + in_off;
            if ((y >= 65536) == hi) w[(y & 0xFFFF) >> 6] |= UINT64_C(1) << (y & 63);
        }
    }
    const int card = words_card(w);
    if (card == 0) return 0;
    if (c->type == T_BITSET) *part = mk_bitset(w, card);
    else if (c->type == T_ARRAY) *part = mk_array(w);
    else *part = mk_run(w);
    return card;
}

/* container_ior(prev, cur) of two disjoint, non-full parts (containers.h:1226-1319), as
 * offset_append_with_merge calls it (roaring.c:2398-2424) */
static oc_t offset_ior(oc_t *prev, oc_t *cur) {
    uint64_t w[WORDS], w2[WORDS];
    to_words(prev, w);
    to_words(cur, w2);
    for (int i = 0; i < WORDS; i++) w[i] |= w2[i];
    const int card = words_card(w);
    oc_t r;
    switch (PAIR(prev->type, cur->type)) {
        case PAIR(T_BITSET, T_BITSET): /* bitset_container_or + OR_BITSET_CONVERSION_TO_FULL (:1233-1244) */
            r = card == 65536 ? mk_run(w) : mk_bitset(w, card);
            break;
        case PAIR(T_ARRAY, T_ARRAY): /* array_array_container_inplace_union (:1246-1254) */
            r = ab_from_words(w);
            break;
        case PAIR(T_BITSET, T_ARRAY): /* :1261-1273, never an array */
        case PAIR(T_ARRAY, T_BITSET):
        case PAIR(T_BITSET, T_RUN): /* :1275-1297, the full-run branches cannot fire */
        case PAIR(T_RUN, T_BITSET):
            r = mk_bitset(w, card);
            break;
        default: /* run with run or array: convert_run_to_efficient_container (:1256-1259, 1299-1313) */
            r = eff_from_words(w);
    }
    oc_free(prev);
    oc_free(cur);
    return r;
}

/* roaring_bitmap_add_offset (roaring.c:2426-2507).  offset == 0: a copy (:2443-2445).  Otherwise
 * co = offset >> 16 (arithmetic), in_off = offset - co * 65536 in [0, 65535] (:2446-2447).
 * in_off == 0: every container unchanged at key + co, keys outside [0, 65535] dropped, no repair
 * (:2454-2468).  Else container k is split into lo (at k + co) and hi (at k + co + 1), parts whose
 * key is out of range are not made (:2476-2485), a lo part landing on the key of the previous hi
 * part is merged into it (:2490-2491), and every container is repaired (:2503).  Writes the
 * portable bytes of the result to out when they fit in cap; returns the size needed, (size_t)-1 on
 * a malformed input. */
size_t oracle_add_offset(const uint8_t *a, size_t na, int64_t offset, uint8_t *out, size_t cap) {
    obm_t x, ans;
    if (!bm_parse(&x, a, na)) return (size_t)-1;
    const int64_t co = offset >> 16;
    const uint16_t in_off = (uint16_t)(offset - co * 65536);
    bm_init(&ans, 2 * x.n);
    for (int i = 0; i < x.n; i++) {
        const int64_t k = (int64_t)x.keys[i] + co;
        const bool lo_ok = k >= 0 && k < 65536, hi_ok = k + 1 >= 0 && k + 1 < 65536;
        if (in_off == 0) {
            if (lo_ok) bm_append(&ans, (uint16_t)k, oc_clone(&x.c[i]));
            continue;
        }
        oc_t lo, hi;
        if (lo_ok && offset_part(&x.c[i], in_off, false, &lo)) {
            if (ans.n > 0 && ans.keys[ans.n - 1] == k) ans.c[ans.n - 1] = offset_ior(&ans.c[ans.n - 1], &lo);
            else bm_append(&ans, (uint16_t)k, lo);
        }
        if (hi_ok && offset_part(&x.c[i], in_off, true, &hi)) bm_append(&ans, (uint16_t)(k + 1), hi);
    }
    if (in_off != 0)
        for (int i = 0; i < ans.n; i++) repair(&ans.c[i]); /* roaring_bitmap_repair_after_lazy, :2845 */
    size_t r = bm_serialize(&ans, out, cap);
    bm_free(&x);
    bm_free(&ans);
    return r;
}
