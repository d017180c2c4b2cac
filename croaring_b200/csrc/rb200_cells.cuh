// rb200_cells.cuh — the container x container grid cells (include/roaring/containers/containers.h:
// 726-1876 and src/containers/mixed_*.c of the reference) as ONE warp-level function, shared by the
// batched kernel (rb200_kernels.cu: k_compute_items) and the single-pair kernel (rb200_fused.cu).
#pragma once
#include "rb200_device.cuh"

namespace rb200 {

#ifndef RB200_FILTER_GLOBAL_MAX
#define RB200_FILTER_GLOBAL_MAX 192   // AND / ANDNOT of an array below this many values with a bitset tests the bits
                                      // in global memory instead of copying the bitset into the accumulator
#endif

// ------------------------------------------------------------------------------ grid cells
// Evaluate one matched cell on the warp's accumulator and write the result payload.
template <int OP, bool LAZY>
__device__ __forceinline__ void
cell_compute(uint32_t *acc, int tA, int tB, const uint8_t *pa, const uint8_t *pb,
             uint32_t cA, uint32_t cB, uint32_t lA, uint32_t lB, uint8_t *out, uint32_t cap,
             int lane, int &otype, uint32_t &ocard, uint32_t &olen, unsigned int *err,
             int rules, bool unkA) {
    // ---- run x run / array x run with few intervals: boundary sweep, no accumulator ---------
    constexpr int op = OP;
    const bool inplace_rules = (rules & RULES_INPLACE) != 0;
    constexpr bool lazy = LAZY && (OP == OP_OR || OP == OP_XOR);
    constexpr uint32_t AV = (OP == OP_OR || OP == OP_XOR) ? APPLY_VECS_OR : APPLY_VECS;   // array rasterise batch
    if (!lazy && (tA == T_RUN || tB == T_RUN) && tA != T_BITSET && tB != T_BITSET &&
        (tA == T_RUN ? lA : cA) + (tB == T_RUN ? lB : cB) <= 512u) {
        if (interval_cell(acc, op, tA, tB, pa, pb, cA, cB, lA, lB, out, cap, lane, otype, ocard, olen))
            return;
    }

    // ---- result is always an array and one side is an array: filter, no re-encode --------
    if (op == OP_AND && (tA == T_ARRAY || tB == T_ARRAY)) {
        // filter the array side through the other side's bits
        const bool arrA = (tA == T_ARRAY) && !(tB == T_ARRAY && cB < cA);  // filter the smaller
        const uint8_t *parr = arrA ? pa : pb;
        const uint32_t narr = arrA ? cA : cB;
        const int to = arrA ? tB : tA;
        const uint8_t *po = arrA ? pb : pa;
        const uint32_t lo = arrA ? lB : lA;
        uint32_t n;
        // (the filter writes only the values it keeps: at most min(cA, cB) of them, in whole 16-byte
        //  words, and the slot is a multiple of 16 bytes)
        if (2 * min(cA, cB) > cap) { if (lane == 0) atomicExch(err, 1u); otype = 0; return; }
        uint16_t *o16 = reinterpret_cast<uint16_t *>(out), *wb = reinterpret_cast<uint16_t *>(acc) + MERGE_WBUF;
        if (to == T_BITSET && narr < (uint32_t)RB200_FILTER_GLOBAL_MAX) {  // few probes: test the bits where they are
            n = filter_array<false, true>(parr, narr, reinterpret_cast<const uint32_t *>(po), o16, wb, lane, false);
        } else {   // a bitset's copy and the array's loads share one trip
            if (to == T_BITSET) acc_copy_bitset_async(acc, po, lane);
            else acc_load<AV>(acc, to, po, lo, lane);
            n = filter_array<false, true>(parr, narr, acc, o16, wb, lane, to == T_BITSET);
        }
        __syncwarp();
        otype = n ? T_ARRAY : 0;
        ocard = olen = n;
        return;
    }
    if (op == OP_ANDNOT && tA == T_ARRAY) {
        uint32_t n;
        if (2 * cA > cap) { if (lane == 0) atomicExch(err, 1u); otype = 0; return; }
        uint16_t *o16 = reinterpret_cast<uint16_t *>(out), *wb = reinterpret_cast<uint16_t *>(acc) + MERGE_WBUF;
        if (tB == T_BITSET && cA < (uint32_t)RB200_FILTER_GLOBAL_MAX) {
            n = filter_array<true, true>(pa, cA, reinterpret_cast<const uint32_t *>(pb), o16, wb, lane, false);
        } else {
            if (tB == T_BITSET) acc_copy_bitset_async(acc, pb, lane);
            else acc_load<AV>(acc, tB, pb, lB, lane);
            n = filter_array<true, true>(pa, cA, acc, o16, wb, lane, tB == T_BITSET);
        }
        __syncwarp();
        otype = n ? T_ARRAY : 0;
        ocard = olen = n;
        return;
    }

    // ---- array x array union / xor whose result is known to stay an array: warp merge path ---
    // (cA + cB <= MAX_ARRAY: the type rule makes the result an array whatever its cardinality)
    // (lazy rules: only unions / xors of at most ARRAY_LAZY_LOWERBOUND values stay arrays)
    const bool lazy_eager = lazy && OP == OP_XOR && inplace_rules;  // container_lazy_ixor A,A is eager
    if ((op == OP_OR || op == OP_XOR) && tA == T_ARRAY && tB == T_ARRAY && cA + cB <= (uint32_t)MAX_ARRAY &&
        (!lazy || lazy_eager || (cA + cB <= 1024u && !(rules & RULES_CONV)))) {
        if (round16(2 * (cA + cB)) > cap) { if (lane == 0) atomicExch(err, 1u); otype = 0; return; }
        const uint32_t n = (op == OP_OR) ? merge_arrays<false>(acc, pa, cA, pb, cB, out, lane)
                                         : merge_arrays<true>(acc, pa, cA, pb, cB, out, lane);
        otype = n ? T_ARRAY : 0;  // cA + cB <= 4096 -> array (mixed_union.c:162-176, mixed_xor.c:196-205)
        ocard = olen = n;
        return;
    }

    // ---- bitset | bitset: the result is a bitset (containers.h:1015-1020), so a | b goes from L2 to
    // the result slot, counted on the way, without the accumulator.  In place, a saturated union
    // becomes the full run unless the left container was full already (see the rules below).
    if (OP == OP_OR && !lazy && tA == T_BITSET && tB == T_BITSET && cap >= (uint32_t)BITSET_BYTES) {
        const int card = acc_bitset_op_bitset<OP_OR>(reinterpret_cast<uint32_t *>(out), pa, pb, lane);
        otype = T_BITSET;
        ocard = (uint32_t)card;
        olen = 1024u;
        if (card == 0) {
            otype = 0;
            olen = 0;
        } else if (inplace_rules && card == 65536 && cA != 65536u) {
            // the run {0, 65535} over the first word of the bitset, which this lane stored itself
            if (lane == 0) reinterpret_cast<uint32_t *>(out)[0] = 0xffff0000u;
            otype = T_RUN;
            olen = 1u;
        }
        return;
    }

    // ---- general path: acc = A op B --------------------------------------------------------
    int card = -1, nruns = 0;
    if (tA == T_BITSET && tB == T_BITSET) {
        switch (op) {
            case OP_AND: card = acc_bitset_op_bitset<OP_AND>(acc, pa, pb, lane); break;
            case OP_OR: card = acc_bitset_op_bitset<OP_OR>(acc, pa, pb, lane); break;
            case OP_XOR: card = acc_bitset_op_bitset<OP_XOR>(acc, pa, pb, lane); break;
            default: card = acc_bitset_op_bitset<OP_ANDNOT>(acc, pa, pb, lane); break;
        }
        __syncwarp();
    } else if ((tA == T_BITSET && tB == T_ARRAY) || (tA == T_ARRAY && tB == T_BITSET)) {
        // bitset with an array (AND and A x B ANDNOT took the filter above): the bitset is copied into
        // the accumulator by cp.async and the array applied on top, its first 512 values staged by
        // cp.async in the same trip.  A x B unions / xors run as B op A, the same set.  The atomics
        // return the words they change, so the result's cardinality is the bitset's plus what the
        // array changed, and the accumulator is not counted again (the lazy rules count it anyway).
        const bool arrA = tA == T_ARRAY;
        const uint8_t *parr = arrA ? pa : pb;
        const uint32_t narr = arrA ? cA : cB;
        acc_copy_bitset_async(acc, arrA ? pb : pa, lane);
        int delta = 0;
        if (op == OP_OR) delta = acc_apply_array_staged<0>(acc, parr, narr, lane);
        else if (op == OP_XOR) delta = acc_apply_array_staged<1>(acc, parr, narr, lane);
        else if (op == OP_ANDNOT) delta = acc_apply_array_staged<2>(acc, parr, narr, lane);
        if (!lazy && op != OP_AND) card = (int)(arrA ? cB : cA) + __reduce_add_sync(FULLMASK, delta);
        __syncwarp();
    } else {
        acc_load<AV>(acc, tA, pa, lA, lane);
        if (tB == T_BITSET) {
            switch (op) {
                case OP_AND: acc_op_bitset<OP_AND>(acc, pb, lane); break;
                case OP_OR: acc_op_bitset<OP_OR>(acc, pb, lane); break;
                case OP_XOR: acc_op_bitset<OP_XOR>(acc, pb, lane); break;
                default: acc_op_bitset<OP_ANDNOT>(acc, pb, lane); break;
            }
        } else if (tB == T_ARRAY) {
            switch (op) {
                case OP_AND: acc_and_array(acc, pb, cB, lane); break;  // not reached (filter path)
                case OP_OR: acc_apply_array<0, APPLY_NONE, AV>(acc, pb, cB, lane); break;
                case OP_XOR: acc_apply_array<1, APPLY_NONE, AV>(acc, pb, cB, lane); break;
                default: acc_apply_array<2, APPLY_NONE, AV>(acc, pb, cB, lane); break;
            }
        } else {
            switch (op) {
                case OP_AND: acc_and_runs(acc, pb, lB, lane); break;
                case OP_OR: acc_apply_runs<0, false>(acc, pb, lB, lane); break;
                case OP_XOR: acc_apply_runs<1, false>(acc, pb, lB, lane); break;
                default: acc_apply_runs<2, false>(acc, pb, lB, lane); break;
            }
        }
        __syncwarp();
    }
    const bool want_runs = lazy ? ((tA == T_RUN || tB == T_RUN) && tA != T_BITSET && tB != T_BITSET)
                                : cell_needs_runs(op, tA, tB);
    if (card < 0 || want_runs) acc_count(acc, lane, want_runs, card, nruns);
    if (card == 0) { otype = 0; ocard = olen = 0; return; }
    bool unknown = false;
    int t = lazy ? decide_type_lazy(op, rules, tA, tB, cA, cB, lA, lB, unkA, card, nruns, unknown)
                 : decide_type(op, tA, tB, cA, cB, lA, lB, card, nruns);
    if (OP == OP_OR && inplace_rules && !lazy) {
        // roaring_bitmap_or_inplace: a full left container is left untouched (roaring.c:1081-1083)
        // and container_ior turns a saturated bitset|bitset into the full run (containers.h:1234-1242)
        const bool a_full = is_full_run(tA, lA, cA) || (tA == T_BITSET && cA == 65536u);
        if (a_full) t = tA;
        else if (tA == T_BITSET && tB == T_BITSET && card == 65536) t = T_RUN;
    }
    if (t == T_RUN && !want_runs) {  // bitset OR full-run -> [0,65535]
        nruns = 1;
    }
    const uint32_t len = (t == T_BITSET) ? 1024u : (t == T_ARRAY ? (uint32_t)card : (uint32_t)nruns);
    if (stored_bytes(t, len) > cap) { if (lane == 0) atomicExch(err, 1u); otype = 0; return; }
    if (t == T_BITSET) acc_store_bitset(acc, out, lane);
    else if (t == T_ARRAY) acc_emit_array(acc, reinterpret_cast<uint16_t *>(out), lane);
    else acc_emit_runs(acc, reinterpret_cast<uint16_t *>(out), lane);
    __syncwarp();
    otype = t;
    ocard = (uint32_t)card | (unknown ? CARD_UNKNOWN : 0u);
    olen = len;
}


}  // namespace rb200
