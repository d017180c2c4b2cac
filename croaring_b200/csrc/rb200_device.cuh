// rb200_device.cuh — warp-level building blocks of the container x container grid (sm_90a).
//
// One warp owns one 65536-bit accumulator `acc` (2048 x u32 = 8 KiB of shared memory) and
// evaluates one grid cell on it:
//   rasterise the left container (bitset copy with 128-bit loads / array scatter /
//   run range-fill) -> apply the right container with the op -> popcount (+ run count)
//   -> pick the reference's result type -> re-encode (bitset copy / ordered bit extraction
//   with a warp scan / run boundary extraction).
// Cells whose result is always an array (AND / ANDNOT with an array on the filtering side)
// skip the accumulator round trip and filter the array through bit tests with
// ballot compaction.
//
// Reference semantics restated here (file:line relative to /root/reference):
//   type rules of the cells      include/roaring/containers/containers.h:726-806 (and),
//                                :1008-1103 (or), :1449-1524 (xor), :1783-1876 (andnot),
//                                src/containers/mixed_*.c, src/containers/convert.c:154-200
#pragma once
#include "rb200_common.h"

namespace rb200 {

constexpr unsigned FULLMASK = 0xffffffffu;

__device__ __forceinline__ unsigned lanemask_lt() {
    unsigned m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ int popc4(const uint4 &q) {
    return __popc(q.x) + __popc(q.y) + __popc(q.z) + __popc(q.w);
}

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t t = __shfl_up_sync(FULLMASK, v, d);
        if (lane >= d) v += t;
    }
    return v;
}

// ---------------------------------------------------------------- type rules
__host__ __device__ __forceinline__ int rule_ab(int card) {
    return card <= MAX_ARRAY ? T_ARRAY : T_BITSET;
}
// convert_run_to_efficient_container, src/containers/convert.c:154-200
__host__ __device__ __forceinline__ int rule_eff(int card, int nruns) {
    int size_run = 2 + 4 * nruns, size_arr = 2 * card;
    int min_non_run = size_arr < BITSET_BYTES ? size_arr : BITSET_BYTES;
    if (size_run <= min_non_run) return T_RUN;
    return rule_ab(card);
}
__host__ __device__ __forceinline__ bool is_full_run(int t, uint32_t len, uint32_t card) {
    return t == T_RUN && len == 1 && card == 65536;
}

// Does the type rule of this cell look at the number of runs of the result?
__host__ __device__ __forceinline__ bool cell_needs_runs(int op, int tA, int tB) {
    if (tA == T_BITSET || tB == T_BITSET) return false;
    if (tA == T_RUN && tB == T_RUN) return true;
    if (op == OP_AND) return false;                // A,R / R,A / A,A -> array
    if (op == OP_ANDNOT) return tA == T_RUN;       // R,A
    return tA == T_RUN || tB == T_RUN;             // OR / XOR with a run
}

// Result container type of a grid cell given the input metadata and the result's
// cardinality / run count.  Mirrors oracle/roaring_oracle.c cell_* (pinned to the reference).
__host__ __device__ inline int decide_type(int op, int tA, int tB, uint32_t cA, uint32_t cB,
                                           uint32_t lA, uint32_t lB, int card, int nruns) {
    const bool fullA = is_full_run(tA, lA, cA), fullB = is_full_run(tB, lB, cB);
    const bool hasB = (tA == T_BITSET) || (tB == T_BITSET);
    const bool bothR = (tA == T_RUN) && (tB == T_RUN);
    const bool bothA = (tA == T_ARRAY) && (tB == T_ARRAY);
    switch (op) {
        case OP_AND:
            if (tA == T_BITSET && tB == T_BITSET) return rule_ab(card);
            if (bothR) return rule_eff(card, nruns);
            if (hasB && (tA == T_RUN || tB == T_RUN)) {  // mixed_intersection.c:117-203
                if (fullA || fullB) return T_BITSET;
                uint32_t cR = (tA == T_RUN) ? cA : cB;
                if (cR <= (uint32_t)MAX_ARRAY) return T_ARRAY;
                return rule_ab(card);
            }
            return T_ARRAY;
        case OP_OR:
            if (bothA) return (cA + cB <= (uint32_t)MAX_ARRAY) ? T_ARRAY : rule_ab(card);
            if (hasB) {
                if (fullA || fullB) return T_RUN;  // containers.h:1056-1080
                return T_BITSET;
            }
            return rule_eff(card, nruns);
        case OP_XOR:
            if (bothA) return (cA + cB <= (uint32_t)MAX_ARRAY) ? T_ARRAY : rule_ab(card);
            if (hasB) return rule_ab(card);
            if (bothR) return rule_eff(card, nruns);
            {  // array_run_container_xor, mixed_xor.c:104-138
                uint32_t ca = (tA == T_ARRAY) ? cA : cB, cr = (tA == T_ARRAY) ? cB : cA;
                if (ca < 32) return rule_eff(card, nruns);
                if (cr <= (uint32_t)MAX_ARRAY)
                    return (cr + ca <= (uint32_t)MAX_ARRAY) ? T_ARRAY : rule_ab(card);
                return rule_ab(card);
            }
        default:  // OP_ANDNOT
            if (tA == T_ARRAY) return T_ARRAY;
            if (bothR) return rule_eff(card, nruns);
            if (tA == T_BITSET) return rule_ab(card);
            // tA == RUN
            if (tB == T_BITSET) return cA <= (uint32_t)MAX_ARRAY ? T_ARRAY : rule_ab(card);
            // R,A: mixed_andnot.c:277-357
            if (cA <= 32) return rule_eff(card, nruns);
            if (cA <= (uint32_t)MAX_ARRAY) return T_ARRAY;
            return rule_ab(card);
    }
}

__host__ __device__ __forceinline__ uint32_t round16(uint32_t x) { return (x + 15u) & ~15u; }

// payload bytes as stored in a slab (runs without the 2-byte n_runs prefix)
__host__ __device__ __forceinline__ uint32_t stored_bytes(int t, uint32_t len) {
    return t == T_BITSET ? (uint32_t)BITSET_BYTES : (t == T_ARRAY ? 2u * len : 4u * len);
}
// container_size_in_bytes, include/roaring/containers/containers.h:402-416
__host__ __device__ __forceinline__ uint32_t portable_bytes(int t, uint32_t len) {
    return t == T_BITSET ? (uint32_t)BITSET_BYTES : (t == T_ARRAY ? 2u * len : 2u + 4u * len);
}

// "Effective bytes" of a container: what it can contribute to the result of a later op on it — its
// stored size, or the size of its values as an array / bitset if that is larger (a run of 4 bytes
// can hold 65536 values).  Summed per bitmap it bounds the result slab of a batch (PairBuf::build).
__host__ __device__ __forceinline__ uint32_t effective_bytes(int t, uint32_t len, uint32_t card) {
    const uint32_t st = stored_bytes(t, len), byc = card > (uint32_t)MAX_ARRAY ? (uint32_t)BITSET_BYTES : 2u * card;
    return round16(st > byc ? st : byc);
}

// Upper bound (bytes, multiple of 16) of the stored result of a COMPUTE cell.
__host__ __device__ inline uint32_t slot_bound(int op, int tA, int tB, uint32_t cA, uint32_t cB,
                                               uint32_t lA, uint32_t lB) {
    const uint32_t FULLB = BITSET_BYTES;
    uint32_t b = FULLB;
    const uint32_t nA = (tA == T_ARRAY) ? cA : lA, nB = (tB == T_ARRAY) ? cB : lB;
    const uint32_t cmin = cA < cB ? cA : cB;
    if (tA == T_BITSET || tB == T_BITSET) {
        if (op == OP_AND) {
            if (tA == T_ARRAY) b = 2 * cA;
            else if (tB == T_ARRAY) b = 2 * cB;
            else if (tA == T_RUN) b = cA <= (uint32_t)MAX_ARRAY ? 2 * cA : FULLB;
            else if (tB == T_RUN) b = cB <= (uint32_t)MAX_ARRAY ? 2 * cB : FULLB;
        } else if (op == OP_ANDNOT) {
            if (tA == T_ARRAY) b = 2 * cA;
            else if (tA == T_RUN) b = cA <= (uint32_t)MAX_ARRAY ? 2 * cA : FULLB;
        }
    } else {
        uint32_t runs_b = 4 * (nA + nB);
        if (op == OP_AND) {
            if (tA == T_ARRAY && tB == T_ARRAY) b = 2 * cmin;
            else if (tA == T_ARRAY) b = 2 * cA;
            else if (tB == T_ARRAY) b = 2 * cB;
            else { uint32_t m = 2 * cmin; b = runs_b > m ? runs_b : m; }
        } else if (op == OP_ANDNOT) {
            if (tA == T_ARRAY) b = 2 * cA;
            else { uint32_t m = 2 * cA; b = runs_b > m ? runs_b : m; }
        } else {
            uint32_t m = 2 * (cA + cB);
            if (tA == T_ARRAY && tB == T_ARRAY) b = (cA + cB <= (uint32_t)MAX_ARRAY) ? m : FULLB;
            else b = runs_b > m ? runs_b : m;
        }
        if (b > FULLB) b = FULLB;
    }
    // Whatever the cell: a non-lazy result is an array (2 * card), a bitset, or a run container that
    // was chosen because it is no larger than either — so min(8192, 2 * card_max) bounds it too.
    const uint32_t cmax = op == OP_AND ? cmin : (op == OP_ANDNOT ? cA : cA + cB);
    const uint32_t g = cmax > (uint32_t)MAX_ARRAY ? FULLB : 2 * cmax;
    if (g < b) b = g;
    return round16(b);
}

// Slot bound of a matched cell under the lazy rules: unions / symmetric differences left as RUN
// (array x run, containers.h:1189-1207) are not capped by the bitset size.
__host__ __device__ inline uint32_t slot_bound_lazy(int tA, int tB, uint32_t cA, uint32_t cB,
                                                    uint32_t lA, uint32_t lB) {
    uint32_t b = BITSET_BYTES;
    if (tA != T_BITSET && tB != T_BITSET && (tA == T_RUN || tB == T_RUN)) {
        const uint32_t nA = (tA == T_ARRAY) ? cA : lA, nB = (tB == T_ARRAY) ? cB : lB;
        const uint32_t r = 4 * (nA + nB);
        if (r > b) b = r;
    }
    return round16(b);
}

// Result type of a matched cell under the public lazy API.  `unknown` = the reference leaves the
// result bitset's cardinality dirty.  Mirrors oracle/roaring_oracle.c cell_lazy_or / cell_lazy_ior /
// cell_lazy_xor / bm_lazy_*  (container_lazy_or containers.h:1113-1215, container_lazy_ior
// :1333-1440, container_lazy_xor :1570-1654, container_lazy_ixor :1749-1776; bitmap level
// roaring.c:2509-2843).  unkA: the left bitset's cardinality is already dirty.
__host__ __device__ inline int decide_type_lazy(int op, int rules, int tA, int tB, uint32_t cA,
                                                uint32_t cB, uint32_t lA, uint32_t lB, bool unkA,
                                                int card, int nruns, bool &unknown) {
    unknown = false;
    // negation (container_not_range, containers.h:2039-2073; mixed_negation.c:79-256): bitset / array
    // input -> by cardinality, run input -> efficient container
    if (rules & RULES_FLIP) return tA == T_RUN ? rule_eff(card, nruns) : rule_ab(card);
    const bool inplace = (rules & RULES_INPLACE) != 0;
    if (op == OP_XOR) {
        if (tA == T_BITSET && tB == T_BITSET) { unknown = true; return T_BITSET; }  // xor_nocard
        if (inplace) return decide_type(OP_XOR, tA, tB, cA, cB, lA, lB, card, nruns);  // container_ixor
        if (tA == T_ARRAY && tB == T_ARRAY) {  // mixed_xor.c:221-252
            if (cA + cB <= 1024u) return T_ARRAY;
            unknown = true;
            return T_BITSET;
        }
        if (tA == T_RUN && tB == T_RUN) return rule_eff(card, nruns);
        if (tA == T_BITSET || tB == T_BITSET) { unknown = true; return T_BITSET; }
        return T_RUN;  // array x run left as RUN (mixed_xor.c:145-174)
    }
    // OP_OR
    const bool fullA = is_full_run(tA, lA, cA), fullB = is_full_run(tB, lB, cB);
    if (inplace && !(rules & RULES_NOFULL)) {  // roaring.c:2621 container_is_full(c1): untouched
        if (fullA || (tA == T_BITSET && !unkA && cA == 65536u)) return tA;
    }
    int a = tA;
    bool ior = inplace;
    if (rules & RULES_CONV) {  // roaring.c:2535-2545, 2622-2633: c1 -> bitset, then lazy_ior
        if (inplace) { if (tA != T_BITSET) a = T_BITSET; }
        else if (tA != T_BITSET && tB != T_BITSET) { a = T_BITSET; ior = true; }
    }
    if (ior) {
        if (a == T_BITSET) {
            if (tB == T_BITSET) return card == 65536 ? T_RUN : T_BITSET;  // :1342-1352, card computed
            if (tB == T_RUN && fullB) return T_RUN;                      // :1394-1399
            unknown = true;
            return T_BITSET;
        }
        if (a == T_ARRAY) {
            if (tB == T_ARRAY) {  // mixed_union.c:285-372
                if (cA + cB <= 1024u) return T_ARRAY;
                unknown = true;
                return T_BITSET;
            }
            if (tB == T_BITSET) { unknown = true; return T_BITSET; }
            return T_RUN;
        }
        // a == RUN
        if (tB == T_RUN) return rule_eff(card, nruns);
        if (tB == T_BITSET) {
            if (fullA) return T_RUN;  // :1409-1412
            unknown = true;
            return T_BITSET;
        }
        return T_RUN;
    }
    // container_lazy_or
    if (tA == T_ARRAY && tB == T_ARRAY) {  // mixed_union.c:247-283
        if (cA + cB <= 1024u) return T_ARRAY;
        unknown = true;
        return T_BITSET;
    }
    if (tA == T_RUN && tB == T_RUN) return rule_eff(card, nruns);
    if (tA == T_BITSET || tB == T_BITSET) {
        if (fullA || fullB) return T_RUN;  // :1165-1170, :1180-1185 copy of the full run
        unknown = true;
        return T_BITSET;
    }
    return T_RUN;  // array x run left as RUN (:1189-1207)
}

// ---------------------------------------------------------------- accumulator primitives
__device__ __forceinline__ void acc_zero(uint32_t *acc, int lane) {
    const uint4 z = make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int i = 0; i < 16; i++) reinterpret_cast<uint4 *>(acc)[i * 32 + lane] = z;
}

// Bitset -> accumulator as 16 cp.async.cg copies of 16 bytes per lane: one trip to L2, no registers
// held.  The copies are only issued here; acc_async_wait() waits for them, so a caller can issue the
// loads of the cell's other operand in between and have both arrive in the same trip.
// acc_async_wait() waits for ALL of the thread's outstanding cp.async groups: in k_compute_items that
// includes the prefetch of the next cell's descriptor, which only makes that wait a little earlier
// (the descriptor slot is read after the loop's own wait + __syncwarp, never before).
__device__ __forceinline__ void acc_copy_bitset_async(uint32_t *acc, const uint8_t *src, int lane) {
    const uint32_t d = smem_u32(acc) + 16u * lane;
    const uint4 *s = reinterpret_cast<const uint4 *>(src) + lane;
#pragma unroll
    for (int i = 0; i < 16; i++)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d + 512u * i), "l"(s + 32 * i) : "memory");
    asm volatile("cp.async.commit_group;\n" ::: "memory");
}
__device__ __forceinline__ void acc_async_wait() {
    asm volatile("cp.async.wait_all;\n" ::: "memory");
    __syncwarp();
}
__device__ __forceinline__ void acc_copy_bitset(uint32_t *acc, const uint8_t *src, int lane) {
    acc_copy_bitset_async(acc, src, lane);
    acc_async_wait();
}

__device__ __forceinline__ void acc_store_bitset(const uint32_t *acc, uint8_t *dst, int lane) {
    uint4 *d = reinterpret_cast<uint4 *>(dst);
#pragma unroll
    for (int i = 0; i < 16; i++) d[i * 32 + lane] = reinterpret_cast<const uint4 *>(acc)[i * 32 + lane];
}

// MODE 0 = set (or), 1 = flip (xor), 2 = clear (andnot)
template <int MODE>
__device__ __forceinline__ void acc_atom(uint32_t *p, uint32_t m) {
    if (MODE == 0) atomicOr(p, m);
    else if (MODE == 1) atomicXor(p, m);
    else atomicAnd(p, ~m);
}
template <int MODE>
__device__ __forceinline__ void acc_plain(uint32_t *p) {
    if (MODE == 0) *p = ~0u;
    else if (MODE == 1) *p = ~*p;
    else *p = 0u;
}

// acc op= {sorted u16 array}.  128-bit loads (8 values per lane); bits that fall in the same
// 32-bit word are merged in registers before the shared-memory atomic.
#ifndef RB200_APPLY_SPARSE_MAX
#define RB200_APPLY_SPARSE_MAX 4097   // arrays below this many values set their bits one atomic per value (merging same-word
                                      // bits in registers first costs more instructions than it saves atomics)
#endif
// Up to VECS vectors per lane (256 values each) are loaded before the first atomic, so an array of up
// to 256 * VECS values costs one trip to L2.  PRE runs between the first loads and the first atomic:
// APPLY_ZERO clears the accumulator (rasterising into a fresh one), APPLY_WAIT waits for an
// acc_copy_bitset_async issued by the caller (the bitset and the array arrive in the same trip).
constexpr int APPLY_NONE = 0, APPLY_ZERO = 1, APPLY_WAIT = 2;
#ifndef RB200_APPLY_VECS
#define RB200_APPLY_VECS 2      // AND / ANDNOT cells, and_cardinality, conversions
#endif
#ifndef RB200_APPLY_VECS_OR
#define RB200_APPLY_VECS_OR 1   // union / xor cells: more registers there spill in the cell kernel's main loop
#endif                          // (measured slower on every union / xor launch of the headline workload)
constexpr uint32_t APPLY_VECS = RB200_APPLY_VECS, APPLY_VECS_OR = RB200_APPLY_VECS_OR;
template <int MODE, int PRE = APPLY_NONE, uint32_t VECS = APPLY_VECS>
__device__ __forceinline__ void acc_apply_array(uint32_t *acc, const uint8_t *__restrict__ src, uint32_t n,
                                                int lane) {
    const uint4 *v4 = reinterpret_cast<const uint4 *>(src);
    const uint32_t nvec = (n + 7) >> 3;
    if (PRE == APPLY_NONE && n >= (uint32_t)RB200_APPLY_SPARSE_MAX) {   // dense: same-word bits merged first
        for (uint32_t i = lane; i < nvec; i += 32) {
            const uint4 q = __ldg(v4 + i);
            const uint32_t w[4] = {q.x, q.y, q.z, q.w};
            const uint32_t left = n - i * 8;           // values valid in this vector (>= 1)
            uint32_t cur_w = (w[0] & 0xffffu) >> 5, cur_m = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const uint32_t v = (k & 1) ? (w[k >> 1] >> 16) : (w[k >> 1] & 0xffffu);
                const uint32_t wi = v >> 5, bit = 1u << (v & 31);
                if (k == 0 || k < (int)left) {         // k == 0 is always valid
                    if (wi != cur_w) {
                        acc_atom<MODE>(acc + cur_w, cur_m);
                        cur_w = wi;
                        cur_m = bit;
                    } else {
                        cur_m |= bit;
                    }
                }
            }
            acc_atom<MODE>(acc + cur_w, cur_m);
        }
        return;
    }
    // sparse: one atomic per value, no merging
    if (VECS == 1 && PRE == APPLY_NONE) {   // one vector per lane in flight (k_or_many2, where more registers spill)
        for (uint32_t i = lane; i < nvec; i += 32) {
            const uint4 q = __ldg(v4 + i);
            const uint32_t w[4] = {q.x, q.y, q.z, q.w};
            const uint32_t left = n - i * 8;
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const uint32_t v = (k & 1) ? (w[k >> 1] >> 16) : (w[k >> 1] & 0xffffu);
                if (k < (int)left) acc_atom<MODE>(acc + (v >> 5), 1u << (v & 31));
            }
        }
        return;
    }
    uint32_t i0 = 0;
    do {
        uint4 q[VECS];
#pragma unroll
        for (uint32_t u = 0; u < VECS; u++) {
            const uint32_t i = i0 + 32 * u + lane;
            if (i < nvec) q[u] = __ldg(v4 + i);
        }
        if (PRE == APPLY_ZERO && i0 == 0) { acc_zero(acc, lane); __syncwarp(); }
        if (PRE == APPLY_WAIT && i0 == 0) acc_async_wait();
#pragma unroll 1
        for (uint32_t u = 0; u < VECS; u++) {   // one vector per pass, the next ones moved down
            const uint32_t i = i0 + 32 * u + lane;
            if (i >= nvec) break;
            const uint32_t w[4] = {q[0].x, q[0].y, q[0].z, q[0].w};
#pragma unroll
            for (uint32_t r = 0; r + 1 < VECS; r++) q[r] = q[r + 1];
            const uint32_t left = n - i * 8;
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const uint32_t v = (k & 1) ? (w[k >> 1] >> 16) : (w[k >> 1] & 0xffffu);
                if (k < (int)left) acc_atom<MODE>(acc + (v >> 5), 1u << (v & 31));
            }
        }
        i0 += 32 * VECS;
    } while (i0 < nvec);
}

// one 16-byte vector (8 values, `left` of them valid, >= 1) of a sorted array into the accumulator
template <int MODE>
__device__ __forceinline__ void acc_apply_vec(uint32_t *acc, uint4 q, uint32_t left) {
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
    uint32_t cur_w = (w[0] & 0xffffu) >> 5, cur_m = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint32_t v = (k & 1) ? (w[k >> 1] >> 16) : (w[k >> 1] & 0xffffu);
        const uint32_t wi = v >> 5, bit = 1u << (v & 31);
        if (k == 0 || k < (int)left) {
            if (wi != cur_w) {
                acc_atom<MODE>(acc + cur_w, cur_m);
                cur_w = wi;
                cur_m = bit;
            } else {
                cur_m |= bit;
            }
        }
    }
    acc_atom<MODE>(acc + cur_w, cur_m);
}

// same for a SPARSE array (values rarely share a 32-bit word: merging them first costs more than it saves)
__device__ __forceinline__ void acc_or_vec_sparse(uint32_t *acc, uint4 q, uint32_t left) {
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint32_t v = (k & 1) ? (w[k >> 1] >> 16) : (w[k >> 1] & 0xffffu);
        if (k < (int)left) atomicOr(acc + (v >> 5), 1u << (v & 31));
    }
}

// Warp-collective: every lane brings one closed range [lo,hi] (valid==false: none).
// Boundary words use shared-memory atomics; interior words are owned by exactly one range
// (ranges of one container never overlap) so they are plain stores; long interiors are
// filled by the whole warp.  ATOMIC_INTERIOR is for accumulators shared by several warps.
template <int MODE, bool ATOMIC_INTERIOR>
__device__ __forceinline__ void acc_apply_ranges(uint32_t *acc, uint32_t lo, uint32_t hi,
                                                 bool valid, int lane) {
    const uint32_t ws = lo >> 5, we = hi >> 5;
    bool longr = false;
    if (valid) {
        const uint32_t m_lo = ~0u << (lo & 31), m_hi = ~0u >> (31 - (hi & 31));
        if (ws == we) {
            acc_atom<MODE>(acc + ws, m_lo & m_hi);
        } else {
            acc_atom<MODE>(acc + ws, m_lo);
            acc_atom<MODE>(acc + we, m_hi);
            if (we - ws - 1 <= 8) {
                for (uint32_t w = ws + 1; w < we; w++) {
                    if (ATOMIC_INTERIOR) acc_atom<MODE>(acc + w, ~0u);
                    else acc_plain<MODE>(acc + w);
                }
            } else {
                longr = true;
            }
        }
    }
    unsigned m = __ballot_sync(FULLMASK, longr);
    while (m) {
        const int r = __ffs(m) - 1;
        m &= m - 1;
        const uint32_t s = __shfl_sync(FULLMASK, ws, r), e = __shfl_sync(FULLMASK, we, r);
        for (uint32_t w = s + 1 + lane; w < e; w += 32) {
            if (ATOMIC_INTERIOR) acc_atom<MODE>(acc + w, ~0u);
            else acc_plain<MODE>(acc + w);
        }
    }
}

// acc op= {run container}: one lane per run ("run-length expansion")
template <int MODE, bool ATOMIC_INTERIOR>
static __device__ __noinline__ void acc_apply_runs(uint32_t *acc, const uint8_t *src, uint32_t n,
                                               int lane) {
    const uint32_t *runs = reinterpret_cast<const uint32_t *>(src);
    for (uint32_t base = 0; base < n; base += 32) {
        const uint32_t i = base + lane;
        const bool valid = i < n;
        const uint32_t r = valid ? __ldg(runs + i) : 0u;
        // (hi is clamped: a run ending past 65535 can only come from a caller-built host bitmap that
        //  breaks the reference's own invariants; it must not write outside the accumulator)
        const uint32_t lo = r & 0xffffu, hi = min(lo + (r >> 16), 65535u);
        acc_apply_ranges<MODE, ATOMIC_INTERIOR>(acc, lo, hi, valid, lane);
    }
}

// acc &= {run container}: clear the n+1 gaps between / around the runs
// (bitset_reset_range over the gaps, src/containers/mixed_intersection.c:171-182)
static __device__ __noinline__ void acc_and_runs(uint32_t *acc, const uint8_t *src, uint32_t n,
                                             int lane) {
    const uint32_t *runs = reinterpret_cast<const uint32_t *>(src);
    for (uint32_t base = 0; base <= n; base += 32) {
        const uint32_t i = base + lane;
        bool valid = i <= n;
        int lo = 0, hi = 65535;
        if (valid) {
            if (i > 0) {
                const uint32_t r = __ldg(runs + i - 1);
                lo = min((int)((r & 0xffffu) + (r >> 16)), 65535) + 1;
            }
            if (i < n) {
                const uint32_t r = __ldg(runs + i);
                hi = (int)(r & 0xffffu) - 1;
            }
            valid = lo <= hi;
        }
        acc_apply_ranges<2, false>(acc, (uint32_t)lo, (uint32_t)hi, valid, lane);
    }
}

// acc &= {sorted array}: clear the gaps between consecutive values
static __device__ __noinline__ void acc_and_array(uint32_t *acc, const uint8_t *src, uint32_t n,
                                              int lane) {
    const uint16_t *arr = reinterpret_cast<const uint16_t *>(src);
    for (uint32_t base = 0; base <= n; base += 32) {
        const uint32_t i = base + lane;
        bool valid = i <= n;
        int lo = 0, hi = 65535;
        if (valid) {
            if (i > 0) lo = (int)arr[i - 1] + 1;
            if (i < n) hi = (int)arr[i] - 1;
            valid = lo <= hi;
        }
        acc_apply_ranges<2, false>(acc, (uint32_t)lo, (uint32_t)hi, valid, lane);
    }
}

// Rasterise any container into the (private) accumulator.
template <uint32_t VECS = APPLY_VECS>
__device__ __forceinline__ void acc_load(uint32_t *acc, int type, const uint8_t *src,
                                         uint32_t len, int lane) {
    if (type == T_BITSET) {
        acc_copy_bitset(acc, src, lane);
    } else if (type == T_ARRAY) {
        acc_apply_array<0, APPLY_ZERO, VECS>(acc, src, len, lane);   // the array's loads overlap the clearing
    } else {
        acc_zero(acc, lane);
        __syncwarp();
        acc_apply_runs<0, false>(acc, src, len, lane);
    }
    __syncwarp();
}

// acc = acc OP bitset(src), returns nothing (cardinality is taken by acc_count)
template <int OP>
__device__ __forceinline__ void acc_op_bitset(uint32_t *acc, const uint8_t *__restrict__ src, int lane) {
    const uint4 *s = reinterpret_cast<const uint4 *>(src);
#pragma unroll
    for (int h = 0; h < 2; h++) {
        uint4 q[8];
#pragma unroll
        for (int i = 0; i < 8; i++) q[i] = __ldg(s + (h * 8 + i) * 32 + lane);
#pragma unroll
        for (int i = 0; i < 8; i++) {
            uint4 *p = reinterpret_cast<uint4 *>(acc) + (h * 8 + i) * 32 + lane;
            uint4 a = *p;
            if (OP == OP_AND) { a.x &= q[i].x; a.y &= q[i].y; a.z &= q[i].z; a.w &= q[i].w; }
            else if (OP == OP_OR) { a.x |= q[i].x; a.y |= q[i].y; a.z |= q[i].z; a.w |= q[i].w; }
            else if (OP == OP_XOR) { a.x ^= q[i].x; a.y ^= q[i].y; a.z ^= q[i].z; a.w ^= q[i].w; }
            else { a.x &= ~q[i].x; a.y &= ~q[i].y; a.z &= ~q[i].z; a.w &= ~q[i].w; }
            *p = a;
        }
    }
}

// acc = bitset(a) OP bitset(b) straight from global memory (the B x B cell): 2 x 8 KiB of
// 128-bit loads per warp, result staged in shared memory, popcount fused.
template <int OP>
__device__ __forceinline__ int acc_bitset_op_bitset(uint32_t *acc, const uint8_t *pa,
                                                    const uint8_t *pb, int lane) {
    const uint4 *a = reinterpret_cast<const uint4 *>(pa);
    const uint4 *b = reinterpret_cast<const uint4 *>(pb);
    int c = 0;
#pragma unroll
    for (int h = 0; h < 4; h++) {
        uint4 qa[4], qb[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            qa[i] = __ldg(a + (h * 4 + i) * 32 + lane);
            qb[i] = __ldg(b + (h * 4 + i) * 32 + lane);
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {
            uint4 r;
            if (OP == OP_AND) { r.x = qa[i].x & qb[i].x; r.y = qa[i].y & qb[i].y; r.z = qa[i].z & qb[i].z; r.w = qa[i].w & qb[i].w; }
            else if (OP == OP_OR) { r.x = qa[i].x | qb[i].x; r.y = qa[i].y | qb[i].y; r.z = qa[i].z | qb[i].z; r.w = qa[i].w | qb[i].w; }
            else if (OP == OP_XOR) { r.x = qa[i].x ^ qb[i].x; r.y = qa[i].y ^ qb[i].y; r.z = qa[i].z ^ qb[i].z; r.w = qa[i].w ^ qb[i].w; }
            else { r.x = qa[i].x & ~qb[i].x; r.y = qa[i].y & ~qb[i].y; r.z = qa[i].z & ~qb[i].z; r.w = qa[i].w & ~qb[i].w; }
            reinterpret_cast<uint4 *>(acc)[(h * 4 + i) * 32 + lane] = r;
            c += popc4(r);
        }
    }
    return __reduce_add_sync(FULLMASK, c);
}

// popcount(bitset(a) & bitset(b)) without materialising (bitset_container_and_justcard)
__device__ __forceinline__ int bitset_and_card(const uint8_t *pa, const uint8_t *pb, int lane) {
    const uint4 *a = reinterpret_cast<const uint4 *>(pa);
    const uint4 *b = reinterpret_cast<const uint4 *>(pb);
    int c = 0;
#pragma unroll
    for (int h = 0; h < 2; h++) {
        uint4 qa[8], qb[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            qa[i] = __ldg(a + (h * 8 + i) * 32 + lane);
            qb[i] = __ldg(b + (h * 8 + i) * 32 + lane);
        }
#pragma unroll
        for (int i = 0; i < 8; i++)
            c += __popc(qa[i].x & qb[i].x) + __popc(qa[i].y & qb[i].y) +
                 __popc(qa[i].z & qb[i].z) + __popc(qa[i].w & qb[i].w);
    }
    return __reduce_add_sync(FULLMASK, c);
}

// popcount(acc & bitset(b))
__device__ __forceinline__ int acc_and_bitset_card(const uint32_t *acc, const uint8_t *pb,
                                                   int lane) {
    const uint4 *b = reinterpret_cast<const uint4 *>(pb);
    int c = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const uint4 q = __ldg(b + i * 32 + lane);
        const uint4 a = reinterpret_cast<const uint4 *>(acc)[i * 32 + lane];
        c += __popc(a.x & q.x) + __popc(a.y & q.y) + __popc(a.z & q.z) + __popc(a.w & q.w);
    }
    return __reduce_add_sync(FULLMASK, c);
}

// cardinality (and number of runs when asked) of the accumulator
__device__ __forceinline__ void acc_count(const uint32_t *acc, int lane, bool want_runs,
                                          int &card, int &nruns) {
    int c = 0, r = 0;
    if (!want_runs) {
#pragma unroll
        for (int i = 0; i < 16; i++) c += popc4(reinterpret_cast<const uint4 *>(acc)[i * 32 + lane]);
    } else {
        for (int i = 0; i < 64; i++) {
            const int w = i * 32 + lane;
            const uint32_t x = acc[w];
            const uint32_t prev = w ? (acc[w - 1] >> 31) : 0u;
            c += __popc(x);
            r += __popc(x & ~((x << 1) | prev));
        }
    }
    card = __reduce_add_sync(FULLMASK, c);
    nruns = __reduce_add_sync(FULLMASK, r);
}

// acc -> sorted u16 list (array_container_from_bitset).  16 stripes of 128 words: every lane
// owns one 128-bit group per stripe (conflict-free LDS.128, value order == lane order),
// per-lane popcount -> warp scan -> every lane emits its bits at its offset, so a stripe's
// output is one contiguous, mostly sector-coalesced range.
// Alternatives tried on weather_sept_85 all-pairs OR, all slower than this layout: 64 stripes of
// one word per lane; cooperative emission of dense halves; one or four 32-bit find-first-set
// loops per lane.
__device__ __forceinline__ uint32_t acc_emit_array(const uint32_t *acc, uint16_t *out, int lane) {
    uint32_t base = 0;
#pragma unroll 1
    for (int it = 0; it < 16; it++) {
        const uint4 q = reinterpret_cast<const uint4 *>(acc)[it * 32 + lane];
        const uint32_t c = popc4(q);
        if (!__any_sync(FULLMASK, c != 0)) continue;
        const uint32_t incl = warp_incl_scan(c, lane);
        const uint32_t total = __shfl_sync(FULLMASK, incl, 31);
        uint16_t *p = out + base + incl - c;
        const uint32_t hi = (uint32_t)(it * 32 + lane) << 7;
        unsigned long long lo64 = ((unsigned long long)q.y << 32) | q.x;
        unsigned long long hi64 = ((unsigned long long)q.w << 32) | q.z;
        while (lo64) {
            const int b = __ffsll((long long)lo64) - 1;
            lo64 &= lo64 - 1;
            *p++ = (uint16_t)(hi | b);
        }
        while (hi64) {
            const int b = __ffsll((long long)hi64) - 1;
            hi64 &= hi64 - 1;
            *p++ = (uint16_t)(hi | 64 | b);
        }
        base += total;
    }
    return base;
}

// acc -> run list {start, length-1}: pass 1 writes run starts, pass 2 run ends, pass 3 turns
// ends into lengths.  Returns the number of runs.
static __device__ __noinline__ uint32_t acc_emit_runs(const uint32_t *acc, uint16_t *out, int lane) {
    uint32_t nr = 0;
    for (int pass = 0; pass < 2; pass++) {
        uint32_t base = 0;
        for (int it = 0; it < 64; it++) {
            const uint32_t w = it * 32 + lane;
            const uint32_t x = acc[w];
            uint32_t e;
            if (pass == 0) {
                const uint32_t prev = w ? (acc[w - 1] >> 31) : 0u;
                e = x & ~((x << 1) | prev);
            } else {
                const uint32_t next = (w < ACC_WORDS - 1) ? (acc[w + 1] & 1u) : 0u;
                e = x & ~((x >> 1) | (next << 31));
            }
            if (!__any_sync(FULLMASK, e != 0)) continue;
            const uint32_t c = __popc(e);
            const uint32_t incl = warp_incl_scan(c, lane);
            const uint32_t total = __shfl_sync(FULLMASK, incl, 31);
            uint32_t k = base + incl - c;
            const uint32_t hi = w << 5;
            while (e) {
                const int b = __ffs(e) - 1;
                e &= e - 1;
                out[2 * k + pass] = (uint16_t)(hi | b);
                k++;
            }
            base += total;
        }
        nr = base;
    }
    __syncwarp();
    for (uint32_t k = lane; k < nr; k += 32) out[2 * k + 1] = (uint16_t)(out[2 * k + 1] - out[2 * k]);
    return nr;
}

// ---------------------------------------------------------------- ordered u16 output through a window
// Both the array filter and the array merge path produce their output 32 lanes x 8 candidate values
// at a time, in order.  A warp scan places the survivors in a shared window buffer `wb` that mirrors
// the output from the last 16-byte boundary below `base`, and the warp stores it as whole 128-bit
// words (u16 stores when `out` is not 16-byte aligned); the partial last word carries into the next
// window.  Every lane brings its 8 candidates in xp (value k in half k & 1 of word k >> 1) and a
// keep mask; returns base + the number kept.  The buffer holds 8 + 256 values.
__device__ __forceinline__ uint32_t window_store(uint16_t *wb, uint16_t *__restrict__ out, bool vec, uint32_t base,
                                                 const uint32_t (&xp)[4], unsigned keep, int lane) {
    const uint32_t c = __popc(keep);
    const uint32_t incl = warp_incl_scan(c, lane);
    const uint32_t total = __shfl_sync(FULLMASK, incl, 31);
    if (total == 0) return base;
    const uint32_t head = base & 7u;   // wb[t] mirrors out[(base & ~7) + t]
    uint32_t o = head + incl - c;
#pragma unroll
    for (int k = 0; k < 8; k++)
        if ((keep >> k) & 1u) wb[o++] = (uint16_t)(xp[k >> 1] >> (16 * (k & 1)));
    __syncwarp();
    if (vec) {
        uint4 *dst = reinterpret_cast<uint4 *>(out + (base - head));
        for (uint32_t v = lane; v < (head + total + 7) / 8; v += 32)
            dst[v] = reinterpret_cast<const uint4 *>(wb)[v];
    } else {
        for (uint32_t v = lane; v < total; v += 32) out[base + v] = wb[head + v];
    }
    __syncwarp();
    const uint32_t end = head + total;
    if (lane == 0 && (end & 7u)) reinterpret_cast<uint4 *>(wb)[0] = reinterpret_cast<const uint4 *>(wb)[end >> 3];
    __syncwarp();
    return base + total;
}

// Filter a sorted array through a bit test (array_bitset_container_intersection /
// _andnot, src/containers/mixed_intersection.c:19-58, mixed_andnot.c:24-38).
// 128-bit loads, 8 values per lane; FILTER_VECS vectors per lane (256 values each) are loaded before
// any bit is tested or any value stored, so an array of up to 256 * FILTER_VECS values waits on L2 once.  With WRITE
// the survivors go out through window_store (wb: the warp's window buffer); without, they are only
// counted.  wait_bits: `bits` is the accumulator and an acc_copy_bitset_async into it is in flight —
// the wait goes after the array's first loads, so both arrive in the same trip.  `out` never aliases
// the operands: it is a result slot (slab, or mapped host memory for k_pair_fused).
#ifndef RB200_FILTER_VECS
#define RB200_FILTER_VECS 2
#endif
constexpr uint32_t FILTER_VECS = RB200_FILTER_VECS;
#ifndef RB200_FILTER_SCALAR_MAX
#define RB200_FILTER_SCALAR_MAX 32   // arrays of at most this many values take the one-u16-per-lane loop: one load
#endif                               // trip as well, and one ballot instead of the window store's scan
template <bool NEG, bool WRITE>
__device__ __forceinline__ uint32_t filter_array(const uint8_t *__restrict__ src, uint32_t n,
                                                 const uint32_t *__restrict__ bits, uint16_t *__restrict__ out,
                                                 uint16_t *wb, int lane, bool wait_bits = false) {
    if ((reinterpret_cast<uintptr_t>(src) & 15) || n <= (uint32_t)RB200_FILTER_SCALAR_MAX) {
        // unaligned source or few values: one u16 per lane, ballot compaction
        if (wait_bits) acc_async_wait();
        const uint16_t *arr = reinterpret_cast<const uint16_t *>(src);
        uint32_t cnt = 0;
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t i = base + lane;
            bool keep = false;
            uint16_t v = 0;
            if (i < n) {
                v = arr[i];
                const bool hit = (bits[v >> 5] >> (v & 31)) & 1u;
                keep = NEG ? !hit : hit;
            }
            const unsigned m = __ballot_sync(FULLMASK, keep);
            if (WRITE && keep) out[cnt + __popc(m & lanemask_lt())] = v;
            cnt += __popc(m);
        }
        return cnt;
    }
    const uint4 *v4 = reinterpret_cast<const uint4 *>(src);
    const uint32_t nvec = (n + 7) >> 3;
    const bool vec = (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    uint32_t base = 0, cnt = 0, i0 = 0;
    do {
        uint4 q[FILTER_VECS];
#pragma unroll
        for (uint32_t u = 0; u < FILTER_VECS; u++) {
            const uint32_t i = i0 + 32 * u + lane;
            if (i < nvec) q[u] = __ldg(v4 + i);
        }
        if (wait_bits && i0 == 0) acc_async_wait();
        // (one vector per pass, the next ones moved down: one copy of the bit tests and the window
        //  store instead of FILTER_VECS)
#pragma unroll 1
        for (uint32_t u = 0; u < FILTER_VECS && i0 + 32 * u < nvec; u++) {   // warp-uniform
            const uint32_t i = i0 + 32 * u + lane;
            const uint32_t xp[4] = {q[0].x, q[0].y, q[0].z, q[0].w};
#pragma unroll
            for (uint32_t r = 0; r + 1 < FILTER_VECS; r++) q[r] = q[r + 1];
            unsigned keep = 0;
            if (i < nvec) {
                const uint32_t left = n - i * 8;
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const uint32_t v = (xp[k >> 1] >> (16 * (k & 1))) & 0xffffu;
                    const bool hit = (bits[v >> 5] >> (v & 31)) & 1u;
                    keep |= (unsigned)((NEG ? !hit : hit) && k < (int)left) << k;
                }
            }
            if (WRITE) base = window_store(wb, out, vec, base, xp, keep, lane);
            else cnt += __popc(keep);
        }
        i0 += 32 * FILTER_VECS;
    } while (i0 < nvec);
    return WRITE ? base : __reduce_add_sync(FULLMASK, cnt);
}

// global -> shared staging of a u16 range (dst 16-byte aligned).  A 16-byte aligned source is copied
// by cp.async.cg, 16 bytes per copy, all of them issued at once and none waited for here: the caller
// issues every range it needs and then waits once (acc_async_wait), so they arrive in one trip to L2.
// An unaligned source is copied one u16 per lane, synchronously.
__device__ __forceinline__ void stage_u16_async(uint16_t *dst, const uint8_t *src, uint32_t n, int lane) {
    if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        const uint32_t d = smem_u32(dst);
        const uint4 *s = reinterpret_cast<const uint4 *>(src);
        for (uint32_t i = lane; i < (n + 7) / 8; i += 32)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d + 16u * i), "l"(s + i) : "memory");
        asm volatile("cp.async.commit_group;\n" ::: "memory");
    } else {
        const uint16_t *s16 = reinterpret_cast<const uint16_t *>(src);
        for (uint32_t i = lane; i < n; i += 32) dst[i] = s16[i];
    }
}

// Union / symmetric difference of two sorted u16 arrays with n + m <= 4096 values, the cells whose
// result the type rule makes an array (array_container_union / xor, src/array_util.c:1104,1198),
// as a windowed warp merge path: no accumulator round trip and no find-first-set emission.
// Both inputs are staged once in the warp's shared block by cp.async, a at 0 and b at round8(n), both
// copies in flight together; the 128-bit staging reaches u16 index round8(n) + round8(m) <= 4104.  The merged sequence is produced in
// windows of 32 * MERGE_PER_LANE positions: every lane finds the split of its diagonal (merge-path
// search between the window's start split and MERGE_PER_LANE more values per lane before it),
// merges its values in registers and decides which survive.  Duplicates (a value present in both
// inputs) are adjacent in the merged order: OR keeps the first, XOR drops both.  window_store places
// the survivors in the window buffer (u16 index MERGE_WBUF, past the staging; the array filter uses
// the same buffer) and stores them at the running output offset as whole 128-bit words.
constexpr uint32_t MERGE_PER_LANE = 8, MERGE_WIN = 32 * MERGE_PER_LANE;
constexpr uint32_t MERGE_WBUF = 4104;
// per-warp shared block: the 8 KiB accumulator, then room for the merge's window buffer (9 KiB)
constexpr int WARP_SMEM_WORDS = ACC_WORDS + 256;
static_assert(2 * MERGE_WBUF + 2 * (MERGE_WIN + 8) <= 4 * WARP_SMEM_WORDS, "merge window buffer");

// Not inlined: the cell kernel's other paths then keep their register allocation (measured faster
// than the inlined merge on the headline workload).
template <bool IS_XOR>
static __device__ __noinline__ uint32_t merge_arrays(uint32_t *acc, const uint8_t *pa, uint32_t n,
                                                     const uint8_t *pb, uint32_t m, uint8_t *out,
                                                     int lane) {
    uint16_t *sa = reinterpret_cast<uint16_t *>(acc);
    uint16_t *sb = sa + ((n + 7) & ~7u);
    uint16_t *wb = sa + MERGE_WBUF;
    uint16_t *o16 = reinterpret_cast<uint16_t *>(out);
    const bool vec = (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    stage_u16_async(sa, pa, n, lane);
    stage_u16_async(sb, pb, m, lane);
    acc_async_wait();   // both inputs in one trip (also waits for the next cell's descriptor prefetch)
    const uint32_t T = n + m, NONE = 0x10000u;   // NONE: past the end of an input, above every value
    uint32_t is = 0;                             // split at the window start: values taken from a
    uint32_t last = NONE + 1;                    // merged value before the window (none yet)
    uint32_t base = 0;                           // values written so far
#pragma unroll 1
    for (uint32_t w0 = 0; w0 < T; w0 += MERGE_WIN) {
        const uint32_t d = w0 + lane * MERGE_PER_LANE;
        // i = how many of the first d merged values come from a (ties: a first); lanes past the end
        // get lo = d - m > n, i.e. both inputs exhausted
        uint32_t lo = max(is, d > m ? d - m : 0u), hi = min(is + lane * MERGE_PER_LANE, n);
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (sa[mid] <= sb[d - 1 - mid]) lo = mid + 1;
            else hi = mid;
        }
        uint32_t i = lo, j = d - lo;
        uint32_t ai = i < n ? sa[i] : NONE, bj = j < m ? sb[j] : NONE;
        // the lane's merged values, two u16 per word; keep bit k: value k survives.  The bits that
        // need a neighbour outside the lane (bit 0, and for XOR also the last) are decided after it.
        uint32_t xp[MERGE_PER_LANE / 2];
        uint32_t x0 = NONE, x1 = NONE, p1 = NONE, p2 = NONE;   // values 0, 1, k-1, k-2
        unsigned keep = 0;
#pragma unroll
        for (int k = 0; k < (int)MERGE_PER_LANE; k++) {
            const bool take_a = ai <= bj;
            const uint32_t v = take_a ? ai : bj;
            if (take_a) { i++; ai = i < n ? sa[i] : NONE; }
            else { j++; bj = j < m ? sb[j] : NONE; }
            if (k & 1) xp[k >> 1] |= v << 16;
            else xp[k >> 1] = v & 0xffffu;
            if (k == 0) x0 = v;
            if (k == 1) x1 = v;
            if (!IS_XOR && k >= 1) keep |= (unsigned)(v < NONE && v != p1) << k;
            if (IS_XOR && k >= 2) keep |= (unsigned)(p1 < NONE && p1 != p2 && p1 != v) << (k - 1);
            p2 = p1;
            p1 = v;
        }
        // neighbours across the lane and window boundaries: the previous lane's last value, and the
        // next merged value (read from the inputs) for XOR's look-ahead
        uint32_t prev = __shfl_up_sync(FULLMASK, p1, 1);
        if (lane == 0) prev = last;
        last = __shfl_sync(FULLMASK, p1, 31);
        is = __shfl_sync(FULLMASK, i, 31);
        keep |= (unsigned)(x0 < NONE && x0 != prev && (!IS_XOR || x0 != x1));
        if (IS_XOR) keep |= (unsigned)(p1 < NONE && p1 != p2 && p1 != min(ai, bj)) << (MERGE_PER_LANE - 1);
        base = window_store(wb, o16, vec, base, xp, keep, lane);
    }
    return base;
}

// ---------------------------------------------------------------- interval (run) algebra
// Cells with a run container on either side and few intervals (run x run, array x run with
// nA' + nB' <= 512, n' = runs or array values) skip the 65536-bit accumulator: both containers
// become sorted lists of interval boundaries {start, end+1} in shared memory, a warp merge path
// walks the merged boundaries with the coverage state (inA, inB) given by the parity of how many
// boundaries of each list were passed, and emits a boundary of the result wherever op(inA, inB)
// flips (run_container_union / _intersection / _xor / _andnot, src/containers/run.c:231-633,
// as one parallel sweep).  Returns false when the reference's type rule wants a bitset
// (card > 4096), in which case the caller takes the general path.
__device__ __forceinline__ bool op_state(int op, bool a, bool b) {
    return op == OP_AND ? (a && b) : op == OP_OR ? (a || b) : op == OP_XOR ? (a != b) : (a && !b);
}

// boundaries of one container into pts[] (2 per interval); returns the number of intervals
__device__ __forceinline__ uint32_t load_boundaries(uint32_t *pts, int type, const uint8_t *src,
                                                    uint32_t len, int lane) {
    if (type == T_RUN) {
        const uint32_t *runs = reinterpret_cast<const uint32_t *>(src);
        for (uint32_t i = lane; i < len; i += 32) {
            const uint32_t r = __ldg(runs + i), s = r & 0xffffu;
            pts[2 * i] = s;
            pts[2 * i + 1] = s + (r >> 16) + 1;
        }
        return len;
    }
    // array: coalesce consecutive values into intervals
    const uint16_t *arr = reinterpret_cast<const uint16_t *>(src);
    uint32_t nint = 0;
    for (uint32_t base = 0; base < len; base += 32) {
        const uint32_t i = base + lane;
        uint32_t v = 0;
        bool st = false, en = false;
        if (i < len) {
            v = arr[i];
            st = (i == 0) || ((uint32_t)arr[i - 1] + 1 != v);
            en = (i + 1 == len) || ((uint32_t)arr[i + 1] != v + 1);
        }
        const unsigned ms = __ballot_sync(FULLMASK, st), me = __ballot_sync(FULLMASK, en);
        // the k-th start pairs with the k-th end; an interval open at the end of this stripe is
        // closed by a later stripe, so count ends seen before this stripe separately
        if (st) pts[2 * (nint + __popc(ms & lanemask_lt()))] = v;
        if (en) {
            // ends so far == starts so far - (1 if an interval is open at stripe start)
            const uint32_t ke = (nint + __popc(ms & (lanemask_lt() | (1u << lane)))) - 1;
            pts[2 * ke + 1] = v + 1;
        }
        nint += __popc(ms);
    }
    return nint;
}

static __device__ __noinline__ bool
interval_cell(uint32_t *acc, int op, int tA, int tB, const uint8_t *pa, const uint8_t *pb,
              uint32_t cA, uint32_t cB, uint32_t lA, uint32_t lB, uint8_t *out, uint32_t cap,
              int lane, int &otype, uint32_t &ocard, uint32_t &olen) {
    uint32_t *pA = acc;
    const uint32_t nA = load_boundaries(pA, tA, pa, lA, lane);
    uint32_t *pB = acc + 2 * nA;
    const uint32_t nB = load_boundaries(pB, tB, pb, lB, lane);
    uint32_t *ev = acc + 1024;
    __syncwarp();
    const uint32_t n = 2 * nA, m = 2 * nB, T = n + m, per = (T + 31) >> 5;
    const uint32_t d0 = min((uint32_t)lane * per, T), d1 = min(d0 + per, T);
    uint32_t lo = d0 > m ? d0 - m : 0u, hi = min(d0, n);
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (pA[mid] <= pB[d0 - 1 - mid]) lo = mid + 1;
        else hi = mid;
    }
    const uint32_t i0 = lo, j0 = d0 - lo;
    const uint32_t NONE = 0x20000u;
    uint32_t prev0 = NONE + 1;
    if (d0 > 0) {
        const uint32_t x = i0 > 0 ? pA[i0 - 1] : 0u, y = j0 > 0 ? pB[j0 - 1] : 0u;
        prev0 = (i0 > 0 && j0 > 0) ? max(x, y) : (i0 > 0 ? x : y);
    }
    uint32_t off = 0, nev = 0;
#pragma unroll 1
    for (int pass = 0; pass < 2; pass++) {
        uint32_t i = i0, j = j0, prev = prev0, c = 0;
        uint32_t ai = i < n ? pA[i] : NONE, bj = j < m ? pB[j] : NONE;
        for (uint32_t p = d0; p < d1; p++) {
            const bool take_a = ai <= bj;
            const uint32_t x = take_a ? ai : bj;
            if (take_a) { i++; ai = i < n ? pA[i] : NONE; }
            else { j++; bj = j < m ? pB[j] : NONE; }
            if (x != min(ai, bj)) {  // last boundary with this value: evaluate the flip
                const bool inA = i & 1, inB = j & 1;
                const bool tie = (x == prev);  // the other list had a boundary at the same value
                const bool wasA = (take_a || tie) ? !inA : inA, wasB = (!take_a || tie) ? !inB : inB;
                if (op_state(op, inA, inB) != op_state(op, wasA, wasB)) {
                    if (pass == 1) ev[off + c] = x;
                    c++;
                }
            }
            prev = x;
        }
        if (pass == 0) {
            const uint32_t incl = warp_incl_scan(c, lane);
            off = incl - c;
            nev = __shfl_sync(FULLMASK, incl, 31);
        }
    }
    __syncwarp();
    const uint32_t nruns = nev >> 1;
    uint32_t card = 0;
    for (uint32_t k = lane; k < nruns; k += 32) card += ev[2 * k + 1] - ev[2 * k];
    card = __reduce_add_sync(FULLMASK, card);
    if (card == 0) { otype = 0; ocard = olen = 0; __syncwarp(); return true; }
    const int t = decide_type(op, tA, tB, cA, cB, lA, lB, (int)card, (int)nruns);
    if (t == T_BITSET) { __syncwarp(); return false; }
    if (t == T_RUN) {
        if (4 * nruns > cap) { __syncwarp(); return false; }
        uint32_t *o = reinterpret_cast<uint32_t *>(out);
        for (uint32_t k = lane; k < nruns; k += 32) {
            const uint32_t s = ev[2 * k], e = ev[2 * k + 1];
            o[k] = s | ((e - s - 1) << 16);
        }
        otype = T_RUN;
        ocard = card;
        olen = nruns;
    } else {  // array: expand the runs at their scanned offsets
        if (2 * card > cap) { __syncwarp(); return false; }
        uint16_t *o = reinterpret_cast<uint16_t *>(out);
        uint32_t base = 0;
        for (uint32_t k0 = 0; k0 < nruns; k0 += 32) {
            const uint32_t k = k0 + lane;
            const uint32_t s = k < nruns ? ev[2 * k] : 0u, len = k < nruns ? ev[2 * k + 1] - s : 0u;
            const uint32_t incl = warp_incl_scan(len, lane);
            uint16_t *p = o + base + incl - len;
            for (uint32_t q = 0; q < len; q++) p[q] = (uint16_t)(s + q);
            base += __shfl_sync(FULLMASK, incl, 31);
        }
        otype = T_ARRAY;
        ocard = olen = card;
    }
    __syncwarp();
    return true;
}

// ---------------------------------------------------------------- TMA bulk copies + mbarrier
// Operand staging with the Hopper TMA unit: ONE elected thread issues cp.async.bulk (global -> shared,
// whole containers, 16-byte granules) against an mbarrier; the bytes land asynchronously while the
// other warps keep working on the previous batch, and nobody holds registers for loads in flight.
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// wait for the phase with the given parity; a bounded spin: a lost transaction traps instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    const uint32_t a = smem_u32(bar);
    for (uint32_t spin = 0;; spin++) {
        uint32_t done;
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}"
            : "=r"(done)
            : "r"(a), "r"(parity)
            : "memory");
        if (done) return;
        if (spin > (1u << 26)) __trap();
    }
}

// shared-memory twins of acc_apply_array / acc_apply_runs (operands staged by bulk copies)
template <int MODE>
__device__ __forceinline__ void acc_apply_array_s(uint32_t *acc, const uint8_t *src, uint32_t n, int lane) {
    const uint4 *v4 = reinterpret_cast<const uint4 *>(src);
    const uint32_t nvec = (n + 7) >> 3;
    for (uint32_t i = lane; i < nvec; i += 32) {
        const uint4 q = v4[i];
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
        const uint32_t left = n - i * 8;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const uint32_t v = (k & 1) ? (w[k >> 1] >> 16) : (w[k >> 1] & 0xffffu);
            if (k < (int)left) acc_atom<MODE>(acc + (v >> 5), 1u << (v & 31));
        }
    }
}
template <int MODE, bool ATOMIC_INTERIOR>
static __device__ __noinline__ void acc_apply_runs_s(uint32_t *acc, const uint8_t *src, uint32_t n, int lane) {
    const uint32_t *runs = reinterpret_cast<const uint32_t *>(src);
    for (uint32_t base = 0; base < n; base += 32) {
        const uint32_t i = base + lane;
        const bool valid = i < n;
        const uint32_t r = valid ? runs[i] : 0u;
        const uint32_t lo = r & 0xffffu, hi = min(lo + (r >> 16), 65535u);
        acc_apply_ranges<MODE, ATOMIC_INTERIOR>(acc, lo, hi, valid, lane);
    }
}

// 16-byte vector copy of a stored payload (pass-through containers)
__device__ __forceinline__ void warp_copy16(uint8_t *dst, const uint8_t *src, uint32_t bytes,
                                            int lane) {
    const uint4 *s = reinterpret_cast<const uint4 *>(src);
    uint4 *d = reinterpret_cast<uint4 *>(dst);
    const uint32_t n = (bytes + 15) >> 4;
    uint32_t i = lane;
    for (; i + 96 < n; i += 128) {
        const uint4 q0 = __ldg(s + i), q1 = __ldg(s + i + 32), q2 = __ldg(s + i + 64),
                    q3 = __ldg(s + i + 96);
        d[i] = q0;
        d[i + 32] = q1;
        d[i + 64] = q2;
        d[i + 96] = q3;
    }
    for (; i < n; i += 32) d[i] = __ldg(s + i);
}

}  // namespace rb200
