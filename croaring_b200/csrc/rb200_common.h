// rb200_common.h — shared between the host engine (rb200_host.cu) and the kernels
// (rb200_kernels.cu).  Internal: nothing here crosses the C ABI.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rb200 {

// ABI constants restated from the reference (SURVEY.md §8b "ABI constants"):
//   typecodes           include/roaring/containers/containers.h:48-51
//   DEFAULT_MAX_SIZE    include/roaring/containers/array.h:38
//   bitset words        include/roaring/containers/bitset.h:40
constexpr int T_BITSET = 1;
constexpr int T_ARRAY = 2;
constexpr int T_RUN = 3;
constexpr int T_SHARED = 4;
constexpr int MAX_ARRAY = 4096;
constexpr int BITSET_BYTES = 8192;
constexpr int ACC_WORDS = 2048;  // 65536 bits as 32-bit words

enum Op { OP_AND = 0, OP_OR = 1, OP_XOR = 2, OP_ANDNOT = 3 };

// work-item kinds produced by the planner
constexpr int K_HOLE = 0;     // nothing to do (slot kept so item order == key order)
constexpr int K_COMPUTE = 1;  // matched key: run the (typeA,typeB) grid cell
constexpr int K_COPY_A = 2;   // pass-through of an unmatched container of the left bitmap
constexpr int K_COPY_B = 3;

// c_src encoding: container index in the left parent, or SRC_B | index in the right parent
// SRC_SHARED (uploaded sets only): the host container was a SHARED (copy-on-write) wrapper — the
// in-place twins then take the FUNCTIONAL cell for it (src/roaring.c:840, 1085-1088, 1235, 1376)
constexpr uint32_t SRC_SHARED = 0xfffffffeu;
constexpr uint32_t SRC_NONE = 0xffffffffu, SRC_B = 0x80000000u;   // pass-through of an unmatched container of the right bitmap

// c_card of a BITSET container produced by a lazy op: the reference leaves its cardinality field
// at BITSET_UNKNOWN_CARDINALITY (bitset.h:42), which later lazy steps can observe
// (container_is_full, containers.h:262-277).  We keep the true cardinality in the low bits and
// the "unknown to the reference" state in the top bit.  Only sets marked lazy carry the bit.
constexpr uint32_t CARD_UNKNOWN = 0x80000000u, CARD_MASK = 0x7fffffffu;

// type-rule variants of the pairwise kernel (bit set):
//   RULES_INPLACE          container_i* outcomes (roaring_bitmap_*_inplace)
//   RULES_LAZY             roaring_bitmap_lazy_or / lazy_xor (+ INPLACE: the _inplace twins)
//   RULES_CONV             lazy_or's bitsetconversion argument
//   RULES_NOFULL           lazy_or_from_lazy_inputs (roaring_priority_queue.c:99): lazy_ior on
//                          every matched key, without lazy_or_inplace's full-container short cut
//   RULES_FLIP             (with RULES_LAZY's kernel instantiation, op XOR) roaring_bitmap_flip: the
//                          right operand is the range as run containers, types follow the
//                          negation cells (mixed_negation.c), see decide_type_lazy
constexpr int RULES_INPLACE = 1, RULES_LAZY = 2, RULES_CONV = 4, RULES_NOFULL = 8, RULES_FLIP = 16;

// Device view of a resident set: SoA container directory + one payload slab.
// Payload of container c starts at payload + c_off[c] (16-byte aligned, padded to 16 B):
//   bitset: 1024 x u64;  array: c_len x u16 (sorted);  run: c_len x {u16 start,u16 len-1}.
// c_card is the true cardinality for every type (runs: sum(len+1), filled at upload).
struct SetView {
    const uint32_t *bm_beg;  // [n_bitmaps] first container of bitmap i
    const uint32_t *bm_cnt;  // [n_bitmaps] number of containers of bitmap i
    const uint16_t *c_key;
    const uint8_t *c_type;
    const uint32_t *c_card;
    const uint32_t *c_len;
    const uint64_t *c_off;
    const uint32_t *c_src;   // provenance of pass-through containers (SRC_NONE = computed here)
    const uint8_t *payload;
};

// Mutable directory of a set being produced by a kernel.
struct SetOut {
    uint32_t *bm_beg;
    uint32_t *bm_cnt;
    uint64_t *bm_card;  // per result bitmap: total cardinality
    uint64_t *bm_bytes;   // per result bitmap: stored payload bytes (16-byte rounded slots)
    uint64_t *bm_ebytes;  // per result bitmap: sum of round16(max(stored, min(8192, 2 * card))) — the
                          // quantity that bounds what a later op on it can produce (see PairBuf::build)
    uint16_t *c_key;
    uint8_t *c_type;
    uint32_t *c_card;
    uint32_t *c_len;
    uint64_t *c_off;
    uint32_t *c_src;
    uint8_t *payload;
};

// Cell descriptor of one pairwise work item: everything k_compute_items needs to run the cell or
// the pass-through copy, so that a warp fetches one 32-byte record instead of walking
// item -> container -> payload.  Two uint4:
//   a = {A payload offset / 16, B payload offset / 16, output slot offset / 16  (low 32 bits each), item id}
//   b.x  cA as stored (CARD_UNKNOWN included)
//   b.y  cB (17 bits) | tA << 17 | tB << 19 | kind << 21 | SHARED left << 23 | (A offset / 16) >> 32 << 24
//   b.z  lA | lB << 16   (at most 32768 runs or 4096 values)
//   b.w  slot capacity / 16 (16 bits) | (B offset / 16) >> 32 << 16 | (slot offset / 16) >> 32 << 24
// Offsets are 16-byte aligned and below 2^44 bytes (16 TiB, more than any device allocation); the
// capacity is at most 4 x 65536 bytes (slot_bound_lazy of two run containers).  A pass-through item
// keeps its source container (of A or B, by kind) in the A fields and leaves the B fields zero;
// a hole is all zero (kind K_HOLE).
struct CellDesc {
    uint64_t offA, offB, off;   // payload offsets of A / B (or the copy's source), output slot offset
    uint32_t item, cA, cB, lA, lB, cap;
    uint32_t tA, tB, kind;
    bool shared;                // the in-place twins' left container is SHARED: take the functional cell
};
__host__ __device__ __forceinline__ void cd_pack(const CellDesc &d, uint4 &a, uint4 &b) {
    const uint64_t oA = d.offA >> 4, oB = d.offB >> 4, oO = d.off >> 4;
    a = make_uint4((uint32_t)oA, (uint32_t)oB, (uint32_t)oO, d.item);
    b = make_uint4(d.cA,
                   d.cB | d.tA << 17 | d.tB << 19 | d.kind << 21 | (d.shared ? 1u : 0u) << 23 | (uint32_t)(oA >> 32) << 24,
                   d.lA | d.lB << 16, (d.cap >> 4) | (uint32_t)(oB >> 32) << 16 | (uint32_t)(oO >> 32) << 24);
}
__host__ __device__ __forceinline__ CellDesc cd_unpack(uint4 a, uint4 b) {
    CellDesc d;
    d.offA = ((uint64_t)(b.y >> 24) << 32 | a.x) << 4;
    d.offB = ((uint64_t)((b.w >> 16) & 0xffu) << 32 | a.y) << 4;
    d.off = ((uint64_t)(b.w >> 24) << 32 | a.z) << 4;
    d.item = a.w;
    d.cA = b.x;
    d.cB = b.y & 0x1ffffu;
    d.tA = (b.y >> 17) & 3u;
    d.tB = (b.y >> 19) & 3u;
    d.kind = (b.y >> 21) & 3u;
    d.shared = (b.y >> 23) & 1u;
    d.lA = b.z & 0xffffu;
    d.lB = b.z >> 16;
    d.cap = (b.w & 0xffffu) << 4;
    return d;
}

// Work items of one batched pairwise op (SoA, W entries; items of pair p occupy
// [item_off[p], item_off[p+1]) in key order with holes).
struct Items {
    uint8_t *kind;
    uint16_t *key;
    uint32_t *ca;        // container index in A (K_COMPUTE, K_COPY_A)
    uint32_t *cb;        // container index in B (K_COMPUTE, K_COPY_B)
    uint64_t *slot_off;  // byte offset of the output slot in the result slab
    uint8_t *cls;        // code-path class of the item (CLS_*), CLS_NONE for holes
    uint4 *desc;         // [2 W] cell descriptors in item order (cd_pack; null: cardinality-only sweeps)
    uint4 *desc_cls;     // [2 W] the live items' descriptors sorted by class (null: tickets walk desc)
    uint8_t *otype;      // result container type (0 = dropped)
    uint32_t *ocard;     // result cardinality
    uint32_t *olen;      // result length (array values / runs)
};

// Counters living in device memory, read back once per op.
struct OpStats {
    unsigned long long slab_cursor;   // bump allocator over the result slab (bytes)
    unsigned long long dir_cursor;    // bump allocator over the result directory (containers)
    unsigned long long algo_bytes;    // SURVEY.md §8(d) algorithmic bytes
    unsigned long long work_counter;  // dynamic scheduler for the compute kernel
    unsigned long long work_counter2;
    unsigned long long out_portable;  // sum over result bitmaps of roaring_bitmap_portable_size_in_bytes
    unsigned int error;               // 0 = ok; 1 = slot overflow; 2 = slab overflow; 3 = malformed blob
    unsigned int nk;                  // or_many: number of distinct keys
    unsigned int units;               // or_many: number of (key, slice) work units
    unsigned int cls_count[8];        // pairwise ops: live work items per code-path class
    unsigned int cls_cursor[8];       //               fill cursors of k_order_items
};

// Code-path classes of the pairwise work items.  k_compute_items is one large kernel (a code path
// per cell family); when the warps of an SM run different families at the same time it is bound
// by INSTRUCTION FETCH (ncu: no_instruction stalls dominate), so
// the tickets are handed out class by class: at any time almost every resident warp executes the
// same few hundred instructions.  Heavy classes first (tail balance).
// (per-item clocks, tools/scale_probe.py: run cells through the accumulator cost an order of
//  magnitude more than the average item under load — they go first)
constexpr int CLS_RUN_ACC = 0;   // run cells through the accumulator
constexpr int CLS_BR = 1;        // bitset x run
constexpr int CLS_AA_ACC = 2;    // array x array through the accumulator (unions / xors above 4096 values)
constexpr int CLS_BA = 3;        // bitset x array (either side)
constexpr int CLS_BB = 4;        // bitset x bitset
constexpr int CLS_AA = 5;        // array x array: filter / merge path
constexpr int CLS_RUN_IV = 6;    // run cells by interval sweep
constexpr int CLS_COPY = 7;      // pass-through
constexpr int CLS_NONE = 0xff;
constexpr int N_CLS = 8;

// Key-major index of one many-way union (rb200_many2.cu): built per call on the device.
//
// Index entry of one participating container, 16 bytes:
//   {payload offset / 16 (low 32 bits), input position, c_len, type | TF_* flags | (payload offset / 16) >> 32 << 8}
constexpr uint32_t TF_FULL_RUN = 16, TF_FULL_BITSET = 32;   // the type takes the low 4 bits, the flags 2 more
__host__ __device__ __forceinline__ uint32_t m2_tf(uint32_t type, uint32_t len, uint32_t card) {
    uint32_t f = type;
    if (type == T_RUN && len == 1 && card == 65536) f |= TF_FULL_RUN;
    if (type == T_BITSET && card == 65536) f |= TF_FULL_BITSET;
    return f;
}
__host__ __device__ __forceinline__ uint4 m2_entry(uint64_t off, uint32_t pos, uint32_t len, uint32_t tf) {
    const uint64_t o16 = off >> 4;
    return make_uint4((uint32_t)o16, pos, len, tf | (uint32_t)(o16 >> 32) << 8);
}
__host__ __device__ __forceinline__ uint64_t m2_entry_off(uint4 e) {
    return (((uint64_t)(e.w >> 8) << 32) | e.x) << 4;
}
__host__ __device__ __forceinline__ uint32_t m2_entry_tf(uint4 e) { return e.w & 0xffu; }

// Per-key counter of the index build (key_cu): participants in the high 32 bits, weight (stored
// bytes) in the low 32 bits in units of 16 << w_shift bytes.  w_shift is the smallest shift that
// keeps n * 2^13 >> w_shift below 2^32 (2^13 x 16 bytes is the largest container, a run container
// of 32768 runs); it is 0 below 2^19 inputs.  Weights are rounded up (m2_weight), so a small
// container still weighs at least one unit; one container weighs at most 2^(13 - w_shift) units, so
// a key's weight stays below n * 2^(13 - w_shift) < 2^32 and never carries into its count.  The
// weight only steers how keys are split into work units, never what they compute.
__host__ __device__ __forceinline__ unsigned long long m2_cu(uint32_t count, uint32_t weight) {
    return ((unsigned long long)count << 32) | weight;
}
__host__ __device__ __forceinline__ uint32_t m2_weight(uint32_t b16, uint32_t w_shift) {   // b16: 16-byte units
    return (b16 + (1u << w_shift) - 1) >> w_shift;
}
__host__ __device__ __forceinline__ uint32_t m2_cu_count(unsigned long long cu) { return (uint32_t)(cu >> 32); }
__host__ __device__ __forceinline__ uint32_t m2_cu_weight_kib(unsigned long long cu, uint32_t w_shift) {
    return (uint32_t)(((cu & 0xffffffffull) << w_shift) >> 6);
}
inline uint32_t m2_weight_shift(uint64_t n) {   // n < 2^32
    uint32_t s = 0;
    while (((n << 13) >> s) >> 32) s++;
    return s;
}

struct Many2Index {
    unsigned long long *key_cu;  // [65536] m2_cu(participants, weight)   (zero on entry)
    uint32_t w_shift;       // weight unit of key_cu: 16 << w_shift bytes
    uint32_t *key_count;    // [65536] participants per key (decoded by k_many2_scan)
    uint32_t *key_fill;     // [65536] fill cursors                    (zero on entry)
    uint32_t *key_start;    // [65536] first index entry of the key
    uint16_t *keys;         // [nk] live keys, increasing
    uint32_t *key_slices;   // [nk] work units of the key
    uint32_t *key_scratch;  // [nk] scratch slot of a split key
    uint32_t *unit_first;   // [nk] first work unit of the key
    unsigned long long *fold_first, *fold_second;   // [nk] order statistics of the fold (k_many2_fold)
    uint32_t *fold_F, *fold_L;                      // [nk]
    uint32_t *unit_ki;      // [max_units] work unit -> live key index
    uint4 *ent;             // [entries] m2_entry(payload offset, input position, c_len, type | flags)
};

// ---- single-pair fused path (rb200_fused.cu): packed input block (host-pinned -> device) and
// output block (mapped pinned host memory the kernel writes directly)
constexpr int FUSED_WARPS = 8;
constexpr uint32_t FUSED_MAX_ITEMS = 512;          // containers of both operands together
constexpr uint32_t FUSED_IN_BYTES = 1u << 20;      // packed operands must fit
constexpr uint32_t FUSED_OUT_BYTES = 2u << 20;     // result slots must fit (else: the batched path)
struct FusedHdr { uint32_t na, nb, o_key, o_type, o_shared, o_card, o_len, o_off, pad[8]; };   // 64 B; offsets from the block start
struct FusedOutHdr { volatile uint32_t seq; uint32_t error, n_out, pad; };
constexpr uint32_t FUSED_OUT_KEY = 64, FUSED_OUT_TYPE = FUSED_OUT_KEY + 2 * FUSED_MAX_ITEMS,
                   FUSED_OUT_CARD = FUSED_OUT_TYPE + FUSED_MAX_ITEMS, FUSED_OUT_LEN = FUSED_OUT_CARD + 4 * FUSED_MAX_ITEMS,
                   FUSED_OUT_OFF = FUSED_OUT_LEN + 4 * FUSED_MAX_ITEMS, FUSED_OUT_PAYLOAD = FUSED_OUT_OFF + 4 * FUSED_MAX_ITEMS;
bool launch_pair_fused(int op, const uint8_t *d_in, uint8_t *out_mapped, uint32_t out_bytes, int rules, uint32_t seq,
                       cudaStream_t s);


// --- launch wrappers (rb200_kernels.cu); every wrapper bumps g_launches -----------------
extern unsigned long long g_launches;

void launch_plan_pairs(const SetView &A, const SetView &B, const uint32_t *ia, const uint32_t *ib,
                       const uint64_t *item_off, uint32_t npairs, int op, bool card_only, int rules,
                       Items it, OpStats *st, cudaStream_t s);
void launch_order_items(Items it, uint64_t W, OpStats *st, cudaStream_t s);
void launch_compute_items(const SetView &A, const SetView &B, Items it, uint64_t W, int op,
                          uint8_t *slab, uint64_t slab_cap, OpStats *st, int rules, int copy_ticket,
                          cudaStream_t s);
void launch_card_items(const SetView &A, const SetView &B, Items it, uint64_t W, OpStats *st,
                       cudaStream_t s);
void launch_finalize_pairs(const SetView &A, const SetView &B, Items it, const uint64_t *item_off,
                           uint32_t npairs, SetOut out, OpStats *st, cudaStream_t s);
void launch_finalize_cards(Items it, const uint64_t *item_off, uint32_t npairs, uint64_t *out,
                           cudaStream_t s);
void launch_sum_cardinalities(const uint64_t *bm_card, uint32_t n, uint64_t *d_acc, cudaStream_t s);
void launch_set_cardinalities(const SetView &S, uint32_t n_bitmaps, uint64_t *out, cudaStream_t s);

// packing for download: measure+scan (off/beg have n+1 entries), then copy
// elide bit 0 / 1: payloads that are pass-through copies of the left / right parent are NOT packed
// (the host rebuilds them from its own copy of the inputs)
void launch_pack(const SetView &S, uint32_t n, int elide, uint64_t *bytes, uint32_t *cnts, uint64_t *off,
                 uint64_t *beg, cudaStream_t s);
void launch_pack_copy(const SetView &S, uint32_t n, int elide, const uint64_t *off, const uint64_t *beg,
                      SetOut out, cudaStream_t s);

// xor_many: mark -> compact keys (then launch_xor_many)
void launch_many_mark(const SetView &S, const uint32_t *idx, uint32_t n, uint32_t key_lo,
                      uint32_t key_hi, uint32_t *flags /*65536*/, cudaStream_t s);
void launch_many_compact(const uint32_t *flags, uint16_t *keys_out, OpStats *st, cudaStream_t s);

// or_many: key-major index, then one pass over the payloads (rb200_many2.cu)
void launch_or_many2(const SetView &S, const uint32_t *idx, uint32_t n, uint32_t key_lo, uint32_t key_hi,
                     const Many2Index &ix, uint32_t max_units, uint32_t *scratch, uint32_t *tickets,
                     uint32_t scratch_slots, SetOut out, uint32_t *card_per_key, OpStats *st, int sms,
                     cudaStream_t s, cudaEvent_t ev_kernel_start, bool use_tma, bool window_index, uint32_t *cnt_tab);
constexpr uint32_t M2W_MAX_CHUNKS = 64;   // key-window index build: chunks of 256 input bitmaps per window

void launch_pack_scan(const uint64_t *bytes, const uint32_t *cnts, uint32_t n, uint64_t *off,
                      uint64_t *beg, cudaStream_t s);
void launch_serialize_measure(const SetView &S, uint32_t n, uint64_t *sizes16, uint32_t *exact,
                              uint32_t *hasrun, cudaStream_t s);
void launch_serialize_write(const SetView &S, uint32_t n, const uint64_t *off, const uint32_t *hasrun,
                            uint8_t *dst, cudaStream_t s);
// device-side roaring_bitmap_portable_deserialize_safe of nb blobs staged in `raw`
void launch_deserialize(const uint8_t *raw, const uint64_t *roff, const uint64_t *rlen,
                        const uint64_t *slab_base, uint32_t nb, uint64_t nc, SetOut out,
                        uint64_t *src_pos, OpStats *st, cudaStream_t s);
void launch_deserialize_frozen(const uint8_t *raw, const uint64_t *roff, const uint64_t *rlen,
                               const uint64_t *slab_base, uint32_t nb, uint64_t nc, SetOut out,
                               uint64_t *src_pos, OpStats *st, cudaStream_t s);
// frozen format emit: sizes32 = blob bytes rounded up to 32 (blob starts stay 32-byte aligned)
void launch_frozen_measure(const SetView &S, uint32_t n, uint64_t *sizes32, uint32_t *exact, uint32_t *cnt,
                           cudaStream_t s);
void launch_frozen_write(const SetView &S, uint32_t n, uint64_t nc, const uint64_t *off, uint8_t *dst,
                         uint64_t *c_dst, cudaStream_t s);
void launch_run_optimize(const SetView &S, uint32_t nb, uint64_t nc, int mode, SetOut out, OpStats *st,
                         cudaStream_t s);
void launch_values_measure(const SetView &S, uint32_t nb, uint64_t *bm_vals, uint32_t *dummy,
                           uint64_t *c_start, uint32_t *c_bitmap, cudaStream_t s);
void launch_values_write(const SetView &S, uint32_t nb, const uint64_t *bm_off, const uint64_t *c_start,
                         const uint32_t *c_bitmap, uint64_t nc, uint32_t *out, cudaStream_t s);
void launch_xor_many(const SetView &S, const uint32_t *idx, uint32_t n, const uint16_t *keys,
                     uint8_t *t_type, uint32_t *t_card, uint32_t *t_len, SetOut out, OpStats *st,
                     int sms, cudaStream_t s);

}  // namespace rb200
