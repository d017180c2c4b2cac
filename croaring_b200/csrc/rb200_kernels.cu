// rb200_kernels.cu — sm_90a kernels of the Roaring set-algebra hot path.
//
//   k_plan_pairs      warp per bitmap pair: key merge by binary-search ranks (the reference's
//                     two-pointer loops, src/roaring.c:742-768, 896-951) -> work items.
//   k_compute_items   (rb200_compute.cu) warp per work item: one container x container grid cell
//                     (include/roaring/containers/containers.h:726-1876) or a pass-through copy.
//   k_card_items      warp per matched item: container_and_cardinality (containers.h:811-859).
//   k_finalize_pairs  warp per pair: drop empty results (roaring.c:756-760), build the
//                     key-sorted result directory.
//   k_many_mark       the live keys of an N-way XOR's inputs (k_xor_many, rb200_many.cu), then
//   k_many_compact    their increasing list.  The N-way union is rb200_many2.cu.
#include "rb200_device.cuh"
#include "rb200_cells.cuh"

namespace rb200 {

unsigned long long g_launches = 0;
int g_sm_count = 132;   // until rb200_init reads the device's
bool g_pdl = []() { const char *e = getenv("RB200_PDL"); return !(e && e[0] == '0'); }();

// code-path class of a matched cell (see rb200_common.h CLS_*); mirrors the branches of cell_compute
__device__ __forceinline__ int cell_class(int op, int rules, int tA, int tB, uint32_t cA, uint32_t cB, uint32_t lA,
                                          uint32_t lB) {
    const bool bA = tA == T_BITSET, bB = tB == T_BITSET;
    if (bA && bB) return CLS_BB;
    if (bA || bB) return (bA ? tB : tA) == T_ARRAY ? CLS_BA : CLS_BR;
    if (tA == T_ARRAY && tB == T_ARRAY) {
        if (op == OP_AND || op == OP_ANDNOT) return CLS_AA;
        const bool lazy = (rules & RULES_LAZY) != 0, lazy_eager = lazy && op == OP_XOR && (rules & RULES_INPLACE);
        return cA + cB <= (uint32_t)MAX_ARRAY && (!lazy || lazy_eager || (cA + cB <= 1024u && !(rules & RULES_CONV)))
                   ? CLS_AA : CLS_AA_ACC;
    }
    return (tA == T_RUN ? lA : cA) + (tB == T_RUN ? lB : cB) <= 512u ? CLS_RUN_IV : CLS_RUN_ACC;
}

// ------------------------------------------------------------------------------ planner
// sh.onA / sh.onB: an unmatched container of that operand is not copied but shared — no slot, no
// cell, its directory entry (type, card, len as in the parent; c_off = sh.dA / sh.dB + the parent's
// c_off) goes straight into the item records for k_finalize_pairs, and st->shared_used[side] is set.
// Own slots are offset by sh.bias (see PassShare).
__global__ void __launch_bounds__(128)
k_plan_pairs(SetView A, SetView B, const uint32_t *__restrict__ ia,
             const uint32_t *__restrict__ ib, const uint64_t *__restrict__ item_off,
             uint32_t npairs, int op, bool card_only, int rules, PassShare sh, Items it, OpStats *st) {
    __shared__ unsigned int s_cls[N_CLS];   // live items per class of this block (one global atomic per class at the end)
    // the four pairs of a block reserve their result slots with ONE atomic per round (the slab cursor
    // is a single address: a returning atomic per pair serialised 19 900 of them per launch)
    __shared__ uint32_t s_tot[4];
    __shared__ unsigned long long s_base;
    __shared__ unsigned int s_used[2];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    // Before the wait: lane r fetches the warp's pair of round r (the first 32 rounds, all loads in
    // flight together) and the sizes of its two bitmaps.  The pair list arrives by a copy queued
    // right before this launch, which is never overlapped, and the operands' directories were
    // complete when the launch was queued (the host settles a pending operand before it plans a
    // batch on it: ensure_mirrors), so none of this depends on the kernel still draining ahead.
    const uint32_t stride = gridDim.x * 4;
    uint32_t r_a0 = 0, r_na = 0, r_b0 = 0, r_nb = 0;
    uint64_t r_off = 0;
    {
        const uint64_t p = (uint64_t)blockIdx.x * 4 + wid + (uint64_t)lane * stride;
        if (p < npairs) {
            const uint32_t a = ia[p], b = ib[p];
            r_off = item_off[p];
            r_a0 = A.bm_beg[a];
            r_na = A.bm_cnt[a];
            r_b0 = B.bm_beg[b];
            r_nb = B.bm_cnt[b];
        }
    }
    // Wait: from here on the kernel writes device buffers (item records, counters), which
    // may have been released by the previous op to the stream-ordered pool while that op's kernels
    // still read them, and the counters of `st` are zeroed by the previous op's k_finalize_pairs.
    pdl_wait();
    if (threadIdx.x == 0) stamp_first(&st->t_begin);
    if (threadIdx.x < N_CLS) s_cls[threadIdx.x] = 0;
    if (threadIdx.x < 2) s_used[threadIdx.x] = 0;
    __syncthreads();
    uint32_t round = 0;
    for (uint32_t p0 = blockIdx.x * 4; p0 < npairs; p0 += stride, round++) {
        const uint32_t p = p0 + wid;
        const bool vp = p < npairs;
        uint32_t a0, na, b0, nb;
        uint64_t base_item;
        if (round < 32) {
            a0 = __shfl_sync(FULLMASK, r_a0, round);
            na = __shfl_sync(FULLMASK, r_na, round);
            b0 = __shfl_sync(FULLMASK, r_b0, round);
            nb = __shfl_sync(FULLMASK, r_nb, round);
            base_item = __shfl_sync(FULLMASK, r_off, round);
        } else {
            const uint32_t a = vp ? ia[p] : 0, b = vp ? ib[p] : 0;
            a0 = vp ? A.bm_beg[a] : 0, na = vp ? A.bm_cnt[a] : 0;
            b0 = vp ? B.bm_beg[b] : 0, nb = vp ? B.bm_cnt[b] : 0;
            base_item = vp ? item_off[p] : 0;
        }
        const uint32_t tot = na + nb;
        for (uint32_t t0 = 0;; t0 += 32) {
            if (!__syncthreads_or(t0 < tot)) break;   // (also keeps the rounds' shared words apart)
            const uint32_t t = t0 + lane;
            int kind = K_HOLE, cls = CLS_NONE;
            uint32_t ca = 0, cb = 0, cap = 0, pos = 0, key = 0;
            CellDesc d = {};
            if (t < tot) {
                if (t < na) {
                    ca = a0 + t;
                    key = A.c_key[ca];
                    const uint32_t lb = lower_bound_u16(B.c_key + b0, nb, key);
                    const bool matched = lb < nb && B.c_key[b0 + lb] == key;
                    pos = t + lb;
                    if (matched) {
                        cb = b0 + lb;
                        kind = K_COMPUTE;
                        if (!card_only) {
                            d.tA = A.c_type[ca];
                            d.tB = B.c_type[cb];
                            d.cA = A.c_card[ca];
                            d.cB = B.c_card[cb] & CARD_MASK;
                            d.lA = A.c_len[ca];
                            d.lB = B.c_len[cb];
                            d.offA = A.c_off[ca];
                            d.offB = B.c_off[cb];
                            // in-place twins: a SHARED left container takes the functional cell (roaring.c:1085-1088),
                            // and so does lazy_xor_inplace (container_lazy_xor, :2794-2797); lazy_or_inplace
                            // works on a writable copy instead (:2624, 2636)
                            d.shared = (rules & RULES_INPLACE) && (!(rules & RULES_LAZY) || op == OP_XOR) &&
                                       A.c_src[ca] == SRC_SHARED;
                            const uint32_t cA = d.cA & CARD_MASK;
                            cap = (rules & RULES_LAZY) ? slot_bound_lazy(d.tA, d.tB, cA, d.cB, d.lA, d.lB)
                                  : (rules & RULES_KEEP_RUN) && d.tA == T_RUN ? slot_bound_keep_run(d.lA, d.cB)
                                                                              : slot_bound(op, d.tA, d.tB, cA, d.cB, d.lA, d.lB);
                            cls = cell_class(op, d.shared ? rules & ~RULES_INPLACE : rules, d.tA, d.tB, cA, d.cB, d.lA, d.lB);
                        }
                    } else if (op != OP_AND && !card_only) {
                        kind = K_COPY_A;
                        cls = sh.onA ? CLS_NONE : CLS_COPY;
                        d.tA = A.c_type[ca];
                        d.cA = A.c_card[ca];
                        d.lA = A.c_len[ca];
                        d.offA = A.c_off[ca];
                        cap = sh.onA ? 0u : round16(stored_bytes(d.tA, d.lA));
                    }
                } else {
                    const uint32_t j = t - na;
                    cb = b0 + j;
                    key = B.c_key[cb];
                    const uint32_t ub = upper_bound_u16(A.c_key + a0, na, key);
                    const bool matched = ub > 0 && A.c_key[a0 + ub - 1] == key;
                    pos = j + ub;
                    if (!matched && (op == OP_OR || op == OP_XOR) && !card_only) {
                        kind = K_COPY_B;
                        cls = sh.onB ? CLS_NONE : CLS_COPY;
                        d.tA = B.c_type[cb];
                        d.cA = B.c_card[cb];
                        d.lA = B.c_len[cb];
                        d.offA = B.c_off[cb];
                        cap = sh.onB ? 0u : round16(stored_bytes(d.tA, d.lA));
                    }
                }
            }
            // warp-aggregated bump allocation of the output slots
            const uint32_t incl = warp_incl_scan(cap, lane);
            const uint32_t total = __shfl_sync(FULLMASK, incl, 31);
            if (lane == 31) s_tot[wid] = total;
            __syncthreads();
            if (threadIdx.x == 0) {
                const unsigned long long sum = (unsigned long long)s_tot[0] + s_tot[1] + s_tot[2] + s_tot[3];
                s_base = sum ? atomicAdd(&st->slab_cursor, sum) : 0ull;
            }
            __syncthreads();
            unsigned long long slab_base = s_base;
            for (int w = 0; w < wid; w++) slab_base += s_tot[w];
            const bool shared = (kind == K_COPY_A && sh.onA) || (kind == K_COPY_B && sh.onB);
            if (shared) s_used[kind == K_COPY_B] = 1u;
            if (t < tot) {
                const uint64_t idx = base_item + pos;
                const int dkind = shared ? K_HOLE : kind;   // nothing for k_compute_items to do
                it.kind[idx] = (uint8_t)kind;
                it.key[idx] = (uint16_t)key;
                it.ca[idx] = ca;
                it.cb[idx] = cb;
                it.slot_off[idx] = shared ? (kind == K_COPY_A ? sh.dA : sh.dB) + d.offA : slab_base + incl - cap + sh.bias;
                // the class-ordered list copies only live descriptors; without it the holes are read too
                if (it.desc && (dkind != K_HOLE || !it.desc_cls)) {
                    d.off = slab_base + incl - cap;
                    d.cap = cap;
                    d.kind = dkind;
                    d.item = (uint32_t)idx;
                    cd_pack(d, it.desc[2 * idx], it.desc[2 * idx + 1]);
                }
                if (it.cls) it.cls[idx] = (uint8_t)cls;
                it.otype[idx] = shared ? (uint8_t)d.tA : 0;
                it.ocard[idx] = shared ? d.cA : 0;
                it.olen[idx] = shared ? d.lA : 0;
            }
            if (it.cls) {   // live items per class
#pragma unroll
                for (int c = 0; c < N_CLS; c++) {
                    const unsigned m = __ballot_sync(FULLMASK, cls == c);
                    if (m && lane == 0) atomicAdd(&s_cls[c], (unsigned)__popc(m));
                }
            }
        }
    }
    // Trigger: what is left is one atomic per class.  The next kernel reads the counters and item
    // records only after its own wait, which waits for this whole grid.
    pdl_trigger();
    __syncthreads();
    if (it.cls && threadIdx.x < N_CLS && s_cls[threadIdx.x]) atomicAdd(&st->cls_count[threadIdx.x], s_cls[threadIdx.x]);
    if (threadIdx.x < 2 && s_used[threadIdx.x]) st->shared_used[threadIdx.x] = 1u;
}

// descriptors of the live items grouped by class: desc_cls[prefix(class) + k].  A block takes chunks of 2048 item slots
// (256 per warp); per chunk ONE global atomic per class reserves the block's range, the ranks
// inside come from ballots and an 8-warp scan in shared memory.
__global__ void __launch_bounds__(256)
k_order_items(Items it, uint64_t W, OpStats *st) {
    __shared__ uint32_t s_wcnt[8][N_CLS], s_base[N_CLS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    // Wait: everything this kernel reads (class counts, classes, descriptors) is k_plan_pairs' output.
    pdl_wait();
    uint32_t pre_l = 0;   // lane c (< N_CLS): first slot of class c in the order list
    for (int c = 0; c < N_CLS; c++)
        if (c < lane) pre_l += st->cls_count[c];
    for (uint64_t chunk = (uint64_t)blockIdx.x * 2048; chunk < W; chunk += (uint64_t)gridDim.x * 2048) {
        const uint64_t w0 = chunk + (uint64_t)wid * 256;
        int cl[8];
        uint32_t mycnt = 0;   // lane c: this warp's items of class c
#pragma unroll
        for (int s8 = 0; s8 < 8; s8++) {
            const uint64_t i = w0 + s8 * 32 + lane;
            cl[s8] = i < W ? (int)it.cls[i] : CLS_NONE;
#pragma unroll
            for (int cc = 0; cc < N_CLS; cc++) {
                const unsigned m = __ballot_sync(FULLMASK, cl[s8] == cc);
                if (lane == cc) mycnt += __popc(m);
            }
        }
        if (lane < N_CLS) s_wcnt[wid][lane] = mycnt;
        __syncthreads();
        if (wid == 0 && lane < N_CLS) {
            uint32_t run = 0;
            for (int w = 0; w < 8; w++) {
                const uint32_t t = s_wcnt[w][lane];
                s_wcnt[w][lane] = run;
                run += t;
            }
            s_base[lane] = run ? atomicAdd(&st->cls_cursor[lane], run) : 0u;
        }
        __syncthreads();
        uint32_t nxt = lane < N_CLS ? pre_l + s_base[lane] + s_wcnt[wid][lane] : 0u;   // lane c: next slot of class c
#pragma unroll
        for (int s8 = 0; s8 < 8; s8++) {
            const uint64_t i = w0 + s8 * 32 + lane;
            uint4 d0 = {}, d1 = {};
            if (cl[s8] != CLS_NONE) {
                d0 = it.desc[2 * i];
                d1 = it.desc[2 * i + 1];
            }
#pragma unroll
            for (int cc = 0; cc < N_CLS; cc++) {
                const unsigned m = __ballot_sync(FULLMASK, cl[s8] == cc);
                if (!m) continue;
                const uint32_t b = __shfl_sync(FULLMASK, nxt, cc);
                if (cl[s8] == cc) {
                    const uint64_t o = b + __popc(m & lanemask_lt());
                    it.desc_cls[2 * o] = d0;
                    it.desc_cls[2 * o + 1] = d1;
                }
                if (lane == cc) nxt += __popc(m);
            }
        }
        __syncthreads();
    }
    // Trigger: this CTA has placed its last descriptor; the cell kernel waits for the whole grid
    // before it reads the order list.
    pdl_trigger();
}

// (the pairwise cell kernel, k_compute_items, is in rb200_compute.cu; the grid cells themselves —
// cell_compute — live in rb200_cells.cuh, shared with rb200_fused.cu)

// container_and_cardinality for one matched cell (containers.h:811-859)
__device__ __forceinline__ uint32_t cell_and_card(uint32_t *acc, int tA, int tB, const uint8_t *pa,
                                                  const uint8_t *pb, uint32_t cA, uint32_t cB,
                                                  uint32_t lA, uint32_t lB, int lane) {
    if (tA == T_BITSET && tB == T_BITSET) return (uint32_t)bitset_and_card(pa, pb, lane);
    if (tA == T_ARRAY || tB == T_ARRAY) {
        const bool arrA = (tA == T_ARRAY) && !(tB == T_ARRAY && cB < cA);
        const uint8_t *parr = arrA ? pa : pb;
        const uint32_t narr = arrA ? cA : cB;
        const int to = arrA ? tB : tA;
        const uint8_t *po = arrA ? pb : pa;
        const uint32_t lo = arrA ? lB : lA;
        if (to == T_BITSET)
            return filter_array<false, false>(parr, narr, reinterpret_cast<const uint32_t *>(po),
                                              nullptr, nullptr, lane);
        acc_load(acc, to, po, lo, lane);
        const uint32_t n = filter_array<false, false>(parr, narr, acc, nullptr, nullptr, lane);
        __syncwarp();
        return n;
    }
    // run x bitset / bitset x run / run x run
    int card, nr;
    if (tA == T_RUN && tB == T_RUN) {
        acc_load(acc, tA, pa, lA, lane);
        acc_and_runs(acc, pb, lB, lane);
        __syncwarp();
        acc_count(acc, lane, false, card, nr);
    } else {
        const bool runA = tA == T_RUN;
        acc_load(acc, T_RUN, runA ? pa : pb, runA ? lA : lB, lane);
        card = acc_and_bitset_card(acc, runA ? pb : pa, lane);
    }
    __syncwarp();
    return (uint32_t)card;
}

__global__ void __launch_bounds__(128)
k_card_items(SetView A, SetView B, Items it, uint64_t W, OpStats *st) {
    __shared__ __align__(16) uint32_t s_acc[4][ACC_WORDS];
    const int lane = threadIdx.x & 31;
    uint32_t *acc = s_acc[threadIdx.x >> 5];
    constexpr unsigned long long TICKET = 8;
    unsigned long long tk = 0;
    if (lane == 0) tk = atomicAdd(&st->work_counter, TICKET);
    tk = __shfl_sync(FULLMASK, tk, 0);
    while (tk < W) {
        unsigned long long next = 0;
        if (lane == 0) next = atomicAdd(&st->work_counter, TICKET);
        const unsigned long long tend = tk + TICKET < W ? tk + TICKET : W;
        for (unsigned long long item = tk; item < tend; item++) {
            if (it.kind[item] != K_COMPUTE) continue;
            const uint32_t ca = it.ca[item], cb = it.cb[item];
            const uint32_t c =
                cell_and_card(acc, A.c_type[ca], B.c_type[cb], A.payload + A.c_off[ca],
                              B.payload + B.c_off[cb], A.c_card[ca], B.c_card[cb], A.c_len[ca],
                              B.c_len[cb], lane);
            if (lane == 0) it.ocard[item] = c;
        }
        tk = __shfl_sync(FULLMASK, next, 0);
    }
}

// ------------------------------------------------------------------------------ finalize
#ifndef RB200_FIN_BLOCKS
#define RB200_FIN_BLOCKS 16
#endif
// deliver (null: the counters stay in st for the caller): the last CTA copies the counters resolve()
// reads into this mapped pinned block, then zeroes st for the next op.
__global__ void __launch_bounds__(128)
k_finalize_pairs(SetView A, SetView B, Items it, const uint64_t *__restrict__ item_off,
                 uint32_t npairs, uint32_t rw_a, uint32_t rw_b, SetOut out, OpStats *st, OpStats *deliver) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    // the four pairs of a block reserve their directory range with ONE atomic (the cursor is a single
    // address: one returning atomic per pair serialised 19 900 of them per launch)
    __shared__ uint32_t s_cnt[4];
    __shared__ unsigned long long s_base;
    unsigned long long acc_bytes = 0, acc_outb = 0;  // per-warp totals: one atomic each at the end
    // Wait before everything: the result records come from the cell kernel still draining ahead.
    pdl_wait();
    for (uint32_t p0 = blockIdx.x * 4; p0 < npairs; p0 += gridDim.x * 4) {
        const uint32_t p = p0 + wid;
        const bool vp = p < npairs;
        const uint64_t i0 = vp ? item_off[p] : 0, i1 = vp ? item_off[p + 1] : 0;
        // pass 1: count surviving containers, cardinality and algorithmic bytes
        uint32_t cnt = 0, anyrun = 0;
        unsigned long long card = 0, bytes = 0, outb = 0, sbytes = 0, ebytes = 0;
        for (uint64_t i = i0 + lane; i < i1; i += 32) {
            const int kind = it.kind[i];
            if (kind == K_HOLE) continue;
            const int ot = it.otype[i];
            const uint32_t osz = ot ? portable_bytes(ot, it.olen[i]) : 0u;
            outb += osz;
            if (ot) {
                sbytes += round16(stored_bytes(ot, it.olen[i]));
                ebytes += effective_bytes(ot, it.olen[i], it.ocard[i] & CARD_MASK);
            }
            anyrun |= (ot == T_RUN) ? 1u : 0u;
            if (kind == K_COMPUTE) {   // (add_offset's cells name a source on one side or none, SRC_NONE)
                const uint32_t ca = it.ca[i], cb = it.cb[i];
                bytes += (ca != SRC_NONE ? portable_bytes(A.c_type[ca], A.c_len[ca]) : 0u) +
                         (cb != SRC_NONE ? portable_bytes(B.c_type[cb], B.c_len[cb]) : 0u) + osz;
            } else {   // a copied pass-through container is read and written, a shared one moves nothing
                bytes += (unsigned long long)(kind == K_COPY_A ? rw_a : rw_b) * osz;
            }
            if (ot) {
                cnt++;
                card += it.ocard[i] & CARD_MASK;
            }
        }
        cnt = __reduce_add_sync(FULLMASK, cnt);
        anyrun = __reduce_or_sync(FULLMASK, anyrun);
        for (int d = 16; d > 0; d >>= 1) {
            card += __shfl_xor_sync(FULLMASK, card, d);
            bytes += __shfl_xor_sync(FULLMASK, bytes, d);
            outb += __shfl_xor_sync(FULLMASK, outb, d);
            sbytes += __shfl_xor_sync(FULLMASK, sbytes, d);
            ebytes += __shfl_xor_sync(FULLMASK, ebytes, d);
        }
        if (lane == 0) s_cnt[wid] = cnt;
        __syncthreads();
        if (threadIdx.x == 0) {
            const unsigned long long tot = (unsigned long long)s_cnt[0] + s_cnt[1] + s_cnt[2] + s_cnt[3];
            s_base = tot ? atomicAdd(&st->dir_cursor, tot) : 0ull;
        }
        __syncthreads();
        unsigned long long base = s_base;
        for (int w = 0; w < wid; w++) base += s_cnt[w];
        __syncthreads();   // s_cnt / s_base are rewritten by the next round
        if (lane == 0 && vp) {
            acc_bytes += bytes;
            acc_outb += outb + portable_header_bytes(cnt, anyrun != 0);
            out.bm_beg[p] = (uint32_t)base;
            out.bm_cnt[p] = cnt;
            out.bm_card[p] = card;
            out.bm_bytes[p] = sbytes;
            out.bm_ebytes[p] = ebytes;
        }
        // pass 2: ordered compaction into the directory
        uint32_t done = 0;
        for (uint64_t i = i0; i < i1; i += 32) {
            const uint64_t idx = i + lane;
            const bool live = idx < i1 && it.kind[idx] != K_HOLE && it.otype[idx] != 0;
            const unsigned m = __ballot_sync(FULLMASK, live);
            if (live) {
                const uint64_t o = base + done + __popc(m & lanemask_lt());
                out.c_key[o] = it.key[idx];
                out.c_type[o] = it.otype[idx];
                out.c_card[o] = it.ocard[idx];
                out.c_len[o] = it.olen[idx];
                out.c_off[o] = it.slot_off[idx];
                const int kd = it.kind[idx];
                out.c_src[o] = kd == K_COPY_A ? it.ca[idx] : (kd == K_COPY_B ? (SRC_B | it.cb[idx]) : SRC_NONE);
            }
            done += __popc(m);
        }
    }
    // Trigger: the directory of this CTA's pairs is written; the next kernel waits for the whole
    // grid before it reads the result.
    pdl_trigger();
    __shared__ unsigned long long s_tot[4][2];
    if (lane == 0) { s_tot[wid][0] = acc_bytes; s_tot[wid][1] = acc_outb; }
    __syncthreads();
    if (threadIdx.x < 2) {
        const unsigned long long v = s_tot[0][threadIdx.x] + s_tot[1][threadIdx.x] + s_tot[2][threadIdx.x] + s_tot[3][threadIdx.x];
        if (v) atomicAdd(threadIdx.x ? &st->out_portable : &st->algo_bytes, v);
    }
    if (!deliver) return;
    // the last CTA to get here sees every other CTA's counters (fence, then the ticket)
    __shared__ bool s_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(&st->fin_blocks, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (threadIdx.x == 0) {
        deliver->slab_cursor = __ldcg(&st->slab_cursor);
        deliver->dir_cursor = __ldcg(&st->dir_cursor);
        deliver->algo_bytes = __ldcg(&st->algo_bytes);
        deliver->out_portable = __ldcg(&st->out_portable);
        deliver->error = __ldcg(&st->error);
        deliver->shared_used[0] = __ldcg(&st->shared_used[0]);
        deliver->shared_used[1] = __ldcg(&st->shared_used[1]);
        deliver->t_begin = __ldcg(&st->t_begin);
        deliver->t_cells0 = __ldcg(&st->t_cells0);
        deliver->t_cells1 = __ldcg(&st->t_cells1);
        deliver->t_end = global_ns();
    }
    __syncthreads();
    // every kernel of the next op that touches st waits for this grid first
    for (uint32_t k = threadIdx.x; k < sizeof(OpStats) / 4; k += blockDim.x) reinterpret_cast<uint32_t *>(st)[k] = 0u;
}

__global__ void __launch_bounds__(128)
k_finalize_cards(Items it, const uint64_t *__restrict__ item_off, uint32_t npairs,
                 uint64_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t p = warp; p < npairs; p += nwarps) {
        const uint64_t i0 = item_off[p], i1 = item_off[p + 1];
        unsigned long long card = 0;
        for (uint64_t i = i0 + lane; i < i1; i += 32)
            if (it.kind[i] == K_COMPUTE) card += it.ocard[i];
        card = warp_sum(card);
        if (lane == 0) out[p] = card;
    }
}

__global__ void k_set_cardinalities(SetView S, uint32_t n, uint64_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t b = warp; b < n; b += nwarps) {
        const uint32_t c0 = S.bm_beg[b], nc = S.bm_cnt[b];
        unsigned long long card = 0;
        for (uint32_t i = lane; i < nc; i += 32) card += S.c_card[c0 + i] & CARD_MASK;
        card = warp_sum(card);
        if (lane == 0) out[b] = card;
    }
}

// *acc += sum of bm_card[0..n) (device-resident checksum of a result set)
__global__ void k_sum_cards(const uint64_t *__restrict__ bm_card, uint32_t n, unsigned long long *acc) {
    // Wait: bm_card is written by the op that produced the set, usually the kernel right ahead.
    pdl_wait();
    unsigned long long v = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) v += bm_card[i];
    // Trigger: only the warp sums and one atomic per warp are left.
    pdl_trigger();
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(acc, v);
}

// ------------------------------------------------------------------------------ xor_many keys
__global__ void k_many_mark(SetView S, const uint32_t *__restrict__ idx, uint32_t n,
                            uint32_t key_lo, uint32_t key_hi, uint32_t *__restrict__ flags) {
    for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
        const uint32_t b = idx ? idx[i] : i;
        const uint32_t c0 = S.bm_beg[b], nc = S.bm_cnt[b];
        for (uint32_t c = threadIdx.x; c < nc; c += blockDim.x) {
            const uint32_t k = S.c_key[c0 + c];
            if (k >= key_lo && k <= key_hi) flags[k] = 1u;
        }
    }
}

// single CTA, 1024 threads: ordered list of the keys whose flag is set
__global__ void __launch_bounds__(1024)
k_many_compact(const uint32_t *__restrict__ flags, uint16_t *__restrict__ keys, OpStats *st) {
    __shared__ uint32_t s_warp[32];
    const int tid = threadIdx.x;
    uint32_t cnt = 0, nk;
    for (int k = 0; k < 64; k++) cnt += flags[tid * 64 + k] ? 1u : 0u;
    uint32_t o = block_excl_scan<1024>(cnt, s_warp, &nk);
    if (tid == 0) st->nk = nk;
    for (int k = 0; k < 64; k++)
        if (flags[tid * 64 + k]) keys[o++] = (uint16_t)(tid * 64 + k);
}

// ------------------------------------------------------------------------------ packing
// Compact a set for download: directory in bitmap order, payload contiguous in bitmap order
// without slot slack, so that any range of bitmaps is one directory range + one payload range
// (chunked D2H overlapped with host materialisation).
__global__ void __launch_bounds__(128)
k_pack_measure(SetView S, uint32_t n, int elide, uint64_t *__restrict__ bytes, uint32_t *__restrict__ cnts) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t b = warp; b < n; b += nwarps) {
        const uint32_t c0 = S.bm_beg[b], nc = S.bm_cnt[b];
        unsigned long long v = 0;
        for (uint32_t i = lane; i < nc; i += 32) {
            const uint32_t src = elide ? S.c_src[c0 + i] : SRC_NONE;
            const bool skip = src != SRC_NONE && ((src & SRC_B) ? (elide & 2) : (elide & 1));
            if (!skip) v += round16(stored_bytes(S.c_type[c0 + i], S.c_len[c0 + i]));
        }
        v = warp_sum(v);
        if (lane == 0) {
            bytes[b] = v;
            cnts[b] = nc;
        }
    }
}

// single CTA: exclusive scan of per-bitmap payload bytes, and of container counts when cnts is given
// (n+1 outputs each: the last entry is the total)
__global__ void __launch_bounds__(1024)
k_pack_scan(const uint64_t *__restrict__ bytes, const uint32_t *__restrict__ cnts, uint32_t n,
            uint64_t *__restrict__ off_out, uint64_t *__restrict__ beg_out) {
    __shared__ unsigned long long s_w[32];
    unsigned long long carry_b = 0, carry_c = 0;
    for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        unsigned long long tot;
        const unsigned long long eb = carry_b + block_excl_scan<1024>(i < n ? bytes[i] : 0ull, s_w, &tot);
        if (i < n) off_out[i] = eb;
        carry_b += tot;
        if (cnts) {
            const unsigned long long ec = carry_c + block_excl_scan<1024>(i < n ? (unsigned long long)cnts[i] : 0ull, s_w, &tot);
            if (i < n) beg_out[i] = ec;
            carry_c += tot;
        }
    }
    if (threadIdx.x == 0) {
        off_out[n] = carry_b;
        if (cnts) beg_out[n] = carry_c;
    }
}

__global__ void __launch_bounds__(128)
k_pack_copy(SetView S, uint32_t n, int elide, const uint64_t *__restrict__ off_in,
            const uint64_t *__restrict__ beg_in, SetOut out) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t b = warp; b < n; b += nwarps) {
        const uint32_t c0 = S.bm_beg[b], nc = S.bm_cnt[b];
        const uint64_t nb = beg_in[b];
        uint64_t run = off_in[b];
        unsigned long long card = 0;
        for (uint32_t i0 = 0; i0 < nc; i0 += 32) {
            const uint32_t i = i0 + lane;
            uint32_t sz = 0, t = 0, len = 0, cd = 0, src = SRC_NONE;
            uint64_t soff = 0;
            if (i < nc) {
                t = S.c_type[c0 + i];
                len = S.c_len[c0 + i];
                cd = S.c_card[c0 + i];
                soff = S.c_off[c0 + i];
                src = elide ? S.c_src[c0 + i] : SRC_NONE;
                const bool skip = src != SRC_NONE && ((src & SRC_B) ? (elide & 2) : (elide & 1));
                if (!skip) src = SRC_NONE;  // payload travels: the host needs no provenance
                sz = skip ? 0u : round16(stored_bytes(t, len));
            }
            const uint32_t incl = warp_incl_scan(sz, lane);
            const uint64_t doff = run + incl - sz;
            if (i < nc) {
                out.c_key[nb + i] = S.c_key[c0 + i];
                out.c_type[nb + i] = (uint8_t)t;
                out.c_card[nb + i] = cd;
                out.c_len[nb + i] = len;
                out.c_off[nb + i] = doff;
                out.c_src[nb + i] = src;
                card += cd;
            }
            // the warp copies the (up to 32) payloads one after the other
            const uint32_t m = nc - i0 < 32 ? nc - i0 : 32;
            for (uint32_t k = 0; k < m; k++) {
                const uint64_t so = __shfl_sync(FULLMASK, soff, k), d_o = __shfl_sync(FULLMASK, doff, k);
                const uint32_t bytes = __shfl_sync(FULLMASK, sz, k);
                if (bytes) warp_copy16(out.payload + d_o, S.payload + so, bytes, lane);
            }
            run += __shfl_sync(FULLMASK, incl, 31);
        }
        card = warp_sum(card);
        if (lane == 0) {
            out.bm_beg[b] = (uint32_t)nb;
            out.bm_cnt[b] = nc;
            out.bm_card[b] = card;
        }
    }
}

// ------------------------------------------------------------------------------ launchers
void launch_plan_pairs(const SetView &A, const SetView &B, const uint32_t *ia, const uint32_t *ib,
                       const uint64_t *item_off, uint32_t npairs, int op, bool card_only, int rules,
                       const PassShare &sh, Items it, OpStats *st, cudaStream_t s) {
    if (!npairs) return;
    launch_kernel_chained(k_plan_pairs, grid_for(npairs, 4, 16), 128, 0, s, A, B, ia, ib, item_off, npairs, op,
                          card_only, rules, sh, it, st);
}

void launch_order_items(Items it, uint64_t W, OpStats *st, cudaStream_t s) {
    if (!W || !it.desc_cls) return;
    launch_kernel_chained(k_order_items, grid_for(W, 2048, 8), 256, 0, s, it, W, st);
}

void launch_card_items(const SetView &A, const SetView &B, Items it, uint64_t W, OpStats *st,
                       cudaStream_t s) {
    if (!W) return;
    // tickets of 8 items, 4 warps per block
    launch_kernel(k_card_items, grid_for(W, 32, 5), 128, 0, s, A, B, it, W, st);
}

void launch_finalize_pairs(const SetView &A, const SetView &B, Items it, const uint64_t *item_off,
                           uint32_t npairs, const PassShare &sh, SetOut out, OpStats *st, OpStats *deliver,
                           cudaStream_t s) {
    if (!npairs) return;
    // a warp per pair, full residency (16 CTAs of 4 warps per SM); counters: one atomic per block
    launch_kernel_chained(k_finalize_pairs, grid_for(npairs, 4, RB200_FIN_BLOCKS), 128, 0, s, A, B, it, item_off,
                          npairs, sh.onA ? 0u : 2u, sh.onB ? 0u : 2u, out, st, deliver);
}

void launch_finalize_cards(Items it, const uint64_t *item_off, uint32_t npairs, uint64_t *out,
                           cudaStream_t s) {
    if (!npairs) return;
    launch_kernel(k_finalize_cards, grid_for(npairs, 4, 16), 128, 0, s, it, item_off, npairs, out);
}

void launch_sum_cardinalities(const uint64_t *bm_card, uint32_t n, uint64_t *d_acc, cudaStream_t s) {
    if (!n) return;
    const uint32_t blocks = (n + 255) / 256 < 592u ? (n + 255) / 256 : 592u;
    launch_kernel_chained(k_sum_cards, blocks, 256, 0, s, bm_card, n, (unsigned long long *)d_acc);
}
void launch_set_cardinalities(const SetView &S, uint32_t n, uint64_t *out, cudaStream_t s) {
    if (!n) return;
    launch_kernel(k_set_cardinalities, grid_for(n, 4, 16), 128, 0, s, S, n, out);
}

void launch_many_mark(const SetView &S, const uint32_t *idx, uint32_t n, uint32_t key_lo,
                      uint32_t key_hi, uint32_t *flags, cudaStream_t s) {
    cudaMemsetAsync(flags, 0, 65536 * sizeof(uint32_t), s);
    if (!n) return;
    launch_kernel(k_many_mark, grid_for(n, 1, 8), 128, 0, s, S, idx, n, key_lo, key_hi, flags);
}

void launch_many_compact(const uint32_t *flags, uint16_t *keys_out, OpStats *st, cudaStream_t s) {
    launch_kernel(k_many_compact, 1, 1024, 0, s, flags, keys_out, st);
}

void launch_pack(const SetView &S, uint32_t n, int elide, uint64_t *bytes, uint32_t *cnts, uint64_t *off,
                 uint64_t *beg, cudaStream_t s) {
    launch_kernel(k_pack_measure, grid_for(n, 4, 16), 128, 0, s, S, n, elide, bytes, cnts);
    launch_pack_scan(bytes, cnts, n, off, beg, s);
}
void launch_pack_copy(const SetView &S, uint32_t n, int elide, const uint64_t *off, const uint64_t *beg,
                      SetOut out, cudaStream_t s) {
    if (!n) return;
    launch_kernel(k_pack_copy, grid_for(n, 4, 16), 128, 0, s, S, n, elide, off, beg, out);
}
void launch_pack_scan(const uint64_t *bytes, const uint32_t *cnts, uint32_t n, uint64_t *off,
                      uint64_t *beg, cudaStream_t s) {
    launch_kernel(k_pack_scan, 1, 1024, 0, s, bytes, cnts, n, off, beg);
}
}  // namespace rb200

// ------------------------------------------------------------------------------ serialization
// Device-side roaring_bitmap_portable_serialize (src/roaring_array.c:469-531): every bitmap of a
// set becomes its portable byte string inside one device buffer (blob starts 16-byte aligned),
// so results can leave the device as bytes — one D2H, no per-container host allocation.
namespace rb200 {

__global__ void __launch_bounds__(128)
k_ser_measure(SetView S, uint32_t n, uint64_t *__restrict__ sizes16, uint32_t *__restrict__ exact,
              uint32_t *__restrict__ hasrun_out) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t b = warp; b < n; b += nwarps) {
        const uint32_t c0 = S.bm_beg[b], nc = S.bm_cnt[b];
        uint32_t bytes = 0, anyrun = 0;
        for (uint32_t i = lane; i < nc; i += 32) {
            const int t = S.c_type[c0 + i];
            bytes += portable_bytes(t, S.c_len[c0 + i]);
            anyrun |= (t == T_RUN) ? 1u : 0u;
        }
        bytes = __reduce_add_sync(FULLMASK, bytes);
        anyrun = __reduce_or_sync(FULLMASK, anyrun);
        if (lane == 0) {
            const uint32_t tot = portable_header_bytes(nc, anyrun != 0) + bytes;
            exact[b] = tot;
            sizes16[b] = (uint64_t)round16(tot);
            hasrun_out[b] = anyrun;
        }
    }
}

// byte-granular warp copy: src 4-byte aligned or not, dst arbitrary
__device__ __forceinline__ void warp_copy_unaligned(uint8_t *dst, const uint8_t *src, uint32_t n, int lane) {
    uint32_t head = (uint32_t)((4u - (uint32_t)(reinterpret_cast<uintptr_t>(dst) & 3u)) & 3u);
    if (head > n) head = n;
    if ((uint32_t)lane < head) dst[lane] = src[lane];
    uint8_t *d = dst + head;
    const uint8_t *s = src + head;
    const uint32_t m = n - head, words = m >> 2;
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(s) & 3u) * 8u;
    const uint32_t *sa = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(s) & ~(uintptr_t)3);
    uint32_t *dw = reinterpret_cast<uint32_t *>(d);
    if (sh == 0) {
        for (uint32_t w = lane; w < words; w += 32) dw[w] = sa[w];
    } else {
        for (uint32_t w = lane; w < words; w += 32) dw[w] = __funnelshift_r(sa[w], sa[w + 1], sh);
    }
    const uint32_t tail = m & 3u;
    if ((uint32_t)lane < tail) d[4 * words + lane] = s[4 * words + lane];
}

__device__ __forceinline__ void store_u16(uint8_t *p, uint32_t v) {
    p[0] = (uint8_t)v;
    p[1] = (uint8_t)(v >> 8);
}
__device__ __forceinline__ void store_u32(uint8_t *p, uint32_t v) {
    p[0] = (uint8_t)v;
    p[1] = (uint8_t)(v >> 8);
    p[2] = (uint8_t)(v >> 16);
    p[3] = (uint8_t)(v >> 24);
}

__global__ void __launch_bounds__(128)
k_ser_write(SetView S, uint32_t n, const uint64_t *__restrict__ off, const uint32_t *__restrict__ hasrun_in,
            uint8_t *__restrict__ dst) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t b = warp; b < n; b += nwarps) {
        const uint32_t c0 = S.bm_beg[b], nc = S.bm_cnt[b];
        const bool hasrun = hasrun_in[b] != 0;
        uint8_t *o = dst + off[b];
        const uint32_t hdr = portable_header_bytes(nc, hasrun);
        uint8_t *kc, *offs = nullptr;
        if (hasrun) {
            if (lane == 0) store_u32(o, SERIAL_COOKIE | ((nc - 1) << 16));
            const uint32_t nfb = (nc + 7) >> 3;
            for (uint32_t j = lane; j < nfb; j += 32) {
                uint32_t byte = 0;
                for (uint32_t k = 0; k < 8 && 8 * j + k < nc; k++)
                    byte |= (S.c_type[c0 + 8 * j + k] == T_RUN ? 1u : 0u) << k;
                o[4 + j] = (uint8_t)byte;
            }
            kc = o + 4 + nfb;
            if (nc >= NO_OFFSET_THRESHOLD) offs = kc + 4 * nc;
        } else {
            if (lane == 0) { store_u32(o, SERIAL_COOKIE_NO_RUN); store_u32(o + 4, nc); }
            kc = o + 8;
            offs = kc + 4 * nc;
        }
        uint32_t run = hdr;
        for (uint32_t i0 = 0; i0 < nc; i0 += 32) {
            const uint32_t i = i0 + lane;
            uint32_t sz = 0, t = 0, len = 0;
            uint64_t soff = 0;
            if (i < nc) {
                t = S.c_type[c0 + i];
                len = S.c_len[c0 + i];
                soff = S.c_off[c0 + i];
                sz = portable_bytes(t, len);
                store_u16(kc + 4 * i, S.c_key[c0 + i]);
                store_u16(kc + 4 * i + 2, S.c_card[c0 + i] - 1);
            }
            const uint32_t incl = warp_incl_scan(sz, lane);
            const uint32_t doff = run + incl - sz;
            if (i < nc && offs) store_u32(offs + 4 * i, doff);
            const uint32_t m = nc - i0 < 32 ? nc - i0 : 32;
            for (uint32_t k = 0; k < m; k++) {
                const uint64_t so = __shfl_sync(FULLMASK, soff, k);
                const uint32_t d_o = __shfl_sync(FULLMASK, doff, k);
                const uint32_t tt = __shfl_sync(FULLMASK, t, k), ll = __shfl_sync(FULLMASK, len, k);
                uint8_t *pd = o + d_o;
                if (tt == T_RUN) {
                    if (lane == 0) store_u16(pd, ll);
                    warp_copy_unaligned(pd + 2, S.payload + so, 4 * ll, lane);
                } else {
                    warp_copy_unaligned(pd, S.payload + so, tt == T_BITSET ? (uint32_t)BITSET_BYTES : 2 * ll, lane);
                }
            }
            run += __shfl_sync(FULLMASK, incl, 31);
        }
    }
}

// ---- 64-bit portable format (src/roaring64.c:2262-2395): a u64 bucket count, then per bucket its
// u32 high 32 bits and the 32-bit portable blob of its low halves.  The buckets are the bitmaps of an
// inner set (k_ser_measure gives their exact sizes, k_ser_write writes them at boff); empty buckets
// are not emitted, as the reference never holds one.  Warp per 64-bit bitmap.
__global__ void __launch_bounds__(128)
k_r64_ser_sizes(const uint32_t *__restrict__ b_beg, const uint32_t *__restrict__ b_cnt, uint32_t n,
                const uint32_t *__restrict__ bm_cnt, const uint32_t *__restrict__ exact,
                uint64_t *__restrict__ sizes16, uint64_t *__restrict__ exact64) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = warp; i < n; i += nwarps) {
        const uint32_t j0 = b_beg[i], c = b_cnt[i];
        unsigned long long sum = 0;
        for (uint32_t k = lane; k < c; k += 32)
            if (bm_cnt[j0 + k]) sum += 4ull + exact[j0 + k];
        sum = warp_sum(sum);
        if (lane == 0) {
            exact64[i] = 8 + sum;
            sizes16[i] = (8 + sum + 15) & ~15ull;
        }
    }
}

__global__ void __launch_bounds__(128)
k_r64_ser_layout(const uint32_t *__restrict__ b_beg, const uint32_t *__restrict__ b_cnt,
                 const uint32_t *__restrict__ high, uint32_t n, uint32_t nbuckets, const uint32_t *__restrict__ bm_cnt,
                 const uint32_t *__restrict__ exact, const uint64_t *__restrict__ off, uint64_t *__restrict__ boff,
                 uint8_t *__restrict__ dst) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    const uint64_t scratch = off[n];
    // the inner set's last bitmap is its empty sentinel, in no 64-bit bitmap
    if (blockIdx.x == 0 && threadIdx.x == 0 && nbuckets) boff[nbuckets - 1] = scratch;
    for (uint32_t i = warp; i < n; i += nwarps) {
        const uint32_t j0 = b_beg[i], c = b_cnt[i];
        const uint64_t o = off[i];
        uint64_t run = o + 8;
        uint32_t kept = 0;
        for (uint32_t k0 = 0; k0 < c; k0 += 32) {
            const uint32_t j = j0 + k0 + lane;
            const bool in = k0 + lane < c, live = in && bm_cnt[j] != 0;
            const unsigned long long sz = live ? 4ull + exact[j] : 0ull;
            const unsigned long long incl = warp_incl_scan(sz, lane);
            const uint64_t pos = run + incl - sz;
            if (live) {
                store_u32(dst + pos, high[j]);
                boff[j] = pos + 4;
            } else if (in) {
                boff[j] = scratch;
            }
            kept += __popc(__ballot_sync(FULLMASK, live));
            run += __shfl_sync(FULLMASK, incl, 31);
        }
        if (lane == 0) *reinterpret_cast<unsigned long long *>(dst + o) = kept;   // blob starts are 16-byte aligned
    }
}

void launch_r64_ser_sizes(const uint32_t *b_beg, const uint32_t *b_cnt, uint32_t n, const uint32_t *bm_cnt,
                          const uint32_t *exact, uint64_t *sizes16, uint64_t *exact64, cudaStream_t s) {
    if (!n) return;
    launch_kernel(k_r64_ser_sizes, grid_for(n, 4, 16), 128, 0, s, b_beg, b_cnt, n, bm_cnt, exact, sizes16, exact64);
}
void launch_r64_ser_layout(const uint32_t *b_beg, const uint32_t *b_cnt, const uint32_t *high, uint32_t n,
                           uint32_t nbuckets, const uint32_t *bm_cnt, const uint32_t *exact, const uint64_t *off,
                           uint64_t *boff, uint8_t *dst, cudaStream_t s) {
    launch_kernel(k_r64_ser_layout, grid_for(n, 4, 16), 128, 0, s, b_beg, b_cnt, high, n, nbuckets, bm_cnt, exact, off,
                  boff, dst);
}

void launch_serialize_measure(const SetView &S, uint32_t n, uint64_t *sizes16, uint32_t *exact,
                              uint32_t *hasrun, cudaStream_t s) {
    if (!n) return;
    launch_kernel(k_ser_measure, grid_for(n, 4, 16), 128, 0, s, S, n, sizes16, exact, hasrun);
}
void launch_serialize_write(const SetView &S, uint32_t n, const uint64_t *off, const uint32_t *hasrun,
                            uint8_t *dst, cudaStream_t s) {
    if (!n) return;
    launch_kernel(k_ser_write, grid_for(n, 4, 16), 128, 0, s, S, n, off, hasrun, dst);
}
}  // namespace rb200

// ------------------------------------------------------------------------------ deserialization
// roaring_bitmap_portable_deserialize_safe (src/roaring_array.c:633-813) of every blob of a batch,
// on the device: the raw bytes arrive in one staging buffer (blob b at raw + roff[b], 16-byte
// aligned); k_deser_dir walks the headers (warp per bitmap) and fills the directory, k_deser_copy
// moves the payloads into the 16-byte aligned slab (warp per container) and counts run cardinalities.
namespace rb200 {

__device__ __forceinline__ uint32_t ld_u16(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
__device__ __forceinline__ uint32_t ld_u32(const uint8_t *p) { return ld_u16(p) | (ld_u16(p + 2) << 16); }

// Do the keys of this chunk of (up to) 32 containers, one per lane, strictly increase, also from
// prev_key, the last key of the previous chunk (-1 before the first)?  (roaring.c:496-503)
// Advances prev_key to the chunk's last key.
__device__ __forceinline__ bool keys_increase(uint32_t key, bool valid, int &prev_key, int lane) {
    int left = __shfl_up_sync(FULLMASK, (int)key, 1);
    if (lane == 0) left = prev_key;
    if (__any_sync(FULLMASK, valid && (int)key <= left)) return false;
    prev_key = __shfl_sync(FULLMASK, (int)key, 31);
    return true;
}

// blob b of nb is malformed: error 3; the host names the first such blob, nb - st->nk
__device__ __forceinline__ void report_malformed(OpStats *st, uint32_t nb, uint32_t b) {
    atomicExch(&st->error, 3u);
    atomicMax(&st->nk, nb - b);
}

__global__ void __launch_bounds__(128)
k_deser_dir(const uint8_t *__restrict__ raw, const uint64_t *__restrict__ roff,
            const uint64_t *__restrict__ rlen, const uint64_t *__restrict__ slab_base, uint32_t nb,
            SetOut out, uint64_t *__restrict__ src_pos, OpStats *st) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t b = warp; b < nb; b += nwarps) {
        const uint8_t *buf = raw + roff[b];
        const uint64_t len = rlen[b];
        const uint32_t c0 = out.bm_beg[b], want = out.bm_cnt[b];  // filled by the host from the cookies
        bool bad = len < 4;
        uint32_t size = 0;
        uint64_t pos = 4;
        bool hasrun = false;
        const uint8_t *runflags = nullptr;
        if (!bad) {
            const uint32_t cookie = ld_u32(buf);
            if ((cookie & 0xFFFFu) == SERIAL_COOKIE) {
                size = (cookie >> 16) + 1;
                hasrun = true;
                runflags = buf + 4;
                pos = 4 + ((size + 7) >> 3);
            } else if (cookie == SERIAL_COOKIE_NO_RUN && len >= 8) {
                size = ld_u32(buf + 4);
                pos = 8;
            } else {
                bad = true;
            }
        }
        if (!bad && (size != want || size > 65536u || pos + 4ull * size > len)) bad = true;
        const uint8_t *kc = buf + pos;
        if (!bad) {
            pos += 4ull * size;
            if (!hasrun || size >= NO_OFFSET_THRESHOLD) pos += 4ull * size;   // offset header, not trusted
        }
        uint64_t off = slab_base[b];
        int prev_key = -1;
        for (uint32_t chunk = 0; chunk < size && !bad; chunk += 32) {
            const uint32_t i = chunk + lane;
            const bool valid = i < size;
            uint32_t key = 0, card = 0, known = 0;
            bool isrun = false;
            if (valid) {
                key = ld_u16(kc + 4 * i);
                card = ld_u16(kc + 4 * i + 2) + 1;
                isrun = hasrun && ((runflags[i >> 3] >> (i & 7)) & 1);
                known = isrun ? 0u : (card > (uint32_t)MAX_ARRAY ? (uint32_t)BITSET_BYTES : 2u * card);
            }
            if (!keys_increase(key, valid, prev_key, lane)) { bad = true; break; }
            // sequential walk over the chunk: a run container's size is in its first two bytes
            uint64_t mypos = 0;
            uint32_t mylen = 0, mystored = 0;
            const uint32_t cnt = size - chunk < 32u ? size - chunk : 32u;
            for (uint32_t j = 0; j < cnt; j++) {
                const bool isr = __shfl_sync(FULLMASK, isrun ? 1 : 0, j) != 0;
                uint32_t sz = __shfl_sync(FULLMASK, known, j), nr = 0, skip = 0;
                if (isr) {
                    if (pos + 2 > len) { bad = true; break; }
                    nr = ld_u16(buf + pos);
                    sz = 2u + 4u * nr;
                    skip = 2;
                }
                if (pos + sz > len) { bad = true; break; }
                if (lane == (int)j) { mypos = pos + skip; mylen = isr ? nr : 0u; mystored = sz - skip; }
                pos += sz;
            }
            if (bad) break;
            const uint32_t r16 = valid ? round16(mystored) : 0u;
            const uint32_t incl = warp_incl_scan(r16, lane);
            if (valid) {
                const uint64_t c = (uint64_t)c0 + i;
                const int t = isrun ? T_RUN : (card > (uint32_t)MAX_ARRAY ? T_BITSET : T_ARRAY);
                out.c_key[c] = (uint16_t)key;
                out.c_type[c] = (uint8_t)t;
                out.c_card[c] = card;                      // runs: recounted by k_deser_copy
                out.c_len[c] = t == T_BITSET ? 1024u : (t == T_ARRAY ? card : mylen);
                out.c_off[c] = off + incl - r16;
                out.c_src[c] = SRC_NONE;
                src_pos[c] = roff[b] + mypos;
            }
            off += __shfl_sync(FULLMASK, incl, 31);
        }
        if (bad && lane == 0) report_malformed(st, nb, b);
    }
}

// The bitmap of nb that holds directory entry c: the last b with bm_beg[b] <= c (empty bitmaps share
// their bm_beg with the next one, so the last such b is the one that owns c).
__device__ __forceinline__ uint32_t bitmap_of(const uint32_t *__restrict__ bm_beg, uint32_t nb, uint64_t c) {
    uint32_t lo = 0, hi = nb;   // bm_beg[lo] <= c < bm_beg[hi]
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (bm_beg[mid] <= c) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(128)
k_deser_copy(const uint8_t *__restrict__ raw, const uint64_t *__restrict__ src_pos, uint64_t nc, uint32_t nb,
             SetOut out, OpStats *st) {
    if (st->error == 3u) return;  // a malformed blob leaves directory entries unwritten: nothing to move
    const int lane = threadIdx.x & 31;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t c = warp; c < nc; c += nwarps) {
        const int t = out.c_type[c];
        const uint32_t len = out.c_len[c];
        const uint32_t n = stored_bytes(t, len);
        uint8_t *dst = out.payload + out.c_off[c];
        const uint8_t *src = raw + src_pos[c];
        warp_copy_unaligned(dst, src, n, lane);
        const uint32_t pad = round16(n) - n;
        if ((uint32_t)lane < pad) dst[n + lane] = 0;
        // Container CONTENTS of an untrusted blob: what roaring_bitmap_internal_validate checks of each
        // container (src/containers/run.c:669-713, array.c:456-487, bitset.c:1023-1042), so the device
        // holds exactly the containers the reference's validator accepts.  The kernels rasterise runs
        // and index by array values without further checks, and take c_card as exact (prefix sums,
        // select, slot bounds, the type rules): nothing else may reach them.
        bool bad = false;
        if (t == T_RUN) {  // run_container_cardinality (run.c:1077) + bounds / order of the runs
            uint32_t card = 0;
            bad = len == 0;
            for (uint32_t k = lane; k < len; k += 32) {
                const uint32_t s0 = ld_u16(src + 4 * k), l0 = ld_u16(src + 4 * k + 2);
                card += l0 + 1u;
                if (s0 + l0 > 65535u) bad = true;
                // after the previous run's end + 1: neither overlapping nor adjacent (those combine)
                if (k > 0 && s0 <= ld_u16(src + 4 * k - 4) + ld_u16(src + 4 * k - 2) + 1u) bad = true;
            }
            card = __reduce_add_sync(FULLMASK, card);
            if (lane == 0) out.c_card[c] = card;
        } else if (t == T_ARRAY) {  // at most 4096 (only a frozen blob can say more) strictly increasing values
            bad = len > (uint32_t)MAX_ARRAY;
            for (uint32_t k = lane + 1; k < len && !bad; k += 32)
                if (ld_u16(src + 2 * k) <= ld_u16(src + 2 * k - 2)) bad = true;
        } else {  // the header's cardinality is the popcount, and above 4096 (a frozen blob may say less)
            __syncwarp();
            const uint64_t *w = (const uint64_t *)dst;
            uint32_t pop = 0;
            for (uint32_t k = lane; k < 1024u; k += 32) pop += __popcll(w[k]);
            pop = __reduce_add_sync(FULLMASK, pop);
            const uint32_t card = out.c_card[c];
            bad = pop != card || card <= (uint32_t)MAX_ARRAY;
        }
        if (__any_sync(FULLMASK, bad) && lane == 0) {  // error 4, and the first such blob as report_malformed names it
            atomicCAS(&st->error, 0u, 4u);
            atomicMax(&st->nk, nb - bitmap_of(out.bm_beg, nb, c));
        }
    }
}

__global__ void k_deser_bitmap_cards(SetOut out, uint32_t nb, const OpStats *st) {
    if (st->error == 3u) return;
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t b = warp; b < nb; b += nwarps) {
        const uint32_t c0 = out.bm_beg[b], n = out.bm_cnt[b];
        unsigned long long card = 0, sbytes = 0, ebytes = 0;
        for (uint32_t i = lane; i < n; i += 32) {
            card += out.c_card[c0 + i];
            sbytes += round16(stored_bytes(out.c_type[c0 + i], out.c_len[c0 + i]));
            ebytes += effective_bytes(out.c_type[c0 + i], out.c_len[c0 + i], out.c_card[c0 + i]);
        }
        card = warp_sum(card);
        sbytes = warp_sum(sbytes);
        ebytes = warp_sum(ebytes);
        if (lane == 0) { out.bm_card[b] = card; out.bm_bytes[b] = sbytes; out.bm_ebytes[b] = ebytes; }
    }
}

// ------------------------------------------------------------------------------ frozen format
// roaring_bitmap_frozen_serialize / roaring_bitmap_frozen_view (src/roaring.c:3180-3456): zones
// [bitset words | runs | array values | keys u16 | counts u16 | typecodes u8 | header u32], the
// header LAST: (n_containers << 15) | FROZEN_COOKIE.  counts = cardinality-1 (bitset, array) or
// n_runs (run).  Blob starts are 32-byte aligned so frozen_view accepts them in place.

// Write cursors of the three payload zones of one blob, zb bytes of bitset words then zr bytes of
// runs then the array values, advanced by a warp over its containers a chunk of 32 at a time.
struct FrozenZones {
    unsigned long long pb, pr, pa;
    __device__ FrozenZones(unsigned long long zb, unsigned long long zr) : pb(0), pr(zb), pa(zb + zr) {}
    // offset of this lane's container (type t, sz payload bytes; sz = 0 past the end) in the zones
    __device__ __forceinline__ unsigned long long next(int t, uint32_t sz, int lane) {
        const uint32_t sb = t == T_BITSET ? sz : 0u, sr = t == T_RUN ? sz : 0u, sa = t == T_ARRAY ? sz : 0u;
        const uint32_t ib = warp_incl_scan(sb, lane), ir = warp_incl_scan(sr, lane), ia = warp_incl_scan(sa, lane);
        const unsigned long long d = t == T_BITSET ? pb + ib - sb : (t == T_RUN ? pr + ir - sr : pa + ia - sa);
        pb += __shfl_sync(FULLMASK, ib, 31);
        pr += __shfl_sync(FULLMASK, ir, 31);
        pa += __shfl_sync(FULLMASK, ia, 31);
        return d;
    }
};

__global__ void __launch_bounds__(128)
k_frozen_measure(SetView S, uint32_t n, uint64_t *__restrict__ sizes32, uint32_t *__restrict__ exact,
                 uint32_t *__restrict__ cnt_out) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t b = warp; b < n; b += nwarps) {
        const uint32_t c0 = S.bm_beg[b], nc = S.bm_cnt[b];
        unsigned long long bytes = 0;
        for (uint32_t i = lane; i < nc; i += 32) bytes += stored_bytes(S.c_type[c0 + i], S.c_len[c0 + i]);
        bytes = warp_sum(bytes);
        if (lane == 0) {
            const unsigned long long tot = bytes + 5ull * nc + 4ull;
            exact[b] = (uint32_t)tot;
            sizes32[b] = (tot + 31ull) & ~31ull;
            cnt_out[b] = nc;
        }
    }
}

__global__ void __launch_bounds__(128)
k_frozen_dir(SetView S, uint32_t n, const uint64_t *__restrict__ off, uint8_t *__restrict__ dst,
             uint64_t *__restrict__ c_dst) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t b = warp; b < n; b += nwarps) {
        const uint32_t c0 = S.bm_beg[b], nc = S.bm_cnt[b];
        unsigned long long zb = 0, zr = 0, za = 0;
        for (uint32_t i = lane; i < nc; i += 32) {
            const int t = S.c_type[c0 + i];
            const uint32_t sz = stored_bytes(t, S.c_len[c0 + i]);
            if (t == T_BITSET) zb += sz; else if (t == T_RUN) zr += sz; else za += sz;
        }
        zb = warp_sum(zb);
        zr = warp_sum(zr);
        za = warp_sum(za);
        uint8_t *base = dst + off[b];
        const unsigned long long k0 = zb + zr + za, n0 = k0 + 2ull * nc, t0 = n0 + 2ull * nc, h0 = t0 + nc;
        FrozenZones z(zb, zr);
        for (uint32_t chunk = 0; chunk < nc; chunk += 32) {
            const uint32_t i = chunk + lane;
            const bool valid = i < nc;
            int t = 0;
            uint32_t sz = 0, card = 0, len = 0;
            if (valid) {
                t = S.c_type[c0 + i];
                len = S.c_len[c0 + i];
                card = S.c_card[c0 + i] & CARD_MASK;
                sz = stored_bytes(t, len);
            }
            const unsigned long long d = z.next(t, sz, lane);
            if (valid) {
                c_dst[c0 + i] = off[b] + d;
                store_u16(base + k0 + 2ull * i, S.c_key[c0 + i]);
                store_u16(base + n0 + 2ull * i, t == T_RUN ? len : card - 1u);
                base[t0 + i] = (uint8_t)t;
            }
        }
        if (lane == 0) store_u32(base + h0, (nc << 15) | FROZEN_COOKIE);
    }
}

__global__ void __launch_bounds__(128)
k_frozen_copy(SetView S, uint64_t nc, const uint64_t *__restrict__ c_dst, uint8_t *__restrict__ dst) {
    const int lane = threadIdx.x & 31;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t c = warp; c < nc; c += nwarps)
        warp_copy_unaligned(dst + c_dst[c], S.payload + S.c_off[c], stored_bytes(S.c_type[c], S.c_len[c]), lane);
}

void launch_frozen_measure(const SetView &S, uint32_t n, uint64_t *sizes32, uint32_t *exact, uint32_t *cnt,
                           cudaStream_t s) {
    if (!n) return;
    launch_kernel(k_frozen_measure, grid_for(n, 4, 16), 128, 0, s, S, n, sizes32, exact, cnt);
}
void launch_frozen_write(const SetView &S, uint32_t n, uint64_t nc, const uint64_t *off, uint8_t *dst,
                         uint64_t *c_dst, cudaStream_t s) {
    if (!n) return;
    launch_kernel(k_frozen_dir, grid_for(n, 4, 16), 128, 0, s, S, n, off, dst, c_dst);
    if (nc) launch_kernel(k_frozen_copy, grid_for(nc, 4, 16), 128, 0, s, S, nc, c_dst, dst);
}

// frozen blobs -> directory (the zones make every payload offset a prefix sum: no sequential walk)
__global__ void __launch_bounds__(128)
k_frozen_parse_dir(const uint8_t *__restrict__ raw, const uint64_t *__restrict__ roff,
                   const uint64_t *__restrict__ rlen, const uint64_t *__restrict__ slab_base, uint32_t nb,
                   SetOut out, uint64_t *__restrict__ src_pos, OpStats *st) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t b = warp; b < nb; b += nwarps) {
        const uint8_t *buf = raw + roff[b];
        const uint64_t len = rlen[b];
        const uint32_t c0 = out.bm_beg[b], want = out.bm_cnt[b];
        bool bad = len < 4;
        uint32_t nc = 0;
        if (!bad) {
            const uint32_t header = ld_u32(buf + len - 4);
            nc = header >> 15;
            bad = (header & 0x7FFFu) != FROZEN_COOKIE || nc != want || len < 4ull + 5ull * nc;
        }
        const uint8_t *tz = buf + len - 4 - nc, *nz = tz - 2ull * nc, *kz = nz - 2ull * nc;
        unsigned long long zb = 0, zr = 0, za = 0;
        if (!bad) {
            for (uint32_t i = lane; i < nc; i += 32) {
                const int t = tz[i];
                const uint32_t cnt = ld_u16(nz + 2ull * i);
                if (t == T_BITSET) zb += BITSET_BYTES;
                else if (t == T_RUN) zr += 4ull * cnt;
                else if (t == T_ARRAY) za += 2ull * (cnt + 1);
                else bad = true;
            }
            bad = __any_sync(FULLMASK, bad);
            zb = warp_sum(zb);
            zr = warp_sum(zr);
            za = warp_sum(za);
            if (zb + zr + za + 5ull * nc + 4ull != len) bad = true;   // roaring.c:3425-3429 exact length
        }
        FrozenZones z(zb, zr);
        unsigned long long off = slab_base[b];
        int prev_key = -1;
        for (uint32_t chunk = 0; chunk < nc && !bad; chunk += 32) {
            const uint32_t i = chunk + lane;
            const bool valid = i < nc;
            int t = 0;
            uint32_t key = 0, cnt = 0, sz = 0;
            if (valid) {
                t = tz[i];
                key = ld_u16(kz + 2ull * i);
                cnt = ld_u16(nz + 2ull * i);
                sz = t == T_BITSET ? (uint32_t)BITSET_BYTES : (t == T_RUN ? 4u * cnt : 2u * (cnt + 1u));
            }
            if (!keys_increase(key, valid, prev_key, lane)) { bad = true; break; }
            const unsigned long long d = z.next(t, sz, lane);
            const uint32_t r16 = valid ? round16(sz) : 0u;
            const uint32_t incl = warp_incl_scan(r16, lane);
            if (valid) {
                const uint64_t c = (uint64_t)c0 + i;
                out.c_key[c] = (uint16_t)key;
                out.c_type[c] = (uint8_t)t;
                out.c_card[c] = cnt + 1u;                    // runs: recounted by k_deser_copy
                out.c_len[c] = t == T_BITSET ? 1024u : (t == T_ARRAY ? cnt + 1u : cnt);
                out.c_off[c] = off + incl - r16;
                out.c_src[c] = SRC_NONE;
                src_pos[c] = roff[b] + d;
            }
            off += __shfl_sync(FULLMASK, incl, 31);
        }
        if (bad && lane == 0) report_malformed(st, nb, b);
    }
}

// the directory parse (k_deser_dir / k_frozen_parse_dir), then the payload moves and the bitmap figures
static void deserialize_tail(const uint8_t *raw, uint32_t nb, uint64_t nc, SetOut out, uint64_t *src_pos, OpStats *st,
                             cudaStream_t s) {
    if (nc) launch_kernel(k_deser_copy, grid_for(nc, 4, 16), 128, 0, s, raw, src_pos, nc, nb, out, st);
    launch_kernel(k_deser_bitmap_cards, grid_for(nb, 4, 16), 128, 0, s, out, nb, st);
}

void launch_deserialize_frozen(const uint8_t *raw, const uint64_t *roff, const uint64_t *rlen,
                               const uint64_t *slab_base, uint32_t nb, uint64_t nc, SetOut out,
                               uint64_t *src_pos, OpStats *st, cudaStream_t s) {
    if (!nb) return;
    launch_kernel(k_frozen_parse_dir, grid_for(nb, 4, 16), 128, 0, s, raw, roff, rlen, slab_base, nb, out, src_pos, st);
    deserialize_tail(raw, nb, nc, out, src_pos, st, s);
}

void launch_deserialize(const uint8_t *raw, const uint64_t *roff, const uint64_t *rlen,
                        const uint64_t *slab_base, uint32_t nb, uint64_t nc, SetOut out,
                        uint64_t *src_pos, OpStats *st, cudaStream_t s) {
    if (!nb) return;
    launch_kernel(k_deser_dir, grid_for(nb, 4, 16), 128, 0, s, raw, roff, rlen, slab_base, nb, out, src_pos, st);
    deserialize_tail(raw, nb, nc, out, src_pos, st, s);
}

void launch_bitmap_figures(SetOut out, uint32_t nb, const OpStats *st, cudaStream_t s) {
    if (!nb) return;
    launch_kernel(k_deser_bitmap_cards, grid_for(nb, 4, 16), 128, 0, s, out, nb, st);
}
}  // namespace rb200
