// rb200_kernels.cu — sm_90a kernels of the Roaring set-algebra hot path.
//
//   k_plan_pairs      warp per bitmap pair: key merge by binary-search ranks (the reference's
//                     two-pointer loops, src/roaring.c:742-768, 896-951) -> work items.
//   k_compute_items   warp per work item: one container x container grid cell
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

static inline int sm_count() {
    static int n = 0;
    if (!n) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

__device__ __forceinline__ uint32_t lower_bound_u16(const uint16_t *a, uint32_t n, uint32_t key) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (a[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ uint32_t upper_bound_u16(const uint16_t *a, uint32_t n, uint32_t key) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (a[mid] <= key) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

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
__global__ void __launch_bounds__(128)
k_plan_pairs(SetView A, SetView B, const uint32_t *__restrict__ ia,
             const uint32_t *__restrict__ ib, const uint64_t *__restrict__ item_off,
             uint32_t npairs, int op, bool card_only, int rules, Items it, OpStats *st) {
    __shared__ unsigned int s_cls[N_CLS];   // live items per class of this block (one global atomic per class at the end)
    // the four pairs of a block reserve their result slots with ONE atomic per round (the slab cursor
    // is a single address: a returning atomic per pair serialised 19 900 of them per launch)
    __shared__ uint32_t s_tot[4];
    __shared__ unsigned long long s_base;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x < N_CLS) s_cls[threadIdx.x] = 0;
    __syncthreads();
    for (uint32_t p0 = blockIdx.x * 4; p0 < npairs; p0 += gridDim.x * 4) {
        const uint32_t p = p0 + wid;
        const bool vp = p < npairs;
        const uint32_t a = vp ? ia[p] : 0, b = vp ? ib[p] : 0;
        const uint32_t a0 = vp ? A.bm_beg[a] : 0, na = vp ? A.bm_cnt[a] : 0;
        const uint32_t b0 = vp ? B.bm_beg[b] : 0, nb = vp ? B.bm_cnt[b] : 0;
        const uint64_t base_item = vp ? item_off[p] : 0;
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
                            // in-place twins: a SHARED left container takes the functional cell (roaring.c:1085-1088);
                            // the lazy in-place twins work on a writable copy instead (roaring.c:2636)
                            d.shared = (rules & (RULES_INPLACE | RULES_LAZY)) == RULES_INPLACE && A.c_src[ca] == SRC_SHARED;
                            const uint32_t cA = d.cA & CARD_MASK;
                            cap = (rules & RULES_LAZY) ? slot_bound_lazy(d.tA, d.tB, cA, d.cB, d.lA, d.lB)
                                                       : slot_bound(op, d.tA, d.tB, cA, d.cB, d.lA, d.lB);
                            cls = cell_class(op, rules, d.tA, d.tB, cA, d.cB, d.lA, d.lB);
                        }
                    } else if (op != OP_AND && !card_only) {
                        kind = K_COPY_A;
                        cls = CLS_COPY;
                        d.tA = A.c_type[ca];
                        d.cA = A.c_card[ca];
                        d.lA = A.c_len[ca];
                        d.offA = A.c_off[ca];
                        cap = round16(stored_bytes(d.tA, d.lA));
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
                        cls = CLS_COPY;
                        d.tA = B.c_type[cb];
                        d.cA = B.c_card[cb];
                        d.lA = B.c_len[cb];
                        d.offA = B.c_off[cb];
                        cap = round16(stored_bytes(d.tA, d.lA));
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
            if (t < tot) {
                const uint64_t idx = base_item + pos;
                it.kind[idx] = (uint8_t)kind;
                it.key[idx] = (uint16_t)key;
                it.ca[idx] = ca;
                it.cb[idx] = cb;
                it.slot_off[idx] = slab_base + incl - cap;
                // the class-ordered list copies only live descriptors; without it the holes are read too
                if (it.desc && (kind != K_HOLE || !it.desc_cls)) {
                    d.off = slab_base + incl - cap;
                    d.cap = cap;
                    d.kind = kind;
                    d.item = (uint32_t)idx;
                    cd_pack(d, it.desc[2 * idx], it.desc[2 * idx + 1]);
                }
                if (it.cls) it.cls[idx] = (uint8_t)cls;
                it.otype[idx] = 0;
                it.ocard[idx] = 0;
                it.olen[idx] = 0;
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
    __syncthreads();
    if (it.cls && threadIdx.x < N_CLS && s_cls[threadIdx.x]) atomicAdd(&st->cls_count[threadIdx.x], s_cls[threadIdx.x]);
}

// descriptors of the live items grouped by class: desc_cls[prefix(class) + k].  A block takes chunks of 2048 item slots
// (256 per warp); per chunk ONE global atomic per class reserves the block's range, the ranks
// inside come from ballots and an 8-warp scan in shared memory.
__global__ void __launch_bounds__(256)
k_order_items(Items it, uint64_t W, OpStats *st) {
    __shared__ uint32_t s_wcnt[8][N_CLS], s_base[N_CLS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
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
}

// (the grid cells themselves — cell_compute — live in rb200_cells.cuh, shared with rb200_fused.cu)

#ifndef RB200_CI_MINBLOCKS
#define RB200_CI_MINBLOCKS 6   // resident CTAs per SM the register allocation is held to (6 = what the 36 KiB of shared memory allow)
#endif
#ifdef RB200_PROBE
// tuning aid (variant builds only, never the product): slowest item / warp of the last launch
__device__ unsigned long long g_probe[24];   // [8 + cls] clocks, [16 + cls] items of the class
extern "C" __attribute__((visibility("default"))) void rb200_debug_probe(unsigned long long *out) {
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out, g_probe, sizeof(g_probe));
    unsigned long long z[24] = {0, 0, ~0ull};
    cudaMemcpyToSymbol(g_probe, z, sizeof(z));
}
#endif
#ifndef RB200_CI_KMAX
#define RB200_CI_KMAX 1   // most cells one ticket claims (measured best: 1, one cell per atomic; DESIGN.md §6)
#endif
// cp.async of one 16-byte piece of a cell descriptor into the warp's shared slot
__device__ __forceinline__ void desc_prefetch(uint4 *slot, const uint4 *src, int lane) {
    if (lane < 2)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"((uint32_t)__cvta_generic_to_shared(slot + lane)),
                     "l"(src + lane) : "memory");
    asm volatile("cp.async.commit_group;\n" ::: "memory");
}
template <int OP, bool LAZY>
__global__ void __launch_bounds__(128, RB200_CI_MINBLOCKS)
k_compute_items(SetView A, SetView B, Items it, uint64_t W, uint8_t *slab,
                uint64_t slab_cap, OpStats *st, int rules, int copy_ticket) {
    __shared__ __align__(16) uint32_t s_acc[4][WARP_SMEM_WORDS];   // accumulator + merge window (rb200_device.cuh)
    __shared__ __align__(16) uint4 s_desc[4][2];                     // the descriptor of the warp's next cell
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t *acc = s_acc[wid];
    // Dynamic scheduling over units: cells [0, n_cells), then pass-through tickets [n_cells, T).
    // One atomic claims a chunk of consecutive cells whose size shrinks with what is left (guided
    // self-scheduling, at most RB200_CI_KMAX): the tail is handed out one cell at a time — four
    // consecutive heavy cells on one warp were the tail of every launch — and the work counter, a
    // single address, sees fewer atomics while the list is long.  A warp keeps one claim in flight and
    // fetches the descriptor of its next cell into shared memory while the current cell runs.
    // (small batches: no order list, the units are the items, holes included)
    // with an order list (big batches) the units walk the live items class by class
    // (tried: a lean kernel of its own for the pass-through class — 40 registers, no accumulator —
    //  launched behind this one: slower, the copies no longer overlap the cells)
    const uint4 *D = it.desc_cls ? it.desc_cls : it.desc;
    // (unit numbers are 32-bit: the host keeps W below 2^32; counter values past T are clamped to T)
    uint32_t n_cells = (uint32_t)W, T = (uint32_t)W;
    if (it.desc_cls) {
        uint32_t live = 0;
#pragma unroll
        for (int c = 0; c < N_CLS; c++) live += st->cls_count[c];
        W = live;
        n_cells = live - st->cls_count[CLS_COPY];
        T = n_cells + (st->cls_count[CLS_COPY] + copy_ticket - 1) / copy_ticket;
    }
    const uint32_t split = 2u * gridDim.x * (blockDim.x >> 5);
    // size of the chunk claimed when the counter was last seen at `seen`
    auto chunk = [&](uint32_t seen) -> uint32_t {
        const uint32_t k = seen < n_cells ? (n_cells - seen) / split : 0u;
        return k < 1u ? 1u : (k > RB200_CI_KMAX ? RB200_CI_KMAX : k);
    };
    auto claim = [&](uint32_t k) -> uint32_t {   // lane 0
        const unsigned long long c = atomicAdd(&st->work_counter, (unsigned long long)k);
        return c < T ? (uint32_t)c : T;
    };
#ifdef RB200_PROBE
    const long long probe_w0 = clock64();
    unsigned long long probe_n = 0;
#endif
    uint32_t u = 0, pend = 0, kc = chunk(0);
    if (lane == 0) u = claim(kc);
    u = __shfl_sync(FULLMASK, u, 0);
    uint32_t e = kc < T - u ? u + kc : T;   // end of the current chunk
    kc = chunk(e);                          // size of the claim in flight
    if (lane == 0) pend = claim(kc);
    if (u < n_cells) desc_prefetch(s_desc[wid], D + 2ull * u, lane);
    while (u < T) {
        uint4 d0, d1;
        if (u < n_cells) {
            asm volatile("cp.async.wait_all;\n" ::: "memory");
            __syncwarp();
            d0 = s_desc[wid][0];
            d1 = s_desc[wid][1];
            __syncwarp();
        }
        uint32_t nu = u + 1;
        if (nu >= e) {   // the chunk in flight becomes current, the next one is claimed
            nu = __shfl_sync(FULLMASK, pend, 0);
            e = kc < T - nu ? nu + kc : T;
            kc = chunk(e);
            if (lane == 0) pend = claim(kc);
        }
        if (nu < n_cells) desc_prefetch(s_desc[wid], D + 2ull * nu, lane);
        if (u >= n_cells) {
            // ---- pass-through ticket: copy_ticket (4 .. 32) items, ONE PER LANE, each lane reading
            // its item's descriptor; then the warp copies the payloads, the first 512 bytes of four
            // items in flight at a time
            const unsigned long long slot = n_cells + (unsigned long long)(u - n_cells) * copy_ticket + lane;
            const bool valid = lane < copy_ticket && slot < W;
            const uint8_t *src = nullptr;
            uint8_t *dst = nullptr;
            uint32_t nvec = 0;
            if (valid) {
                const CellDesc d = cd_unpack(D[2 * slot], D[2 * slot + 1]);
                int otype = d.tA;
                uint32_t ocard = d.cA, olen = d.lA;
                // roaring_bitmap_flip on an absent key: container_range_of_ones (containers.h:300-312)
                // makes a one-value range an ARRAY; {start, 0} and {start} share their first 2 bytes
                if (LAZY && (rules & RULES_FLIP) && d.kind == K_COPY_B && (ocard & CARD_MASK) == 1u) {
                    otype = T_ARRAY;
                    olen = 1;
                }
                if (d.off + d.cap > slab_cap) {
                    atomicExch(&st->error, 2u);
                    otype = 0;
                    ocard = olen = 0;
                } else {
                    src = (d.kind == K_COPY_A ? A.payload : B.payload) + d.offA;
                    dst = slab + d.off;
                    nvec = (stored_bytes(otype, olen) + 15) >> 4;
                }
                it.otype[d.item] = (uint8_t)otype;
                it.ocard[d.item] = ocard;
                it.olen[d.item] = olen;
            }
            const int cnt = __popc(__ballot_sync(FULLMASK, valid));   // valid lanes are 0 .. cnt-1
            for (int j0 = 0; j0 < cnt; j0 += 4) {
                const uint4 *sp[4];
                uint4 *dp[4];
                uint32_t nv[4];
                uint4 v[4];
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const int j = (j0 + k) & 31;
                    sp[k] = reinterpret_cast<const uint4 *>(__shfl_sync(FULLMASK, (unsigned long long)src, j));
                    dp[k] = reinterpret_cast<uint4 *>(__shfl_sync(FULLMASK, (unsigned long long)dst, j));
                    nv[k] = __shfl_sync(FULLMASK, nvec, j);
                    if (j0 + k >= cnt) nv[k] = 0;
                }
#pragma unroll
                for (int k = 0; k < 4; k++)
                    if ((uint32_t)lane < nv[k]) v[k] = __ldg(sp[k] + lane);
#pragma unroll
                for (int k = 0; k < 4; k++)
                    if ((uint32_t)lane < nv[k]) dp[k][lane] = v[k];
#pragma unroll
                for (int k = 0; k < 4; k++)
                    if (nv[k] > 32)
                        warp_copy16(reinterpret_cast<uint8_t *>(dp[k] + 32), reinterpret_cast<const uint8_t *>(sp[k] + 32),
                                    (nv[k] - 32) * 16, lane);
            }
            u = nu;
            continue;
        }
        // (tried in round 2: fetching the metadata of 8 items with the first lanes and passing the
        //  fields by shuffle — 17 more live registers, spills at the 6-CTA register budget and
        //  8-item tickets made every launch 15-60 % SLOWER; one descriptor per cell, prefetched
        //  into shared memory, replaces that chain)
        const CellDesc d = cd_unpack(d0, d1);
        u = nu;
        if (d.kind == K_HOLE) continue;
#ifdef RB200_PROBE
        const long long probe_t0 = clock64();
#endif
        int otype = 0;
        uint32_t ocard = 0, olen = 0;
        if (d.off + d.cap > slab_cap) {
            if (lane == 0) atomicExch(&st->error, 2u);
        } else if (d.kind == K_COMPUTE) {
            cell_compute<OP, LAZY>(acc, d.tA, d.tB, A.payload + d.offA, B.payload + d.offB, d.cA & CARD_MASK, d.cB,
                                   d.lA, d.lB, slab + d.off, d.cap, lane, otype, ocard, olen, &st->error,
                                   d.shared ? rules & ~RULES_INPLACE : rules, (d.cA & CARD_UNKNOWN) != 0);
        } else {
            otype = d.tA;
            ocard = d.cA;
            olen = d.lA;
            // roaring_bitmap_flip on an absent key: see the pass-through tickets above
            if (LAZY && (rules & RULES_FLIP) && d.kind == K_COPY_B && (ocard & CARD_MASK) == 1u) {
                otype = T_ARRAY;
                olen = 1;
            }
            warp_copy16(slab + d.off, (d.kind == K_COPY_A ? A.payload : B.payload) + d.offA, stored_bytes(otype, olen), lane);
        }
        if (lane == 0) {
            it.otype[d.item] = (uint8_t)otype;
            it.ocard[d.item] = ocard;
            it.olen[d.item] = olen;
        }
#ifdef RB200_PROBE
        if (lane == 0) {
            const unsigned long long dt = (unsigned long long)(clock64() - probe_t0);
            unsigned long long tag = (unsigned long long)d.kind << 28;
            if (d.kind == K_COMPUTE)
                tag |= (unsigned long long)d.tA << 26 | (unsigned long long)d.tB << 24 |
                       (unsigned long long)((d.cA & CARD_MASK) >> 5) << 12 | (d.cB >> 5);
            atomicMax(&g_probe[0], dt << 32 | tag);
            atomicAdd(&g_probe[3], dt);
            atomicAdd(&g_probe[4], 1ull);
            atomicAdd(&g_probe[5 + (d.kind == K_COMPUTE ? 0 : 1)], dt);
            const int pc = it.cls ? it.cls[d.item] & 7 : 0;
            atomicAdd(&g_probe[8 + pc], dt);
            atomicAdd(&g_probe[16 + pc], 1ull);
            probe_n++;
        }
#endif
    }
#ifdef RB200_PROBE
    if (lane == 0) {
        const unsigned long long dt = (unsigned long long)(clock64() - probe_w0);
        atomicMax(&g_probe[1], dt << 32 | probe_n);
        atomicMin(&g_probe[2], dt << 32 | probe_n);
        atomicAdd(&g_probe[7], dt);
    }
#endif
}

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
// header bytes of the portable format (roaring_array.c:469-500)
__device__ __forceinline__ uint32_t portable_header_bytes(uint32_t n, bool hasrun) {
    if (!hasrun) return 8u + 8u * n;
    return 4u + ((n + 7u) >> 3) + (n < 4u ? 4u * n : 8u * n);
}

#ifndef RB200_FIN_BLOCKS
#define RB200_FIN_BLOCKS 16
#endif
__global__ void __launch_bounds__(128)
k_finalize_pairs(SetView A, SetView B, Items it, const uint64_t *__restrict__ item_off,
                 uint32_t npairs, SetOut out, OpStats *st) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    // the four pairs of a block reserve their directory range with ONE atomic (the cursor is a single
    // address: one returning atomic per pair serialised 19 900 of them per launch)
    __shared__ uint32_t s_cnt[4];
    __shared__ unsigned long long s_base;
    unsigned long long acc_bytes = 0, acc_outb = 0;  // per-warp totals: one atomic each at the end
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
            if (kind == K_COMPUTE) {
                const uint32_t ca = it.ca[i], cb = it.cb[i];
                bytes += portable_bytes(A.c_type[ca], A.c_len[ca]) +
                         portable_bytes(B.c_type[cb], B.c_len[cb]) + osz;
            } else {
                bytes += 2ull * osz;
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
    __shared__ unsigned long long s_tot[4][2];
    if (lane == 0) { s_tot[wid][0] = acc_bytes; s_tot[wid][1] = acc_outb; }
    __syncthreads();
    if (threadIdx.x < 2) {
        const unsigned long long v = s_tot[0][threadIdx.x] + s_tot[1][threadIdx.x] + s_tot[2][threadIdx.x] + s_tot[3][threadIdx.x];
        if (v) atomicAdd(threadIdx.x ? &st->out_portable : &st->algo_bytes, v);
    }
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
        for (int d = 16; d > 0; d >>= 1) card += __shfl_xor_sync(FULLMASK, card, d);
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
        for (int d = 16; d > 0; d >>= 1) card += __shfl_xor_sync(FULLMASK, card, d);
        if (lane == 0) out[b] = card;
    }
}

// *acc += sum of bm_card[0..n) (device-resident checksum of a result set)
__global__ void k_sum_cards(const uint64_t *__restrict__ bm_card, uint32_t n, unsigned long long *acc) {
    unsigned long long v = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) v += bm_card[i];
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULLMASK, v, d);
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
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    uint32_t cnt = 0;
    for (int k = 0; k < 64; k++) cnt += flags[tid * 64 + k] ? 1u : 0u;
    const uint32_t incl = warp_incl_scan(cnt, lane);
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        const uint32_t v = s_warp[lane];
        const uint32_t s = warp_incl_scan(v, lane);
        s_warp[lane] = s - v;
        if (lane == 31) st->nk = s;
    }
    __syncthreads();
    uint32_t o = s_warp[wid] + incl - cnt;
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
        for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULLMASK, v, d);
        if (lane == 0) {
            bytes[b] = v;
            cnts[b] = nc;
        }
    }
}

// single CTA: exclusive scans of per-bitmap container counts and payload bytes
// (n+1 outputs each: the last entry is the total)
__global__ void __launch_bounds__(1024)
k_pack_scan(const uint64_t *__restrict__ bytes, const uint32_t *__restrict__ cnts, uint32_t n,
            uint64_t *__restrict__ off_out, uint64_t *__restrict__ beg_out) {
    __shared__ unsigned long long s_b[32], s_c[32];
    __shared__ unsigned long long carry_b, carry_c;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) carry_b = carry_c = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t i = base + tid;
        unsigned long long vb = i < n ? bytes[i] : 0ull, vc = i < n ? cnts[i] : 0ull;
        unsigned long long ib = vb, ic = vc;
        for (int d = 1; d < 32; d <<= 1) {
            unsigned long long tb = __shfl_up_sync(FULLMASK, ib, d), tc = __shfl_up_sync(FULLMASK, ic, d);
            if (lane >= d) { ib += tb; ic += tc; }
        }
        if (lane == 31) { s_b[wid] = ib; s_c[wid] = ic; }
        __syncthreads();
        if (wid == 0) {
            unsigned long long wb = s_b[lane], wc = s_c[lane], xb = wb, xc = wc;
            for (int d = 1; d < 32; d <<= 1) {
                unsigned long long tb = __shfl_up_sync(FULLMASK, xb, d), tc = __shfl_up_sync(FULLMASK, xc, d);
                if (lane >= d) { xb += tb; xc += tc; }
            }
            s_b[lane] = xb - wb;
            s_c[lane] = xc - wc;
        }
        __syncthreads();
        const unsigned long long eb = carry_b + s_b[wid] + ib - vb, ec = carry_c + s_c[wid] + ic - vc;
        if (i < n) { off_out[i] = eb; beg_out[i] = ec; }
        __syncthreads();
        if (tid == 1023) { carry_b = eb + vb; carry_c = ec + vc; }
        __syncthreads();
    }
    if (tid == 0) { off_out[n] = carry_b; beg_out[n] = carry_c; }
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
        for (int d = 16; d > 0; d >>= 1) card += __shfl_xor_sync(FULLMASK, card, d);
        if (lane == 0) {
            out.bm_beg[b] = (uint32_t)nb;
            out.bm_cnt[b] = nc;
            out.bm_card[b] = card;
        }
    }
}

// ------------------------------------------------------------------------------ launchers
static inline uint32_t blocks_for_warps(uint64_t warps, int warps_per_block, int max_blocks) {
    uint64_t b = (warps + warps_per_block - 1) / warps_per_block;
    if (b < 1) b = 1;
    if (b > (uint64_t)max_blocks) b = max_blocks;
    return (uint32_t)b;
}

void launch_plan_pairs(const SetView &A, const SetView &B, const uint32_t *ia, const uint32_t *ib,
                       const uint64_t *item_off, uint32_t npairs, int op, bool card_only, int rules,
                       Items it, OpStats *st, cudaStream_t s) {
    if (!npairs) return;
    const uint32_t g = blocks_for_warps(npairs, 4, sm_count() * 16);
    k_plan_pairs<<<g, 128, 0, s>>>(A, B, ia, ib, item_off, npairs, op, card_only, rules, it, st);
    g_launches++;
}

void launch_order_items(Items it, uint64_t W, OpStats *st, cudaStream_t s) {
    if (!W || !it.desc_cls) return;
    const uint64_t chunks = (W + 2047) / 2048;
    const uint32_t g = (uint32_t)(chunks < (uint64_t)sm_count() * 8 ? chunks : (uint64_t)sm_count() * 8);
    k_order_items<<<g, 256, 0, s>>>(it, W, st);
    g_launches++;
}

void launch_compute_items(const SetView &A, const SetView &B, Items it, uint64_t W, int op,
                          uint8_t *slab, uint64_t slab_cap, OpStats *st, int rules, int copy_ticket,
                          cudaStream_t s) {
    if (!W) return;
    const uint32_t g = blocks_for_warps(W, 4, sm_count() * 6);
    switch (op) {
        case OP_AND: k_compute_items<OP_AND, false><<<g, 128, 0, s>>>(A, B, it, W, slab, slab_cap, st, rules, copy_ticket); break;
        case OP_OR:
            if (rules & RULES_LAZY) k_compute_items<OP_OR, true><<<g, 128, 0, s>>>(A, B, it, W, slab, slab_cap, st, rules, copy_ticket);
            else k_compute_items<OP_OR, false><<<g, 128, 0, s>>>(A, B, it, W, slab, slab_cap, st, rules, copy_ticket);
            break;
        case OP_XOR:
            if (rules & RULES_LAZY) k_compute_items<OP_XOR, true><<<g, 128, 0, s>>>(A, B, it, W, slab, slab_cap, st, rules, copy_ticket);
            else k_compute_items<OP_XOR, false><<<g, 128, 0, s>>>(A, B, it, W, slab, slab_cap, st, rules, copy_ticket);
            break;
        default: k_compute_items<OP_ANDNOT, false><<<g, 128, 0, s>>>(A, B, it, W, slab, slab_cap, st, rules, copy_ticket); break;
    }
    g_launches++;
}

void launch_card_items(const SetView &A, const SetView &B, Items it, uint64_t W, OpStats *st,
                       cudaStream_t s) {
    if (!W) return;
    const uint32_t g = blocks_for_warps((W + 7) / 8, 4, sm_count() * 5);
    k_card_items<<<g, 128, 0, s>>>(A, B, it, W, st);
    g_launches++;
}

void launch_finalize_pairs(const SetView &A, const SetView &B, Items it, const uint64_t *item_off,
                           uint32_t npairs, SetOut out, OpStats *st, cudaStream_t s) {
    if (!npairs) return;
    // a warp per pair, full residency (16 CTAs of 4 warps per SM); counters: one atomic per block
    const uint32_t g = blocks_for_warps(npairs, 4, sm_count() * RB200_FIN_BLOCKS);
    k_finalize_pairs<<<g, 128, 0, s>>>(A, B, it, item_off, npairs, out, st);
    g_launches++;
}

void launch_finalize_cards(Items it, const uint64_t *item_off, uint32_t npairs, uint64_t *out,
                           cudaStream_t s) {
    if (!npairs) return;
    const uint32_t g = blocks_for_warps(npairs, 4, sm_count() * 16);
    k_finalize_cards<<<g, 128, 0, s>>>(it, item_off, npairs, out);
    g_launches++;
}

void launch_sum_cardinalities(const uint64_t *bm_card, uint32_t n, uint64_t *d_acc, cudaStream_t s) {
    if (!n) return;
    const uint32_t blocks = (n + 255) / 256 < 592u ? (n + 255) / 256 : 592u;
    k_sum_cards<<<blocks, 256, 0, s>>>(bm_card, n, (unsigned long long *)d_acc);
    g_launches++;
}
void launch_set_cardinalities(const SetView &S, uint32_t n, uint64_t *out, cudaStream_t s) {
    if (!n) return;
    const uint32_t g = blocks_for_warps(n, 4, sm_count() * 16);
    k_set_cardinalities<<<g, 128, 0, s>>>(S, n, out);
    g_launches++;
}

void launch_many_mark(const SetView &S, const uint32_t *idx, uint32_t n, uint32_t key_lo,
                      uint32_t key_hi, uint32_t *flags, cudaStream_t s) {
    cudaMemsetAsync(flags, 0, 65536 * sizeof(uint32_t), s);
    if (!n) return;
    const uint32_t g = n < (uint32_t)sm_count() * 8 ? n : (uint32_t)sm_count() * 8;
    k_many_mark<<<g, 128, 0, s>>>(S, idx, n, key_lo, key_hi, flags);
    g_launches++;
}

void launch_many_compact(const uint32_t *flags, uint16_t *keys_out, OpStats *st, cudaStream_t s) {
    k_many_compact<<<1, 1024, 0, s>>>(flags, keys_out, st);
    g_launches++;
}

}  // namespace rb200

namespace rb200 {
void launch_pack(const SetView &S, uint32_t n, int elide, uint64_t *bytes, uint32_t *cnts, uint64_t *off,
                 uint64_t *beg, cudaStream_t s) {
    const uint32_t g = blocks_for_warps(n ? n : 1, 4, sm_count() * 16);
    k_pack_measure<<<g, 128, 0, s>>>(S, n, elide, bytes, cnts);
    k_pack_scan<<<1, 1024, 0, s>>>(bytes, cnts, n, off, beg);
    g_launches += 2;
}
void launch_pack_copy(const SetView &S, uint32_t n, int elide, const uint64_t *off, const uint64_t *beg,
                      SetOut out, cudaStream_t s) {
    if (!n) return;
    const uint32_t g = blocks_for_warps(n, 4, sm_count() * 16);
    k_pack_copy<<<g, 128, 0, s>>>(S, n, elide, off, beg, out);
    g_launches++;
}
}  // namespace rb200

// ------------------------------------------------------------------------------ serialization
// Device-side roaring_bitmap_portable_serialize (src/roaring_array.c:469-531): every bitmap of a
// set becomes its portable byte string inside one device buffer (blob starts 16-byte aligned),
// so results can leave the device as bytes — one D2H, no per-container host allocation.
namespace rb200 {

__device__ __forceinline__ uint32_t ser_header_bytes(uint32_t n, bool hasrun) {
    if (!hasrun) return 8u + 8u * n;
    return 4u + ((n + 7u) >> 3) + (n < 4u ? 4u * n : 8u * n);
}

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
            const uint32_t tot = ser_header_bytes(nc, anyrun != 0) + bytes;
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
        const uint32_t hdr = ser_header_bytes(nc, hasrun);
        uint8_t *kc, *offs = nullptr;
        if (hasrun) {
            if (lane == 0) store_u32(o, 12347u | ((nc - 1) << 16));  // SERIAL_COOKIE, roaring_array.h:35-40
            const uint32_t nfb = (nc + 7) >> 3;
            for (uint32_t j = lane; j < nfb; j += 32) {
                uint32_t byte = 0;
                for (uint32_t k = 0; k < 8 && 8 * j + k < nc; k++)
                    byte |= (S.c_type[c0 + 8 * j + k] == T_RUN ? 1u : 0u) << k;
                o[4 + j] = (uint8_t)byte;
            }
            kc = o + 4 + nfb;
            if (nc >= 4) offs = kc + 4 * nc;  // NO_OFFSET_THRESHOLD
        } else {
            if (lane == 0) { store_u32(o, 12346u); store_u32(o + 4, nc); }
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

void launch_serialize_measure(const SetView &S, uint32_t n, uint64_t *sizes16, uint32_t *exact,
                              uint32_t *hasrun, cudaStream_t s) {
    if (!n) return;
    const uint32_t g = blocks_for_warps(n, 4, sm_count() * 16);
    k_ser_measure<<<g, 128, 0, s>>>(S, n, sizes16, exact, hasrun);
    g_launches++;
}
void launch_serialize_write(const SetView &S, uint32_t n, const uint64_t *off, const uint32_t *hasrun,
                            uint8_t *dst, cudaStream_t s) {
    if (!n) return;
    const uint32_t g = blocks_for_warps(n, 4, sm_count() * 16);
    k_ser_write<<<g, 128, 0, s>>>(S, n, off, hasrun, dst);
    g_launches++;
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
            if ((cookie & 0xFFFFu) == 12347u) {          // SERIAL_COOKIE, roaring_array.h:35-40
                size = (cookie >> 16) + 1;
                hasrun = true;
                runflags = buf + 4;
                pos = 4 + ((size + 7) >> 3);
            } else if (cookie == 12346u && len >= 8) {   // SERIAL_COOKIE_NO_RUN
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
            if (!hasrun || size >= 4u) pos += 4ull * size;   // offset header (NO_OFFSET_THRESHOLD), not trusted
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
            // keys strictly increasing (roaring.c:496-503)
            int left = __shfl_up_sync(FULLMASK, (int)key, 1);
            if (lane == 0) left = prev_key;
            if (__any_sync(FULLMASK, valid && (int)key <= left)) { bad = true; break; }
            prev_key = __shfl_sync(FULLMASK, (int)key, 31);
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
        if (bad && lane == 0) {
            atomicExch(&st->error, 3u);
            atomicMax(&st->nk, nb - b);  // host: first malformed blob = nb - nk
        }
    }
}

__global__ void __launch_bounds__(128)
k_deser_copy(const uint8_t *__restrict__ raw, const uint64_t *__restrict__ src_pos, uint64_t nc,
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
        // Container CONTENTS of an untrusted blob (the device-side counterpart of the payload checks of
        // roaring_bitmap_internal_validate, src/containers/run.c:693-713, array.c:469-487): the
        // kernels rasterise runs and index by array values without further checks, so a run that
        // ends past 65535 or unsorted data must never reach them.
        bool bad = false;
        if (t == T_RUN) {  // run_container_cardinality (run.c:1077) + bounds / order of the runs
            uint32_t card = 0;
            bad = len == 0;
            for (uint32_t k = lane; k < len; k += 32) {
                const uint32_t s0 = ld_u16(src + 4 * k), l0 = ld_u16(src + 4 * k + 2);
                card += l0 + 1u;
                if (s0 + l0 > 65535u) bad = true;
                if (k > 0 && s0 <= ld_u16(src + 4 * k - 4) + ld_u16(src + 4 * k - 2)) bad = true;
            }
            card = __reduce_add_sync(FULLMASK, card);
            if (lane == 0) out.c_card[c] = card;
        } else if (t == T_ARRAY) {  // strictly increasing values
            for (uint32_t k = lane + 1; k < len; k += 32)
                if (ld_u16(src + 2 * k) <= ld_u16(src + 2 * k - 2)) bad = true;
        }
        if (__any_sync(FULLMASK, bad) && lane == 0) atomicCAS(&st->error, 0u, 4u);
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
        for (int d = 16; d > 0; d >>= 1) {
            card += __shfl_xor_sync(FULLMASK, card, d);
            sbytes += __shfl_xor_sync(FULLMASK, sbytes, d);
            ebytes += __shfl_xor_sync(FULLMASK, ebytes, d);
        }
        if (lane == 0) { out.bm_card[b] = card; out.bm_bytes[b] = sbytes; out.bm_ebytes[b] = ebytes; }
    }
}

// ------------------------------------------------------------------------------ frozen format
// roaring_bitmap_frozen_serialize / roaring_bitmap_frozen_view (src/roaring.c:3180-3456): zones
// [bitset words | runs | array values | keys u16 | counts u16 | typecodes u8 | header u32], the
// header LAST: (n_containers << 15) | FROZEN_COOKIE (13766).  counts = cardinality-1 (bitset,
// array) or n_runs (run).  Blob starts are 32-byte aligned so frozen_view accepts them in place.
constexpr uint32_t FROZEN_COOKIE = 13766u;

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
        for (int d = 16; d > 0; d >>= 1) bytes += __shfl_xor_sync(FULLMASK, bytes, d);
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
        for (int d = 16; d > 0; d >>= 1) {
            zb += __shfl_xor_sync(FULLMASK, zb, d);
            zr += __shfl_xor_sync(FULLMASK, zr, d);
            za += __shfl_xor_sync(FULLMASK, za, d);
        }
        uint8_t *base = dst + off[b];
        const unsigned long long k0 = zb + zr + za, n0 = k0 + 2ull * nc, t0 = n0 + 2ull * nc, h0 = t0 + nc;
        unsigned long long pb = 0, pr = zb, pa = zb + zr;  // running write cursors of the three zones
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
            const uint32_t sb = t == T_BITSET ? sz : 0u, sr = t == T_RUN ? sz : 0u, sa = t == T_ARRAY ? sz : 0u;
            const uint32_t ib = warp_incl_scan(sb, lane), ir = warp_incl_scan(sr, lane), ia = warp_incl_scan(sa, lane);
            if (valid) {
                const unsigned long long d = t == T_BITSET ? pb + ib - sb : (t == T_RUN ? pr + ir - sr : pa + ia - sa);
                c_dst[c0 + i] = off[b] + d;
                store_u16(base + k0 + 2ull * i, S.c_key[c0 + i]);
                store_u16(base + n0 + 2ull * i, t == T_RUN ? len : card - 1u);
                base[t0 + i] = (uint8_t)t;
            }
            pb += __shfl_sync(FULLMASK, ib, 31);
            pr += __shfl_sync(FULLMASK, ir, 31);
            pa += __shfl_sync(FULLMASK, ia, 31);
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
    k_frozen_measure<<<blocks_for_warps(n, 4, sm_count() * 16), 128, 0, s>>>(S, n, sizes32, exact, cnt);
    g_launches++;
}
void launch_frozen_write(const SetView &S, uint32_t n, uint64_t nc, const uint64_t *off, uint8_t *dst,
                         uint64_t *c_dst, cudaStream_t s) {
    if (!n) return;
    k_frozen_dir<<<blocks_for_warps(n, 4, sm_count() * 16), 128, 0, s>>>(S, n, off, dst, c_dst);
    g_launches++;
    if (nc) {
        k_frozen_copy<<<blocks_for_warps(nc, 4, sm_count() * 16), 128, 0, s>>>(S, nc, c_dst, dst);
        g_launches++;
    }
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
            for (int d = 16; d > 0; d >>= 1) {
                zb += __shfl_xor_sync(FULLMASK, zb, d);
                zr += __shfl_xor_sync(FULLMASK, zr, d);
                za += __shfl_xor_sync(FULLMASK, za, d);
            }
            if (zb + zr + za + 5ull * nc + 4ull != len) bad = true;   // roaring.c:3425-3429 exact length
        }
        unsigned long long pb = 0, pr = zb, pa = zb + zr, off = slab_base[b];
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
            int left = __shfl_up_sync(FULLMASK, (int)key, 1);
            if (lane == 0) left = prev_key;
            if (__any_sync(FULLMASK, valid && (int)key <= left)) { bad = true; break; }
            prev_key = __shfl_sync(FULLMASK, (int)key, 31);
            const uint32_t sb = t == T_BITSET ? sz : 0u, sr = t == T_RUN ? sz : 0u, sa = t == T_ARRAY ? sz : 0u;
            const uint32_t ib = warp_incl_scan(sb, lane), ir = warp_incl_scan(sr, lane), ia = warp_incl_scan(sa, lane);
            const uint32_t r16 = valid ? round16(sz) : 0u;
            const uint32_t incl = warp_incl_scan(r16, lane);
            if (valid) {
                const uint64_t c = (uint64_t)c0 + i;
                const unsigned long long d = t == T_BITSET ? pb + ib - sb : (t == T_RUN ? pr + ir - sr : pa + ia - sa);
                out.c_key[c] = (uint16_t)key;
                out.c_type[c] = (uint8_t)t;
                out.c_card[c] = cnt + 1u;                    // runs: recounted by k_deser_copy
                out.c_len[c] = t == T_BITSET ? 1024u : (t == T_ARRAY ? cnt + 1u : cnt);
                out.c_off[c] = off + incl - r16;
                out.c_src[c] = SRC_NONE;
                src_pos[c] = roff[b] + d;
            }
            pb += __shfl_sync(FULLMASK, ib, 31);
            pr += __shfl_sync(FULLMASK, ir, 31);
            pa += __shfl_sync(FULLMASK, ia, 31);
            off += __shfl_sync(FULLMASK, incl, 31);
        }
        if (bad && lane == 0) {
            atomicExch(&st->error, 3u);
            atomicMax(&st->nk, nb - b);
        }
    }
}

void launch_deserialize_frozen(const uint8_t *raw, const uint64_t *roff, const uint64_t *rlen,
                               const uint64_t *slab_base, uint32_t nb, uint64_t nc, SetOut out,
                               uint64_t *src_pos, OpStats *st, cudaStream_t s) {
    if (!nb) return;
    k_frozen_parse_dir<<<blocks_for_warps(nb, 4, sm_count() * 16), 128, 0, s>>>(raw, roff, rlen, slab_base, nb, out, src_pos, st);
    g_launches++;
    if (nc) {
        k_deser_copy<<<blocks_for_warps(nc, 4, sm_count() * 16), 128, 0, s>>>(raw, src_pos, nc, out, st);
        g_launches++;
    }
    k_deser_bitmap_cards<<<blocks_for_warps(nb, 4, sm_count() * 16), 128, 0, s>>>(out, nb, st);
    g_launches++;
}

void launch_deserialize(const uint8_t *raw, const uint64_t *roff, const uint64_t *rlen,
                        const uint64_t *slab_base, uint32_t nb, uint64_t nc, SetOut out,
                        uint64_t *src_pos, OpStats *st, cudaStream_t s) {
    if (!nb) return;
    k_deser_dir<<<blocks_for_warps(nb, 4, sm_count() * 16), 128, 0, s>>>(raw, roff, rlen, slab_base, nb, out, src_pos, st);
    g_launches++;
    if (nc) {
        k_deser_copy<<<blocks_for_warps(nc, 4, sm_count() * 16), 128, 0, s>>>(raw, src_pos, nc, out, st);
        g_launches++;
    }
    k_deser_bitmap_cards<<<blocks_for_warps(nb, 4, sm_count() * 16), 128, 0, s>>>(out, nb, st);
    g_launches++;
}
}  // namespace rb200

namespace rb200 {
void launch_pack_scan(const uint64_t *bytes, const uint32_t *cnts, uint32_t n, uint64_t *off,
                      uint64_t *beg, cudaStream_t s) {
    k_pack_scan<<<1, 1024, 0, s>>>(bytes, cnts, n, off, beg);
    g_launches++;
}
}  // namespace rb200
