// rb200_compute.cu — k_compute_items, the pairwise cell kernel (one warp per container x container
// cell of a batch, or a ticket of pass-through copies; the cells themselves are cell_compute() in
// rb200_cells.cuh).
//
// A translation unit of its own so that build.py can give it evict-first as the default for global
// stores (ptxas -dscm=cs): every global store of this kernel writes a result that it never reads
// again (payloads and item records), and with write-back stores the results streaming out (1.25 GB
// per weather_sept_85 OR launch of the headline workload) pushed the operands, which every cell
// reads, out of L2.  The store instructions are unchanged, so the register allocation is too.
#include "rb200_device.cuh"
#include "rb200_cells.cuh"

namespace rb200 {

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
    // Wait: the class counts, the descriptors and the work counter are written by the kernels ahead
    // (k_plan_pairs, k_order_items), and the result slab may still be read by an earlier op.
    pdl_wait();
    if (threadIdx.x == 0) stamp_first(&st->t_cells0);
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
            // Trigger: the claim came back past T, so every unit is handed out and this warp has only
            // its current one left.  k_finalize_pairs may launch into the drain; it reads the results
            // after its wait, which waits for this whole grid.
            if (nu >= T) pdl_trigger();
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
    if (lane == 0) atomicMax(&st->t_cells1, global_ns());
#ifdef RB200_PROBE
    if (lane == 0) {
        const unsigned long long dt = (unsigned long long)(clock64() - probe_w0);
        atomicMax(&g_probe[1], dt << 32 | probe_n);
        atomicMin(&g_probe[2], dt << 32 | probe_n);
        atomicAdd(&g_probe[7], dt);
    }
#endif
}

void launch_compute_items(const SetView &A, const SetView &B, Items it, uint64_t W, int op,
                          uint8_t *slab, uint64_t slab_cap, OpStats *st, int rules, int copy_ticket,
                          cudaStream_t s) {
    if (!W) return;
    const bool lazy = (rules & RULES_LAZY) != 0;
    auto *k = op == OP_AND  ? k_compute_items<OP_AND, false>
            : op == OP_OR   ? (lazy ? k_compute_items<OP_OR, true> : k_compute_items<OP_OR, false>)
            : op == OP_XOR  ? (lazy ? k_compute_items<OP_XOR, true> : k_compute_items<OP_XOR, false>)
                            : k_compute_items<OP_ANDNOT, false>;
    // a warp per unit, 4 per block, at most 6 resident blocks per SM
    launch_kernel_chained(k, grid_for(W, 4, 6), 128, 0, s, A, B, it, W, slab, slab_cap, st, rules, copy_ticket);
}

}  // namespace rb200
