// rb200_range.cu — roaring_bitmap_add_range_closed / remove_range_closed over a batch of resident
// bitmaps (sm_90a).
//
//   k_range_plan   warp per result bitmap: the item records in key order.  Keys outside the range
//                  keep their container (shared with S, or copied when S shares containers itself);
//                  keys the range covers whole become full runs (add) or holes (remove); keys an add
//                  creates with part of the range get their container_range_of_ones here; the at most
//                  two boundary keys S holds become cells.
//   k_range_cells  warp per boundary cell: container_add_range / container_remove_range of one
//                  container, typed by range_type (rb200_device.cuh).
// The result directory is then compacted by k_finalize_pairs (rb200_kernels.cu), as for add_offset.
//
// Reference semantics restated here (file:line relative to the reference's source tree):
//   roaring_bitmap_add_range_closed       src/roaring.c:251-300
//   roaring_bitmap_remove_range_closed    src/roaring.c:302-340
//   container_add_range / _remove_range   include/roaring/containers/containers.h:2280-2430
//   container_range_of_ones               include/roaring/containers/containers.h:300
//   run merge and cut                     include/roaring/containers/run.h:156-196, 607-700
#include "rb200_device.cuh"

namespace rb200 {

namespace {

// first index of runs[0, n) for which pred(start, end) is false; pred is true on a prefix
template <typename P>
__device__ __forceinline__ uint32_t run_partition(const uint32_t *runs, uint32_t n, P pred) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1, r = __ldg(runs + mid), s = r & 0xffffu;
        if (pred(s, s + (r >> 16))) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// the 16-byte slot of container_range_of_ones [lo, hi] of a key S lacks, which the plan writes itself:
// an array of one value, else one run (range_type)
__device__ __forceinline__ void small_container(uint32_t lo, uint32_t hi, uint32_t &type, uint32_t &card,
                                                uint32_t &len, uint32_t &word) {
    card = hi - lo + 1;
    if (range_type(true, 0, (int)card, 0) == T_ARRAY) {
        type = T_ARRAY;
        len = 1;
        word = lo;
    } else {
        type = T_RUN;
        len = 1;
        word = lo | (hi - lo) << 16;
    }
}

}  // namespace

// Cell record of a boundary key: {S's container (SRC_NONE: no cell), item slot, lo | hi << 16 (the
// range on the key), 0}.  Two per item: the first and the last key of its range.
__global__ void __launch_bounds__(128)
k_range_plan(SetView S, const uint32_t *__restrict__ idx, const uint32_t *__restrict__ mins,
             const uint32_t *__restrict__ maxs, const uint64_t *__restrict__ item_off, uint32_t n, bool add,
             PassShare sh, Items it, uint4 *__restrict__ cell, uint8_t *slab, uint64_t slab_cap, OpStats *st) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    if (threadIdx.x == 0) stamp_first(&st->t_begin);
    bool used = false;
    for (uint32_t p = warp; p < n; p += nwarps) {
        const uint32_t b = idx[p];
        const uint32_t c0 = S.bm_beg[b], nc = S.bm_cnt[b];
        const uint32_t lo = mins[p], hi = maxs[p];
        const bool live = lo <= hi;   // roaring.c:253, 305: min > max changes nothing
        const uint32_t kmin = lo >> 16, kmax = hi >> 16, lo16 = lo & 0xffffu, hi16 = hi & 0xffffu;
        // S's containers with keys in [kmin, kmax] are [i_lo, i_hi)
        const uint16_t *keys = S.c_key + c0;
        const uint32_t i_lo = live ? lower_bound_u16(keys, nc, kmin) : nc;
        const uint32_t i_hi = live ? upper_bound_u16(keys, nc, kmax) : nc;
        const bool has_min = i_lo < i_hi && keys[i_lo] == kmin, has_max = i_lo < i_hi && keys[i_hi - 1] == kmax;
        const bool part_min = lo16 != 0 || (kmin == kmax && hi16 != 0xffffu);
        const bool part_max = hi16 != 0xffffu || (kmin == kmax && lo16 != 0);
        const uint32_t nk = add && live ? kmax - kmin + 1 : 0u;
        const uint64_t s0 = item_off[p], ns = item_off[p + 1] - s0;
        if (lane < 2) {   // the boundary cells: the first key of the range, then the last
            const bool first = lane == 0;
            const bool want = live && (first || kmax != kmin) && (first ? has_min && part_min : has_max && part_max);
            const uint32_t c = first ? i_lo : i_hi - 1;
            const uint32_t slot = !add ? c : first ? i_lo : i_lo + nk - 1;
            const uint32_t clo = first ? lo16 : 0u, chi = first && kmin != kmax ? 0xffffu : hi16;
            cell[2ull * p + lane] = want ? make_uint4(c0 + c, (uint32_t)(s0 + slot), clo | chi << 16, 0u)
                                         : make_uint4(SRC_NONE, 0u, 0u, 0u);
        }
        for (uint64_t q0 = 0; q0 < ns; q0 += 32) {
            const uint64_t q = q0 + lane;
            const bool v = q < ns;
            uint32_t kind = K_HOLE, ca = SRC_NONE, key = 0, otype = 0, ocard = 0, olen = 0, cap = 0, word = 0;
            uint32_t src = SRC_NONE;   // a container of S that stays as it is
            bool direct = false;       // the plan writes the container (word) itself
            if (v) {
                const uint32_t qq = (uint32_t)q;
                if (!live) {
                    src = qq;
                } else if (add) {
                    if (qq < i_lo) {
                        src = qq;
                    } else if (qq < i_lo + nk) {   // roaring.c:273-297: one container per key of the range
                        key = kmin + (qq - i_lo);
                        const bool at_min = key == kmin, at_max = key == kmax;
                        const uint32_t clo = at_min ? lo16 : 0u, chi = at_max ? hi16 : 0xffffu;
                        kind = K_COMPUTE;
                        if ((at_min && part_min && has_min) || (at_max && part_max && has_max)) {
                            ca = c0 + (at_min ? i_lo : i_hi - 1);
                            cap = BITSET_BYTES;   // the cell's: every result type is at most 8 KiB
                        } else if (clo == 0 && chi == 0xffffu) {   // whatever S held: a full run
                            otype = T_RUN;
                            ocard = 65536;
                            olen = 1;
                            word = 0xffff0000u;
                            direct = true;
                            cap = 16;
                        } else {
                            small_container(clo, chi, otype, ocard, olen, word);
                            direct = true;
                            cap = 16;
                        }
                    } else if (qq < i_lo + nk + (nc - i_hi)) {
                        src = i_hi + (qq - i_lo - nk);
                    }
                } else if (qq < i_lo || qq >= i_hi) {
                    src = qq;
                } else {   // roaring.c:311-331: a key the range covers whole is dropped
                    key = keys[qq];
                    if ((key == kmin && part_min) || (key == kmax && part_max)) {
                        kind = K_COMPUTE;
                        ca = c0 + qq;
                        cap = BITSET_BYTES;
                    }
                }
                if (src != SRC_NONE) {
                    const uint32_t c = c0 + src;
                    kind = K_COPY_A;
                    ca = c;
                    key = S.c_key[c];
                    otype = S.c_type[c];
                    ocard = S.c_card[c];
                    olen = S.c_len[c];
                    if (sh.onA) used = true;
                    else cap = round16(stored_bytes(otype, olen));
                }
            }
            // warp-aggregated reservation of the slots of these 32 items
            const uint32_t incl = warp_incl_scan(cap, lane), total = __shfl_sync(FULLMASK, incl, 31);
            unsigned long long base = 0;
            if (lane == 31 && total) base = atomicAdd(&st->slab_cursor, (unsigned long long)total);
            base = __shfl_sync(FULLMASK, base, 31) + incl - cap;
            if (cap && base + cap > slab_cap) {   // the host's bound was wrong: fail loudly
                st->error = 2u;
                kind = K_HOLE;
                direct = false;
                src = SRC_NONE;
            }
            if (v) {
                const uint64_t j = s0 + q;
                it.kind[j] = (uint8_t)kind;
                it.key[j] = (uint16_t)key;
                it.ca[j] = ca;
                it.cb[j] = SRC_NONE;
                it.slot_off[j] = kind == K_COPY_A && sh.onA ? sh.dA + S.c_off[ca] : base + sh.bias;
                it.otype[j] = (uint8_t)otype;
                it.ocard[j] = ocard;
                it.olen[j] = olen;
                if (direct) *reinterpret_cast<uint4 *>(slab + base) = make_uint4(word, 0u, 0u, 0u);
            }
            // copies of S's containers when S shares containers itself (holds never chain)
            unsigned m = __ballot_sync(FULLMASK, kind == K_COPY_A && !sh.onA);
            while (m) {
                const int r = __ffs(m) - 1;
                m &= m - 1;
                const uint32_t c = __shfl_sync(FULLMASK, ca, r);
                const unsigned long long o = __shfl_sync(FULLMASK, base, r);
                warp_copy16(slab + o, S.payload + S.c_off[c], stored_bytes(S.c_type[c], S.c_len[c]), lane);
            }
        }
    }
    if (used) st->shared_used[0] = 1u;
}

// container_add_range / container_remove_range of one boundary container, straight into its slot
__global__ void __launch_bounds__(128)
k_range_cells(SetView S, Items it, const uint4 *__restrict__ cell, uint64_t W, bool add, uint64_t bias,
              uint8_t *slab, OpStats *st) {
    __shared__ __align__(16) uint32_t s_acc[4][ACC_WORDS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t *acc = s_acc[wid];
    const uint64_t warp = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * (uint64_t)blockDim.x) >> 5;
    if (threadIdx.x == 0) stamp_first(&st->t_cells0);
    for (uint64_t e0 = warp * 32; e0 < W; e0 += nwarps * 32) {
        const uint64_t el = e0 + lane;
        bool live = false;
        if (el < W) {
            const uint4 d = cell[el];
            live = d.x != SRC_NONE && it.kind[d.y] == K_COMPUTE;   // (a hole: the slab bound failed)
        }
        unsigned m = __ballot_sync(FULLMASK, live);
        while (m) {
            const uint64_t e = e0 + __ffs(m) - 1;
            m &= m - 1;
            const uint4 d = cell[e];
            const uint32_t c = d.x, j = d.y, clo = d.z & 0xffffu, chi = d.z >> 16;
            uint8_t *out = slab + (it.slot_off[j] - bias);
            const int t = S.c_type[c];
            const uint32_t len = S.c_len[c];
            const uint8_t *p = S.payload + S.c_off[c];
            uint32_t ot = 0, card = 0, olen = 0;
            int nruns = 0;   // range_type's nruns of a run add
            bool via_acc = true;
            if (t == T_ARRAY) {
                // the three spans "below, range, above" (array_container_add_range_nvals), or the two
                // outside the range (array_container_remove_range)
                const uint16_t *a = reinterpret_cast<const uint16_t *>(p);
                const uint32_t nl = lower_bound_u16(a, len, clo), g0 = upper_bound_u16(a, len, chi);
                const uint32_t mid = add ? chi - clo + 1 : 0u, u = nl + mid + (len - g0);
                const int tt = range_type(add, T_ARRAY, (int)u, 0);
                if (tt != T_BITSET) {
                    via_acc = false;
                    card = u;
                    if (tt == T_RUN) {   // 65536 values: the full run
                        if (lane == 0) *reinterpret_cast<uint32_t *>(out) = 0xffff0000u;
                        olen = 1;
                    } else if (tt == T_ARRAY) {
                        uint16_t *o = reinterpret_cast<uint16_t *>(out);
                        for (uint32_t i = lane; i < u; i += 32)
                            o[i] = i < nl ? a[i] : i < nl + mid ? (uint16_t)(clo + (i - nl)) : a[g0 + (i - nl - mid)];
                        olen = u;
                    }
                    ot = (uint32_t)tt;
                }
            } else if (t == T_RUN && add) {
                // rle16_count_less / rle16_count_greater: the runs that neither meet nor touch the range
                const uint32_t *runs = reinterpret_cast<const uint32_t *>(p);
                const uint32_t less = run_partition(runs, len, [&](uint32_t, uint32_t e) { return e + 1 < clo; });
                const uint32_t g0 = run_partition(runs, len, [&](uint32_t s, uint32_t) { return s <= chi + 1; });
                const uint32_t greater = len - g0, common = g0 - less;
                nruns = (int)(less + 1 + greater);
                if (4 * nruns <= BITSET_BYTES) {   // run_container_add_range_nruns: prefix, merged run, suffix
                    via_acc = false;
                    uint32_t mlo = clo, mhi = chi, ccard = 0;
                    if (common) {
                        const uint32_t rf = __ldg(runs + less), rl = __ldg(runs + g0 - 1);
                        mlo = min(clo, rf & 0xffffu);
                        mhi = max(chi, (rl & 0xffffu) + (rl >> 16));
                        for (uint32_t i = less + lane; i < g0; i += 32) ccard += (__ldg(runs + i) >> 16) + 1;
                        ccard = __reduce_add_sync(FULLMASK, ccard);
                    }
                    uint32_t *o = reinterpret_cast<uint32_t *>(out);
                    for (uint32_t i = lane; i < (uint32_t)nruns; i += 32)
                        o[i] = i < less ? __ldg(runs + i) : i == less ? (mlo | (mhi - mlo) << 16) : __ldg(runs + g0 + (i - less - 1));
                    ot = T_RUN;
                    card = (S.c_card[c] & CARD_MASK) - ccard + (mhi - mlo + 1);
                    olen = (uint32_t)nruns;
                }
            }
            if (via_acc) {   // a bitset, an array past 4096 values, a run add of too many runs, a run removal
                acc_load(acc, t, p, len, lane);
                if (add) acc_apply_ranges<0, false>(acc, clo, chi, lane == 0, lane);
                else acc_apply_ranges<2, false>(acc, clo, chi, lane == 0, lane);
                __syncwarp();
                int cc = 0, nr = 0;
                acc_count(acc, lane, !add && t == T_RUN, cc, nr);
                ot = (uint32_t)range_type(add, t, cc, add ? nruns : nr);
                card = (uint32_t)cc;
                if (ot == T_BITSET) {
                    acc_store_bitset(acc, out, lane);
                    olen = 1024;
                } else if (ot == T_ARRAY) {
                    olen = acc_emit_array(acc, reinterpret_cast<uint16_t *>(out), lane);
                } else if (ot == T_RUN) {
                    olen = acc_emit_runs(acc, reinterpret_cast<uint16_t *>(out), lane);
                }
                __syncwarp();   // the accumulator is reused by the next cell
            }
            if (lane == 0) {
                it.otype[j] = (uint8_t)ot;
                it.ocard[j] = card;
                it.olen[j] = olen;
            }
        }
    }
    if (lane == 0) atomicMax(&st->t_cells1, global_ns());
}

void launch_range_plan(const SetView &S, const uint32_t *idx, const uint32_t *mins, const uint32_t *maxs,
                       const uint64_t *item_off, uint32_t n, bool add, const PassShare &sh, Items it, uint4 *cell,
                       uint8_t *slab, uint64_t slab_cap, OpStats *st, cudaStream_t s) {
    if (!n) return;
    launch_kernel(k_range_plan, grid_for(n, 4, 16), 128, 0, s, S, idx, mins, maxs, item_off, n, add, sh, it, cell,
                  slab, slab_cap, st);
}

void launch_range_cells(const SetView &S, Items it, const uint4 *cell, uint32_t n, bool add, uint64_t bias,
                        uint8_t *slab, OpStats *st, cudaStream_t s) {
    if (!n) return;
    // a warp per 32 cell records at a time, 4 warps (32 KiB of accumulators) per block
    const uint64_t W = 2ull * n;
    launch_kernel(k_range_cells, grid_for(W, 128, 6), 128, 0, s, S, it, cell, W, add, bias, slab, st);
}

}  // namespace rb200
