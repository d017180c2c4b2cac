// rb200_offset.cu — roaring_bitmap_add_offset over a batch of resident bitmaps (sm_90a).
//
//   k_offset_plan   warp per result bitmap: two output slots per source container (its lo part, merged
//                   with the previous container's hi part when their keys are adjacent, and its hi
//                   part), keys, holes, slot reservation; key-aligned shifts share or copy the source.
//   k_offset_cells  warp per live slot: the shifted parts of at most two source containers, merged
//                   and typed as the reference's split + container_ior + repair leave them.
// The result directory is then compacted by k_finalize_pairs (rb200_kernels.cu), which reads the
// item records the plan writes: kind, key, slot_off, ca / cb (what the algorithmic bytes count)
// and the otype / ocard / olen the plan (shared and copied slots) or the cells kernel writes.
//
// Reference semantics restated here (file:line relative to /root/reference):
//   roaring_bitmap_add_offset             src/roaring.c:2426-2507
//   container_add_offset and its parts    include/roaring/containers/containers.h:1536,
//                                         src/containers/bitset.c:182, array.c:103, run.c:133
//   merge of adjacent parts               src/roaring.c:2398 offset_append_with_merge,
//                                         containers.h:1226-1319 container_ior
//   final types                           offset_type (rb200_device.cuh)
#include "rb200_device.cuh"

namespace rb200 {

namespace {

// One source container's shifted parts (in_off > 0): the values v < top = 65536 - in_off (lo part,
// v + in_off at the container's key + co) and the rest (hi part, v - top at the next key).  For an
// array the cardinalities are exact; for a run or a bitset they bound the part (0: the part is
// certainly empty).
__device__ __forceinline__ void part_cards(const SetView &S, uint32_t c, uint32_t top, uint32_t &lo, uint32_t &hi) {
    const int t = S.c_type[c];
    const uint32_t len = S.c_len[c], card = S.c_card[c] & CARD_MASK;
    const uint8_t *p = S.payload + S.c_off[c];
    if (t == T_ARRAY) {
        lo = lower_bound_u16(reinterpret_cast<const uint16_t *>(p), len, top);
        hi = len - lo;
    } else if (t == T_RUN) {
        const uint32_t *runs = reinterpret_cast<const uint32_t *>(p);
        const uint32_t first = len ? runs[0] & 0xffffu : 65536u;
        const uint32_t last = len ? (runs[len - 1] & 0xffffu) + (runs[len - 1] >> 16) : 0u;
        lo = len && first < top ? card : 0u;
        hi = len && last >= top ? card : 0u;
    } else {
        lo = hi = card;
    }
}

}  // namespace

// Slot record of the cells kernel: {lo-part container, hi-part container (SRC_NONE: none),
// in_off | path << 16, slot capacity in bytes}.
constexpr uint32_t OFS_NONE = 0, OFS_COPY = 1, OFS_ARRAY = 2, OFS_ACC = 3;

__global__ void __launch_bounds__(128)
k_offset_plan(SetView S, const uint32_t *__restrict__ idx, const int64_t *__restrict__ offsets,
              const uint64_t *__restrict__ item_off, uint32_t n, PassShare sh, Items it, uint4 *__restrict__ cell,
              uint64_t slab_cap, OpStats *st) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    if (threadIdx.x == 0) stamp_first(&st->t_begin);
    bool used = false;
    for (uint32_t p = warp; p < n; p += nwarps) {
        const uint32_t b = idx ? idx[p] : p;
        const uint32_t c0 = S.bm_beg[b], nc = S.bm_cnt[b];
        const int64_t off = offsets[p];
        const int64_t co = off >> 16;                   // roaring.c:2446-2447 (arithmetic shift)
        const uint32_t in_off = (uint32_t)(off - co * 65536), top = 65536u - in_off;
        const uint64_t s0 = item_off[p];
        for (uint32_t t0 = 0; t0 < nc; t0 += 32) {
            const uint32_t i = t0 + lane;
            const bool v = i < nc;
            const uint32_t c = c0 + i;
            uint32_t kind[2] = {K_HOLE, K_HOLE}, ca[2] = {SRC_NONE, SRC_NONE}, cb[2] = {SRC_NONE, SRC_NONE};
            uint32_t otype[2] = {0, 0}, ocard[2] = {0, 0}, olen[2] = {0, 0}, cap[2] = {0, 0};
            uint4 d[2] = {make_uint4(SRC_NONE, SRC_NONE, 0, 0), make_uint4(SRC_NONE, SRC_NONE, 0, 0)};
            uint64_t shared_off = 0;
            bool shared = false;
            int64_t key = 0;
            if (v) {
                key = (int64_t)S.c_key[c] + co;
                const bool in_lo = key >= 0 && key < 65536, in_hi = key + 1 >= 0 && key + 1 < 65536;
                if (in_off == 0) {   // roaring.c:2454-2468: the container as it is, at key + co
                    if (in_lo) {
                        kind[0] = K_COPY_A;
                        ca[0] = c;
                        otype[0] = S.c_type[c];
                        ocard[0] = S.c_card[c];
                        olen[0] = S.c_len[c];
                        if (sh.onA) {
                            shared_off = sh.dA + S.c_off[c];
                            shared = used = true;
                        } else {
                            cap[0] = round16(stored_bytes(otype[0], olen[0]));
                            d[0] = make_uint4(c, SRC_NONE, OFS_COPY << 16, cap[0]);
                        }
                    }
                } else {
                    uint32_t lo_i, hi_i, lo_p = 0, hi_p = 0;
                    part_cards(S, c, top, lo_i, hi_i);
                    const bool adj_prev = i > 0 && S.c_key[c - 1] + 1u == S.c_key[c];
                    const bool adj_next = i + 1 < nc && S.c_key[c] + 1u == S.c_key[c + 1];
                    if (adj_prev && in_lo) part_cards(S, c - 1, top, lo_p, hi_p);
                    const int64_t key_p = key - 1;   // the previous container's key + co (adjacent)
                    const bool prev_lo_kept = key_p >= 0 && lo_p > 0;
                    // slot 2i: lo(i) and the hi part of i - 1 when it lands on the same key
                    const uint32_t L = in_lo && lo_i ? c : SRC_NONE, H = in_lo && hi_p ? c - 1 : SRC_NONE;
                    // slot 2i + 1: hi(i), unless the next container's lo part takes it in
                    const uint32_t H1 = !adj_next && in_hi && hi_i ? c : SRC_NONE;
                    for (int s = 0; s < 2; s++) {
                        const uint32_t lc = s == 0 ? L : SRC_NONE, hc = s == 0 ? H : H1;
                        if (lc == SRC_NONE && hc == SRC_NONE) continue;
                        const uint32_t lcard = lc != SRC_NONE ? (s == 0 ? lo_i : 0u) : 0u;
                        const uint32_t hcard = hc != SRC_NONE ? (s == 0 ? hi_p : hi_i) : 0u;
                        const int tl = lc != SRC_NONE ? S.c_type[lc] : T_ARRAY, th = hc != SRC_NONE ? S.c_type[hc] : T_ARRAY;
                        const uint32_t sum = lcard + hcard;
                        const bool one = lc == SRC_NONE || hc == SRC_NONE;
                        const bool direct = tl == T_ARRAY && th == T_ARRAY && (one || sum <= (uint32_t)MAX_ARRAY);
                        kind[s] = K_COMPUTE;
                        // algorithmic bytes: each source once, with its lo part if that is computed
                        ca[s] = lc;
                        cb[s] = hc != SRC_NONE && !(s == 0 ? prev_lo_kept : (L != SRC_NONE)) ? hc : SRC_NONE;
                        cap[s] = round16(direct ? 2u * sum : min(2u * sum, (uint32_t)BITSET_BYTES));
                        d[s] = make_uint4(lc, hc, in_off | (direct ? OFS_ARRAY : OFS_ACC) << 16, cap[s]);
                    }
                }
            }
            // warp-aggregated reservation of the slots of these 32 containers
            const uint32_t own = cap[0] + cap[1];
            const uint32_t incl = warp_incl_scan(own, lane), total = __shfl_sync(FULLMASK, incl, 31);
            unsigned long long base = 0;
            if (lane == 31 && total) base = atomicAdd(&st->slab_cursor, (unsigned long long)total);
            base = __shfl_sync(FULLMASK, base, 31) + incl - own;
            if (v) {
                for (int s = 0; s < 2; s++) {
                    const uint64_t j = s0 + 2ull * i + s;
                    uint64_t slot = base + (s ? cap[0] : 0u);
                    if (cap[s] && slot + cap[s] > slab_cap) {   // the host's bound was wrong: fail loudly
                        st->error = 2u;
                        kind[s] = K_HOLE;
                        d[s].z = 0;
                    }
                    it.kind[j] = (uint8_t)kind[s];
                    it.key[j] = (uint16_t)(key + s);
                    it.ca[j] = ca[s];
                    it.cb[j] = cb[s];
                    it.slot_off[j] = s == 0 && shared ? shared_off : slot + sh.bias;
                    it.otype[j] = (uint8_t)otype[s];
                    it.ocard[j] = ocard[s];
                    it.olen[j] = olen[s];
                    cell[j] = d[s];
                }
            }
        }
    }
    if (used) st->shared_used[0] = 1u;
}

// bits [p, p + 64) of a 65536-bit bitset in global memory, zero outside [0, 65536)
__device__ __forceinline__ uint64_t bits_at(const uint64_t *__restrict__ w, int p) {
    const int q = p >> 6, r = p & 63;   // arithmetic shift: p may be negative
    const uint64_t a = q >= 0 && q < 1024 ? __ldg(w + q) : 0ull;
    const uint64_t b = q + 1 >= 0 && q + 1 < 1024 ? __ldg(w + q + 1) : 0ull;
    return r ? (a >> r) | (b << (64 - r)) : a;
}

// acc |= one shifted part of an array or run container: hi == false the values v < top (+ in_off),
// hi == true the others (- top).  The accumulator's bitset words are already in place.
__device__ __forceinline__ void acc_or_part(uint32_t *acc, const SetView &S, uint32_t c, bool hi, uint32_t in_off,
                                            int lane) {
    const uint32_t top = 65536u - in_off, len = S.c_len[c];
    const uint8_t *p = S.payload + S.c_off[c];
    if (S.c_type[c] == T_ARRAY) {
        const uint16_t *a = reinterpret_cast<const uint16_t *>(p);
        const uint32_t split = lower_bound_u16(a, len, top);
        const uint32_t b = hi ? split : 0u, e = hi ? len : split;
        for (uint32_t j = b + lane; j < e; j += 32) {
            const uint32_t y = (a[j] + in_off) & 0xffffu;
            atomicOr(acc + (y >> 5), 1u << (y & 31));
        }
        return;
    }
    const uint32_t *runs = reinterpret_cast<const uint32_t *>(p);
    for (uint32_t base = 0; base < len; base += 32) {   // run.c:133-190: the run across top is cut
        const uint32_t j = base + lane;
        const uint32_t r = j < len ? __ldg(runs + j) : 0u;
        const uint32_t s = r & 0xffffu, e = min(s + (r >> 16), 65535u);
        bool valid = j < len;
        uint32_t lo, hv;
        if (hi) {
            valid = valid && e >= top;
            lo = max(s, top) - top;
            hv = e - top;
        } else {
            valid = valid && s < top;
            lo = s + in_off;
            hv = min(e, top - 1) + in_off;
        }
        acc_apply_ranges<0, false>(acc, valid ? lo : 0u, valid ? hv : 0u, valid, lane);
    }
}

__global__ void __launch_bounds__(128)
k_offset_cells(SetView S, Items it, const uint4 *__restrict__ cell, uint64_t W, uint64_t bias, uint8_t *slab,
               OpStats *st) {
    __shared__ __align__(16) uint32_t s_acc[4][ACC_WORDS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t *acc = s_acc[wid];
    const uint64_t warp = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * (uint64_t)blockDim.x) >> 5;
    if (threadIdx.x == 0) stamp_first(&st->t_cells0);
    for (uint64_t j0 = warp * 32; j0 < W; j0 += nwarps * 32) {
        const uint64_t jl = j0 + lane;
        unsigned m = __ballot_sync(FULLMASK, jl < W && (cell[jl].z >> 16) != OFS_NONE);
        while (m) {
            const uint64_t j = j0 + __ffs(m) - 1;
            m &= m - 1;
            const uint4 d = cell[j];
            const uint32_t path = d.z >> 16, in_off = d.z & 0xffffu, top = 65536u - in_off, cap = d.w;
            uint8_t *out = slab + (it.slot_off[j] - bias);
            if (path == OFS_COPY) {   // a key-aligned shift from a set that shares containers itself
                warp_copy16(out, S.payload + S.c_off[d.x], stored_bytes(S.c_type[d.x], S.c_len[d.x]), lane);
                continue;
            }
            const uint32_t lc = d.x, hc = d.y;
            uint32_t ot = 0, card = 0, len = 0;
            if (path == OFS_ARRAY) {
                // the hi part of the previous container (values [0, in_off)), then the lo part of this
                // one ([in_off, 65536)): v + in_off in u16 arithmetic keeps them in order
                const uint16_t *ah = hc != SRC_NONE ? reinterpret_cast<const uint16_t *>(S.payload + S.c_off[hc]) : nullptr;
                const uint16_t *al = lc != SRC_NONE ? reinterpret_cast<const uint16_t *>(S.payload + S.c_off[lc]) : nullptr;
                const uint32_t nh_all = ah ? S.c_len[hc] : 0u, sh = ah ? lower_bound_u16(ah, nh_all, top) : 0u;
                const uint32_t nh = nh_all - sh, nl = al ? lower_bound_u16(al, S.c_len[lc], top) : 0u;
                card = len = nh + nl;
                if (2 * card > cap) {
                    if (lane == 0) st->error = 1u;
                    card = len = 0;
                } else {
                    ot = T_ARRAY;
                    uint16_t *o = reinterpret_cast<uint16_t *>(out);
                    for (uint32_t q = lane; 8 * q < card; q += 32) {
                        uint16_t x[8];
#pragma unroll
                        for (int k = 0; k < 8; k++) {
                            const uint32_t jj = 8 * q + k;
                            x[k] = jj < card ? (uint16_t)((jj < nh ? ah[sh + jj] : al[jj - nh]) + in_off) : 0;
                        }
                        if (8 * q + 8 <= card) {
                            reinterpret_cast<uint4 *>(o)[q] = make_uint4(x[0] | (uint32_t)x[1] << 16, x[2] | (uint32_t)x[3] << 16,
                                                                         x[4] | (uint32_t)x[5] << 16, x[6] | (uint32_t)x[7] << 16);
                        } else {
                            for (uint32_t k = 0; 8 * q + k < card; k++) o[8 * q + k] = x[k];
                        }
                    }
                }
            } else {   // OFS_ACC
                int tl = lc != SRC_NONE ? S.c_type[lc] : 0, th = hc != SRC_NONE ? S.c_type[hc] : 0;
                // bitset parts first, as whole words (bitset.c:182-235 funnel shift), then the others
                if (tl == T_BITSET || th == T_BITSET) {
                    const uint64_t *wl = tl == T_BITSET ? reinterpret_cast<const uint64_t *>(S.payload + S.c_off[lc]) : nullptr;
                    const uint64_t *wh = th == T_BITSET ? reinterpret_cast<const uint64_t *>(S.payload + S.c_off[hc]) : nullptr;
                    uint64_t *acc64 = reinterpret_cast<uint64_t *>(acc);
                    int cl = 0, ch = 0;
#pragma unroll 4
                    for (int w = lane; w < 1024; w += 32) {
                        const uint64_t xl = wl ? bits_at(wl, 64 * w - (int)in_off) : 0ull;
                        const uint64_t xh = wh ? bits_at(wh, 64 * w + (int)top) : 0ull;
                        cl += __popcll(xl);
                        ch += __popcll(xh);
                        acc64[w] = xl | xh;
                    }
                    // an empty bitset part is no part at all (bitset.c:206, 233: it is freed, not appended)
                    if (wl && !__reduce_add_sync(FULLMASK, cl)) tl = 0;
                    if (wh && !__reduce_add_sync(FULLMASK, ch)) th = 0;
                } else {
                    acc_zero(acc, lane);
                }
                __syncwarp();
                if (tl && tl != T_BITSET) acc_or_part(acc, S, lc, false, in_off, lane);
                if (th && th != T_BITSET) acc_or_part(acc, S, hc, true, in_off, lane);
                __syncwarp();
                int c = 0, nr = 0;
                acc_count(acc, lane, tl == T_RUN || th == T_RUN, c, nr);
                card = (uint32_t)c;
                if (card) {
                    ot = offset_type(tl ? tl : th, tl ? th : 0, c, nr);
                    const uint32_t need = ot == T_BITSET ? (uint32_t)BITSET_BYTES : ot == T_ARRAY ? 2u * card : 4u * (uint32_t)nr;
                    if (need > cap) {
                        if (lane == 0) st->error = 1u;
                        ot = 0;
                        card = 0;
                    } else if (ot == T_BITSET) {
                        acc_store_bitset(acc, out, lane);
                        len = 1024;
                    } else if (ot == T_ARRAY) {
                        len = acc_emit_array(acc, reinterpret_cast<uint16_t *>(out), lane);
                    } else {
                        len = acc_emit_runs(acc, reinterpret_cast<uint16_t *>(out), lane);
                    }
                }
                __syncwarp();   // the accumulator is reused by the next slot
            }
            if (lane == 0) {
                it.otype[j] = (uint8_t)ot;
                it.ocard[j] = card;
                it.olen[j] = len;
            }
        }
    }
    if (lane == 0) atomicMax(&st->t_cells1, global_ns());
}

void launch_offset_plan(const SetView &S, const uint32_t *idx, const int64_t *offsets, const uint64_t *item_off,
                        uint32_t n, const PassShare &sh, Items it, uint4 *cell, uint64_t slab_cap, OpStats *st,
                        cudaStream_t s) {
    if (!n) return;
    launch_kernel(k_offset_plan, grid_for(n, 4, 16), 128, 0, s, S, idx, offsets, item_off, n, sh, it, cell, slab_cap, st);
}

void launch_offset_cells(const SetView &S, Items it, const uint4 *cell, uint64_t W, uint64_t bias, uint8_t *slab,
                         OpStats *st, cudaStream_t s) {
    if (!W) return;
    // a warp per 32 slots at a time, 4 warps (32 KiB of accumulators) per block
    launch_kernel(k_offset_cells, grid_for(W, 128, 6), 128, 0, s, S, it, cell, W, bias, slab, st);
}

}  // namespace rb200
