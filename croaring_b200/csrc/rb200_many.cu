// rb200_many.cu — N-way union (roaring_bitmap_or_many, src/roaring.c:775-790) on sm_90a.
//
// The reference folds the inputs left to right with lazy cells (roaring_bitmap_lazy_or
// :2509-2598, roaring_bitmap_lazy_or_inplace :2600-2682, container_lazy_or / container_lazy_ior
// include/roaring/containers/containers.h:1113-1215, 1333-1442) and repairs once
// (roaring_bitmap_repair_after_lazy :2845).  OR is associative, so on the GPU each KEY is
// reduced independently:
//
//   work unit = (key, slice of the input list).  A CTA gathers the containers carrying the key
//   (binary search in every bitmap's sorted key array, ordered compaction into shared memory),
//   ORs bitset containers into a per-thread register slice (two 128-bit words per thread, loads
//   batched four containers deep), flattens all array values / runs of the slice into one work
//   list spread over the 256 threads (shared-memory atomics on a 65536-bit accumulator), and
//   — when the key was split over several CTAs for parallelism — merges into a global scratch
//   accumulator; the last CTA of a key finalises: popcount, result type, re-encode.
//
// Result types follow the reference's fold exactly: the metadata of the participants is
// replayed through the fold's state machine (full runs / full bitsets short-circuit the fold,
// a bitset x bitset in-place step converts a saturated accumulator to the full run,
// containers.h:1342-1352); the rare saturated-with-bitsets case is decided by an ordered
// replay of the prefix unions.
#include <stdlib.h>

#include "rb200_device.cuh"

namespace rb200 {

__device__ __forceinline__ uint32_t lower_bound_key(const uint16_t *a, uint32_t n, uint32_t key) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (a[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

constexpr int OM_THREADS = 256;
constexpr int OM_CHUNK = 512;  // bitmaps gathered per round: two per thread
constexpr uint32_t PF_FULL_RUN = 16, PF_FULL_BITSET = 32;

// The reference's fold, metadata only (lives in thread 0's registers).
struct FoldState {
    uint32_t m_total = 0, first_pos = 0, second_pos = 0, first_tf = 0, last_ib_pos = 0;
    bool any_inplace_bitset = false, run_full = false, decided_skip = false,
         first_is_full_bitset = false;
};

// (roaring.c:2535-2545 first combine; :2621-2640 in-place steps; containers.h:1342-1404)
__device__ __forceinline__ void fold_step(FoldState &f, uint32_t tf, uint32_t pos) {
    const int t = tf & 15;
    const bool full_run = tf & PF_FULL_RUN, full_bitset = tf & PF_FULL_BITSET;
    if (f.m_total == 0) {
        f.first_tf = tf;
        f.first_pos = pos;
        if (full_run) { f.run_full = true; f.decided_skip = true; }
        if (full_bitset) { f.first_is_full_bitset = true; f.decided_skip = true; }
    } else {
        if (f.m_total == 1) f.second_pos = pos;
        const bool non_inplace = f.m_total == 1 && f.first_pos == 0 && f.second_pos == 1;
        if (non_inplace) {
            // first combine of x[0], x[1]: no "is full" skip (roaring.c:2535-2550)
            const int t1 = f.first_tf & 15;
            f.first_is_full_bitset = false;
            if (t1 != T_BITSET && t != T_BITSET) f.run_full = full_run;  // c1 -> bitset, lazy_ior(B, c2)
            else f.run_full = full_run || (f.first_tf & PF_FULL_RUN);    // container_lazy_or copies a full run
            f.decided_skip = f.run_full;
        } else if (!f.decided_skip) {
            if (full_run) { f.run_full = true; f.decided_skip = true; }
            else if (t == T_BITSET) { f.any_inplace_bitset = true; f.last_ib_pos = pos; }
        }
    }
    f.m_total++;
}

struct ManySmem {
    uint32_t acc[ACC_WORDS];
    unsigned long long poff[OM_CHUNK];
    uint32_t plen[OM_CHUNK];
    uint32_t ppos[OM_CHUNK];
    uint32_t pustart[OM_CHUNK + 1];  // exclusive prefix of flattened work units (array vectors / runs)
    uint8_t ptf[OM_CHUNK];           // type | PF_* flags
    uint32_t pcard[OM_CHUNK];        // cardinality of each participant (xor_many)
    uint32_t warp_a[OM_THREADS / 32], warp_b[OM_THREADS / 32];
    int red[OM_THREADS / 32][2];
    uint32_t np, ki, flag, anyfull, aux, rfull;
};

// Gather the participants of `key` among bitmaps [c0, c0+OM_CHUNK) ∩ [0,n) in input order.
__device__ __forceinline__ uint32_t many_gather(ManySmem &sm, const SetView &S,
                                                const uint32_t *__restrict__ idx, uint32_t n,
                                                uint32_t key, uint32_t c0, uint32_t c1) {
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    uint32_t cont[2], tf[2], len[2], units[2];
    unsigned long long off[2];
    uint32_t cnt = 0, ucnt = 0;
    // two lower_bound searches per thread, advanced in lockstep so their loads overlap
    uint32_t b0[2], nb[2], lo[2], hi[2];
#pragma unroll
    for (int k = 0; k < 2; k++) {
        const uint32_t i = c0 + tid * 2 + k;
        cont[k] = 0xffffffffu;
        units[k] = 0;
        b0[k] = nb[k] = 0;
        if (i < c1) {
            const uint32_t b = idx ? idx[i] : i;
            b0[k] = S.bm_beg[b];
            nb[k] = S.bm_cnt[b];
        }
        lo[k] = 0;
        hi[k] = nb[k];
    }
    while (lo[0] < hi[0] || lo[1] < hi[1]) {
        uint32_t mid[2], kv[2];
#pragma unroll
        for (int k = 0; k < 2; k++) {
            mid[k] = (lo[k] + hi[k]) >> 1;
            kv[k] = lo[k] < hi[k] ? (uint32_t)S.c_key[b0[k] + mid[k]] : 0u;
        }
#pragma unroll
        for (int k = 0; k < 2; k++)
            if (lo[k] < hi[k]) {
                if (kv[k] < key) lo[k] = mid[k] + 1;
                else hi[k] = mid[k];
            }
    }
    uint32_t ct[2], cl[2], cc[2];
    bool hit[2];
#pragma unroll
    for (int k = 0; k < 2; k++) {
        hit[k] = lo[k] < nb[k] && S.c_key[b0[k] + lo[k]] == key;
        const uint32_t c = b0[k] + lo[k];
        ct[k] = hit[k] ? (uint32_t)S.c_type[c] : 0u;
        cl[k] = hit[k] ? S.c_len[c] : 0u;
        cc[k] = hit[k] ? S.c_card[c] : 0u;
        off[k] = hit[k] ? S.c_off[c] : 0ull;
    }
#pragma unroll
    for (int k = 0; k < 2; k++)
        if (hit[k]) {
            const uint32_t t = ct[k], l = cl[k], cd = cc[k];
            cont[k] = b0[k] + lo[k];
            len[k] = l;
            uint32_t f = t;
            if (t == T_RUN && l == 1 && cd == 65536) f |= PF_FULL_RUN;
            if (t == T_BITSET && cd == 65536) f |= PF_FULL_BITSET;
            tf[k] = f;
            if (t == T_ARRAY) units[k] = (l + 7) >> 3;
            else if (t == T_RUN && !(f & PF_FULL_RUN)) units[k] = l;
            cnt++;
            ucnt += units[k];
        }
    const uint32_t incl = warp_incl_scan(cnt, lane), uincl = warp_incl_scan(ucnt, lane);
    if (lane == 31) { sm.warp_a[wid] = incl; sm.warp_b[wid] = uincl; }
    __syncthreads();
    if (wid == 0) {
        const uint32_t va = lane < OM_THREADS / 32 ? sm.warp_a[lane] : 0u;
        const uint32_t vb = lane < OM_THREADS / 32 ? sm.warp_b[lane] : 0u;
        const uint32_t sa = warp_incl_scan(va, lane), sb = warp_incl_scan(vb, lane);
        if (lane < OM_THREADS / 32) { sm.warp_a[lane] = sa - va; sm.warp_b[lane] = sb - vb; }
        if (lane == 31) { sm.np = sa; sm.pustart[sa] = sb; }
    }
    __syncthreads();
    uint32_t o = sm.warp_a[wid] + incl - cnt, u = sm.warp_b[wid] + uincl - ucnt;
#pragma unroll
    for (int k = 0; k < 2; k++)
        if (cont[k] != 0xffffffffu) {
            sm.poff[o] = off[k];
            sm.plen[o] = len[k];
            sm.ppos[o] = c0 + tid * 2 + k;
            sm.ptf[o] = (uint8_t)tf[k];
            sm.pcard[o] = cc[k];
            sm.pustart[o] = u;
            u += units[k];
            o++;
        }
    __syncthreads();
    return sm.np;
}

// OR the payloads of the gathered participants into (r0,r1) registers + shared accumulator.
__device__ __forceinline__ void many_accumulate(ManySmem &sm, const SetView &S, uint32_t np,
                                                uint4 &r0, uint4 &r1) {
    const int tid = threadIdx.x;
    // bitset containers: registers, four containers in flight per thread
    uint32_t j = 0;
    while (j < np) {
        const uint4 *src[4];
        int nb4 = 0;
        while (j < np && nb4 < 4) {
            if ((sm.ptf[j] & 15) == T_BITSET)
                src[nb4++] = reinterpret_cast<const uint4 *>(S.payload + sm.poff[j]);
            j++;
        }
        uint4 qa[4], qb[4];
#pragma unroll
        for (int k = 0; k < 4; k++)
            if (k < nb4) {
                qa[k] = __ldg(src[k] + tid);
                qb[k] = __ldg(src[k] + tid + OM_THREADS);
            }
#pragma unroll
        for (int k = 0; k < 4; k++)
            if (k < nb4) {
                r0.x |= qa[k].x; r0.y |= qa[k].y; r0.z |= qa[k].z; r0.w |= qa[k].w;
                r1.x |= qb[k].x; r1.y |= qb[k].y; r1.z |= qb[k].z; r1.w |= qb[k].w;
            }
    }
    // arrays and runs: one flat list of work units over all participants; a thread takes four
    // consecutive units (one participant search, then a linear advance) and issues their loads
    // together so several are in flight per thread
    const uint32_t V = sm.pustart[np];
    for (uint32_t u0 = tid * 4; u0 < V; u0 += OM_THREADS * 4) {
        uint32_t lo = 0, hi = np;  // last participant with pustart <= u0
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (sm.pustart[mid] <= u0) lo = mid;
            else hi = mid;
        }
        uint4 q[4];
        uint32_t left[4];
        int kind[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint32_t u = u0 + k;
            kind[k] = 0;
            left[k] = 0;
            q[k] = make_uint4(0, 0, 0, 0);
            if (u < V) {
                while (lo + 1 < np && sm.pustart[lo + 1] <= u) lo++;
                const uint32_t local = u - sm.pustart[lo];
                const uint8_t *p = S.payload + sm.poff[lo];
                if ((sm.ptf[lo] & 15) == T_ARRAY) {
                    q[k] = __ldg(reinterpret_cast<const uint4 *>(p) + local);
                    left[k] = sm.plen[lo] - local * 8;
                    kind[k] = 1;
                } else {
                    q[k].x = __ldg(reinterpret_cast<const uint32_t *>(p) + local);
                    kind[k] = 2;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (kind[k] == 1) {
                const uint32_t w[4] = {q[k].x, q[k].y, q[k].z, q[k].w};
                uint32_t cur_w = (w[0] & 0xffffu) >> 5, cur_m = 0;
#pragma unroll
                for (int e = 0; e < 8; e++) {
                    const uint32_t v = (e & 1) ? (w[e >> 1] >> 16) : (w[e >> 1] & 0xffffu);
                    const uint32_t wi = v >> 5, bit = 1u << (v & 31);
                    if (e == 0 || e < (int)left[k]) {
                        if (wi != cur_w) {
                            atomicOr(sm.acc + cur_w, cur_m);
                            cur_w = wi;
                            cur_m = bit;
                        } else {
                            cur_m |= bit;
                        }
                    }
                }
                atomicOr(sm.acc + cur_w, cur_m);
            } else if (kind[k] == 2) {  // one run
                const uint32_t r = q[k].x;
                const uint32_t s0 = r & 0xffffu, e0 = min(s0 + (r >> 16), 65535u);
                const uint32_t ws = s0 >> 5, we = e0 >> 5;
                const uint32_t m_lo = ~0u << (s0 & 31), m_hi = ~0u >> (31 - (e0 & 31));
                if (ws == we) {
                    atomicOr(sm.acc + ws, m_lo & m_hi);
                } else {
                    atomicOr(sm.acc + ws, m_lo);
                    for (uint32_t w2 = ws + 1; w2 < we; w2++) atomicOr(sm.acc + w2, ~0u);
                    atomicOr(sm.acc + we, m_hi);
                }
            }
        }
    }
}

__device__ __forceinline__ void
or_many_body(SetView S, const uint32_t *__restrict__ idx, uint32_t n,
          const uint16_t *__restrict__ keys, uint32_t want_slices, uint32_t *scratch_acc,
          uint32_t *scratch_tickets, uint32_t scratch_keys, SetOut out,
          uint32_t *__restrict__ card_per_key, OpStats *st) {
    __shared__ __align__(16) ManySmem sm;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t nk = st->nk;
    // split a key over several CTAs only when there are few keys and the scratch can hold them
    const uint32_t ns = (want_slices > 1 && nk <= scratch_keys) ? want_slices : 1u;
    const uint32_t per_slice = (n + ns - 1) / ns;
    const unsigned long long total_units = (unsigned long long)nk * ns;

    for (;;) {
        if (tid == 0) sm.ki = (uint32_t)atomicAdd(&st->work_counter2, 1ull);
        __syncthreads();
        const uint32_t unit = sm.ki;
        __syncthreads();
        if (unit >= total_units) break;
        const uint32_t ki = unit / ns, sl = unit % ns;
        const uint32_t key = keys[ki];
        const uint32_t i_lo = min(sl * per_slice, n), i_hi = min(i_lo + per_slice, n);

        uint4 r0 = make_uint4(0, 0, 0, 0), r1 = make_uint4(0, 0, 0, 0);
        for (int i = tid; i < ACC_WORDS / 4; i += OM_THREADS)
            reinterpret_cast<uint4 *>(sm.acc)[i] = make_uint4(0, 0, 0, 0);
        if (tid == 0) sm.anyfull = 0;
        FoldState f;
        __syncthreads();

        for (uint32_t c0 = i_lo; c0 < i_hi; c0 += OM_CHUNK) {
            const uint32_t np = many_gather(sm, S, idx, n, key, c0, min(c0 + OM_CHUNK, i_hi));
            if (tid == 0) {
                uint32_t af = 0;
                for (uint32_t j = 0; j < np; j++) {
                    fold_step(f, sm.ptf[j], sm.ppos[j]);
                    af |= sm.ptf[j] & (PF_FULL_RUN | PF_FULL_BITSET);
                }
                if (af) sm.anyfull = 1;
            }
            many_accumulate(sm, S, np, r0, r1);
            __syncthreads();
        }
        // merge the register slice into the shared accumulator
        {
            uint4 *a4 = reinterpret_cast<uint4 *>(sm.acc);
            uint4 a = a4[tid], b = a4[tid + OM_THREADS];
            a.x |= r0.x; a.y |= r0.y; a.z |= r0.z; a.w |= r0.w;
            b.x |= r1.x; b.y |= r1.y; b.z |= r1.z; b.w |= r1.w;
            if (sm.anyfull) a = b = make_uint4(~0u, ~0u, ~0u, ~0u);  // a full container took part
            a4[tid] = a;
            a4[tid + OM_THREADS] = b;
        }
        __syncthreads();

        if (ns > 1) {
            // ---- split key: publish the partial union, the last slice finalises --------------
            uint32_t *g = scratch_acc + (size_t)ki * ACC_WORDS;
            for (int w = tid; w < ACC_WORDS; w += OM_THREADS) {
                const uint32_t v = sm.acc[w];
                if (v) atomicOr(g + w, v);
            }
            __threadfence();
            __syncthreads();
            if (tid == 0) sm.flag = (atomicAdd(scratch_tickets + ki, 1u) == ns - 1) ? 1u : 0u;
            __syncthreads();
            const bool last = sm.flag != 0;
            __syncthreads();
            if (!last) continue;
            __threadfence();
            for (int w = tid; w < ACC_WORDS; w += OM_THREADS) {
                sm.acc[w] = __ldcg(g + w);
                g[w] = 0;  // leave the scratch clean for the next call
            }
            if (tid == 0) scratch_tickets[ki] = 0;
            // the fold needs every participant's metadata, in input order
            f = FoldState();
            for (uint32_t c0 = 0; c0 < n; c0 += OM_CHUNK) {
                const uint32_t np = many_gather(sm, S, idx, n, key, c0, min(c0 + OM_CHUNK, n));
                if (tid == 0)
                    for (uint32_t j = 0; j < np; j++) fold_step(f, sm.ptf[j], sm.ppos[j]);
                __syncthreads();
            }
        }

        // ---- count -------------------------------------------------------------------------
        int c = 0, r = 0;
        for (int w = tid; w < ACC_WORDS; w += OM_THREADS) {
            const uint32_t x = sm.acc[w];
            const uint32_t prev = w ? (sm.acc[w - 1] >> 31) : 0u;
            c += __popc(x);
            r += __popc(x & ~((x << 1) | prev));
        }
        c = __reduce_add_sync(FULLMASK, c);
        r = __reduce_add_sync(FULLMASK, r);
        if (lane == 0) { sm.red[wid][0] = c; sm.red[wid][1] = r; }
        __syncthreads();
        int card = 0, nruns = 0;
        for (int w = 0; w < OM_THREADS / 32; w++) { card += sm.red[w][0]; nruns += sm.red[w][1]; }

        // ---- result type (thread 0 holds the fold state) ---------------------------------------
        if (tid == 0) {
            int t;
            if (f.m_total == 1) {
                // one input carries the key: clone, then container_repair_after_lazy
                // (containers.h:344-371); n == 1 is a plain copy (roaring.c:780-782)
                const int t1 = f.first_tf & 15;
                if (n == 1) t = t1;
                else if (t1 == T_RUN) t = rule_eff(card, nruns);
                else if (t1 == T_ARRAY) t = T_ARRAY;
                else t = rule_ab(card);
            } else if (f.run_full) {
                t = T_RUN;
            } else if (card == 65536 && f.any_inplace_bitset && !f.first_is_full_bitset) {
                t = 0x80;  // saturated with bitset steps: ordered replay decides
            } else {
                t = rule_ab(card);
            }
            sm.flag = (uint32_t)t;
            sm.aux = f.last_ib_pos;
        }
        __syncthreads();
        int otype = (int)sm.flag;
        __syncthreads();

        if (otype == 0x80) {
            // Saturated accumulator with in-place bitset steps: the reference turns it into the
            // full run iff some in-place bitset x bitset step observes cardinality 65536
            // (containers.h:1345-1352).  Prefix unions only grow, so that happens iff the union
            // of the inputs up to and including the LAST in-place bitset participant is already
            // full: one more (order-free) accumulation over that prefix decides.
            const uint32_t L = sm.aux;
            for (int i = tid; i < ACC_WORDS; i += OM_THREADS) sm.acc[i] = 0;
            uint4 q0 = make_uint4(0, 0, 0, 0), q1 = make_uint4(0, 0, 0, 0);
            __syncthreads();
            if (tid == 0) sm.rfull = 0;
            for (uint32_t c0 = 0; c0 <= L; c0 += OM_CHUNK) {
                const uint32_t np = many_gather(sm, S, idx, n, key, c0, min(c0 + OM_CHUNK, L + 1));
                if (tid == 0) {  // a full container in the prefix (its payload is not rasterised)
                    uint32_t af = 0;
                    for (uint32_t j = 0; j < np; j++) af |= sm.ptf[j] & (PF_FULL_RUN | PF_FULL_BITSET);
                    if (af) sm.rfull = 1;
                }
                many_accumulate(sm, S, np, q0, q1);
                __syncthreads();
            }
            const uint4 *a4 = reinterpret_cast<const uint4 *>(sm.acc);
            const uint4 a = a4[tid], b = a4[tid + OM_THREADS];
            const bool full = ((a.x | q0.x) & (a.y | q0.y) & (a.z | q0.z) & (a.w | q0.w) &
                               (b.x | q1.x) & (b.y | q1.y) & (b.z | q1.z) & (b.w | q1.w)) == 0xffffffffu;
            const bool became_run = __syncthreads_and(full) || sm.rfull != 0;
            for (int i = tid; i < ACC_WORDS; i += OM_THREADS) sm.acc[i] = 0xffffffffu;
            __syncthreads();
            otype = became_run ? T_RUN : T_BITSET;
        }

        // ---- emit ----------------------------------------------------------------------------
        const uint64_t off = (uint64_t)ki * BITSET_BYTES;
        uint8_t *dst = out.payload + off;
        uint32_t olen;
        if (otype == T_BITSET) {
            olen = 1024;
            for (int i = tid; i < ACC_WORDS / 4; i += OM_THREADS)
                reinterpret_cast<uint4 *>(dst)[i] = reinterpret_cast<const uint4 *>(sm.acc)[i];
        } else if (otype == T_ARRAY) {
            olen = (uint32_t)card;
            if (wid == 0) acc_emit_array(sm.acc, reinterpret_cast<uint16_t *>(dst), lane);
        } else {
            olen = (uint32_t)nruns;
            if (wid == 0) acc_emit_runs(sm.acc, reinterpret_cast<uint16_t *>(dst), lane);
        }
        if (tid == 0) {
            out.c_key[ki] = (uint16_t)key;
            out.c_type[ki] = (uint8_t)otype;
            out.c_card[ki] = (uint32_t)card;
            out.c_len[ki] = olen;
            out.c_off[ki] = off;
            out.c_src[ki] = SRC_NONE;
            if (card_per_key) card_per_key[key] = (uint32_t)card;
        }
        __syncthreads();
    }
    if (blockIdx.x == 0 && tid == 0) {
        out.bm_beg[0] = 0;
        out.bm_cnt[0] = nk;
    }
}

// Two register budgets of the same body: 2 CTAs/SM (no spills) and 3 CTAs/SM (more warps in
// flight to cover the gather / payload latency, a few spills).  RB200_OM_CTAS=2|3 selects.
__global__ void __launch_bounds__(OM_THREADS, 2)
k_or_many(SetView S, const uint32_t *__restrict__ idx, uint32_t n, const uint16_t *__restrict__ keys,
          uint32_t want_slices, uint32_t *scratch_acc, uint32_t *scratch_tickets, uint32_t scratch_keys,
          SetOut out, uint32_t *__restrict__ card_per_key, OpStats *st) {
    or_many_body(S, idx, n, keys, want_slices, scratch_acc, scratch_tickets, scratch_keys, out, card_per_key, st);
}
__global__ void __launch_bounds__(OM_THREADS, 3)
k_or_many_occ3(SetView S, const uint32_t *__restrict__ idx, uint32_t n, const uint16_t *__restrict__ keys,
               uint32_t want_slices, uint32_t *scratch_acc, uint32_t *scratch_tickets, uint32_t scratch_keys,
               SetOut out, uint32_t *__restrict__ card_per_key, OpStats *st) {
    or_many_body(S, idx, n, keys, want_slices, scratch_acc, scratch_tickets, scratch_keys, out, card_per_key, st);
}

// total cardinality of the one-bitmap result of or_many
__global__ void k_sum_cards(const uint32_t *__restrict__ c_card, const OpStats *st,
                            uint64_t *__restrict__ out) {
    __shared__ unsigned long long s[32];
    const uint32_t n = st->nk;
    unsigned long long v = 0;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) v += c_card[i];
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULLMASK, v, d);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int i = 0; i < (int)(blockDim.x >> 5); i++) t += s[i];
        out[0] = t;
    }
}

// ------------------------------------------------------------------------------ xor_many
// roaring_bitmap_xor_many (src/roaring.c:795-809): lazy_xor of x[0], x[1] (:2684-2761), then
// lazy_xor_inplace of every further input (:2763-2843), then repair (:2845).  Unlike OR, the
// container TYPE after each step depends on the type and cardinality of the accumulator before
// it (container_lazy_xor containers.h:1570-1654; container_lazy_ixor :1749-1776 -> eager
// container_ixor rules for everything but bitset x bitset), and a key whose accumulator
// becomes empty is removed and re-inserted as a clone by a later input.  So the fold is kept
// sequential per key: a CTA owns the key, applies one participant at a time to the shared
// 65536-bit accumulator (bitsets: word xor; arrays: atomicXor; runs: range flips), recounts
// cardinality and run starts, and thread 0 advances the (type, cardinality, runs) state with
// the same decide_type() rules as the pairwise XOR cells.
__global__ void __launch_bounds__(OM_THREADS, 2)
k_xor_many(SetView S, const uint32_t *__restrict__ idx, uint32_t n,
           const uint16_t *__restrict__ keys, uint8_t *__restrict__ t_type,
           uint32_t *__restrict__ t_card, uint32_t *__restrict__ t_len, uint8_t *slab, OpStats *st) {
    __shared__ __align__(16) ManySmem sm;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t nk = st->nk;
    for (;;) {
        if (tid == 0) sm.ki = (uint32_t)atomicAdd(&st->work_counter2, 1ull);
        __syncthreads();
        const uint32_t ki = sm.ki;
        __syncthreads();
        if (ki >= nk) break;
        const uint32_t key = keys[ki];
        for (int i = tid; i < ACC_WORDS; i += OM_THREADS) sm.acc[i] = 0;
        // fold state (thread 0): accumulator present?, its type, cardinality, run count
        bool have = false;
        int t_acc = 0;
        uint32_t card_acc = 0, nruns_acc = 0, m_total = 0, first_pos = 0;
        int card = 0, nruns = 0;
        __syncthreads();
        for (uint32_t c0 = 0; c0 < n; c0 += OM_CHUNK) {
            const uint32_t np = many_gather(sm, S, idx, n, key, c0, min(c0 + OM_CHUNK, n));
            for (uint32_t j = 0; j < np; j++) {
                const int t2 = sm.ptf[j] & 15;
                const uint32_t l2 = sm.plen[j];
                const uint8_t *p = S.payload + sm.poff[j];
                // ---- acc ^= participant j ------------------------------------------------
                if (t2 == T_BITSET) {
                    const uint4 *src = reinterpret_cast<const uint4 *>(p);
                    uint4 *a4 = reinterpret_cast<uint4 *>(sm.acc);
                    for (int k = tid; k < ACC_WORDS / 4; k += OM_THREADS) {
                        uint4 a = a4[k];
                        const uint4 q = __ldg(src + k);
                        a.x ^= q.x; a.y ^= q.y; a.z ^= q.z; a.w ^= q.w;
                        a4[k] = a;
                    }
                } else if (t2 == T_ARRAY) {
                    const uint16_t *arr = reinterpret_cast<const uint16_t *>(p);
                    for (uint32_t i = tid; i < l2; i += OM_THREADS) {
                        const uint32_t v = arr[i];
                        atomicXor(sm.acc + (v >> 5), 1u << (v & 31));
                    }
                } else {
                    const uint32_t *runs = reinterpret_cast<const uint32_t *>(p);
                    for (uint32_t i = tid; i < l2; i += OM_THREADS) {
                        const uint32_t r = __ldg(runs + i), s0 = r & 0xffffu, e0 = min(s0 + (r >> 16), 65535u);
                        const uint32_t ws = s0 >> 5, we = e0 >> 5;
                        const uint32_t m_lo = ~0u << (s0 & 31), m_hi = ~0u >> (31 - (e0 & 31));
                        if (ws == we) {
                            atomicXor(sm.acc + ws, m_lo & m_hi);
                        } else {
                            atomicXor(sm.acc + ws, m_lo);
                            for (uint32_t w = ws + 1; w < we; w++) atomicXor(sm.acc + w, ~0u);
                            atomicXor(sm.acc + we, m_hi);
                        }
                    }
                }
                __syncthreads();
                // ---- recount -----------------------------------------------------------------
                int c = 0, r = 0;
                for (int w = tid; w < ACC_WORDS; w += OM_THREADS) {
                    const uint32_t x = sm.acc[w];
                    const uint32_t prev = w ? (sm.acc[w - 1] >> 31) : 0u;
                    c += __popc(x);
                    r += __popc(x & ~((x << 1) | prev));
                }
                c = __reduce_add_sync(FULLMASK, c);
                r = __reduce_add_sync(FULLMASK, r);
                if (lane == 0) { sm.red[wid][0] = c; sm.red[wid][1] = r; }
                __syncthreads();
                card = 0;
                nruns = 0;
                for (int w = 0; w < OM_THREADS / 32; w++) { card += sm.red[w][0]; nruns += sm.red[w][1]; }
                // ---- advance the fold state (every thread computes the same values) ------------
                const uint32_t c2 = sm.pcard[j], pos = sm.ppos[j];
                if (!have) {
                    have = true;  // clone (roaring.c:2724-2745 / :2822-2834)
                    t_acc = t2;
                } else {
                    const bool non_inplace = (m_total == 1) && first_pos == 0 && pos == 1;
                    int t;
                    if (t_acc == T_BITSET && t2 == T_BITSET) {
                        t = T_BITSET;  // lazy in both variants (containers.h:1579-1585, 1757-1761)
                    } else if (non_inplace) {
                        // container_lazy_xor, containers.h:1570-1654
                        if (t_acc == T_ARRAY && t2 == T_ARRAY)
                            t = (card_acc + c2 <= 1024u) ? T_ARRAY : T_BITSET;  // mixed_xor.c:221-252
                        else if (t_acc == T_RUN && t2 == T_RUN)
                            t = rule_eff(card, nruns);
                        else if (t_acc == T_BITSET || t2 == T_BITSET)
                            t = T_BITSET;
                        else
                            t = T_RUN;  // array x run left as run (mixed_xor.c:145-174)
                    } else {
                        // container_lazy_ixor -> container_ixor: the eager cell rules
                        t = decide_type(OP_XOR, t_acc, t2, card_acc, c2, nruns_acc, l2, card, nruns);
                    }
                    t_acc = t;
                }
                if (m_total == 0) first_pos = pos;
                m_total++;
                if (card == 0) have = false;  // emptied: key removed (roaring.c:2714-2718, 2803-2808)
                card_acc = (uint32_t)card;
                nruns_acc = (t_acc == T_RUN) ? (uint32_t)nruns : (t_acc == T_ARRAY ? (uint32_t)card : 1024u);
                __syncthreads();
            }
        }
        // ---- repair (containers.h:344-371) and emit ---------------------------------------------
        int otype = 0;
        if (have) {
            if (n == 1) otype = t_acc;  // plain copy
            else if (t_acc == T_BITSET) otype = rule_ab(card);
            else if (t_acc == T_RUN) otype = rule_eff(card, nruns);
            else otype = T_ARRAY;
        }
        uint8_t *dst = slab + (uint64_t)ki * BITSET_BYTES;
        uint32_t olen = 0;
        if (otype == T_BITSET) {
            olen = 1024;
            for (int i = tid; i < ACC_WORDS / 4; i += OM_THREADS)
                reinterpret_cast<uint4 *>(dst)[i] = reinterpret_cast<const uint4 *>(sm.acc)[i];
        } else if (otype == T_ARRAY) {
            olen = (uint32_t)card;
            if (wid == 0) acc_emit_array(sm.acc, reinterpret_cast<uint16_t *>(dst), lane);
        } else if (otype == T_RUN) {
            olen = (uint32_t)nruns;
            if (wid == 0) acc_emit_runs(sm.acc, reinterpret_cast<uint16_t *>(dst), lane);
        }
        if (tid == 0) {
            t_type[ki] = (uint8_t)otype;
            t_card[ki] = (uint32_t)card;
            t_len[ki] = olen;
        }
        __syncthreads();
    }
}

// single CTA: drop the keys whose result is empty, build the one-bitmap directory
__global__ void __launch_bounds__(1024)
k_compact_dir(const uint16_t *__restrict__ keys, const uint8_t *__restrict__ t_type,
              const uint32_t *__restrict__ t_card, const uint32_t *__restrict__ t_len,
              SetOut out, OpStats *st) {
    __shared__ uint32_t s_w[32];
    __shared__ unsigned long long s_c[32];
    __shared__ uint32_t s_carry, s_total;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t nk = st->nk;
    if (tid == 0) s_carry = 0;
    unsigned long long csum = 0;
    __syncthreads();
    for (uint32_t base = 0; base < nk; base += 1024) {
        const uint32_t i = base + tid;
        const bool live = i < nk && t_type[i] != 0;
        const uint32_t v = live ? 1u : 0u;
        const uint32_t incl = warp_incl_scan(v, lane);
        if (lane == 31) s_w[wid] = incl;
        __syncthreads();
        if (wid == 0) {
            const uint32_t x = s_w[lane];
            const uint32_t sx = warp_incl_scan(x, lane);
            s_w[lane] = sx - x;
            if (lane == 31) s_total = sx;
        }
        __syncthreads();
        if (live) {
            const uint32_t o = s_carry + s_w[wid] + incl - v;
            out.c_key[o] = keys[i];
            out.c_type[o] = t_type[i];
            out.c_card[o] = t_card[i];
            out.c_len[o] = t_len[i];
            out.c_off[o] = (uint64_t)i * BITSET_BYTES;
            out.c_src[o] = SRC_NONE;
            csum += t_card[i];
        }
        __syncthreads();
        if (tid == 0) s_carry += s_total;
        __syncthreads();
    }
    for (int d = 16; d > 0; d >>= 1) csum += __shfl_xor_sync(FULLMASK, csum, d);
    if (lane == 0) s_c[wid] = csum;
    __syncthreads();
    if (tid == 0) {
        unsigned long long t = 0;
        for (int w = 0; w < 32; w++) t += s_c[w];
        out.bm_beg[0] = 0;
        out.bm_cnt[0] = s_carry;
        out.bm_card[0] = t;
        st->dir_cursor = s_carry;
    }
}

void launch_xor_many(const SetView &S, const uint32_t *idx, uint32_t n, const uint16_t *keys,
                     uint8_t *t_type, uint32_t *t_card, uint32_t *t_len, SetOut out, OpStats *st,
                     int sms, cudaStream_t s) {
    k_xor_many<<<sms * 2, OM_THREADS, 0, s>>>(S, idx, n, keys, t_type, t_card, t_len, out.payload, st);
    g_launches++;
    k_compact_dir<<<1, 1024, 0, s>>>(keys, t_type, t_card, t_len, out, st);
    g_launches++;
}

void launch_or_many(const SetView &S, const uint32_t *idx, uint32_t n, const uint16_t *keys,
                    uint32_t want_slices, uint32_t *scratch_acc, uint32_t *scratch_tickets,
                    uint32_t scratch_keys, SetOut out, uint32_t *card_per_key, OpStats *st,
                    int sms, cudaStream_t s) {
    static int ctas = 0;
    if (!ctas) {
        const char *e = getenv("RB200_OM_CTAS");
        ctas = (e && atoi(e) == 3) ? 3 : 2;
    }
    if (ctas == 3)
        k_or_many_occ3<<<sms * 3, OM_THREADS, 0, s>>>(S, idx, n, keys, want_slices, scratch_acc,
                                                      scratch_tickets, scratch_keys, out, card_per_key, st);
    else
        k_or_many<<<sms * 2, OM_THREADS, 0, s>>>(S, idx, n, keys, want_slices, scratch_acc,
                                                 scratch_tickets, scratch_keys, out, card_per_key, st);
    g_launches++;
    k_sum_cards<<<1, 1024, 0, s>>>(out.c_card, st, out.bm_card);
    g_launches++;
}

}  // namespace rb200
