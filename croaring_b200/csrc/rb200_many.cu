// rb200_many.cu — N-way XOR (roaring_bitmap_xor_many, src/roaring.c:795-809) on sm_90a.
//
//   k_xor_many      CTA per key: gathers the participants in input order and folds them one at a
//                   time, with the reference's type rules at every step (details below)
//   k_compact_dir   single CTA: drops the keys whose result is empty, builds the directory
//
// (the N-way union, roaring_bitmap_or_many, is rb200_many2.cu)
#include "rb200_device.cuh"

namespace rb200 {

constexpr int OM_THREADS = 256;
constexpr int OM_CHUNK = 512;  // bitmaps gathered per round: two per thread

struct ManySmem {
    uint32_t acc[ACC_WORDS];
    unsigned long long poff[OM_CHUNK];
    uint32_t plen[OM_CHUNK];
    uint32_t ppos[OM_CHUNK];
    uint8_t ptype[OM_CHUNK];
    uint32_t pcard[OM_CHUNK];
    uint32_t warp_a[OM_THREADS / 32];
    int red[OM_THREADS / 32][2];
    uint32_t np, ki;
};

// Gather the participants of `key` among bitmaps [c0, c0+OM_CHUNK) ∩ [0,n) in input order.
__device__ __forceinline__ uint32_t many_gather(ManySmem &sm, const SetView &S,
                                                const uint32_t *__restrict__ idx, uint32_t n,
                                                uint32_t key, uint32_t c0, uint32_t c1) {
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    uint32_t cnt = 0;
    // two lower_bound searches per thread, advanced in lockstep so their loads overlap
    uint32_t b0[2], nb[2], lo[2], hi[2];
#pragma unroll
    for (int k = 0; k < 2; k++) {
        const uint32_t i = c0 + tid * 2 + k;
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
    unsigned long long off[2];
    bool hit[2];
#pragma unroll
    for (int k = 0; k < 2; k++) {
        hit[k] = lo[k] < nb[k] && S.c_key[b0[k] + lo[k]] == key;
        const uint32_t c = b0[k] + lo[k];
        ct[k] = hit[k] ? (uint32_t)S.c_type[c] : 0u;
        cl[k] = hit[k] ? S.c_len[c] : 0u;
        cc[k] = hit[k] ? S.c_card[c] : 0u;
        off[k] = hit[k] ? S.c_off[c] : 0ull;
        cnt += hit[k] ? 1u : 0u;
    }
    const uint32_t incl = warp_incl_scan(cnt, lane);
    if (lane == 31) sm.warp_a[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        const uint32_t va = lane < OM_THREADS / 32 ? sm.warp_a[lane] : 0u;
        const uint32_t sa = warp_incl_scan(va, lane);
        if (lane < OM_THREADS / 32) sm.warp_a[lane] = sa - va;
        if (lane == 31) sm.np = sa;
    }
    __syncthreads();
    uint32_t o = sm.warp_a[wid] + incl - cnt;
#pragma unroll
    for (int k = 0; k < 2; k++)
        if (hit[k]) {
            sm.poff[o] = off[k];
            sm.plen[o] = cl[k];
            sm.ppos[o] = c0 + tid * 2 + k;
            sm.ptype[o] = (uint8_t)ct[k];
            sm.pcard[o] = cc[k];
            o++;
        }
    __syncthreads();
    return sm.np;
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
                const int t2 = sm.ptype[j];
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

}  // namespace rb200
