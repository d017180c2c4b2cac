// rb200_many2.cu — N-way union (roaring_bitmap_or_many, src/roaring.c:775-790), second generation:
// a key-major index built once per call, then one streaming pass over the payloads.
//
//   k_many2_count   histogram of the participating containers per high-16 key (+ their bytes)
//   k_many2_scan    exclusive scan -> per-key segment of the index, list of live keys, and the
//                   work units: a key whose participants weigh more than SLICE_BYTES is split
//                   into several units (slices of its participant list) merged through a global
//                   scratch accumulator
//   k_many2_fill    index entries (m2_entry, rb200_common.h), grouped by key
//                   (order inside a key is arbitrary: nothing below needs it)
//   k_or_many2      work unit = (key, slice): the participants' payloads are staged into shared
//                   memory by TMA bulk copies (cp.async.bulk + one mbarrier per half of a 64 KiB
//                   ping-pong buffer, issued by one thread, whole containers per copy), so the
//                   loads of the next batch are in flight while the CTA consumes the current one:
//                   bitsets are ORed into registers (every thread owns 32 bytes of the 8 KiB),
//                   arrays and runs are rasterised into a shared accumulator by one warp each; the
//                   last slice of a key counts, picks the reference's result type and re-encodes.
//
// The reference folds the inputs left to right with lazy cells (roaring_bitmap_lazy_or :2509-2598,
// roaring_bitmap_lazy_or_inplace :2600-2682, container_lazy_or / container_lazy_ior
// include/roaring/containers/containers.h:1113-1215, 1333-1442) and repairs once (:2845).  The
// VALUE is order free; the result TYPE depends on the order only through a few order statistics
// of the participants' metadata, which are computed by reductions instead of a sequential replay:
//     first / second participant (smallest input positions), whether they are x[0], x[1] (their
//     combine is the non-in-place container_lazy_or, roaring.c:2535-2550: no "is full" shortcut),
//     F = the first in-place step that brings a full run (containers.h:1394-1399: the accumulator
//         becomes the full RUN and later inputs are skipped, roaring.c:2621),
//     L = the last in-place step before F whose input is a bitset: container_lazy_ior B,B computes
//         the cardinality and turns a saturated accumulator into the full run (:1342-1352) — so a
//         saturated union ends as RUN iff the union of the inputs up to and including L is
//         already full.  Inputs after L (arrays / runs only) go to a second accumulator, which
//         makes that test a popcount instead of a second pass over the payloads.
#include <stdlib.h>

#include "rb200_device.cuh"

namespace rb200 {

constexpr int M2_THREADS = 256;
constexpr int M2_STAGE = 256;                    // index entries staged per round
constexpr uint32_t M2_SLICE_BYTES = 384u << 10;  // payload bytes per work unit before a key is split
constexpr uint32_t M2_MAX_SLICES = 64;
constexpr uint32_t POS_NONE = 0xffffffffu;
#ifndef RB200_M2_FLAT_VECS
#define RB200_M2_FLAT_VECS 513
#endif
// Arrays of at least RB200_M2_MERGE_MIN values would merge same-word bits before the atomic.  Only
// arrays below 8 * M2_FLAT_VECS values reach that test, so with this default the merging arm never
// runs; deleting it still changes how the direct path of k_or_many2 is compiled and made that path
// ~4 % slower on configs[2] (H100 80GB HBM3, 700 W), so it stays until the flat list is retuned.
#ifndef RB200_M2_MERGE_MIN
#define RB200_M2_MERGE_MIN 100000
#endif
constexpr uint32_t M2_FLAT_VECS = RB200_M2_FLAT_VECS;   // arrays below this many 16-byte vectors go through the flat list

// ------------------------------------------------------------------------------ index
__global__ void __launch_bounds__(128)
k_many2_count(SetView S, const uint32_t *__restrict__ idx, uint32_t n, uint32_t key_lo, uint32_t key_hi,
              Many2Index ix) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = warp; i < n; i += nwarps) {
        const uint32_t b = idx ? idx[i] : i;
        const uint32_t c0 = S.bm_beg[b], nc = S.bm_cnt[b];
        for (uint32_t c = lane; c < nc; c += 32) {
            const uint32_t k = S.c_key[c0 + c];
            if (k < key_lo || k > key_hi) continue;
            // one atomic per container
            atomicAdd(ix.key_cu + k, m2_cu(1, m2_weight(round16(stored_bytes(S.c_type[c0 + c], S.c_len[c0 + c])) >> 4, ix.w_shift)));
        }
    }
}

// key-window form of the index build (inputs with long directories): a CTA owns windows of 32
// consecutive keys; thread t finds where window w starts in the (sorted) directory of bitmap t —
// keys are distinct, so position <= key - first key: a galloping search from that bound, 1-3 probes
// on dense directories — then a warp reads the <= 32 containers of (window, bitmap) in one
// coalesced access and counts them with SHARED-memory atomics.  No global atomic anywhere
// (the bitmap-major kernels above spend one L2 atomic per container, which dominates on the 13 M
// containers of config 3 at density 0.003).
constexpr int M2W_KEYS = 32, M2W_THREADS = 256;

// live key span of the participants -> key_fill[0] = largest key, key_fill[1] = 65535 - smallest key
__global__ void __launch_bounds__(256)
k_many2_span(SetView S, const uint32_t *__restrict__ idx, uint32_t n, uint32_t *__restrict__ span) {
    uint32_t hi = 0, lo_c = 0;
    bool any = false;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t b = idx ? idx[i] : i;
        const uint32_t nc = S.bm_cnt[b];
        if (!nc) continue;
        const uint32_t c0 = S.bm_beg[b];
        hi = max(hi, (uint32_t)S.c_key[c0 + nc - 1]);
        lo_c = max(lo_c, 65535u - (uint32_t)S.c_key[c0]);
        any = true;
    }
    hi = __reduce_max_sync(FULLMASK, hi);
    lo_c = __reduce_max_sync(FULLMASK, lo_c);
    if (__any_sync(FULLMASK, any) && (threadIdx.x & 31) == 0) {
        atomicMax(span, hi);
        atomicMax(span + 1, lo_c);
    }
}

// first directory position of bitmap (c0, nc) whose key is >= k0
__device__ __forceinline__ uint32_t window_lower_bound(const uint16_t *__restrict__ keys, uint32_t nc, uint32_t k0) {
    const uint32_t kfirst = keys[0];
    if (k0 <= kfirst) return 0;
    uint32_t lo = 0, hi = min(nc, k0 - kfirst), w = 1;
    while (lo < hi) {                      // gallop down from the bound
        uint32_t p = hi > w ? hi - w : 0u;
        if (p < lo) p = lo;
        if (keys[p] < k0) { lo = p + 1; break; }
        hi = p;
        w <<= 1;
    }
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (keys[mid] < k0) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

template <bool FILL>
__global__ void __launch_bounds__(M2W_THREADS)
k_many2_window(SetView S, const uint32_t *__restrict__ idx, uint32_t n, uint32_t key_lo, uint32_t key_hi,
               Many2Index ix, uint32_t nchunks, uint32_t *__restrict__ cnt_tab) {
    // work unit = (window of 32 keys, chunk of 256 input bitmaps); with several chunks the count pass
    // leaves the unit's per-key counts in cnt_tab and the fill pass starts a key's entries of chunk c
    // behind those of the chunks before it — still no atomic per container
    __shared__ uint32_t s_cnt[M2W_KEYS], s_b16[M2W_KEYS], s_start[M2W_KEYS];
    __shared__ uint32_t s_seg[M2W_THREADS], s_c0[M2W_THREADS], s_nc[M2W_THREADS];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t span_hi = min(ix.key_fill[0], key_hi), span_lo = max(65535u - ix.key_fill[1], key_lo);
    if (span_lo > span_hi) return;
    const uint32_t w0 = span_lo / M2W_KEYS, w1 = span_hi / M2W_KEYS;
    const uint32_t units = (w1 - w0 + 1) * nchunks;
    for (uint32_t u = blockIdx.x; u < units; u += gridDim.x) {
        const uint32_t w = w0 + u / nchunks, c = u % nchunks;
        const uint32_t k0 = w * M2W_KEYS, base = c * M2W_THREADS;
        if (tid < M2W_KEYS) {
            s_cnt[tid] = 0;
            s_b16[tid] = 0;
            if (FILL) {
                uint32_t st = ix.key_start[k0 + tid];
                for (uint32_t cc = 0; cc < c; cc++) st += cnt_tab[(size_t)(u - c + cc) * M2W_KEYS + tid];
                s_start[tid] = st;
            }
        }
        {   // every thread: where the window starts in one bitmap's directory
            const uint32_t i = base + tid;
            uint32_t nc = 0, c0 = 0, seg = 0;
            if (i < n) {
                const uint32_t b = idx ? idx[i] : i;
                nc = S.bm_cnt[b];
                c0 = S.bm_beg[b];
                if (nc) {
                    if ((uint32_t)S.c_key[c0 + nc - 1] < k0) nc = 0;   // directory ends before the window
                    else seg = window_lower_bound(S.c_key + c0, nc, k0);
                }
            }
            s_seg[tid] = seg;
            s_c0[tid] = c0;
            s_nc[tid] = nc;
        }
        __syncthreads();
        const uint32_t m = min((uint32_t)M2W_THREADS, n - base);
        for (uint32_t q = wid; q < m; q += M2W_THREADS / 32) {
            const uint32_t nc = s_nc[q], p = s_seg[q] + lane;
            if (p >= nc) continue;                     // (whole warp when the bitmap has nothing here)
            const uint32_t cix = s_c0[q] + p;
            const uint32_t k = S.c_key[cix];
            if (k >= k0 + M2W_KEYS || k < key_lo || k > key_hi) continue;
            const uint32_t t = S.c_type[cix], l = S.c_len[cix];
            if (!FILL) {
                atomicAdd(&s_cnt[k - k0], 1u);
                atomicAdd(&s_b16[k - k0], round16(stored_bytes(t, l)) >> 4);
            } else {
                const uint32_t slot = s_start[k - k0] + atomicAdd(&s_cnt[k - k0], 1u);
                ix.ent[slot] = m2_entry(S.c_off[cix], base + q, l, m2_tf(t, l, S.c_card[cix] & CARD_MASK));
            }
        }
        __syncthreads();
        if (!FILL && tid < M2W_KEYS && k0 + tid <= 65535u) {
            const unsigned long long packed = m2_cu(s_cnt[tid], m2_weight(s_b16[tid], ix.w_shift));
            if (nchunks == 1) {
                ix.key_cu[k0 + tid] = packed;
            } else {
                if (packed) atomicAdd(ix.key_cu + k0 + tid, packed);   // one atomic per (unit, live key)
                cnt_tab[(size_t)u * M2W_KEYS + tid] = s_cnt[tid];
            }
        }
        __syncthreads();
    }
}

// single CTA, 1024 threads: tiles of 4096 keys, 4 consecutive keys per thread (coalesced), running carries
__device__ __forceinline__ uint32_t key_units(unsigned long long cu, uint32_t w_shift, uint32_t slice_kib) {
    const uint32_t c = m2_cu_count(cu);
    if (!c) return 0;
    const uint32_t kib = m2_cu_weight_kib(cu, w_shift);
    uint32_t s = (kib + slice_kib - 1) / slice_kib;
    const uint32_t by_cnt = (c + 3) >> 2;
    if (s > by_cnt) s = by_cnt;
    if (s > M2_MAX_SLICES) s = M2_MAX_SLICES;
    if (s < 1) s = 1;
    return s;
}

__global__ void __launch_bounds__(1024)
k_many2_scan(Many2Index ix, uint32_t scratch_slots, uint32_t max_units, uint32_t want_parallel, SetOut out,
             OpStats *st, int has_span) {
    __shared__ uint32_t s_w[32][4];
    __shared__ uint32_t s_carry[4];
    __shared__ uint32_t s_split;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t ntiles = has_span ? (min(ix.key_fill[0], 65535u) >> 12) + 1 : 16u;
    // pass 1: total weight -> slice size
    uint32_t w16 = 0;
    for (uint32_t t = 0; t < ntiles; t++) {
        const ulonglong2 *p = reinterpret_cast<const ulonglong2 *>(ix.key_cu + t * 4096 + tid * 4);
        const ulonglong2 a = p[0], b = p[1];
        const uint32_t ws = ix.w_shift;
        w16 += m2_cu_weight_kib(a.x, ws) + m2_cu_weight_kib(a.y, ws) + m2_cu_weight_kib(b.x, ws) + m2_cu_weight_kib(b.y, ws);   // KiB, to stay inside 32 bits
    }
    w16 = __reduce_add_sync(FULLMASK, w16);
    if (lane == 0) s_w[wid][0] = w16;
    if (tid < 4) s_carry[tid] = 0;
    __syncthreads();
    if (tid == 0) {
        uint32_t total_kib = 0;
        for (int i = 0; i < 32; i++) total_kib += s_w[i][0];
        // few heavy keys: split them so that the grid has ~want_parallel units (measured: units of
        // ~384 KiB beat both finer and coarser ones at every density of config 3)
        uint32_t slice_kib = M2_SLICE_BYTES >> 10;
        if (want_parallel && total_kib / slice_kib < want_parallel) {
            slice_kib = total_kib / want_parallel;
            if (slice_kib < 32) slice_kib = 32;
        }
        s_split = slice_kib;
    }
    __syncthreads();
    const uint32_t slice_kib = s_split;
    // pass 2: per key start / live index / slices / units, tile by tile
    for (uint32_t t = 0; t < 16; t++) {
        const uint32_t key0 = t * 4096 + tid * 4;
        if (t >= ntiles) {   // beyond the span: empty keys
            *reinterpret_cast<uint4 *>(ix.key_count + key0) = make_uint4(0, 0, 0, 0);
            continue;
        }
        const ulonglong2 *p = reinterpret_cast<const ulonglong2 *>(ix.key_cu + key0);
        const ulonglong2 a = p[0], b = p[1];
        const unsigned long long cu[4] = {a.x, a.y, b.x, b.y};
        uint32_t c[4], s[4];
        uint32_t cnt = 0, live = 0, units = 0, nsplit = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            c[k] = m2_cu_count(cu[k]);
            s[k] = key_units(cu[k], ix.w_shift, slice_kib);
            cnt += c[k];
            live += c[k] ? 1u : 0u;
            units += s[k];
            nsplit += s[k] > 1 ? 1u : 0u;
        }
        const uint32_t icnt = warp_incl_scan(cnt, lane), ilive = warp_incl_scan(live, lane),
                       iu = warp_incl_scan(units, lane), is = warp_incl_scan(nsplit, lane);
        __syncthreads();                       // s_w of the previous tile consumed
        if (lane == 31) { s_w[wid][0] = icnt; s_w[wid][1] = ilive; s_w[wid][2] = iu; s_w[wid][3] = is; }
        __syncthreads();
        uint32_t e = s_carry[0] + icnt - cnt, ki = s_carry[1] + ilive - live, u = s_carry[2] + iu - units,
                 sp = s_carry[3] + is - nsplit;
        for (int w = 0; w < wid; w++) { e += s_w[w][0]; ki += s_w[w][1]; u += s_w[w][2]; sp += s_w[w][3]; }
        __syncthreads();                       // carries read by everyone
        if (tid == 1023) { s_carry[0] = e + cnt; s_carry[1] = ki + live; s_carry[2] = u + units; s_carry[3] = sp + nsplit; }
        uint32_t st4[4];
#pragma unroll
        for (int k = 0; k < 4; k++) { st4[k] = e; e += c[k]; }
        *reinterpret_cast<uint4 *>(ix.key_start + key0) = make_uint4(st4[0], st4[1], st4[2], st4[3]);
        *reinterpret_cast<uint4 *>(ix.key_count + key0) = make_uint4(c[0], c[1], c[2], c[3]);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (!c[k]) continue;
            uint32_t slot = POS_NONE;
            if (s[k] > 1) {
                // a split key needs a scratch slot and room in the unit table; else it stays whole
                // (the unit numbering must not depend on this decision: units were reserved)
                if (sp < scratch_slots && u + s[k] <= max_units) slot = sp;
                sp++;
            }
            ix.keys[ki] = (uint16_t)(key0 + k);
            ix.key_slices[ki] = slot == POS_NONE ? 1u : s[k];
            ix.key_scratch[ki] = slot;
            ix.unit_first[ki] = u;
            // reserved-but-unused units of an unsplit heavy key are marked idle
            for (uint32_t q = 0; q < s[k] && u + q < max_units; q++)
                ix.unit_ki[u + q] = (slot == POS_NONE && q > 0) ? POS_NONE : ki;
            u += s[k];
            ki++;
        }
    }
    __syncthreads();
    if (tid == 0) {
        st->nk = s_carry[1];
        st->units = s_carry[2] < max_units ? s_carry[2] : max_units;
        out.bm_beg[0] = 0;
        out.bm_cnt[0] = s_carry[1];
    }
}

__global__ void __launch_bounds__(128)
k_many2_fill(SetView S, const uint32_t *__restrict__ idx, uint32_t n, uint32_t key_lo, uint32_t key_hi,
             Many2Index ix) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = warp; i < n; i += nwarps) {
        const uint32_t b = idx ? idx[i] : i;
        const uint32_t c0 = S.bm_beg[b], nc = S.bm_cnt[b];
        for (uint32_t c = lane; c < nc; c += 32) {
            const uint32_t k = S.c_key[c0 + c];
            if (k < key_lo || k > key_hi) continue;
            const uint32_t slot = ix.key_start[k] + atomicAdd(ix.key_fill + k, 1u);
            const uint32_t l = S.c_len[c0 + c];
            ix.ent[slot] = m2_entry(S.c_off[c0 + c], i, l, m2_tf(S.c_type[c0 + c], l, S.c_card[c0 + c] & CARD_MASK));   // ONE 16-byte store
        }
    }
}

// Order statistics of the reference's fold, once per key (warp per live key): the main kernel's
// work units (several per heavy key) only read the four words.
//   fold_first / fold_second : (position << 8 | type flags) of the two earliest participants
//   fold_F : first in-place step that brings a full run (POS_NONE: none)
//   fold_L : last in-place bitset step before F (POS_NONE: none)
__global__ void __launch_bounds__(128)
k_many2_fold(Many2Index ix, const OpStats *st) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t nk = st->nk;
    for (uint32_t ki = warp; ki < nk; ki += nwarps) {
        const uint32_t key = ix.keys[ki];
        const uint32_t e0 = ix.key_start[key], m = ix.key_count[key];
        unsigned long long m1 = ~0ull, m2 = ~0ull;
        for (uint32_t e = lane; e < m; e += 32) {
            const uint4 en = ix.ent[e0 + e];
            const unsigned long long v = ((unsigned long long)en.y << 8) | m2_entry_tf(en);
            if (v < m1) { m2 = m1; m1 = v; }
            else if (v < m2) m2 = v;
        }
        unsigned long long first = m1;
        for (int d = 16; d > 0; d >>= 1) { const unsigned long long o = __shfl_xor_sync(FULLMASK, first, d); first = o < first ? o : first; }
        unsigned long long second = m1 == first ? m2 : m1;
        for (int d = 16; d > 0; d >>= 1) { const unsigned long long o = __shfl_xor_sync(FULLMASK, second, d); second = o < second ? o : second; }
        const uint32_t pos1 = (uint32_t)(first >> 8), tf1 = (uint32_t)(first & 0xff);
        const uint32_t pos2 = (uint32_t)(second >> 8), tf2 = (uint32_t)(second & 0xff);
        const int t1 = tf1 & 15, t2 = tf2 & 15;
        bool decided = (tf1 & (TF_FULL_RUN | TF_FULL_BITSET)) != 0;
        const bool non_inplace = m >= 2 && pos1 == 0 && pos2 == 1;   // roaring.c:2535-2550
        uint32_t inplace_from = pos1;
        if (non_inplace) {
            decided = (t1 != T_BITSET && t2 != T_BITSET) ? (tf2 & TF_FULL_RUN) != 0 : ((tf2 | tf1) & TF_FULL_RUN) != 0;
            inplace_from = pos2;
        }
        uint32_t F = POS_NONE, L = POS_NONE;
        if (m >= 2 && !decided) {
            uint32_t f = POS_NONE;
            for (uint32_t e = lane; e < m; e += 32) {
                const uint4 en = ix.ent[e0 + e];
                const uint32_t p = en.y;
                if (p > inplace_from && (m2_entry_tf(en) & TF_FULL_RUN)) f = min(f, p);
            }
            F = __reduce_min_sync(FULLMASK, f);
            uint32_t l = 0;   // position + 1, 0 = none
            for (uint32_t e = lane; e < m; e += 32) {
                const uint4 en = ix.ent[e0 + e];
                const uint32_t p = en.y;
                if (p > inplace_from && p < F && (m2_entry_tf(en) & 15) == T_BITSET) l = max(l, p + 1);
            }
            l = __reduce_max_sync(FULLMASK, l);
            if (l) L = l - 1;
        }
        if (lane == 0) {
            ix.fold_first[ki] = first;
            ix.fold_second[ki] = second;
            ix.fold_F[ki] = F;
            ix.fold_L[ki] = L;
        }
    }
}

// ------------------------------------------------------------------------------ reduction
constexpr uint32_t M2_HALF = 32u << 10;   // bytes of one staging half (two halves: ping / pong)
constexpr uint32_t M2_HALF_ENTRIES = 128;  // participants staged per half at most

struct Many2Smem {
    uint32_t acc[ACC_WORDS];    // union of the inputs up to L (or of all of them when L is not needed)
    uint32_t acc2[ACC_WORDS];   // union of the inputs after L
    uint64_t bar[2];            // mbarriers of the two halves: "the bytes have landed"
    uint64_t ebar[2];           // mbarriers of the two halves: "all eight warps are done with the half"
    uint32_t h_last[2];         // the half holds the last entries of the round
    uint16_t h_bs[2][M2_HALF_ENTRIES], h_ar[2][M2_HALF_ENTRIES];   // staged bitsets / arrays+runs of a half (entry ids)
    uint32_t h_soff[M2_STAGE];  // byte offset of a staged entry inside its half
    uint32_t h_nbs[2], h_nar[2], h_big[2];
    uint16_t bs_list[M2_STAGE], ar_list[M2_STAGE];   // direct path: staged bitsets / runs + larger arrays of a round
    uint32_t nbs, nar;
    uint32_t s_vend[M2_STAGE];  // direct path: inclusive prefix of the 16-byte vectors of the staged ARRAYS (entry order)
    unsigned long long s_off[M2_STAGE];
    uint32_t s_len[M2_STAGE];
    uint32_t s_pos[M2_STAGE];
    uint8_t s_tf[M2_STAGE];
    unsigned long long red64[M2_THREADS / 32];
    uint32_t red32[M2_THREADS / 32][2];
    uint32_t unit, flag;
    unsigned long long first, second;
    uint32_t F, L, any_ib;
};

// min over the block of a u64 (all threads get the result); two barriers
__device__ __forceinline__ unsigned long long block_min64(Many2Smem &sm, unsigned long long v) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int d = 16; d > 0; d >>= 1) {
        const unsigned long long o = __shfl_xor_sync(FULLMASK, v, d);
        v = o < v ? o : v;
    }
    __syncthreads();
    if (lane == 0) sm.red64[wid] = v;
    __syncthreads();
    unsigned long long r = sm.red64[0];
#pragma unroll
    for (int w = 1; w < M2_THREADS / 32; w++) r = sm.red64[w] < r ? sm.red64[w] : r;
    return r;
}

// TMA = true: operands staged by bulk copies (bitset-dominated inputs); false: direct global loads
// (array-dominated inputs, where a bulk copy per small container costs more than it hides)
#ifndef RB200_M2_MINB
#define RB200_M2_MINB 4   // resident CTAs per SM of the direct path (register budget 64 at 4)
#endif
template <bool TMA>
__global__ void __launch_bounds__(M2_THREADS, TMA ? 2 : RB200_M2_MINB)
k_or_many2(SetView S, Many2Index ix, uint32_t n, uint32_t *__restrict__ scratch, uint32_t *__restrict__ tickets,
           SetOut out, uint32_t *__restrict__ card_per_key, OpStats *st) {
    extern __shared__ __align__(128) uint8_t m2_smem_raw[];
    Many2Smem &sm = *reinterpret_cast<Many2Smem *>(m2_smem_raw);
    uint8_t(*ring)[M2_HALF] = reinterpret_cast<uint8_t(*)[M2_HALF]>(m2_smem_raw + ((sizeof(Many2Smem) + 127) & ~(size_t)127));
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t nunits = st->units;
    if (TMA && tid == 0) {
        mbar_init(&sm.bar[0], 1);
        mbar_init(&sm.bar[1], 1);
        mbar_init(&sm.ebar[0], M2_THREADS / 32);
        mbar_init(&sm.ebar[1], M2_THREADS / 32);
        mbar_fence_init();
    }
    uint32_t ph0 = 0, ph1 = 0;   // phase parity of the two staging halves (every thread tracks both)
    uint32_t fills0 = 0, fills1 = 0;   // fills issued per half (thread 0)
    __syncthreads();
    if (tid == 0) sm.unit = (uint32_t)atomicAdd(&st->work_counter2, 1ull);
    for (;;) {
        __syncthreads();
        const uint32_t unit = sm.unit;
        __syncthreads();
        // the next ticket is drawn now: its latency hides behind this unit's work
        if (tid == 0) sm.unit = (uint32_t)atomicAdd(&st->work_counter2, 1ull);
        if (unit >= nunits) break;
        const uint32_t ki = ix.unit_ki[unit];
        if (ki == POS_NONE) continue;   // reserved for a key that could not be split
        const uint32_t key = ix.keys[ki], ns = ix.key_slices[ki], sl = unit - ix.unit_first[ki];
        const uint32_t e0 = ix.key_start[key], m = ix.key_count[key];

        // ---- order statistics of the fold: computed once per key by k_many2_fold ------------------
        const unsigned long long first = ix.fold_first[ki], second = ix.fold_second[ki];
        const uint32_t pos1 = (uint32_t)(first >> 8), tf1 = (uint32_t)(first & 0xff);
        const uint32_t pos2 = (uint32_t)(second >> 8), tf2 = (uint32_t)(second & 0xff);
        const int t1 = tf1 & 15, t2 = tf2 & 15;
        bool run_full = (tf1 & TF_FULL_RUN) != 0;
        bool decided = (tf1 & (TF_FULL_RUN | TF_FULL_BITSET)) != 0;
        bool first_full_bitset = (tf1 & TF_FULL_BITSET) != 0;
        const bool non_inplace = m >= 2 && pos1 == 0 && pos2 == 1;   // roaring.c:2535-2550
        if (non_inplace) {
            first_full_bitset = false;
            if (t1 != T_BITSET && t2 != T_BITSET) run_full = (tf2 & TF_FULL_RUN) != 0;   // c1 -> bitset, lazy_ior(B, c2)
            else run_full = ((tf2 | tf1) & TF_FULL_RUN) != 0;                            // container_lazy_or copies a full run
            decided = run_full;
        }
        uint32_t L = POS_NONE;             // POS_NONE: no prefix test needed, everything goes to acc
        bool any_ib = false;
        if (m >= 2 && !decided) {
            if (ix.fold_F[ki] != POS_NONE) run_full = true;
            const uint32_t l = ix.fold_L[ki];
            if (l != POS_NONE) {
                any_ib = true;
                if (!run_full) L = l;
            }
        }

        // ---- accumulate this unit's slice of the participants ---------------------------------
        uint4 r0 = make_uint4(0, 0, 0, 0), r1 = make_uint4(0, 0, 0, 0);
        for (int i = tid; i < ACC_WORDS / 4; i += M2_THREADS) {
            reinterpret_cast<uint4 *>(sm.acc)[i] = make_uint4(0, 0, 0, 0);
            reinterpret_cast<uint4 *>(sm.acc2)[i] = make_uint4(0, 0, 0, 0);
        }
        const uint32_t per = (m + ns - 1) / ns;
        const uint32_t s_lo = min(sl * per, m), s_hi = min(s_lo + per, m);
        uint32_t anyfull = 0, anyfull_pre = 0;   // bit flags, merged over the block at the end
        for (uint32_t base = s_lo; base < s_hi; base += M2_STAGE) {
            __syncthreads();
            const uint32_t e = base + tid;
            const uint32_t R = min((uint32_t)M2_STAGE, s_hi - base);   // entries of this round
            if (!TMA && tid == 0) { sm.nbs = 0; sm.nar = 0; }
            if (!TMA) __syncthreads();
            uint32_t my_vec = 0;
            if (tid < M2_STAGE && e < s_hi) {
                const uint4 en = ix.ent[e0 + e];
                const uint32_t tf = m2_entry_tf(en), p = en.y;
                sm.s_off[tid] = m2_entry_off(en);
                sm.s_len[tid] = en.z;
                sm.s_pos[tid] = p;
                sm.s_tf[tid] = (uint8_t)tf;
                if (tf & (TF_FULL_RUN | TF_FULL_BITSET)) {
                    anyfull = 1;
                    if (L != POS_NONE && p <= L) anyfull_pre = 1;
                }
                if (!TMA) {
                    if ((tf & 15) == T_BITSET) sm.bs_list[atomicAdd(&sm.nbs, 1u)] = (uint16_t)tid;
                    else if ((tf & 15) == T_ARRAY && en.z < 8 * M2_FLAT_VECS) my_vec = (en.z + 7) >> 3;
                    else if (!(tf & TF_FULL_RUN)) sm.ar_list[atomicAdd(&sm.nar, 1u)] = (uint16_t)tid;
                }
            }
            if (!TMA) {   // block scan of the array vectors (entry order)
                const uint32_t inc = warp_incl_scan(my_vec, lane);
                if (lane == 31) sm.red32[wid][0] = inc;
                __syncthreads();
                uint32_t pre = 0;
                for (int w = 0; w < wid; w++) pre += sm.red32[w][0];
                sm.s_vend[tid] = pre + inc;
            }
            __syncthreads();
            if (!TMA) {
                // bitsets: registers, four containers in flight per thread (all of them are <= L)
                const uint32_t nbs = sm.nbs;
                for (uint32_t j = 0; j < nbs; j += 4) {
                    uint4 qa[4], qb[4];
#pragma unroll
                    for (int k = 0; k < 4; k++)
                        if (j + k < nbs) {
                            const uint4 *src = reinterpret_cast<const uint4 *>(S.payload + sm.s_off[sm.bs_list[j + k]]);
                            qa[k] = __ldg(src + tid);
                            qb[k] = __ldg(src + tid + M2_THREADS);
                        }
#pragma unroll
                    for (int k = 0; k < 4; k++)
                        if (j + k < nbs) {
                            r0.x |= qa[k].x; r0.y |= qa[k].y; r0.z |= qa[k].z; r0.w |= qa[k].w;
                            r1.x |= qb[k].x; r1.y |= qb[k].y; r1.z |= qb[k].z; r1.w |= qb[k].w;
                        }
                }
                // small arrays: the 16-byte vectors of ALL of them as one flat list, a thread per vector
                // (two in flight): every lane loads whatever the container sizes are — a warp per
                // container left 18 of 32 lanes idle on the ~110-value arrays of the sparse densities
                // (arrays that fill a warp's 32 lanes anyway stay on the warp path below: the flat
                //  list for all sizes was slower at d = 0.03)
                const uint32_t V = sm.s_vend[M2_STAGE - 1];
                for (uint32_t x0 = 4 * tid; x0 < V; x0 += 4 * M2_THREADS) {
                    // four CONSECUTIVE vectors per thread: one search, then a linear walk; all four loads in flight
                    uint32_t q = 0, hi = R;   // first entry whose inclusive prefix exceeds x0
                    while (q < hi) {
                        const uint32_t mid = (q + hi) >> 1;
                        if (sm.s_vend[mid] > x0) hi = mid;
                        else q = mid + 1;
                    }
                    uint4 qv[4];
                    uint32_t left[4], ent[4];
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const uint32_t x = x0 + k;
                        left[k] = 0;
                        if (x < V) {
                            while (sm.s_vend[q] <= x) q++;
                            const uint32_t n = sm.s_len[q], i = x - (sm.s_vend[q] - ((n + 7) >> 3));
                            ent[k] = q;
                            left[k] = n - i * 8;
                            qv[k] = __ldg(reinterpret_cast<const uint4 *>(S.payload + sm.s_off[q]) + i);
                        }
                    }
#pragma unroll
                    for (int k = 0; k < 4; k++)
                        if (left[k]) {
                            uint32_t *dst = (L != POS_NONE && sm.s_pos[ent[k]] > L) ? sm.acc2 : sm.acc;
                            if (sm.s_len[ent[k]] < (uint32_t)RB200_M2_MERGE_MIN) acc_or_vec_sparse(dst, qv[k], left[k]);
                            else acc_apply_vec<0>(dst, qv[k], left[k]);
                        }
                }
                // runs and larger arrays: one warp per container, shared-memory atomics on the accumulator
                const uint32_t nar = sm.nar;
                for (uint32_t j = wid; j < nar; j += M2_THREADS / 32) {
                    const uint32_t q = sm.ar_list[j];
                    uint32_t *dst = (L != POS_NONE && sm.s_pos[q] > L) ? sm.acc2 : sm.acc;
                    const uint8_t *p = S.payload + sm.s_off[q];
                    if ((sm.s_tf[q] & 15) == T_ARRAY) acc_apply_array<0, APPLY_NONE, 1>(dst, p, sm.s_len[q], lane);
                    else acc_apply_runs<0, true>(dst, p, sm.s_len[q], lane);
                }
                continue;
            }
            // ---- two-half pipeline without block-wide barriers: thread 0 is the producer (packs entries
            // into a half, arms its "full" mbarrier with the byte count, issues the bulk copies); every
            // warp consumes a half as soon as its bytes have landed and then arrives on the half's
            // "empty" mbarrier; thread 0 refills the half once all eight warps have arrived.
            uint32_t next = 0;   // next entry of the round to stage (thread 0 only)
            auto fill = [&](int h) {   // thread 0 only
                const uint32_t fills = h ? fills1 : fills0;
                if (fills) mbar_wait(&sm.ebar[h], (fills - 1) & 1);   // the previous content has been consumed
                uint32_t bytes = 0, nbs = 0, nar = 0, big = POS_NONE;
                while (next < R && nbs + nar < M2_HALF_ENTRIES) {
                    const uint32_t tf = sm.s_tf[next], t = tf & 15;
                    const uint32_t sz = (tf & TF_FULL_RUN) ? 0u : round16(stored_bytes((int)t, sm.s_len[next]));
                    if (sz > M2_HALF) {   // an oversized run container (unoptimised input): straight from global
                        if (nbs + nar == 0 && big == POS_NONE) { big = next; next++; }
                        break;
                    }
                    if (bytes + sz > M2_HALF) break;
                    sm.h_soff[next] = bytes;
                    if (sz) {
                        if (t == T_BITSET) sm.h_bs[h][nbs++] = (uint16_t)next;
                        else sm.h_ar[h][nar++] = (uint16_t)next;
                    }
                    bytes += sz;
                    next++;
                }
                sm.h_nbs[h] = nbs;
                sm.h_nar[h] = nar;
                sm.h_big[h] = big;
                sm.h_last[h] = next >= R ? 1u : 0u;
                mbar_arrive_expect_tx(&sm.bar[h], bytes);
                for (uint32_t k = 0; k < nbs; k++) {
                    const uint32_t q = sm.h_bs[h][k];
                    bulk_copy_g2s(ring[h] + sm.h_soff[q], S.payload + sm.s_off[q], BITSET_BYTES, &sm.bar[h]);
                }
                for (uint32_t k = 0; k < nar; k++) {
                    const uint32_t q = sm.h_ar[h][k];
                    bulk_copy_g2s(ring[h] + sm.h_soff[q], S.payload + sm.s_off[q],
                                  round16(stored_bytes(sm.s_tf[q] & 15, sm.s_len[q])), &sm.bar[h]);
                }
                if (h) fills1++; else fills0++;
            };
            if (tid == 0) {
                fill(0);
                if (next < R) fill(1);
            }
            for (int h = 0;; h ^= 1) {
                mbar_wait(&sm.bar[h], h ? ph1 : ph0);
                if (h) ph1 ^= 1; else ph0 ^= 1;
                const uint32_t nbs = sm.h_nbs[h], nar = sm.h_nar[h];
                for (uint32_t j = 0; j < nbs; j += 2) {
                    const uint4 *s0 = reinterpret_cast<const uint4 *>(ring[h] + sm.h_soff[sm.h_bs[h][j]]);
                    const uint4 a0 = s0[tid], b0 = s0[tid + M2_THREADS];
                    r0.x |= a0.x; r0.y |= a0.y; r0.z |= a0.z; r0.w |= a0.w;
                    r1.x |= b0.x; r1.y |= b0.y; r1.z |= b0.z; r1.w |= b0.w;
                    if (j + 1 < nbs) {
                        const uint4 *s1 = reinterpret_cast<const uint4 *>(ring[h] + sm.h_soff[sm.h_bs[h][j + 1]]);
                        const uint4 a1 = s1[tid], b1 = s1[tid + M2_THREADS];
                        r0.x |= a1.x; r0.y |= a1.y; r0.z |= a1.z; r0.w |= a1.w;
                        r1.x |= b1.x; r1.y |= b1.y; r1.z |= b1.z; r1.w |= b1.w;
                    }
                }
                for (uint32_t j = wid; j < nar; j += M2_THREADS / 32) {
                    const uint32_t q = sm.h_ar[h][j];
                    uint32_t *dst = (L != POS_NONE && sm.s_pos[q] > L) ? sm.acc2 : sm.acc;
                    const uint8_t *p = ring[h] + sm.h_soff[q];
                    if ((sm.s_tf[q] & 15) == T_ARRAY) acc_apply_array_s<0>(dst, p, sm.s_len[q], lane);
                    else acc_apply_runs_s<0, true>(dst, p, sm.s_len[q], lane);
                }
                const uint32_t big = sm.h_big[h];
                if (big != POS_NONE) {   // oversized run container: every warp takes a share, from global
                    uint32_t *dst = (L != POS_NONE && sm.s_pos[big] > L) ? sm.acc2 : sm.acc;
                    const uint32_t nr = sm.s_len[big], per_w = (nr + M2_THREADS / 32 - 1) / (M2_THREADS / 32);
                    const uint32_t r_lo = min((uint32_t)wid * per_w, nr), r_hi = min(r_lo + per_w, nr);
                    if (r_hi > r_lo)
                        acc_apply_runs<0, true>(dst, S.payload + sm.s_off[big] + 4ull * r_lo, r_hi - r_lo, lane);
                }
                const uint32_t last = sm.h_last[h];
                __syncwarp();
                if (lane == 0) mbar_arrive(&sm.ebar[h]);          // this warp is done with the half
                if (tid == 0 && !last && next < R) fill(h);       // (waits for all eight warps first)
                __syncwarp();
                if (last) break;
            }
        }
        __syncthreads();
        anyfull = __syncthreads_or(anyfull);
        anyfull_pre = __syncthreads_or(anyfull_pre);
        // registers -> shared accumulator
        {
            uint4 *a4 = reinterpret_cast<uint4 *>(sm.acc);
            uint4 a = a4[tid], b = a4[tid + M2_THREADS];
            a.x |= r0.x; a.y |= r0.y; a.z |= r0.z; a.w |= r0.w;
            b.x |= r1.x; b.y |= r1.y; b.z |= r1.z; b.w |= r1.w;
            a4[tid] = a;
            a4[tid + M2_THREADS] = b;
        }
        __syncthreads();

        if (ns > 1) {
            // ---- split key: publish the partial unions, the last slice finalises --------------
            uint32_t *g = scratch + (size_t)ix.key_scratch[ki] * (2 * ACC_WORDS + 32);
            for (int w = tid; w < ACC_WORDS; w += M2_THREADS) {
                const uint32_t v = sm.acc[w], v2 = sm.acc2[w];
                if (v) atomicOr(g + w, v);
                if (v2) atomicOr(g + ACC_WORDS + w, v2);
            }
            if (tid == 0 && (anyfull | anyfull_pre)) atomicOr(g + 2 * ACC_WORDS, (anyfull ? 1u : 0u) | (anyfull_pre ? 2u : 0u));
            __threadfence();
            __syncthreads();
            if (tid == 0) sm.flag = (atomicAdd(tickets + ix.key_scratch[ki], 1u) == ns - 1) ? 1u : 0u;
            __syncthreads();
            if (!sm.flag) continue;
            __threadfence();
            for (int w = tid; w < ACC_WORDS; w += M2_THREADS) {
                sm.acc[w] = __ldcg(g + w);
                sm.acc2[w] = __ldcg(g + ACC_WORDS + w);
                g[w] = 0;   // leave the scratch clean for the next call
                g[ACC_WORDS + w] = 0;
            }
            const uint32_t fl = __ldcg(g + 2 * ACC_WORDS);
            anyfull = fl & 1u;
            anyfull_pre = fl & 2u;
            __syncthreads();
            if (tid == 0) { g[2 * ACC_WORDS] = 0; tickets[ix.key_scratch[ki]] = 0; }
        }

        // ---- count: cardinality of the prefix union, then of the whole union (+ run starts) -----
        int cpre = 0;
        if (L != POS_NONE)
            for (int w = tid; w < ACC_WORDS; w += M2_THREADS) cpre += __popc(sm.acc[w]);
        __syncthreads();
        for (int w = tid; w < ACC_WORDS; w += M2_THREADS) {
            uint32_t x = sm.acc[w] | sm.acc2[w];
            if (anyfull) x = ~0u;   // a full container took part (full runs are not rasterised)
            sm.acc[w] = x;
        }
        __syncthreads();
        int c = 0, r = 0;
        for (int w = tid; w < ACC_WORDS; w += M2_THREADS) {
            const uint32_t x = sm.acc[w];
            const uint32_t prev = w ? (sm.acc[w - 1] >> 31) : 0u;
            c += __popc(x);
            r += __popc(x & ~((x << 1) | prev));
        }
        c = __reduce_add_sync(FULLMASK, c);
        r = __reduce_add_sync(FULLMASK, r);
        cpre = __reduce_add_sync(FULLMASK, cpre);
        if (lane == 0) { sm.red32[wid][0] = (uint32_t)c; sm.red32[wid][1] = (uint32_t)r; sm.red64[wid] = (unsigned long long)cpre; }
        __syncthreads();
        int card = 0, nruns = 0, card_pre = 0;
        for (int w = 0; w < M2_THREADS / 32; w++) {
            card += (int)sm.red32[w][0];
            nruns += (int)sm.red32[w][1];
            card_pre += (int)sm.red64[w];
        }

        // ---- result type (every thread computes the same value) ------------------------------
        int otype;
        if (m == 1) {
            // one input carries the key: clone, then container_repair_after_lazy
            // (containers.h:344-371); n == 1 is a plain copy (roaring.c:780-782)
            if (n == 1) otype = t1;
            else if (t1 == T_RUN) otype = rule_eff(card, nruns);
            else if (t1 == T_ARRAY) otype = T_ARRAY;
            else otype = rule_ab(card);
        } else if (run_full) {
            otype = T_RUN;
        } else if (card == 65536 && any_ib && !first_full_bitset) {
            // saturated with in-place bitset steps: full run iff the union up to L was already full
            otype = (anyfull_pre || card_pre == 65536) ? T_RUN : T_BITSET;
        } else {
            otype = rule_ab(card);
        }

        // ---- emit ----------------------------------------------------------------------------
        const uint64_t off = (uint64_t)ki * BITSET_BYTES;
        uint8_t *dst = out.payload + off;
        uint32_t olen;
        if (otype == T_BITSET) {
            olen = 1024;
            for (int i = tid; i < ACC_WORDS / 4; i += M2_THREADS)
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
    }
}

// total cardinality of the one-bitmap result
__global__ void k_many2_sum_cards(const uint32_t *__restrict__ c_card, const OpStats *st, uint64_t *__restrict__ out) {
    __shared__ unsigned long long s[32];
    const uint32_t n = st->nk;
    unsigned long long v = 0;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) v += c_card[i];
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int i = 0; i < (int)(blockDim.x >> 5); i++) t += s[i];
        out[0] = t;
    }
}

void launch_or_many2(const SetView &S, const uint32_t *idx, uint32_t n, uint32_t key_lo, uint32_t key_hi,
                     const Many2Index &ix, uint32_t max_units, uint32_t *scratch, uint32_t *tickets,
                     uint32_t scratch_slots, SetOut out, uint32_t *card_per_key, OpStats *st, cudaStream_t s,
                     cudaEvent_t ev_kernel_start, bool use_tma, bool window_index, uint32_t *cnt_tab) {
    const uint32_t gw = (uint32_t)g_sm_count * 8;
    if (window_index) {
        // long directories: key-window index build, shared-memory counting, no global atomics
        launch_kernel(k_many2_span, grid_for(n, 256, 4), 256, 0, s, S, idx, n, ix.key_fill);
        const uint32_t nchunks = (n + M2W_THREADS - 1) / M2W_THREADS;
        launch_kernel(k_many2_window<false>, g_sm_count * 6, M2W_THREADS, 0, s, S, idx, n, key_lo, key_hi, ix, nchunks,
                      cnt_tab);
        launch_kernel(k_many2_scan, 1, 1024, 0, s, ix, scratch_slots, max_units, gw, out, st, 1);
        launch_kernel(k_many2_window<true>, g_sm_count * 6, M2W_THREADS, 0, s, S, idx, n, key_lo, key_hi, ix, nchunks,
                      cnt_tab);
    } else {
        launch_kernel(k_many2_count, gw, 128, 0, s, S, idx, n, key_lo, key_hi, ix);
        launch_kernel(k_many2_scan, 1, 1024, 0, s, ix, scratch_slots, max_units, gw, out, st, 0);
        launch_kernel(k_many2_fill, gw, 128, 0, s, S, idx, n, key_lo, key_hi, ix);
    }
    launch_kernel(k_many2_fold, gw, 128, 0, s, ix, st);
    if (ev_kernel_start) cudaEventRecord(ev_kernel_start, s);
    const size_t smem_direct = (sizeof(Many2Smem) + 127) & ~(size_t)127, smem_tma = smem_direct + 2 * M2_HALF;
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(k_or_many2<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_tma);
        cudaFuncSetAttribute(k_or_many2<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_direct);
        attr = true;
    }
    if (use_tma)
        launch_kernel(k_or_many2<true>, g_sm_count * 2, M2_THREADS, smem_tma, s, S, ix, n, scratch, tickets, out,
                      card_per_key, st);
    else
        launch_kernel(k_or_many2<false>, g_sm_count * RB200_M2_MINB, M2_THREADS, smem_direct, s, S, ix, n, scratch,
                      tickets, out, card_per_key, st);
    launch_kernel(k_many2_sum_cards, 1, 1024, 0, s, out.c_card, st, out.bm_card);
}

}  // namespace rb200
