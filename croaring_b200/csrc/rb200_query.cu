// rb200_query.cu — batched point queries against a resident set (sm_90a): contains, rank, get_index
// and select of one value (or rank) per query, one warp per query.
//
//   k_query_cards  c_card & CARD_MASK of every directory entry as u64, the input of the set's
//                  c_cum scan (exclusive, n_containers + 1 entries; built once per set by the host)
//   k_query<KIND>  warp per query: the container by a 32-ary search of the bitmap's keys (SELECT: of
//                  its c_cum range), then the answer inside it —
//                    array   32-ary lower / upper bound over the u16 values, or the r-th value
//                    bitset  a lane per 32 words: popcounts summed (rank) or scanned (select), then
//                            the bit inside the found word
//                    run     the lanes stride the {start, len - 1} pairs, a scan of len + 1 gives
//                            rank, get_index and select in one pass
// Inside bitmap b the values before container c number c_cum[c] - c_cum[bm_beg[b]] (u64, modular:
// only entries inside the bitmap enter the difference), so no count is ever held in 32 bits.
//
// 64-bit sets: a 64-bit bitmap is a run of inner bitmaps, one per high-32 bucket.
//   k_query64_cards  the values of every inner bitmap from the inner c_cum, the input of the set's b_cum
//                    scan (exclusive, nbuckets + 1 entries; built once per set by the host)
//   k_query64<KIND>  warp per query: the bucket by a 32-ary search of the bitmap's highs (SELECT: of its
//                    b_cum range), then answer<KIND> on that inner bitmap, plus the buckets before it
//
// Reference semantics restated here (file:line relative to /root/reference):
//   roaring_bitmap_contains    include/roaring/roaring.h:478
//   roaring_bitmap_rank        src/roaring.c:2862 (values <= x)
//   roaring_bitmap_get_index   src/roaring.c:2916 (-1 when x is absent)
//   roaring_bitmap_select      src/roaring.c:2974 (0-based rank; false -> -1 here)
//   roaring64_bitmap_contains / rank / get_index / select   src/roaring64.c:682, 804, 827, 779 (a false
//                              return is found = 0, with the answer 2^64 - 1)
#include "rb200_device.cuh"

namespace rb200 {

namespace {

// The first i in [0, m) for which pred(i) is false, pred being true on a prefix of [0, m); m when it
// holds everywhere.  Every lane of the warp calls it with the same arguments and gets the answer.
// Each round tests 32 evenly spaced positions and keeps the gap after the last true one: a range of
// m shrinks to below m / 32, so 65536 positions take at most four rounds.
template <typename P>
__device__ __forceinline__ uint32_t warp_partition(uint32_t m, int lane, P pred) {
    uint32_t lo = 0, hi = m;
    while (lo < hi) {
        const uint32_t step = (hi - lo + 31) >> 5, p = lo + lane * step;
        const uint32_t t = __popc(__ballot_sync(FULLMASK, p < hi && pred(p)));
        if (!t) break;
        const uint32_t nhi = lo + t * step;
        lo += (t - 1) * step + 1;
        hi = nhi < hi ? nhi : hi;
    }
    return lo;
}

__device__ __forceinline__ uint32_t run_start(uint32_t r) { return r & 0xffffu; }
__device__ __forceinline__ uint32_t run_last(uint32_t r) { return (r & 0xffffu) + (r >> 16); }

// 0-based position of the (r + 1)-th set bit of w (r < popcount(w))
__device__ __forceinline__ uint32_t nth_bit(uint64_t w, uint32_t r) {
    const uint32_t lo = (uint32_t)w, hi = (uint32_t)(w >> 32), pl = __popc(lo);
    return r < pl ? __fns(lo, 0, (int)r + 1) : 32 + __fns(hi, 0, (int)(r - pl) + 1);
}

// Whether container c holds the low half v.
__device__ __forceinline__ bool contains_in(const SetView &S, uint32_t c, uint32_t v, int lane) {
    const int t = S.c_type[c];
    const uint32_t len = S.c_len[c];
    const uint8_t *p = S.payload + S.c_off[c];
    if (t == T_BITSET) return (reinterpret_cast<const uint64_t *>(p)[v >> 6] >> (v & 63)) & 1;
    if (t == T_ARRAY) {
        const uint16_t *a = reinterpret_cast<const uint16_t *>(p);
        const uint32_t i = warp_partition(len, lane, [&](uint32_t j) { return a[j] < v; });
        return i < len && a[i] == v;
    }
    const uint32_t *runs = reinterpret_cast<const uint32_t *>(p);
    const uint32_t k = warp_partition(len, lane, [&](uint32_t j) { return run_start(runs[j]) <= v; });
    return k && v <= run_last(runs[k - 1]);
}

// Values <= v in container c (0 .. 65536), and whether v is one of them.
__device__ __forceinline__ uint32_t rank_in(const SetView &S, uint32_t c, uint32_t v, int lane, bool &has) {
    const int t = S.c_type[c];
    const uint32_t len = S.c_len[c];
    const uint8_t *p = S.payload + S.c_off[c];
    if (t == T_ARRAY) {
        const uint16_t *a = reinterpret_cast<const uint16_t *>(p);
        const uint32_t u = warp_partition(len, lane, [&](uint32_t j) { return a[j] <= v; });
        has = u && a[u - 1] == v;
        return u;
    }
    if (t == T_BITSET) {
        // lane l counts words [32 l, 32 l + 32) up to word v >> 6, that word up to bit v & 63
        const uint4 *w4 = reinterpret_cast<const uint4 *>(p) + lane * 16;
        const uint32_t wv = v >> 6, first = lane * 32;
        uint32_t cnt = 0;
        if (first <= wv) {
            for (uint32_t k = 0; k < 16; k++) {
                const uint4 q = w4[k];
                const uint32_t j = first + 2 * k;   // words j and j + 1
                const uint64_t a = (uint64_t)q.y << 32 | q.x, b = (uint64_t)q.w << 32 | q.z;
                const uint64_t keep = (v & 63) == 63 ? ~0ull : (2ull << (v & 63)) - 1;
                cnt += j < wv ? __popcll(a) : j == wv ? __popcll(a & keep) : 0;
                cnt += j + 1 < wv ? __popcll(b) : j + 1 == wv ? __popcll(b & keep) : 0;
            }
        }
        has = (reinterpret_cast<const uint64_t *>(p)[wv] >> (v & 63)) & 1;
        return (uint32_t)warp_sum(cnt);
    }
    const uint32_t *runs = reinterpret_cast<const uint32_t *>(p);
    uint32_t cnt = 0;
    bool in = false;
    for (uint32_t i0 = 0; i0 < len; i0 += 32) {
        const uint32_t i = i0 + lane;
        const uint32_t r = i < len ? runs[i] : 0u;
        const bool live = i < len && run_start(r) <= v;
        if (live) {
            const uint32_t e = run_last(r) < v ? run_last(r) : v;
            cnt += e - run_start(r) + 1;
            in |= v <= run_last(r);
        }
        if (__ballot_sync(FULLMASK, i < len && run_start(r) > v)) break;   // the runs past v start here
    }
    has = __any_sync(FULLMASK, in);
    return (uint32_t)warp_sum(cnt);
}

// The low half of the value of rank r (0-based, r < the container's cardinality) in container c.
__device__ __forceinline__ uint32_t select_in(const SetView &S, uint32_t c, uint32_t r, int lane) {
    const int t = S.c_type[c];
    const uint32_t len = S.c_len[c];
    const uint8_t *p = S.payload + S.c_off[c];
    if (t == T_ARRAY) return reinterpret_cast<const uint16_t *>(p)[r];
    if (t == T_BITSET) {
        const uint64_t *w = reinterpret_cast<const uint64_t *>(p) + lane * 32;
        const uint4 *w4 = reinterpret_cast<const uint4 *>(w);
        uint32_t cnt = 0;
        for (uint32_t k = 0; k < 16; k++) cnt += popc4(w4[k]);
        const uint32_t incl = warp_incl_scan(cnt, lane);
        const unsigned owner = __ffs(__ballot_sync(FULLMASK, incl > r)) - 1;
        uint32_t out = 0;
        if ((unsigned)lane == owner) {
            uint32_t left = r - (incl - cnt);
            for (uint32_t j = 0; j < 32; j++) {
                const uint32_t pc = __popcll(w[j]);
                if (left < pc) {
                    out = lane * 2048 + j * 64 + nth_bit(w[j], left);
                    break;
                }
                left -= pc;
            }
        }
        return __shfl_sync(FULLMASK, out, owner);
    }
    const uint32_t *runs = reinterpret_cast<const uint32_t *>(p);
    uint32_t carry = 0;
    for (uint32_t i0 = 0; i0 < len; i0 += 32) {
        const uint32_t i = i0 + lane;
        const uint32_t rr = i < len ? runs[i] : 0u, n = i < len ? (rr >> 16) + 1 : 0u;
        const uint32_t incl = carry + warp_incl_scan(n, lane);
        const unsigned hit = __ballot_sync(FULLMASK, incl > r);
        if (hit) {
            const unsigned owner = __ffs(hit) - 1;
            return __shfl_sync(FULLMASK, run_start(rr) + (r - (incl - n)), owner);
        }
        carry = __shfl_sync(FULLMASK, incl, 31);
    }
    return 0;   // not reached: r is below the cardinality
}

template <int KIND>
__device__ __forceinline__ int64_t answer(const SetView &S, const uint64_t *c_cum, uint32_t b, uint32_t x, int lane) {
    const uint32_t beg = S.bm_beg[b], cnt = S.bm_cnt[b];
    if (KIND == Q_SELECT) {
        if (!cnt) return -1;
        const uint64_t base = c_cum[beg];
        if (x >= c_cum[beg + cnt] - base) return -1;
        // the container whose values reach past rank x
        const uint32_t i = warp_partition(cnt, lane, [&](uint32_t j) { return c_cum[beg + j + 1] - base <= x; });
        const uint32_t c = beg + i;
        const uint32_t lowv = select_in(S, c, (uint32_t)(x - (c_cum[c] - base)), lane);
        return (int64_t)((uint32_t)S.c_key[c] << 16 | lowv);
    }
    const uint32_t hk = x >> 16, v = x & 0xffffu;
    const uint32_t i = warp_partition(cnt, lane, [&](uint32_t j) { return S.c_key[beg + j] < hk; });
    const bool present = i < cnt && S.c_key[beg + i] == hk;
    if (KIND == Q_CONTAINS) return present && contains_in(S, beg + i, v, lane) ? 1 : 0;
    if (KIND == Q_GET_INDEX && !present) return -1;
    const uint64_t before = cnt ? c_cum[beg + i] - c_cum[beg] : 0;
    if (!present) return (int64_t)before;
    bool has;
    const uint32_t in = rank_in(S, beg + i, v, lane, has);
    if (KIND == Q_RANK) return (int64_t)(before + in);
    return has ? (int64_t)(before + in - 1) : -1;
}

template <int KIND>
__global__ void __launch_bounds__(256)
k_query(SetView S, const uint64_t *__restrict__ c_cum, uint32_t n_bitmaps, const uint32_t *__restrict__ idx,
        const uint32_t *__restrict__ vals, uint32_t n, int64_t *__restrict__ out, unsigned long long *bad) {
    const int lane = threadIdx.x & 31;
    const uint64_t nwarps = (gridDim.x * (uint64_t)blockDim.x) >> 5;
    for (uint64_t q = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5; q < n; q += nwarps) {
        const uint32_t b = idx ? idx[q] : (uint32_t)q, x = vals[q];
        int64_t r = -1;
        if (b < n_bitmaps) r = answer<KIND>(S, c_cum, b, x, lane);
        else if (lane == 0) atomicMin(bad, (unsigned long long)q);   // no directory read
        if (lane == 0) out[q] = r;
    }
}

__global__ void __launch_bounds__(256)
k_query_cards(const uint32_t *__restrict__ c_card, uint64_t nc, uint64_t *__restrict__ out) {
    const uint64_t stride = gridDim.x * (uint64_t)blockDim.x;
    for (uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; c <= nc; c += stride)
        out[c] = c < nc ? (uint64_t)(c_card[c] & CARD_MASK) : 0ull;
}

// The answer about x of the 64-bit bitmap whose buckets are [beg, beg + cnt) of the inner set (bucket j
// holding the values high[j] << 32 | v of the inner bitmap j): the bucket by a 32-ary search of the highs (SELECT:
// of the bucket prefix b_cum), then answer<KIND> inside it.  Empty buckets (results of x XOR x, of a
// removal) hold no container: contains and rank find nothing in them and their b_cum step is 0, so
// select never stops on one.  r: the answer, left as it is on a get_index or select miss, which returns
// false; contains returns its answer, rank true.
template <int KIND>
__device__ __forceinline__ bool answer64(const SetView &S, const uint64_t *c_cum, const uint64_t *b_cum,
                                         const uint32_t *high, uint32_t beg, uint32_t cnt, uint64_t x, int lane,
                                         uint64_t &r) {
    if (KIND == Q_SELECT) {
        const uint64_t base = b_cum[beg];
        if (x >= b_cum[beg + cnt] - base) return false;
        const uint32_t i = warp_partition(cnt, lane, [&](uint32_t j) { return b_cum[beg + j + 1] - base <= x; });
        // a bucket holds at most 2^32 values, so the rank inside it fits 32 bits
        const int64_t lo = answer<Q_SELECT>(S, c_cum, beg + i, (uint32_t)(x - (b_cum[beg + i] - base)), lane);
        r = (uint64_t)high[beg + i] << 32 | (uint32_t)lo;
        return true;
    }
    const uint32_t hx = (uint32_t)(x >> 32);
    const uint32_t i = warp_partition(cnt, lane, [&](uint32_t j) { return high[beg + j] < hx; });
    const bool present = i < cnt && high[beg + i] == hx;
    if (KIND == Q_CONTAINS) {
        r = present ? (uint64_t)answer<Q_CONTAINS>(S, c_cum, beg + i, (uint32_t)x, lane) : 0ull;
        return r != 0;
    }
    if (KIND == Q_GET_INDEX && !present) return false;
    const int64_t in = present ? answer<KIND>(S, c_cum, beg + i, (uint32_t)x, lane) : 0;
    if (in < 0) return false;   // get_index: x's bucket is there, x is not
    r = b_cum[beg + i] - b_cum[beg] + (uint64_t)in;   // (read after the inner answer: fewer live registers)
    return true;
}

// (256, 6): at most 42 registers, where ptxas's own choice of 32 for (256) spills the get_index path
template <int KIND>
__global__ void __launch_bounds__(256, 6)
k_query64(SetView S, const uint64_t *__restrict__ c_cum, const uint64_t *__restrict__ b_cum,
          const uint32_t *__restrict__ b_beg, const uint32_t *__restrict__ b_cnt, const uint32_t *__restrict__ high,
          uint32_t n64, const uint32_t *__restrict__ idx, const uint64_t *__restrict__ vals, uint32_t n,
          uint64_t *__restrict__ out, uint8_t *__restrict__ found, unsigned long long *bad) {
    const int lane = threadIdx.x & 31;
    const uint64_t nwarps = (gridDim.x * (uint64_t)blockDim.x) >> 5;
    for (uint64_t q = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5; q < n; q += nwarps) {
        const uint32_t b = idx ? idx[q] : (uint32_t)q;
        uint64_t r = ~0ull;   // a miss, and an index out of range
        bool hit = false;
        if (b < n64) hit = answer64<KIND>(S, c_cum, b_cum, high, b_beg[b], b_cnt[b], vals[q], lane, r);
        else if (lane == 0) atomicMin(bad, (unsigned long long)q);   // no directory read
        if (lane == 0) {
            out[q] = r;
            if (found) found[q] = hit;
        }
    }
}

// Values of every inner bitmap (bucket) from the inner set's c_cum, 0 for an empty one; nb + 1 entries,
// the last zero, the input of the set's b_cum scan.
__global__ void __launch_bounds__(256)
k_query64_cards(const uint32_t *__restrict__ bm_beg, const uint32_t *__restrict__ bm_cnt,
                const uint64_t *__restrict__ c_cum, uint64_t nb, uint64_t *__restrict__ out) {
    const uint64_t stride = gridDim.x * (uint64_t)blockDim.x;
    for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j <= nb; j += stride) {
        const uint32_t cnt = j < nb ? bm_cnt[j] : 0u;
        out[j] = cnt ? c_cum[bm_beg[j] + cnt] - c_cum[bm_beg[j]] : 0ull;   // (no c_cum without containers)
    }
}

}  // namespace

void launch_query(int kind, const SetView &S, const uint64_t *c_cum, uint32_t n_bitmaps, const uint32_t *idx,
                  const uint32_t *vals, uint32_t n, int64_t *out, unsigned long long *bad, cudaStream_t s) {
    if (!n) return;
    // a warp per query, 8 warps per block
    const dim3 grid = grid_for(n, 8, 8);
    switch (kind) {
        case Q_CONTAINS: launch_kernel(k_query<Q_CONTAINS>, grid, 256, 0, s, S, c_cum, n_bitmaps, idx, vals, n, out, bad); break;
        case Q_RANK: launch_kernel(k_query<Q_RANK>, grid, 256, 0, s, S, c_cum, n_bitmaps, idx, vals, n, out, bad); break;
        case Q_GET_INDEX: launch_kernel(k_query<Q_GET_INDEX>, grid, 256, 0, s, S, c_cum, n_bitmaps, idx, vals, n, out, bad); break;
        default: launch_kernel(k_query<Q_SELECT>, grid, 256, 0, s, S, c_cum, n_bitmaps, idx, vals, n, out, bad); break;
    }
}

void launch_query_cards(const uint32_t *c_card, uint64_t nc, uint64_t *out, cudaStream_t s) {
    launch_kernel(k_query_cards, grid_for(nc + 1, 256, 8), 256, 0, s, c_card, nc, out);
}

void launch_query64(int kind, const SetView &S, const uint64_t *c_cum, const uint64_t *b_cum, const uint32_t *b_beg,
                    const uint32_t *b_cnt, const uint32_t *high, uint32_t n64, const uint32_t *idx,
                    const uint64_t *vals, uint32_t n, uint64_t *out, uint8_t *found, unsigned long long *bad,
                    cudaStream_t s) {
    if (!n) return;
    const dim3 grid = grid_for(n, 8, 6);   // a warp per query, 8 warps per block
    const auto go = [&](auto kernel) {
        launch_kernel(kernel, grid, 256, 0, s, S, c_cum, b_cum, b_beg, b_cnt, high, n64, idx, vals, n, out, found, bad);
    };
    switch (kind) {
        case Q_CONTAINS: go(k_query64<Q_CONTAINS>); break;
        case Q_RANK: go(k_query64<Q_RANK>); break;
        case Q_GET_INDEX: go(k_query64<Q_GET_INDEX>); break;
        default: go(k_query64<Q_SELECT>); break;
    }
}

void launch_query64_cards(const uint32_t *bm_beg, const uint32_t *bm_cnt, const uint64_t *c_cum, uint64_t nb,
                          uint64_t *out, cudaStream_t s) {
    launch_kernel(k_query64_cards, grid_for(nb + 1, 256, 8), 256, 0, s, bm_beg, bm_cnt, c_cum, nb, out);
}

}  // namespace rb200
