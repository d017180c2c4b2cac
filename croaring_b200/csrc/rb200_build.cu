// rb200_build.cu — roaring_bitmap_of_ptr (src/roaring.c:195) for every bitmap of a batch, on the device.
//
// of_ptr inserts value by value through container_add (containers.h:489-521): a new key starts as an
// array, array_container_try_add (array.h:291-320) turns it into a bitset only when a NEW value meets
// a full array, a bitset never turns back and no run container is made.  So the result depends only
// on the set of distinct values: keys ascending, per key an array of the sorted distinct low halves
// when there are at most 4096 of them (rule_ab), a bitset otherwise.
//
// Input: values vals[off[b] .. off[b+1]) of bitmap b, any order, duplicates allowed.  Steps:
//   k_build_measure  tiles of BUILD_TILE positions: container starts per tile (valid once the
//                    values are sorted) and a flag when some bitmap's values decrease
//   (sort)           only when flagged: cub::DeviceSegmentedSort into a scratch buffer
//   k_build_emit     first position and key of every container (tile counts scanned to offsets)
//   k_build_slots    payload slot of every container, round16(min(2 * values, 8192)): never less than
//                    what is stored (an array holds <= values distinct u16, a bitset needs > 4096)
//   k_build_bitmaps  bm_beg / bm_cnt by binary search of the bitmap's first position
//   k_build_write    warp per container: distinct low halves compacted by ballot + scan into an
//                    array, or OR-ed into the warp's 8 KiB accumulator and stored as a bitset
// roaring64_bitmap_of_ptr (src/roaring64.c:523-620) adds through the same container_add per 48-bit
// key, so a 64-bit batch is first split into high-32 buckets (k_build_measure<uint64_t> counts them
// and flags unsorted input, k_build64_split writes the low halves and the bucket starts) and every
// bucket is then one sorted segment of the 32-bit steps above.
// CUB (NVIDIA's library shipped with the toolkit) is used for the sort and the two scans only, and
// only in this file.
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include "rb200_device.cuh"

namespace rb200 {

constexpr int BUILD_THREADS = 256, BUILD_ITEMS = 8;
constexpr uint64_t BUILD_TILE = (uint64_t)BUILD_THREADS * BUILD_ITEMS;
constexpr int BUILD_WARPS = BUILD_THREADS / 32;

// largest b in [lo, hi] with off[b] <= p (off[lo] <= p): the bitmap holding position p
__device__ __forceinline__ uint32_t find_bitmap(const uint64_t *__restrict__ off, uint32_t lo, uint32_t hi,
                                                uint64_t p) {
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo + 1) / 2;
        if (off[mid] <= p) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// Bitmaps of the first and last position of this block's tile, for every thread of the block.
__device__ __forceinline__ void tile_bitmaps(const uint64_t *__restrict__ off, uint32_t n, uint64_t N, uint64_t t0,
                                             uint32_t &b_lo, uint32_t &b_hi) {
    __shared__ uint32_t s_b[2];
    if (threadIdx.x == 0) {
        const uint64_t last = (t0 + BUILD_TILE < N ? t0 + BUILD_TILE : N) - 1;
        s_b[0] = find_bitmap(off, 0, n - 1, t0);
        s_b[1] = find_bitmap(off, s_b[0], n - 1, last);
    }
    __syncthreads();
    b_lo = s_b[0];
    b_hi = s_b[1];
}

// Position p (< N) of bitmap *b (advanced from the previous position of this thread): does it start
// a container (first value of its bitmap or a new high half), and do the values decrease there?
// T = uint32_t: the high half is the 16-bit key of a container; T = uint64_t: the high 32 bits of a
// 64-bit value, the bucket of roaring64's portable format.
template <typename T>
__device__ __forceinline__ bool position_starts(const T *__restrict__ v, const uint64_t *__restrict__ off,
                                                uint32_t &b, uint32_t b_hi, uint64_t p, T &x, bool &decreases) {
    constexpr int HALF = 4 * sizeof(T);
    if (off[b + 1] <= p) b = find_bitmap(off, b + 1, b_hi, p);
    x = v[p];
    const bool first = p == off[b];
    const T prev = first ? (T)0 : v[p - 1];
    decreases = !first && x < prev;
    return first || (x >> HALF) != (prev >> HALF);
}

// Container (T = uint32_t) or bucket (T = uint64_t) starts per tile (tile_cnt[tile]); *unsorted |= 1
// when some bitmap's values decrease, | 2 when that bitmap holds 2^31 values or more (more than one
// sort call can take).
template <typename T>
__global__ void __launch_bounds__(BUILD_THREADS)
k_build_measure(const T *__restrict__ v, const uint64_t *__restrict__ off, uint32_t n, uint64_t N,
                uint64_t *__restrict__ tile_cnt, uint32_t *unsorted) {
    __shared__ uint32_t s_cnt[BUILD_WARPS];
    const uint64_t t0 = (uint64_t)blockIdx.x * BUILD_TILE;
    uint32_t b, b_hi;
    tile_bitmaps(off, n, N, t0, b, b_hi);
    uint32_t starts = 0, bad = 0;
#pragma unroll 4
    for (int k = 0; k < BUILD_ITEMS; k++) {
        const uint64_t p = t0 + (uint64_t)k * BUILD_THREADS + threadIdx.x;
        if (p >= N) break;
        T x;
        bool dec;
        starts += position_starts(v, off, b, b_hi, p, x, dec) ? 1u : 0u;
        if (dec) bad |= (off[b + 1] - off[b] >= (1ull << 31)) ? 3u : 1u;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    starts = __reduce_add_sync(FULLMASK, starts);
    bad = __reduce_or_sync(FULLMASK, bad);
    // read before the atomic: a fully shuffled input would otherwise send one atomic per warp to one word
    if (lane == 0 && bad && (*(volatile uint32_t *)unsorted & bad) != bad) atomicOr(unsorted, bad);
    if (lane == 0) s_cnt[warp] = starts;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t s = 0;
        for (int w = 0; w < BUILD_WARPS; w++) s += s_cnt[w];
        tile_cnt[blockIdx.x] = s;
    }
}

// First position and key of every container; tile_base = exclusive scan of tile_cnt.
__global__ void __launch_bounds__(BUILD_THREADS)
k_build_emit(const uint32_t *__restrict__ v, const uint64_t *__restrict__ off, uint32_t n, uint64_t N,
             const uint64_t *__restrict__ tile_base, uint16_t *__restrict__ c_key, uint64_t *__restrict__ c_pos) {
    __shared__ uint32_t s_w[2][BUILD_WARPS];
    const uint64_t t0 = (uint64_t)blockIdx.x * BUILD_TILE;
    uint32_t b, b_hi;
    tile_bitmaps(off, n, N, t0, b, b_hi);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t base = tile_base[blockIdx.x];
    for (int k = 0; k < BUILD_ITEMS; k++) {   // striped: chunk k is positions t0 + k * 256 + [0, 256)
        const uint64_t p = t0 + (uint64_t)k * BUILD_THREADS + threadIdx.x;
        uint32_t x = 0;
        bool dec, start = false;
        if (p < N) start = position_starts<uint32_t>(v, off, b, b_hi, p, x, dec);
        const unsigned m = __ballot_sync(FULLMASK, start);
        if (lane == 0) s_w[k & 1][warp] = __popc(m);
        __syncthreads();   // s_w[k & 1] is rewritten two chunks later, after the next chunk's barrier
        uint32_t pre = 0, tot = 0;
#pragma unroll
        for (int w = 0; w < BUILD_WARPS; w++) {
            const uint32_t c = s_w[k & 1][w];
            pre += w < warp ? c : 0u;
            tot += c;
        }
        if (start) {
            const uint64_t c = base + pre + __popc(m & lanemask_lt());
            c_pos[c] = p;
            c_key[c] = (uint16_t)(x >> 16);
        }
        base += tot;
    }
}

// 64-bit values (tile_base = exclusive scan of k_build_measure<uint64_t>'s bucket starts): the low
// halves of every position go to lo[p]; the first position and the high 32 bits of every bucket to
// b_pos / b_high, compacted by ballot in position order.  The buckets of a sorted batch are then
// sorted 32-bit segments, the input of the 32-bit builder.
__global__ void __launch_bounds__(BUILD_THREADS)
k_build64_split(const uint64_t *__restrict__ v, const uint64_t *__restrict__ off, uint32_t n, uint64_t N,
                const uint64_t *__restrict__ tile_base, uint32_t *__restrict__ lo, uint64_t *__restrict__ b_pos,
                uint32_t *__restrict__ b_high) {
    __shared__ uint32_t s_w[2][BUILD_WARPS];
    const uint64_t t0 = (uint64_t)blockIdx.x * BUILD_TILE;
    uint32_t b, b_hi;
    tile_bitmaps(off, n, N, t0, b, b_hi);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t base = tile_base[blockIdx.x];
    for (int k = 0; k < BUILD_ITEMS; k++) {   // striped as in k_build_emit
        const uint64_t p = t0 + (uint64_t)k * BUILD_THREADS + threadIdx.x;
        uint64_t x = 0;
        bool dec, start = false;
        if (p < N) {
            start = position_starts<uint64_t>(v, off, b, b_hi, p, x, dec);
            lo[p] = (uint32_t)x;
        }
        const unsigned m = __ballot_sync(FULLMASK, start);
        if (lane == 0) s_w[k & 1][warp] = __popc(m);
        __syncthreads();
        uint32_t pre = 0, tot = 0;
#pragma unroll
        for (int w = 0; w < BUILD_WARPS; w++) {
            const uint32_t c = s_w[k & 1][w];
            pre += w < warp ? c : 0u;
            tot += c;
        }
        if (start) {
            const uint64_t c = base + pre + __popc(m & lanemask_lt());
            b_pos[c] = p;
            b_high[c] = (uint32_t)(x >> 32);
        }
        base += tot;
    }
}

__global__ void k_build_slots(const uint64_t *__restrict__ c_pos, uint64_t nc, uint64_t N, uint64_t *__restrict__ slot) {
    const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nc) return;
    const uint64_t cnt = (c + 1 < nc ? c_pos[c + 1] : N) - c_pos[c];
    slot[c] = round16(cnt < (uint64_t)MAX_ARRAY ? 2u * (uint32_t)cnt : (uint32_t)BITSET_BYTES);
}

// first container at or after position p
__device__ __forceinline__ uint64_t first_container(const uint64_t *__restrict__ c_pos, uint64_t lo, uint64_t hi,
                                                    uint64_t p) {
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (c_pos[mid] < p) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

__global__ void k_build_bitmaps(const uint64_t *__restrict__ off, uint32_t n, const uint64_t *__restrict__ c_pos,
                                uint64_t nc, uint32_t *__restrict__ bm_beg, uint32_t *__restrict__ bm_cnt) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    const uint64_t c0 = first_container(c_pos, 0, nc, off[b]);
    const uint64_t c1 = first_container(c_pos, c0, nc, off[b + 1]);
    bm_beg[b] = (uint32_t)c0;
    bm_cnt[b] = (uint32_t)(c1 - c0);
}

// Distinct values of positions [p0, p1) of a sorted run (the first position always counts):
// WRITE = false counts them, WRITE = true also stores their low halves at dst in order.
template <bool WRITE>
__device__ __forceinline__ uint32_t distinct_run(const uint32_t *__restrict__ v, uint64_t p0, uint64_t p1,
                                                 uint16_t *__restrict__ dst, int lane) {
    uint32_t d = 0, carry = 0;
    for (uint64_t i0 = p0; i0 < p1; i0 += 32) {
        const uint64_t i = i0 + lane;
        const bool valid = i < p1;
        const uint32_t x = valid ? __ldg(v + i) : 0u;
        uint32_t prev = __shfl_up_sync(FULLMASK, x, 1);
        if (lane == 0) prev = carry;
        const bool keep = valid && (i == p0 || x != prev);
        const unsigned m = __ballot_sync(FULLMASK, keep);
        if (WRITE && keep) dst[d + __popc(m & lanemask_lt())] = (uint16_t)x;
        d += __popc(m);
        carry = __shfl_sync(FULLMASK, x, 31);
    }
    return d;
}

// Warp per container (atomic tickets on st->work_counter).  Container c holds the sorted positions
// [c_pos[c], c_pos[c + 1]) (the last one ends at N); its slot starts at out.c_off[c].
__global__ void __launch_bounds__(128)
k_build_write(const uint32_t *__restrict__ v, const uint64_t *__restrict__ c_pos, uint64_t nc, uint64_t N,
              SetOut out, uint64_t slab_cap, OpStats *st) {
    __shared__ __align__(16) uint32_t s_acc[4][ACC_WORDS];
    const int lane = threadIdx.x & 31;
    uint32_t *acc = s_acc[threadIdx.x >> 5];
    unsigned long long payload = 0;   // container_size_in_bytes of this warp's containers
    for (;;) {
        unsigned long long c = 0;
        if (lane == 0) c = atomicAdd(&st->work_counter, 1ull);
        c = __shfl_sync(FULLMASK, c, 0);
        if (c >= nc) break;
        const uint64_t p0 = c_pos[c], p1 = c + 1 < nc ? c_pos[c + 1] : N, cnt = p1 - p0;
        const uint64_t off = out.c_off[c];
        const uint32_t slot = round16(cnt < (uint64_t)MAX_ARRAY ? 2u * (uint32_t)cnt : (uint32_t)BITSET_BYTES);
        if (off + slot > slab_cap) {   // cannot happen with the host's bound; never write past the slab
            if (lane == 0) atomicExch(&st->error, 2u);
            continue;
        }
        uint8_t *dst = out.payload + off;
        // more than 4096 positions: count first, duplicates may still leave an array (array.h:291-320)
        uint32_t d = cnt > (uint64_t)MAX_ARRAY ? distinct_run<false>(v, p0, p1, nullptr, lane) : 0u;
        int t;
        if (d <= (uint32_t)MAX_ARRAY) {
            t = T_ARRAY;
            d = distinct_run<true>(v, p0, p1, reinterpret_cast<uint16_t *>(dst), lane);
            for (uint32_t j = 2 * d + 2 * lane; j < round16(2 * d); j += 64)   // zero the 16-byte padding
                *reinterpret_cast<uint16_t *>(dst + j) = 0;
        } else {
            t = T_BITSET;
            acc_zero(acc, lane);
            __syncwarp();
            for (uint64_t i0 = p0; i0 < p1; i0 += 32) {
                const uint64_t i = i0 + lane;
                const bool valid = i < p1;
                const uint32_t x = valid ? __ldg(v + i) : 0u;
                const uint32_t w = valid ? (x & 0xffffu) >> 5 : 0xffffffffu;
                // sorted values: neighbouring lanes mostly share a word, so merge them before the atomic
                const unsigned grp = __match_any_sync(FULLMASK, w);
                const uint32_t bits = __reduce_or_sync(grp, valid ? 1u << (x & 31) : 0u);
                if (valid && lane == __ffs(grp) - 1) atomicOr(acc + w, bits);
            }
            __syncwarp();
            acc_store_bitset(acc, dst, lane);
            __syncwarp();
        }
        if (lane == 0) {
            out.c_type[c] = (uint8_t)t;
            out.c_card[c] = d;
            out.c_len[c] = t == T_BITSET ? 1024u : d;
            out.c_src[c] = SRC_NONE;
            payload += portable_bytes(t, d);
            if (c + 1 == nc) st->slab_cursor = off + slot;
        }
    }
    if (lane == 0 && payload) atomicAdd(&st->payload_bytes, payload);
}

__global__ void k_build_rel_offsets(const uint64_t *__restrict__ off, uint32_t nseg, int *__restrict__ rel) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= nseg) rel[i] = (int)(off[i] - off[0]);
}

// ------------------------------------------------------------------------------ launch wrappers
static inline uint32_t build_tiles(uint64_t N) { return (uint32_t)((N + BUILD_TILE - 1) / BUILD_TILE); }

uint64_t build_tile_count(uint64_t N) { return build_tiles(N); }

void launch_build_measure(const uint32_t *v, const uint64_t *off, uint32_t n, uint64_t N, uint64_t *tile_cnt,
                          uint32_t *unsorted, cudaStream_t s) {
    if (!N) return;
    launch_kernel(k_build_measure<uint32_t>, build_tiles(N), BUILD_THREADS, 0, s, v, off, n, N, tile_cnt, unsorted);
}

void launch_build64_measure(const uint64_t *v, const uint64_t *off, uint32_t n, uint64_t N, uint64_t *tile_cnt,
                            uint32_t *unsorted, cudaStream_t s) {
    if (!N) return;
    launch_kernel(k_build_measure<uint64_t>, build_tiles(N), BUILD_THREADS, 0, s, v, off, n, N, tile_cnt, unsorted);
}

void launch_build64_split(const uint64_t *v, const uint64_t *off, uint32_t n, uint64_t N, const uint64_t *tile_base,
                          uint32_t *lo, uint64_t *b_pos, uint32_t *b_high, cudaStream_t s) {
    if (!N) return;
    launch_kernel(k_build64_split, build_tiles(N), BUILD_THREADS, 0, s, v, off, n, N, tile_base, lo, b_pos, b_high);
}

void launch_build_emit(const uint32_t *v, const uint64_t *off, uint32_t n, uint64_t N, const uint64_t *tile_base,
                       uint16_t *c_key, uint64_t *c_pos, cudaStream_t s) {
    if (!N) return;
    launch_kernel(k_build_emit, build_tiles(N), BUILD_THREADS, 0, s, v, off, n, N, tile_base, c_key, c_pos);
}

void launch_build_slots(const uint64_t *c_pos, uint64_t nc, uint64_t N, uint64_t *slot, cudaStream_t s) {
    if (!nc) return;
    launch_kernel(k_build_slots, (uint32_t)((nc + 255) / 256), 256, 0, s, c_pos, nc, N, slot);
}

void launch_build_bitmaps(const uint64_t *off, uint32_t n, const uint64_t *c_pos, uint64_t nc, uint32_t *bm_beg,
                          uint32_t *bm_cnt, cudaStream_t s) {
    if (!n) return;
    launch_kernel(k_build_bitmaps, (n + 255) / 256, 256, 0, s, off, n, c_pos, nc, bm_beg, bm_cnt);
}

void launch_build_write(const uint32_t *v, const uint64_t *c_pos, uint64_t nc, uint64_t N, SetOut out,
                        uint64_t slab_cap, OpStats *st, cudaStream_t s) {
    if (!nc) return;
    // 6 x 32 KiB of accumulators per SM
    launch_kernel(k_build_write, grid_for(nc, 4, 6), 128, 0, s, v, c_pos, nc, N, out, slab_cap, st);
}

// Exclusive sum of n u64 (n < 2^31).  temp == nullptr: *temp_bytes receives the scratch size.
bool build_scan(void *temp, size_t *temp_bytes, const uint64_t *in, uint64_t *out, uint64_t n, cudaStream_t s) {
    const cudaError_t e = cub::DeviceScan::ExclusiveSum(temp, *temp_bytes, in, out, (int)n, s);
    if (temp) g_launches++;
    return e == cudaSuccess;
}

// Sort the values of segments [0, nseg) of a chunk (off: nseg + 1 absolute offsets in device memory,
// off[nseg] - off[0] < 2^31) from in + off[0] into out + off[0].  rel: nseg + 1 ints of scratch.
// temp == nullptr: *temp_bytes receives the scratch size (items = off[nseg] - off[0]).
template <typename T>
static bool sort_chunk(void *temp, size_t *temp_bytes, const T *in, T *out, const uint64_t *off, uint64_t first,
                       uint64_t items, uint32_t nseg, int *rel, cudaStream_t s) {
    if (temp) launch_kernel(k_build_rel_offsets, (nseg + 256) / 256, 256, 0, s, off, nseg, rel);
    const cudaError_t e = cub::DeviceSegmentedSort::SortKeys(temp, *temp_bytes, in + first, out + first, (int)items,
                                                             (int)nseg, rel, rel + 1, s);
    if (temp) g_launches++;
    return e == cudaSuccess;
}
bool build_sort_chunk(void *temp, size_t *temp_bytes, const uint32_t *in, uint32_t *out, const uint64_t *off,
                      uint64_t first, uint64_t items, uint32_t nseg, int *rel, cudaStream_t s) {
    return sort_chunk(temp, temp_bytes, in, out, off, first, items, nseg, rel, s);
}
bool build_sort_chunk(void *temp, size_t *temp_bytes, const uint64_t *in, uint64_t *out, const uint64_t *off,
                      uint64_t first, uint64_t items, uint32_t nseg, int *rel, cudaStream_t s) {
    return sort_chunk(temp, temp_bytes, in, out, off, first, items, nseg, rel, s);
}

}  // namespace rb200
