// rb200_convert.cu — the producers / consumers next to the set-algebra path (SURVEY.md §8(f) row 3)
// as batch kernels over a whole resident set:
//
//   k_run_optimize   roaring_bitmap_run_optimize (src/roaring.c:1530 -> convert_run_optimize,
//                    src/containers/convert.c:217-321) and roaring_bitmap_remove_run_compression
//                    (src/roaring.c:1490): warp per container, choose the smallest encoding with the
//                    reference's size rule, re-encode.
//   k_values_*       roaring_bitmap_to_uint32_array (src/roaring_array.c:426): every bitmap of the
//                    set decoded to its sorted uint32 values in one device buffer.
#include "rb200_device.cuh"

namespace rb200 {

// number of maximal runs of a bitset container held in global memory
__device__ __forceinline__ int bitset_nruns_global(const uint8_t *p, int lane) {
    const uint32_t *w = reinterpret_cast<const uint32_t *>(p);
    int r = 0;
    for (int i = lane; i < ACC_WORDS; i += 32) {
        const uint32_t x = __ldg(w + i);
        const uint32_t prev = i ? (__ldg(w + i - 1) >> 31) : 0u;
        r += __popc(x & ~((x << 1) | prev));
    }
    return __reduce_add_sync(FULLMASK, r);
}

// number of runs of a sorted array (array_container_number_of_runs)
__device__ __forceinline__ int array_nruns_global(const uint8_t *p, uint32_t n, int lane) {
    const uint16_t *a = reinterpret_cast<const uint16_t *>(p);
    int r = 0;
    for (uint32_t i = lane; i < n; i += 32) r += (i == 0 || (uint32_t)a[i - 1] + 1 != a[i]) ? 1 : 0;
    return __reduce_add_sync(FULLMASK, r);
}

// mode 1: run_optimize; mode 0: remove_run_compression; mode 2: roaring_bitmap_repair_after_lazy
// (roaring.c:2845 -> container_repair_after_lazy, containers.h:344-371)
__global__ void __launch_bounds__(128)
k_run_optimize(SetView S, uint64_t nc, int mode, SetOut out, OpStats *st) {
    __shared__ __align__(16) uint32_t s_acc[4][ACC_WORDS];
    const int lane = threadIdx.x & 31;
    uint32_t *acc = s_acc[threadIdx.x >> 5];
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t c = warp; c < nc; c += nwarps) {
        const int t = S.c_type[c];
        const uint32_t len = S.c_len[c], card = S.c_card[c] & CARD_MASK;
        const uint8_t *p = S.payload + S.c_off[c];
        int nt = t;       // new type
        int nruns = 0;
        if (mode == 1) {  // convert.c:217-321
            if (t == T_RUN) {
                nt = rule_eff((int)card, (int)len);
            } else if (t == T_ARRAY) {
                nruns = array_nruns_global(p, len, lane);
                nt = (2 + 4 * nruns >= 2 * (int)card) ? T_ARRAY : T_RUN;
            } else {
                nruns = bitset_nruns_global(p, lane);
                nt = (BITSET_BYTES <= 2 + 4 * nruns) ? T_BITSET : T_RUN;
            }
        } else if (mode == 2) {  // bitset: recount, <= 4096 -> array; run: efficient container; array: as is
            if (t == T_BITSET) nt = rule_ab((int)card);
            else if (t == T_RUN) nt = rule_eff((int)card, (int)len);
        } else {  // remove_run_compression: runs -> array / bitset by cardinality (roaring.c:1490-1528)
            if (t == T_RUN) nt = rule_ab((int)card);
        }
        const uint32_t nlen = nt == T_BITSET ? 1024u : (nt == T_ARRAY ? card : (t == T_RUN ? len : (uint32_t)nruns));
        const uint32_t bytes = round16(stored_bytes(nt, nlen));
        unsigned long long off = 0;
        if (lane == 0) off = atomicAdd(&st->slab_cursor, (unsigned long long)bytes);
        off = __shfl_sync(FULLMASK, off, 0);
        uint8_t *dst = out.payload + off;
        if (nt == t) {
            warp_copy16(dst, p, stored_bytes(t, len), lane);
        } else {
            acc_load(acc, t, p, len, lane);
            if (nt == T_BITSET) acc_store_bitset(acc, dst, lane);
            else if (nt == T_ARRAY) acc_emit_array(acc, reinterpret_cast<uint16_t *>(dst), lane);
            else acc_emit_runs(acc, reinterpret_cast<uint16_t *>(dst), lane);
            __syncwarp();
        }
        if (lane == 0) {
            out.c_key[c] = S.c_key[c];
            out.c_type[c] = (uint8_t)nt;
            out.c_card[c] = card;
            out.c_len[c] = nlen;
            out.c_off[c] = off;
            out.c_src[c] = SRC_NONE;
        }
    }
}

__global__ void k_copy_bitmap_dir(SetView S, uint32_t nb, SetOut out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nb) {
        out.bm_beg[i] = S.bm_beg[i];
        out.bm_cnt[i] = S.bm_cnt[i];
        unsigned long long card = 0;
        const uint32_t c0 = S.bm_beg[i], n = S.bm_cnt[i];
        for (uint32_t k = 0; k < n; k++) card += S.c_card[c0 + k] & CARD_MASK;
        out.bm_card[i] = card;
    }
}

void launch_run_optimize(const SetView &S, uint32_t nb, uint64_t nc, int mode, SetOut out, OpStats *st,
                         cudaStream_t s) {
    if (nb) launch_kernel(k_copy_bitmap_dir, (nb + 127) / 128, 128, 0, s, S, nb, out);
    if (nc) launch_kernel(k_run_optimize, grid_for(nc, 4, 6), 128, 0, s, S, nc, mode, out, st);
}

// ------------------------------------------------------------------------------ to_uint32_array
// per bitmap: cardinality (for the caller's exclusive scan) ; per container: start index of its
// values inside the bitmap's output range
__global__ void __launch_bounds__(128)
k_values_measure(SetView S, uint32_t nb, uint64_t *__restrict__ bm_vals, uint64_t *__restrict__ c_start) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t b = warp; b < nb; b += nwarps) {
        const uint32_t c0 = S.bm_beg[b], n = S.bm_cnt[b];
        unsigned long long run = 0;
        for (uint32_t i0 = 0; i0 < n; i0 += 32) {
            const uint32_t i = i0 + lane;
            const uint32_t cd = i < n ? S.c_card[c0 + i] : 0u;
            const unsigned long long incl = warp_incl_scan((unsigned long long)cd, lane);
            if (i < n) c_start[(uint64_t)c0 + i] = run + incl - cd;
            run += __shfl_sync(FULLMASK, incl, 31);
        }
        if (lane == 0) bm_vals[b] = run;
    }
}

// warp per container: decode to uint32 values (key << 16 | low) at out[bm_off[b] + c_start[c]]
__global__ void __launch_bounds__(128)
k_values_write(SetView S, uint32_t nb, const uint64_t *__restrict__ bm_off,
               const uint64_t *__restrict__ c_start, const uint32_t *__restrict__ c_bitmap,
               uint64_t nc, uint32_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t c = warp; c < nc; c += nwarps) {
        const uint32_t b = c_bitmap[c];
        uint32_t *o = out + bm_off[b] + c_start[c];
        const int t = S.c_type[c];
        const uint32_t len = S.c_len[c];
        const uint32_t hi = (uint32_t)S.c_key[c] << 16;
        const uint8_t *p = S.payload + S.c_off[c];
        if (t == T_ARRAY) {
            const uint16_t *a = reinterpret_cast<const uint16_t *>(p);
            for (uint32_t i = lane; i < len; i += 32) o[i] = hi | a[i];
        } else if (t == T_RUN) {
            const uint32_t *runs = reinterpret_cast<const uint32_t *>(p);
            uint32_t base = 0;
            for (uint32_t k0 = 0; k0 < len; k0 += 32) {
                const uint32_t k = k0 + lane;
                const uint32_t r = k < len ? __ldg(runs + k) : 0u;
                const uint32_t s0 = r & 0xffffu, l = k < len ? (r >> 16) + 1 : 0u;
                const uint32_t incl = warp_incl_scan(l, lane);
                // long runs are written by the whole warp, short ones by their lane
                const bool big = l > 64;
                if (!big) { uint32_t *q = o + base + incl - l; for (uint32_t x = 0; x < l; x++) q[x] = hi | (s0 + x); }
                unsigned m = __ballot_sync(FULLMASK, big);
                while (m) {
                    const int src = __ffs(m) - 1;
                    m &= m - 1;
                    const uint32_t ss = __shfl_sync(FULLMASK, s0, src), ll = __shfl_sync(FULLMASK, l, src);
                    const uint32_t oo = __shfl_sync(FULLMASK, base + incl - l, src);
                    for (uint32_t x = lane; x < ll; x += 32) o[oo + x] = hi | (ss + x);
                }
                base += __shfl_sync(FULLMASK, incl, 31);
            }
        } else {
            const uint32_t *w = reinterpret_cast<const uint32_t *>(p);
            uint32_t base = 0;
            for (int it = 0; it < 64; it++) {
                const uint32_t wi = it * 32 + lane;
                uint32_t x = __ldg(w + wi);
                if (!__any_sync(FULLMASK, x != 0)) continue;
                const uint32_t cnt = __popc(x);
                const uint32_t incl = warp_incl_scan(cnt, lane);
                uint32_t *q = o + base + incl - cnt;
                const uint32_t vb = hi | (wi << 5);
                while (x) {
                    const int bit = __ffs(x) - 1;
                    x &= x - 1;
                    *q++ = vb | bit;
                }
                base += __shfl_sync(FULLMASK, incl, 31);
            }
        }
    }
}

// container -> bitmap index table
__global__ void k_container_bitmap(SetView S, uint32_t nb, uint32_t *__restrict__ c_bitmap) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t b = warp; b < nb; b += nwarps) {
        const uint32_t c0 = S.bm_beg[b], n = S.bm_cnt[b];
        for (uint32_t i = lane; i < n; i += 32) c_bitmap[c0 + i] = b;
    }
}

void launch_values_measure(const SetView &S, uint32_t nb, uint64_t *bm_vals, uint64_t *c_start,
                           uint32_t *c_bitmap, cudaStream_t s) {
    if (!nb) return;
    const uint32_t g = grid_for(nb, 4, 16);
    launch_kernel(k_values_measure, g, 128, 0, s, S, nb, bm_vals, c_start);
    launch_kernel(k_container_bitmap, g, 128, 0, s, S, nb, c_bitmap);
}

void launch_values_write(const SetView &S, uint32_t nb, const uint64_t *bm_off, const uint64_t *c_start,
                         const uint32_t *c_bitmap, uint64_t nc, uint32_t *out, cudaStream_t s) {
    if (!nc) return;
    launch_kernel(k_values_write, grid_for(nc, 4, 16), 128, 0, s, S, nb, bm_off, c_start, c_bitmap, nc, out);
}

}  // namespace rb200
