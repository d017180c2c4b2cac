// rb200_fused.cu — ONE launch for a single small pair: the drop-in entry points
// roaring_bitmap_{and,or,xor,andnot}[_inplace] (src/roaring.c:731, 877, 1121, 1275, 812, 1063, 1200,
// 1342) called on one pair of host bitmaps.
//
// The batched path costs a single pair three launches, four copies and two host round trips
// (all latency).  Here the host packs both operands into one pinned block, ONE
// cudaMemcpyAsync moves it, ONE kernel — a single CTA, eight warps — plans the key merge
// (src/roaring.c:742-768, 896-951 as binary-search ranks, like k_plan_pairs), evaluates the cells
// with the very same cell_compute() as the batched kernel (one warp per cell, eight 8 KiB
// accumulators), compacts the result directory and writes directory AND payloads straight into
// mapped pinned host memory; a sequence word written last (after __threadfence_system) tells the
// host that everything has landed.  No intermediate set object, no download.
#include "rb200_device.cuh"
#include "rb200_cells.cuh"

namespace rb200 {

struct FusedSmem {
    uint32_t acc[FUSED_WARPS][WARP_SMEM_WORDS];   // accumulator + merge window (rb200_device.cuh)
    uint16_t keys[FUSED_MAX_ITEMS];          // keys of A then B
    uint32_t i_slot[FUSED_MAX_ITEMS], i_cap[FUSED_MAX_ITEMS], i_ocard[FUSED_MAX_ITEMS], i_olen[FUSED_MAX_ITEMS];
    uint16_t i_ca[FUSED_MAX_ITEMS], i_cb[FUSED_MAX_ITEMS], i_key[FUSED_MAX_ITEMS];
    uint8_t i_kind[FUSED_MAX_ITEMS], i_otype[FUSED_MAX_ITEMS];
    uint32_t scan[FUSED_WARPS * 32 / 32 + 1];
    uint32_t err;
};

template <int OP>
__global__ void __launch_bounds__(FUSED_WARPS * 32, 1)
k_pair_fused(const uint8_t *__restrict__ in, uint8_t *out, uint32_t out_bytes, int rules, uint32_t seq) {
    extern __shared__ __align__(128) uint8_t fused_smem_raw[];
    FusedSmem &sm = *reinterpret_cast<FusedSmem *>(fused_smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const FusedHdr hdr = *reinterpret_cast<const FusedHdr *>(in);
    const uint32_t na = hdr.na, nb = hdr.nb, n = na + nb;
    const uint16_t *c_key = reinterpret_cast<const uint16_t *>(in + hdr.o_key);
    const uint8_t *c_type = in + hdr.o_type, *c_shared = in + hdr.o_shared;
    const uint32_t *c_card = reinterpret_cast<const uint32_t *>(in + hdr.o_card);
    const uint32_t *c_len = reinterpret_cast<const uint32_t *>(in + hdr.o_len);
    const uint32_t *c_off = reinterpret_cast<const uint32_t *>(in + hdr.o_off);
    FusedOutHdr *oh = reinterpret_cast<FusedOutHdr *>(out);

    for (uint32_t i = tid; i < n; i += blockDim.x) sm.keys[i] = c_key[i];
    if (tid == 0) sm.err = 0;
    __syncthreads();

    // ---- plan: item position = rank in the merged key order (holes keep the order stable) -------
    for (uint32_t t = tid; t < n; t += blockDim.x) {
        int kind = K_HOLE;
        uint32_t ca = 0, cb = 0, cap = 0, pos, key;
        if (t < na) {
            ca = t;
            key = sm.keys[t];
            const uint32_t lb = lower_bound_u16(sm.keys + na, nb, key);
            const bool matched = lb < nb && sm.keys[na + lb] == key;
            pos = t + lb;
            if (matched) {
                cb = na + lb;
                kind = K_COMPUTE;
                cap = slot_bound(OP, c_type[ca], c_type[cb], c_card[ca], c_card[cb], c_len[ca], c_len[cb]);
            } else if (OP != OP_AND) {
                kind = K_COPY_A;
                cap = round16(stored_bytes(c_type[ca], c_len[ca]));
            }
        } else {
            const uint32_t j = t - na;
            cb = t;
            key = sm.keys[t];
            const uint32_t lo = upper_bound_u16(sm.keys, na, key);
            const bool matched = lo > 0 && sm.keys[lo - 1] == key;
            pos = j + lo;
            if (!matched && (OP == OP_OR || OP == OP_XOR)) {
                kind = K_COPY_B;
                cap = round16(stored_bytes(c_type[cb], c_len[cb]));
            }
        }
        sm.i_kind[pos] = (uint8_t)kind;
        sm.i_ca[pos] = (uint16_t)ca;
        sm.i_cb[pos] = (uint16_t)cb;
        sm.i_key[pos] = (uint16_t)key;
        sm.i_cap[pos] = cap;
        sm.i_otype[pos] = 0;
        sm.i_ocard[pos] = 0;
        sm.i_olen[pos] = 0;
    }
    __syncthreads();
    // output slots: exclusive scan of the caps in item order (warp 0, n <= FUSED_MAX_ITEMS)
    if (wid == 0) {
        uint32_t run = FUSED_OUT_PAYLOAD;
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t i = base + lane, c = i < n ? sm.i_cap[i] : 0u;
            const uint32_t incl = warp_incl_scan(c, lane);
            if (i < n) sm.i_slot[i] = run + incl - c;
            run += __shfl_sync(FULLMASK, incl, 31);
        }
        if (lane == 0 && run > out_bytes) sm.err = 2;   // result would not fit the mapped block
    }
    __syncthreads();
    if (sm.err) {
        if (tid == 0) { oh->error = sm.err; oh->n_out = 0; __threadfence_system(); oh->seq = seq; }
        return;
    }

    // ---- compute: one warp per item ---------------------------------------------------------------
    for (uint32_t item = wid; item < n; item += FUSED_WARPS) {
        const int kind = sm.i_kind[item];
        if (kind == K_HOLE) continue;
        int otype = 0;
        uint32_t ocard = 0, olen = 0;
        uint8_t *dst = out + sm.i_slot[item];
        if (kind == K_COMPUTE) {
            const uint32_t ca = sm.i_ca[item], cb = sm.i_cb[item];
            int cell_rules = rules;
            if ((rules & RULES_INPLACE) && c_shared[ca]) cell_rules &= ~RULES_INPLACE;   // roaring.c:1085-1088
            cell_compute<OP, false>(sm.acc[wid], c_type[ca], c_type[cb], in + c_off[ca], in + c_off[cb],
                                    c_card[ca], c_card[cb], c_len[ca], c_len[cb], dst, sm.i_cap[item], lane, otype,
                                    ocard, olen, &sm.err, cell_rules, false);
        } else {
            const uint32_t c = kind == K_COPY_A ? sm.i_ca[item] : sm.i_cb[item];
            otype = c_type[c];
            ocard = c_card[c];
            olen = c_len[c];
            warp_copy16(dst, in + c_off[c], stored_bytes(otype, olen), lane);
        }
        if (lane == 0) { sm.i_otype[item] = (uint8_t)otype; sm.i_ocard[item] = ocard; sm.i_olen[item] = olen; }
    }
    __syncthreads();

    // ---- finalize: drop empty results (roaring.c:756-760), ordered directory into the output block
    if (wid == 0) {
        uint16_t *o_key = reinterpret_cast<uint16_t *>(out + FUSED_OUT_KEY);
        uint8_t *o_type = out + FUSED_OUT_TYPE;
        uint32_t *o_card = reinterpret_cast<uint32_t *>(out + FUSED_OUT_CARD);
        uint32_t *o_len = reinterpret_cast<uint32_t *>(out + FUSED_OUT_LEN);
        uint32_t *o_off = reinterpret_cast<uint32_t *>(out + FUSED_OUT_OFF);
        uint32_t done = 0;
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t i = base + lane;
            const bool live = i < n && sm.i_kind[i] != K_HOLE && sm.i_otype[i] != 0;
            const unsigned m = __ballot_sync(FULLMASK, live);
            if (live) {
                const uint32_t o = done + __popc(m & lanemask_lt());
                o_key[o] = sm.i_key[i];
                o_type[o] = sm.i_otype[i];
                o_card[o] = sm.i_ocard[i];
                o_len[o] = sm.i_olen[i];
                o_off[o] = sm.i_slot[i];
            }
            done += __popc(m);
        }
        if (lane == 0) { oh->n_out = done; oh->error = sm.err; }
    }
    __syncthreads();
    __threadfence_system();
    __syncthreads();
    if (tid == 0) {
        __threadfence_system();
        oh->seq = seq;   // last: everything above is visible to the host when it sees this
    }
}

bool launch_pair_fused(int op, const uint8_t *d_in, uint8_t *out_mapped, uint32_t out_bytes, int rules, uint32_t seq,
                       cudaStream_t s) {
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(k_pair_fused<OP_AND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FusedSmem));
        cudaFuncSetAttribute(k_pair_fused<OP_OR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FusedSmem));
        cudaFuncSetAttribute(k_pair_fused<OP_XOR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FusedSmem));
        cudaFuncSetAttribute(k_pair_fused<OP_ANDNOT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FusedSmem));
        attr = true;
    }
    auto *k = op == OP_AND ? k_pair_fused<OP_AND> : op == OP_OR ? k_pair_fused<OP_OR>
            : op == OP_XOR ? k_pair_fused<OP_XOR> : k_pair_fused<OP_ANDNOT>;
    launch_kernel(k, 1, FUSED_WARPS * 32, sizeof(FusedSmem), s, d_in, out_mapped, out_bytes, rules, seq);
    return cudaGetLastError() == cudaSuccess;
}

}  // namespace rb200
