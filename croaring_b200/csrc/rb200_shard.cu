// rb200_shard.cu — the multi-GPU side of the many-way union (SURVEY.md §8(e)): one process per GPU.
//
//   * NCCL communicator handle.  libnccl is resolved at RUN time (dlopen of the copy already in
//     the process — torch's — or the system one), so libroaring_b200.so has no link-time
//     dependency on it and single-GPU users never load it.  The only collective of the path is
//     ONE ncclAllReduce(sum) over the per-key result cardinalities uint32[K] (K = keys between the
//     first and the last live key), issued on the library's stream right behind k_or_many2 — the
//     counters never leave the device before they are reduced.
//   * Host-side key-range planning and slicing of portable-serialized bitmaps
//     (format: /root/reference/src/roaring_array.c:469-531), plain C ABI, no CUDA involved:
//     histogram of container bytes per high-16 key -> contiguous ranges balanced by bytes ->
//     every rank uploads only the containers of its range -> results are concatenated in rank
//     order (disjoint increasing key ranges).
#include <dlfcn.h>
#include <nccl.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

#include "../../include/roaring_b200.h"
#include "rb200_common.h"
#include "rb200_internal.h"

#define RB_API extern "C" __attribute__((visibility("default")))

namespace {

struct NcclApi {
    void *h = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t,
                              cudaStream_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    std::string why;
};

NcclApi &nccl() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, []() {
        const char *env = getenv("RB200_NCCL_LIB");
        const char *names[] = {env, "libnccl.so.2", "libnccl.so"};
        for (const char *n : names) {
            if (!n || !*n) continue;
            api.h = dlopen(n, RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);   // the copy already loaded (torch's)
            if (!api.h) api.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.h) break;
        }
        if (!api.h) {
            // torch loads its bundled copy RTLD_LOCAL under a versioned path: look the symbols up globally
            if (dlsym(RTLD_DEFAULT, "ncclAllReduce")) api.h = RTLD_DEFAULT;
        }
        if (!api.h) { api.why = "libnccl.so.2 not found (set RB200_NCCL_LIB)"; return; }
        api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(api.h, "ncclGetUniqueId");
        api.CommInitRank = (decltype(api.CommInitRank))dlsym(api.h, "ncclCommInitRank");
        api.CommDestroy = (decltype(api.CommDestroy))dlsym(api.h, "ncclCommDestroy");
        api.AllReduce = (decltype(api.AllReduce))dlsym(api.h, "ncclAllReduce");
        api.GetErrorString = (decltype(api.GetErrorString))dlsym(api.h, "ncclGetErrorString");
        if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllReduce) {
            api.why = "libnccl is missing ncclGetUniqueId / ncclCommInitRank / ncclAllReduce";
            api.h = nullptr;
        }
    });
    return api;
}

std::string nccl_err(ncclResult_t r) {
    NcclApi &a = nccl();
    return std::string("NCCL: ") + (a.GetErrorString ? a.GetErrorString(r) : "error");
}

}  // namespace

struct rb200_comm {
    ncclComm_t comm = nullptr;
    int nranks = 1, rank = 0;
    bool owned = false;
};

namespace rb200 {

bool comm_allreduce_sum(rb200_comm *c, void *buf, size_t count, bool u64, cudaStream_t s, std::string &err) {
    if (!c || c->nranks <= 1 || count == 0) return true;
    NcclApi &a = nccl();
    if (!a.h) { err = a.why; return false; }
    const ncclResult_t r = a.AllReduce(buf, buf, count, u64 ? ncclUint64 : ncclUint32, ncclSum, c->comm, s);
    if (r != ncclSuccess) { err = nccl_err(r); return false; }
    return true;
}

}  // namespace rb200

RB_API int rb200_comm_unique_id(char *id128) {
    NcclApi &a = nccl();
    if (!a.h) { rb200::set_error(a.why); return -1; }
    ncclUniqueId id;
    static_assert(sizeof(id) == RB200_COMM_ID_BYTES, "ncclUniqueId size");
    const ncclResult_t r = a.GetUniqueId(&id);
    if (r != ncclSuccess) { rb200::set_error(nccl_err(r)); return -1; }
    memcpy(id128, &id, sizeof(id));
    return 0;
}

RB_API rb200_comm_t *rb200_comm_init_rank(const char *id128, int nranks, int rank) {
    if (nranks < 1 || rank < 0 || rank >= nranks) { rb200::set_error("comm_init_rank: bad rank / size"); return nullptr; }
    rb200_comm *c = new rb200_comm();
    c->nranks = nranks;
    c->rank = rank;
    if (nranks == 1) return c;   // no collective is ever issued: NCCL is not even loaded
    NcclApi &a = nccl();
    if (!a.h) { rb200::set_error(a.why); delete c; return nullptr; }
    if (rb200_init(-1) != 0) { delete c; return nullptr; }   // the communicator lives on the library's device
    ncclUniqueId id;
    memcpy(&id, id128, sizeof(id));
    const ncclResult_t r = a.CommInitRank(&c->comm, nranks, id, rank);
    if (r != ncclSuccess) { rb200::set_error(nccl_err(r)); delete c; return nullptr; }
    c->owned = true;
    return c;
}

RB_API rb200_comm_t *rb200_comm_adopt(void *nccl_comm, int nranks, int rank) {
    if (nranks < 1 || rank < 0 || rank >= nranks || (nranks > 1 && !nccl_comm)) {
        rb200::set_error("comm_adopt: bad arguments");
        return nullptr;
    }
    rb200_comm *c = new rb200_comm();
    c->comm = (ncclComm_t)nccl_comm;
    c->nranks = nranks;
    c->rank = rank;
    return c;
}

RB_API int rb200_comm_size(const rb200_comm_t *c) { return c ? c->nranks : 1; }
RB_API int rb200_comm_rank(const rb200_comm_t *c) { return c ? c->rank : 0; }

RB_API void rb200_comm_destroy(rb200_comm_t *c) {
    if (!c) return;
    if (c->owned && c->comm) {
        rb200_synchronize();
        nccl().CommDestroy(c->comm);
    }
    delete c;
}

// =================================================================== host-side blob algebra
namespace {

constexpr uint32_t COOKIE_NO_RUN = 12346, COOKIE_RUN = 12347;   // roaring_array.h:35-40
constexpr int NO_OFFSET_THRESHOLD_ = 4;

// header-level view: keys, cardinalities, run flags, payload spans (run sizes are read from the
// payload: the walk is sequential).  false = malformed.
struct BlobIndex {
    uint32_t n = 0;
    bool hasrun = false;
    std::vector<uint16_t> key, cm1;
    std::vector<uint8_t> isrun;
    std::vector<uint64_t> start;
    std::vector<uint32_t> size;
};

bool index_blob(const uint8_t *buf, size_t len, BlobIndex &ix) {
    if (len < 4) return false;
    uint32_t cookie;
    memcpy(&cookie, buf, 4);
    size_t pos = 4;
    const uint8_t *flags = nullptr;
    if ((cookie & 0xFFFF) == COOKIE_RUN) {
        ix.n = (cookie >> 16) + 1;
        ix.hasrun = true;
        flags = buf + 4;
        pos = 4 + (ix.n + 7) / 8;
    } else if (cookie == COOKIE_NO_RUN && len >= 8) {
        memcpy(&ix.n, buf + 4, 4);
        pos = 8;
    } else {
        return false;
    }
    const uint32_t n = ix.n;
    if (n > 65536 || pos + 4ull * n > len) return false;
    const uint8_t *kc = buf + pos;
    pos += 4ull * n;
    if (!ix.hasrun || n >= (uint32_t)NO_OFFSET_THRESHOLD_) pos += 4ull * n;
    ix.key.resize(n); ix.cm1.resize(n); ix.isrun.resize(n); ix.start.resize(n); ix.size.resize(n);
    for (uint32_t i = 0; i < n; i++) {
        memcpy(&ix.key[i], kc + 4 * i, 2);
        memcpy(&ix.cm1[i], kc + 4 * i + 2, 2);
        if (i && ix.key[i] <= ix.key[i - 1]) return false;
        const bool r = ix.hasrun && ((flags[i >> 3] >> (i & 7)) & 1);
        ix.isrun[i] = r;
        uint32_t sz;
        if (r) {
            if (pos + 2 > len) return false;
            uint16_t nr;
            memcpy(&nr, buf + pos, 2);
            sz = 2u + 4u * nr;
        } else {
            const uint32_t card = (uint32_t)ix.cm1[i] + 1;
            sz = card > 4096u ? 8192u : 2u * card;
        }
        if (pos + sz > len) return false;
        ix.start[i] = pos;
        ix.size[i] = sz;
        pos += sz;
    }
    return true;
}

// serialize containers [i0, i1) of several indexed blobs (in order) as ONE portable bitmap
struct Piece { const uint8_t *buf; const BlobIndex *ix; uint32_t i0, i1; };

bool build_blob(const std::vector<Piece> &pieces, char **out, size_t *outlen) {
    uint32_t n = 0;
    bool hasrun = false;
    uint64_t payload = 0;
    for (const Piece &p : pieces)
        for (uint32_t i = p.i0; i < p.i1; i++) {
            n++;
            hasrun |= p.ix->isrun[i] != 0;
            payload += p.ix->size[i];
        }
    const size_t hdr = hasrun ? 4 + (n + 7) / 8 + (n < (uint32_t)NO_OFFSET_THRESHOLD_ ? 4ull : 8ull) * n : 8 + 8ull * n;
    uint8_t *o = (uint8_t *)malloc(hdr + payload + 16);
    if (!o) return false;
    memset(o, 0, hdr);
    uint8_t *kc, *offs = nullptr;
    if (hasrun) {
        const uint32_t cookie = COOKIE_RUN | ((n - 1) << 16);
        memcpy(o, &cookie, 4);
        kc = o + 4 + (n + 7) / 8;
        if (n >= (uint32_t)NO_OFFSET_THRESHOLD_) offs = kc + 4ull * n;
    } else {
        memcpy(o, &COOKIE_NO_RUN, 4);
        memcpy(o + 4, &n, 4);
        kc = o + 8;
        offs = kc + 4ull * n;
    }
    uint64_t pos = hdr;
    uint32_t k = 0;
    for (const Piece &p : pieces)
        for (uint32_t i = p.i0; i < p.i1; i++, k++) {
            memcpy(kc + 4ull * k, &p.ix->key[i], 2);
            memcpy(kc + 4ull * k + 2, &p.ix->cm1[i], 2);
            if (p.ix->isrun[i]) o[4 + (k >> 3)] |= (uint8_t)(1u << (k & 7));
            if (offs) { const uint32_t o32 = (uint32_t)pos; memcpy(offs + 4ull * k, &o32, 4); }
            memcpy(o + pos, p.buf + p.ix->start[i], p.ix->size[i]);
            pos += p.ix->size[i];
        }
    *out = (char *)o;
    *outlen = (size_t)pos;
    return true;
}

}  // namespace

// Contiguous key ranges [key_lo[g], key_hi[g]], g < nranks, covering 0..65535 and balanced by the
// work the blobs hold per key: container bytes + 512 per container (Zipfian data concentrates the
// bytes in the low keys and the container count in the high ones).
// span[0], span[1] = first / last key present in any blob (span[0] > span[1]: no container at all).
RB_API int rb200_plan_key_ranges(const char *const *bufs, const size_t *lens, size_t n, int nranks,
                                 uint32_t *key_lo, uint32_t *key_hi, uint32_t *span) {
    if (nranks < 1 || nranks > 65536) { rb200::set_error("plan_key_ranges: bad rank count"); return -1; }
    std::vector<uint64_t> hist(65536, 0);
    uint32_t first = 65536, last = 0;
    bool any = false;
    for (size_t b = 0; b < n; b++) {
        BlobIndex ix;
        if (!index_blob((const uint8_t *)bufs[b], lens[b], ix)) {
            rb200::set_error("plan_key_ranges: malformed portable bitmap at index " + std::to_string(b));
            return -1;
        }
        // weight of a container = its bytes + a fixed per-container cost (k_or_many2 on config 3: a
        // container costs about as much as 0.5 KiB of payload)
        for (uint32_t i = 0; i < ix.n; i++) hist[ix.key[i]] += (uint64_t)ix.size[i] + 512;
        if (ix.n) {
            any = true;
            if (ix.key[0] < first) first = ix.key[0];
            if (ix.key[ix.n - 1] > last) last = ix.key[ix.n - 1];
        }
    }
    uint64_t total = 0;
    for (uint64_t h : hist) total += h;
    // bound g = smallest key count whose prefix reaches g/nranks of the bytes, at least one key per rank
    std::vector<uint32_t> bound(nranks + 1, 0);
    bound[nranks] = 65536;
    uint64_t acc = 0;
    uint32_t k = 0;
    for (int g = 1; g < nranks; g++) {
        const long double target = (long double)total * g / nranks;
        while (k < 65536 && (long double)acc < target) acc += hist[k++];
        uint32_t b = k;
        if (b < bound[g - 1] + 1) b = bound[g - 1] + 1;
        const uint32_t maxb = 65536u - (uint32_t)(nranks - g);
        if (b > maxb) b = maxb;
        bound[g] = b;
        while (k < b) acc += hist[k++];
    }
    for (int g = 0; g < nranks; g++) {
        key_lo[g] = bound[g];
        key_hi[g] = bound[g + 1] - 1;
    }
    if (span) {
        span[0] = any ? first : 1;
        span[1] = any ? last : 0;
    }
    return 0;
}

// The bitmap restricted to the containers whose key lies in [key_lo, key_hi] (malloc'd portable
// blob; release with rb200_blob_free).
RB_API int rb200_blob_slice_keys(const char *buf, size_t len, uint32_t key_lo, uint32_t key_hi, char **out,
                                 size_t *outlen) {
    BlobIndex ix;
    if (!index_blob((const uint8_t *)buf, len, ix)) { rb200::set_error("blob_slice_keys: malformed portable bitmap"); return -1; }
    uint32_t i0 = 0, i1 = ix.n;
    while (i0 < ix.n && ix.key[i0] < key_lo) i0++;
    while (i1 > i0 && ix.key[i1 - 1] > key_hi) i1--;
    std::vector<Piece> p{Piece{(const uint8_t *)buf, &ix, i0, i1}};
    if (!build_blob(p, out, outlen)) { rb200::set_error("blob_slice_keys: out of memory"); return -1; }
    return 0;
}

// Concatenation of bitmaps living on disjoint, increasing key ranges (per-rank results in rank order).
RB_API int rb200_blobs_concat(const char *const *bufs, const size_t *lens, size_t n, char **out, size_t *outlen) {
    std::vector<BlobIndex> ix(n);
    std::vector<Piece> pieces;
    int last = -1;
    for (size_t b = 0; b < n; b++) {
        if (!index_blob((const uint8_t *)bufs[b], lens[b], ix[b])) {
            rb200::set_error("blobs_concat: malformed portable bitmap at index " + std::to_string(b));
            return -1;
        }
        if (ix[b].n) {
            if ((int)ix[b].key[0] <= last) { rb200::set_error("blobs_concat: shards are not on increasing disjoint key ranges"); return -1; }
            last = ix[b].key[ix[b].n - 1];
        }
        pieces.push_back(Piece{(const uint8_t *)bufs[b], &ix[b], 0, ix[b].n});
    }
    if (!build_blob(pieces, out, outlen)) { rb200::set_error("blobs_concat: out of memory"); return -1; }
    return 0;
}

RB_API void rb200_blob_free(char *p) { free(p); }

// Resident set holding, for every input blob, only the containers with key in [key_lo, key_hi]
// (what rank g of a key-sharded union uploads: host slicing, then the ordinary streamed H2D).
RB_API rb200_set_t *rb200_set_upload_serialized_keyrange(const char *const *bufs, const size_t *lens, size_t n,
                                                         uint32_t key_lo, uint32_t key_hi) {
    std::vector<char *> part(n, nullptr);
    std::vector<size_t> plen(n, 0);
    std::vector<int> rc(n, 0);
    rb200::parallel_for(n, [&](size_t b) {
        rc[b] = rb200_blob_slice_keys(bufs[b], lens[b], key_lo, key_hi, &part[b], &plen[b]);
    });
    rb200_set_t *S = nullptr;
    bool ok = true;
    for (size_t b = 0; b < n && ok; b++)
        if (rc[b] != 0) {
            // the slices ran on worker threads and rb200_last_error() is per thread: report on the caller's
            rb200::set_error("set_upload_serialized_keyrange: malformed portable bitmap at index " + std::to_string(b));
            ok = false;
        }
    if (ok) S = rb200_set_upload_serialized(part.data(), plen.data(), n);
    for (char *p : part) free(p);
    return S;
}
