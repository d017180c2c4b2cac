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
#include "rb200_portable.h"

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

using rb200::PortableEntry;

// the containers as ONE malloc'd portable bitmap
bool write_blob(const std::vector<PortableEntry> &c, char **out, size_t *outlen) {
    const auto at = [&c](uint32_t i) { return c[i]; };
    uint8_t *o = (uint8_t *)malloc(rb200::portable_size((uint32_t)c.size(), at));
    if (!o) return false;
    *outlen = rb200::write_portable(o, (uint32_t)c.size(), at);
    *out = (char *)o;
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
        // weight of a container = its bytes + a fixed per-container cost (k_or_many2 on config 3: a
        // container costs about as much as 0.5 KiB of payload)
        const auto weigh = [&](const PortableEntry &e) {
            hist[e.key] += (uint64_t)rb200::portable_bytes(e.type, e.len) + 512;
            any = true;
            if (e.key < first) first = e.key;
            if (e.key > last) last = e.key;
        };
        if (!rb200::walk_portable((const uint8_t *)bufs[b], lens[b], weigh)) {
            rb200::set_error("plan_key_ranges: malformed portable bitmap at index " + std::to_string(b));
            return -1;
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
    std::vector<PortableEntry> c;
    const auto keep = [&](const PortableEntry &e) { if (e.key >= key_lo && e.key <= key_hi) c.push_back(e); };
    if (!rb200::walk_portable((const uint8_t *)buf, len, keep)) { rb200::set_error("blob_slice_keys: malformed portable bitmap"); return -1; }
    if (!write_blob(c, out, outlen)) { rb200::set_error("blob_slice_keys: out of memory"); return -1; }
    return 0;
}

// Concatenation of bitmaps living on disjoint, increasing key ranges (per-rank results in rank order).
RB_API int rb200_blobs_concat(const char *const *bufs, const size_t *lens, size_t n, char **out, size_t *outlen) {
    std::vector<PortableEntry> c;
    for (size_t b = 0; b < n; b++) {
        const size_t c0 = c.size();
        if (!rb200::walk_portable((const uint8_t *)bufs[b], lens[b], [&c](const PortableEntry &e) { c.push_back(e); })) {
            rb200::set_error("blobs_concat: malformed portable bitmap at index " + std::to_string(b));
            return -1;
        }
        if (c0 && c.size() > c0 && c[c0].key <= c[c0 - 1].key) {
            rb200::set_error("blobs_concat: shards are not on increasing disjoint key ranges");
            return -1;
        }
    }
    if (!write_blob(c, out, outlen)) { rb200::set_error("blobs_concat: out of memory"); return -1; }
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
