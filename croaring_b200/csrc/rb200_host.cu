// rb200_host.cu — host side of libroaring_b200.so: context, memory pools, the device mirror
// of roaring_bitmap_t ("set" upload), the batched-op drivers, host materialisation of
// results in the reference's memory layout, portable (de)serialisation, and the C ABI of
// include/roaring_b200.h.  Plain C++ + CUDA runtime; no torch, no reference code.
//
// Reference layout / behaviour restated here (file:line relative to /root/reference):
//   roaring_array_t single-block directory     src/roaring_array.c:42-78
//   container structs                          include/roaring/containers/{array,bitset,run}.h
//   ownership of returned bitmaps              src/roaring.c:552-560, src/containers/containers.c:58-77
//   portable format                            src/roaring_array.c:469-531, :633-813
#include <ctype.h>
#include <dlfcn.h>
#include <pthread.h>
#include <sched.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <stdio.h>
#include <thread>
#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#pragma GCC visibility push(default)
#include "../../include/roaring_b200.h"
#pragma GCC visibility pop
#include "rb200_common.h"
#include "rb200_device.cuh"
#include "rb200_internal.h"

using namespace rb200;

// ------------------------------------------------------------------ reference-compatible structs
namespace {

struct array_container_t { int32_t cardinality; int32_t capacity; uint16_t *array; };   // array.h:46-50
struct bitset_container_t { int32_t cardinality; uint64_t *words; };                     // bitset.h:45-48
struct rle16_t { uint16_t value, length; };                                              // run.h:48-51
struct run_container_t { int32_t n_runs; int32_t capacity; rle16_t *runs; };            // run.h:69-73
struct shared_container_t { void *container; uint8_t typecode; uint32_t counter; };      // containers.h:71-75

constexpr uint8_t FLAG_COW = 1, FLAG_FROZEN = 2;  // roaring_types.h:46-49
constexpr uint32_t SERIAL_COOKIE_NO_RUN = 12346, SERIAL_COOKIE = 12347;  // roaring_array.h:35-40
constexpr int32_t NO_OFFSET_THRESHOLD = 4;
constexpr uint32_t M2_SCRATCH_SLOTS = 2048, M2_SCRATCH_WORDS = 2 * ACC_WORDS + 32;  // rb200_many2.cu split keys

// ------------------------------------------------------------------ host allocation hooks
// If the reference library is loaded in this process (drop-in deployment) every host object we
// hand out is allocated with ITS roaring_malloc / roaring_aligned_malloc so roaring_bitmap_free
// and user memory hooks (src/memory.c:35-60) keep working; otherwise libc, like the defaults.
typedef void *(*malloc_fn)(size_t);
typedef void (*free_fn)(void *);
typedef void *(*amalloc_fn)(size_t, size_t);
struct HostAlloc {
    malloc_fn m = nullptr;
    free_fn f = nullptr;
    amalloc_fn am = nullptr;
    free_fn af = nullptr;
    bool looked = false;
    void look() {
        if (looked) return;
        looked = true;
        m = (malloc_fn)dlsym(RTLD_DEFAULT, "roaring_malloc");
        f = (free_fn)dlsym(RTLD_DEFAULT, "roaring_free");
        am = (amalloc_fn)dlsym(RTLD_DEFAULT, "roaring_aligned_malloc");
        af = (free_fn)dlsym(RTLD_DEFAULT, "roaring_aligned_free");
        if (!m || !f || !am || !af) m = nullptr;
    }
} g_halloc;

inline void *h_malloc(size_t n) {
    g_halloc.look();
    return g_halloc.m ? g_halloc.m(n) : malloc(n);
}
inline void h_free(void *p) {
    g_halloc.look();
    if (g_halloc.m) g_halloc.f(p); else free(p);
}
inline void *h_aligned_malloc(size_t align, size_t n) {
    g_halloc.look();
    if (g_halloc.m) return g_halloc.am(align, n);
    void *p = nullptr;
    if (posix_memalign(&p, align, n) != 0) return nullptr;
    return p;
}
inline void h_aligned_free(void *p) {
    g_halloc.look();
    if (g_halloc.m) g_halloc.af(p); else free(p);
}

// ------------------------------------------------------------------ context
struct Ctx {
    std::recursive_mutex mu;
    bool inited = false;
    int device = 0;
    cudaStream_t own_stream = nullptr, stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, evk0 = nullptr, evk1 = nullptr;
    OpStats *d_stats = nullptr;
    OpStats *h_stats = nullptr;  // pinned
    uint32_t *d_flags = nullptr;   // 65536 key flags (xor_many)
    uint16_t *d_keys = nullptr;    // 65536 compacted keys
    uint32_t *d_cardkey = nullptr; // 65536 per-key cardinalities
    // or_many (rb200_many2.cu): per-key tables + split-key scratch (kept zeroed)
    uint32_t *d_m2_tables = nullptr;   // 14 x 65536 u32: key_cu(2) | fill | count | units16 | fill | start | slices | scratch | unit_first | fold_first(2) | fold_second(2) | fold_F | fold_L
    uint32_t *d_m2_scratch = nullptr, *d_m2_tickets = nullptr;
    // single-pair fused path (rb200_fused.cu): packed operands (pinned + device), mapped result block
    uint8_t *h_fused_in = nullptr, *d_fused_in = nullptr, *h_fused_out = nullptr, *d_fused_out = nullptr;
    uint32_t fused_seq = 0;
    int sms = 132;
    std::multimap<size_t, void *> dpool, hpool;
    std::mutex alloc_mu;  // dpool / hpool are also used by the background downloader thread
    uint64_t last_algo_bytes = 0;
    float last_ms = 0.f, last_compute_ms = 0.f;
    uint64_t last_download_bytes = 0;
    uint64_t last_out_portable = 0;  // portable bytes of the last batch's results (all pairs)
    std::vector<cudaEvent_t> evpool;  // timing events recycled between batch ops (under alloc_mu)
    struct rb200_set *last_op = nullptr;  // result of the most recent batch op (counters may be pending)
} g;
// rb200_last_error() is per calling thread: concurrent callers do not read each other's failures
thread_local std::string t_err;
std::map<uint8_t *, size_t> g_serialized_sizes;  // pinned blobs handed out by rb200_set_serialize

#define CK(call)                                                                    \
    do {                                                                            \
        cudaError_t e_ = (call);                                                    \
        if (e_ != cudaSuccess) {                                                    \
            t_err = std::string(#call) + ": " + cudaGetErrorString(e_);             \
            return false;                                                           \
        }                                                                           \
    } while (0)

bool stats_reset();
bool stats_fetch();

// size classes of the device / pinned pools: 8 per octave (<= 12.5 % slack; the power-of-two
// classes of round 1 could double a multi-GB result slab)
size_t bucket(size_t n) {
    size_t b = 512;
    while (b < n) b <<= 1;
    if (b <= 4096) return b;
    const size_t step = b >> 4;            // b/2 < n <= b: classes b/2 + k * b/16
    return (b >> 1) + ((n - (b >> 1) + step - 1) / step) * step;
}

bool ctx_init(int device = -1) {
    if (g.inited) return true;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        t_err = "no CUDA device visible: libroaring_b200 has no CPU fallback";
        return false;
    }
    if (device >= 0) CK(cudaSetDevice(device));
    CK(cudaGetDevice(&g.device));
    CK(cudaStreamCreateWithFlags(&g.own_stream, cudaStreamNonBlocking));
    g.stream = g.own_stream;
    CK(cudaEventCreate(&g.ev0));
    CK(cudaEventCreate(&g.ev1));
    CK(cudaEventCreate(&g.evk0));
    CK(cudaEventCreate(&g.evk1));
    CK(cudaMalloc(&g.d_stats, sizeof(OpStats)));
    CK(cudaHostAlloc(&g.h_stats, sizeof(OpStats), cudaHostAllocDefault));
    CK(cudaMalloc(&g.d_flags, 65536 * sizeof(uint32_t)));
    CK(cudaMalloc(&g.d_keys, 65536 * sizeof(uint16_t)));
    CK(cudaMalloc(&g.d_cardkey, 65536 * sizeof(uint32_t)));
    CK(cudaMalloc(&g.d_m2_tables, 14 * 65536 * sizeof(uint32_t)));
    CK(cudaMalloc(&g.d_m2_scratch, (size_t)M2_SCRATCH_SLOTS * M2_SCRATCH_WORDS * sizeof(uint32_t)));
    CK(cudaMalloc(&g.d_m2_tickets, M2_SCRATCH_SLOTS * sizeof(uint32_t)));
    CK(cudaMemset(g.d_m2_scratch, 0, (size_t)M2_SCRATCH_SLOTS * M2_SCRATCH_WORDS * sizeof(uint32_t)));
    CK(cudaMemset(g.d_m2_tickets, 0, M2_SCRATCH_SLOTS * sizeof(uint32_t)));
    CK(cudaHostAlloc(&g.h_fused_in, FUSED_IN_BYTES, cudaHostAllocDefault));
    CK(cudaMalloc(&g.d_fused_in, FUSED_IN_BYTES));
    CK(cudaHostAlloc(&g.h_fused_out, FUSED_OUT_BYTES, cudaHostAllocMapped));
    CK(cudaHostGetDevicePointer(&g.d_fused_out, g.h_fused_out, 0));
    memset(g.h_fused_out, 0, 64);
    CK(cudaDeviceGetAttribute(&g.sms, cudaDevAttrMultiProcessorCount, g.device));
    g_halloc.look();  // resolve the host allocator once, before any worker thread exists
    g.inited = true;
    return true;
}

void *dev_alloc(size_t n) {
    std::lock_guard<std::mutex> alk(g.alloc_mu);
    if (n == 0) n = 1;
    const size_t b = bucket(n);
    auto it = g.dpool.find(b);
    if (it != g.dpool.end()) {
        void *p = it->second;
        g.dpool.erase(it);
        return p;
    }
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, b);
    if (e != cudaSuccess) {
        // drop the cache and retry once; the failure is reported through t_err, so it must not stay
        // behind as the runtime's last error for the next launch check to find
        (void)cudaGetLastError();
        for (auto &kv : g.dpool) cudaFree(kv.second);
        g.dpool.clear();
        e = cudaMalloc(&p, b);
        if (e != cudaSuccess) {
            (void)cudaGetLastError();
            t_err = std::string("cudaMalloc: ") + cudaGetErrorString(e);
            return nullptr;
        }
    }
    return p;
}
void dev_free(void *p, size_t n) {
    if (!p) return;
    std::lock_guard<std::mutex> alk(g.alloc_mu);
    if (n == 0) n = 1;
    g.dpool.insert({bucket(n), p});
}
bool enter_local_cpus(cpu_set_t *saved);
void *pin_alloc(size_t n) {
    std::lock_guard<std::mutex> alk(g.alloc_mu);
    if (n == 0) n = 1;
    const size_t b = bucket(n);
    auto it = g.hpool.find(b);
    if (it != g.hpool.end()) {
        void *p = it->second;
        g.hpool.erase(it);
        return p;
    }
    // Staging buffers belong on the GPU's NUMA node: the D2H stream and the (node-bound) workers
    // that read them then never cross the socket interconnect.  Pages are placed when they are
    // pinned, in the calling thread's context, so the caller is moved to the local CPUs for the
    // duration of the allocation.
    cpu_set_t saved;
    const bool moved = b >= (1u << 20) && enter_local_cpus(&saved);
    void *p = nullptr;
    cudaError_t e = cudaHostAlloc(&p, b, cudaHostAllocDefault);
    if (moved) pthread_setaffinity_np(pthread_self(), sizeof(saved), &saved);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();   // reported through t_err, not left for the next launch check
        t_err = std::string("cudaHostAlloc: ") + cudaGetErrorString(e);
        return nullptr;
    }
    return p;
}
void pin_free(void *p, size_t n) {
    if (!p) return;
    std::lock_guard<std::mutex> alk(g.alloc_mu);
    if (n == 0) n = 1;
    g.hpool.insert({bucket(n), p});
}

// ------------------------------------------------------------------ set object
inline size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

// Directory arrays carved out of one block (device and, mirrored, pinned host).
struct DirLayout {
    size_t o_beg, o_cnt, o_bcard, o_bbytes, o_bebytes, o_key, o_type, o_card, o_len, o_off, o_src, total;
    void compute(size_t nb, size_t nc) {
        size_t o = 0;
        o_beg = o; o += al256(4 * nb);
        o_cnt = o; o += al256(4 * nb);        // [cnt | bcard | bbytes | bebytes] are fetched with ONE copy
        o_bcard = o; o += al256(8 * nb);
        o_bbytes = o; o += al256(8 * nb);
        o_bebytes = o; o += al256(8 * nb);
        o_off = o; o += al256(8 * nc);
        o_card = o; o += al256(4 * nc);
        o_len = o; o += al256(4 * nc);
        o_src = o; o += al256(4 * nc);
        o_key = o; o += al256(2 * nc);
        o_type = o; o += al256(nc);
        total = o ? o : 256;
    }
};

}  // namespace

struct rb200_set {
    uint32_t n_bitmaps = 0;
    uint64_t dir_cap = 0;      // directory entries allocated
    uint64_t n_containers = 0; // directory entries in use
    uint64_t slab_cap = 0, slab_used = 0;
    uint64_t portable_bytes = 0;  // sum of container_size_in_bytes
    DirLayout L;
    uint8_t *d_dir = nullptr;   // one block
    uint8_t *d_slab = nullptr;
    std::vector<uint32_t> h_cnt;    // host mirror: containers per bitmap
    std::vector<uint64_t> h_card;   // host mirror: cardinality per bitmap (empty = not cached)
    bool mirrors_pending = false;   // batch results: h_cnt / h_bytes / h_card are fetched on first use
    bool lazy = false;              // produced by a lazy op: needs rb200_set_repair_after_lazy
    // Deferred counters of the batch op that produced this set: the op returns as soon as its
    // kernels and the D2H copy of its counters are queued; resolve() waits for them on first use,
    // so consecutive batch calls pipeline on the stream without a host round trip.
    bool pending = false, failed = false;
    OpStats *pstats = nullptr;                  // pinned
    uint8_t *staging = nullptr;                 // pinned pair list of the op (alive until it ran)
    size_t staging_bytes = 0;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};  // op start, kernel start, kernel end, op end
    float ms = 0.f, compute_ms = 0.f;
    uint64_t algo_bytes = 0, out_portable = 0;
    // payload address of every container in the caller's host bitmaps (sets made by
    // rb200_set_upload; valid while the caller keeps those bitmaps alive) and, for a batch result,
    // the tables of its two parents: pass-through containers can then be rebuilt on the host from
    // the inputs instead of crossing PCIe again
    std::shared_ptr<std::vector<const void *>> h_ptr_all, h_ptr, parentA, parentB;  // h_ptr: bound (opt-in)
    std::vector<uint64_t> h_bytes;  // host mirror: upper bound of stored payload bytes per bitmap
    std::vector<uint64_t> h_ebytes; // host mirror: upper bound of the "effective bytes" (rb200_device.cuh) per bitmap
    std::vector<uint8_t> h_flags;   // per bitmap: COW flag to propagate
    // lazily downloaded host mirror (pinned)
    uint8_t *m_dir = nullptr, *m_slab = nullptr;

    SetView view() const {
        SetView v;
        v.bm_beg = (const uint32_t *)(d_dir + L.o_beg);
        v.bm_cnt = (const uint32_t *)(d_dir + L.o_cnt);
        v.c_key = (const uint16_t *)(d_dir + L.o_key);
        v.c_type = (const uint8_t *)(d_dir + L.o_type);
        v.c_card = (const uint32_t *)(d_dir + L.o_card);
        v.c_len = (const uint32_t *)(d_dir + L.o_len);
        v.c_off = (const uint64_t *)(d_dir + L.o_off);
        v.c_src = (const uint32_t *)(d_dir + L.o_src);
        v.payload = d_slab;
        return v;
    }
    SetOut out() {
        SetOut v;
        v.bm_beg = (uint32_t *)(d_dir + L.o_beg);
        v.bm_cnt = (uint32_t *)(d_dir + L.o_cnt);
        v.bm_card = (uint64_t *)(d_dir + L.o_bcard);
        v.bm_bytes = (uint64_t *)(d_dir + L.o_bbytes);
        v.bm_ebytes = (uint64_t *)(d_dir + L.o_bebytes);
        v.c_key = (uint16_t *)(d_dir + L.o_key);
        v.c_type = (uint8_t *)(d_dir + L.o_type);
        v.c_card = (uint32_t *)(d_dir + L.o_card);
        v.c_len = (uint32_t *)(d_dir + L.o_len);
        v.c_off = (uint64_t *)(d_dir + L.o_off);
        v.c_src = (uint32_t *)(d_dir + L.o_src);
        v.payload = d_slab;
        return v;
    }
};

namespace {

rb200_set *set_new(uint32_t nb, uint64_t dir_cap, uint64_t slab_cap) {
    rb200_set *s = new rb200_set();
    s->n_bitmaps = nb;
    s->dir_cap = dir_cap;
    s->slab_cap = slab_cap;
    s->L.compute(nb, dir_cap);
    s->d_dir = (uint8_t *)dev_alloc(s->L.total);
    s->d_slab = (uint8_t *)dev_alloc(slab_cap);
    if (!s->d_dir || !s->d_slab) {
        dev_free(s->d_dir, s->L.total);
        dev_free(s->d_slab, slab_cap);
        delete s;
        return nullptr;
    }
    s->h_cnt.assign(nb, 0);
    s->h_bytes.assign(nb, 0);
    s->h_ebytes.assign(nb, 0);
    s->h_flags.assign(nb, 0);
    return s;
}

void set_drop_mirror(rb200_set *s) {
    pin_free(s->m_dir, s->L.total);
    pin_free(s->m_slab, s->slab_used);
    s->m_dir = s->m_slab = nullptr;
}

cudaEvent_t ev_get() {
    {
        std::lock_guard<std::mutex> alk(g.alloc_mu);
        if (!g.evpool.empty()) {
            cudaEvent_t e = g.evpool.back();
            g.evpool.pop_back();
            return e;
        }
    }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
}
void ev_put(cudaEvent_t e) {
    if (!e) return;
    std::lock_guard<std::mutex> alk(g.alloc_mu);
    g.evpool.push_back(e);
}

// Wait for the op that produced `cs` (if it is still in flight) and take over its counters.
// false: the op failed (t_err says why); the set must not be used.
bool resolve(const rb200_set *cs) {
    rb200_set *s = const_cast<rb200_set *>(cs);
    if (!s->pending) {
        if (s->failed && t_err.empty()) t_err = "the operation that produced this set failed";
        return !s->failed;
    }
    s->pending = false;
    cudaError_t e = cudaEventSynchronize(s->ev[3]);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) {
        t_err = std::string("batch op: ") + cudaGetErrorString(e);
        s->failed = true;
    } else if (s->pstats->error) {
        t_err = s->pstats->error == 2 ? "internal: result slab bound exceeded" : "internal: result slot bound exceeded";
        s->failed = true;
    } else {
        cudaEventElapsedTime(&s->ms, s->ev[0], s->ev[3]);
        cudaEventElapsedTime(&s->compute_ms, s->ev[1], s->ev[2]);
        s->algo_bytes = s->pstats->algo_bytes;
        s->out_portable = s->pstats->out_portable;
        s->n_containers = s->pstats->dir_cursor;
        s->slab_used = s->pstats->slab_cursor;
        if (s->n_bitmaps == 1) {  // a single result: its mirrors are the op's counters, no extra D2H
            s->h_cnt[0] = (uint32_t)s->n_containers;
            s->h_bytes[0] = s->slab_used;
            s->h_ebytes[0] = std::max<uint64_t>(s->slab_used, s->n_containers * (uint64_t)BITSET_BYTES);
            s->mirrors_pending = false;
        }
    }
    for (int k = 0; k < 4; k++) { ev_put(s->ev[k]); s->ev[k] = nullptr; }
    pin_free(s->pstats, sizeof(OpStats));
    pin_free(s->staging, s->staging_bytes);
    s->pstats = nullptr;
    s->staging = nullptr;
    if (g.last_op == s) {
        g.last_ms = s->ms;
        g.last_compute_ms = s->compute_ms;
        g.last_algo_bytes = s->algo_bytes;
        g.last_out_portable = s->out_portable;
    }
    return !s->failed;
}

void set_delete(rb200_set *s) {
    if (!s) return;
    if (s->pending) resolve(s);  // pinned staging / counters must not be recycled under a pending DMA
    for (int k = 0; k < 4; k++) { ev_put(s->ev[k]); s->ev[k] = nullptr; }  // (only set if the enqueue failed half way)
    pin_free(s->pstats, sizeof(OpStats));
    pin_free(s->staging, s->staging_bytes);
    s->pstats = nullptr;
    s->staging = nullptr;
    if (g.last_op == s) g.last_op = nullptr;
    set_drop_mirror(s);
    dev_free(s->d_dir, s->L.total);
    dev_free(s->d_slab, s->slab_cap);
    delete s;
}

// ------------------------------------------------------------------ host containers
inline const void *unwrap_shared(const void *c, uint8_t &type) {  // containers.h:105-114
    if (type == T_SHARED) {
        const shared_container_t *sc = (const shared_container_t *)c;
        type = sc->typecode;
        return sc->container;
    }
    return c;
}

void container_free_host(void *c, uint8_t type) {  // containers.c:58-77
    if (!c) return;
    switch (type) {
        case T_BITSET: {
            bitset_container_t *b = (bitset_container_t *)c;
            h_aligned_free(b->words);
            h_free(b);
            break;
        }
        case T_ARRAY: {
            array_container_t *a = (array_container_t *)c;
            h_free(a->array);
            h_free(a);
            break;
        }
        case T_RUN: {
            run_container_t *r = (run_container_t *)c;
            h_free(r->runs);
            h_free(r);
            break;
        }
        case T_SHARED: {
            shared_container_t *sc = (shared_container_t *)c;
            if (__atomic_sub_fetch(&sc->counter, 1, __ATOMIC_ACQ_REL) == 0) {
                container_free_host(sc->container, sc->typecode);
                h_free(sc);
            }
            break;
        }
    }
}

// roaring_bitmap_create_with_capacity + ra_init_with_capacity (roaring.c:86, roaring_array.c:80)
roaring_bitmap_t *bitmap_alloc(int32_t cap) {
    roaring_bitmap_t *r = (roaring_bitmap_t *)h_malloc(sizeof(roaring_bitmap_t));
    if (!r) return nullptr;
    roaring_array_t *ra = &r->high_low_container;
    ra->size = 0;
    ra->allocation_size = 0;
    ra->containers = nullptr;
    ra->keys = nullptr;
    ra->typecodes = nullptr;
    ra->flags = 0;
    if (cap > 0) {
        const size_t need = (size_t)cap * (sizeof(void *) + sizeof(uint16_t) + sizeof(uint8_t));
        void *big = h_malloc(need);
        if (!big) {
            h_free(r);
            return nullptr;
        }
        ra->containers = (void **)big;
        ra->keys = (uint16_t *)(ra->containers + cap);
        ra->typecodes = (uint8_t *)(ra->keys + cap);
        ra->allocation_size = cap;
    }
    return r;
}

void bitmap_free_host(roaring_bitmap_t *r) {  // roaring.c:552-560
    if (!r) return;
    roaring_array_t *ra = &r->high_low_container;
    if (!(ra->flags & FLAG_FROZEN)) {
        for (int32_t i = 0; i < ra->size; i++) container_free_host(ra->containers[i], ra->typecodes[i]);
        h_free(ra->containers);
    }
    h_free(r);
}

// make a host container from a stored payload (type, card, len)
void *container_from_payload(uint8_t type, uint32_t card, uint32_t len, const uint8_t *p) {
    if (type == T_BITSET) {
        bitset_container_t *b = (bitset_container_t *)h_malloc(sizeof(bitset_container_t));
        if (!b) return nullptr;
        b->words = (uint64_t *)h_aligned_malloc(64, BITSET_BYTES);
        if (!b->words) { h_free(b); return nullptr; }
        memcpy(b->words, p, BITSET_BYTES);
        b->cardinality = (card & CARD_UNKNOWN) ? -1 : (int32_t)card;  // bitset.h:42 BITSET_UNKNOWN_CARDINALITY
        return b;
    }
    if (type == T_ARRAY) {
        array_container_t *a = (array_container_t *)h_malloc(sizeof(array_container_t));
        if (!a) return nullptr;
        a->array = (uint16_t *)h_malloc(2 * (size_t)(len ? len : 1));
        if (!a->array) { h_free(a); return nullptr; }
        memcpy(a->array, p, 2 * (size_t)len);
        a->cardinality = (int32_t)len;
        a->capacity = (int32_t)(len ? len : 1);
        return a;
    }
    run_container_t *r = (run_container_t *)h_malloc(sizeof(run_container_t));
    if (!r) return nullptr;
    r->runs = (rle16_t *)h_malloc(4 * (size_t)(len ? len : 1));
    if (!r->runs) { h_free(r); return nullptr; }
    memcpy(r->runs, p, 4 * (size_t)len);
    r->n_runs = (int32_t)len;
    r->capacity = (int32_t)(len ? len : 1);
    return r;
}

inline uint32_t host_container_card(const void *c, uint8_t type) {
    if (type == T_ARRAY) return (uint32_t)((const array_container_t *)c)->cardinality;
    if (type == T_RUN) {
        const run_container_t *r = (const run_container_t *)c;
        uint32_t s = 0;
        for (int32_t i = 0; i < r->n_runs; i++) s += (uint32_t)r->runs[i].length + 1;
        return s;
    }
    const bitset_container_t *b = (const bitset_container_t *)c;
    if (b->cardinality >= 0) return (uint32_t)b->cardinality;
    uint32_t s = 0;
    for (int i = 0; i < 1024; i++) s += (uint32_t)__builtin_popcountll(b->words[i]);
    return s;
}

}  // namespace

// =================================================================== C ABI: helpers
extern "C" {

const char *rb200_last_error(void) { return t_err.c_str(); }
uint64_t rb200_kernel_launches(void) { return g_launches; }
static void settle_last_op() {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (g.last_op && g.last_op->pending) resolve(g.last_op);
}
uint64_t rb200_last_algorithmic_bytes(void) { settle_last_op(); return g.last_algo_bytes; }
float rb200_last_device_ms(void) { settle_last_op(); return g.last_ms; }
float rb200_last_compute_ms(void) { settle_last_op(); return g.last_compute_ms; }
uint64_t rb200_last_download_bytes(void) { return g.last_download_bytes; }

int rb200_init(int device) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return ctx_init(device) ? 0 : -1;
}

void rb200_set_stream(void *cuda_stream) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return;
    cudaStream_t next = cuda_stream ? (cudaStream_t)cuda_stream : g.own_stream;
    if (next == g.stream) return;
    // The device pools hand buffers back as soon as the work using them is ENQUEUED (stream-ordered
    // reuse), which is only sound on one stream: drain the old stream before work moves to the new one.
    cudaStreamSynchronize(g.stream);
    g.stream = next;
}

void rb200_synchronize(void) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (g.inited) cudaStreamSynchronize(g.stream);
}

void rb200_bitmap_free(roaring_bitmap_t *r) { bitmap_free_host(r); }

uint64_t rb200_bitmap_get_cardinality(const roaring_bitmap_t *r) {
    const roaring_array_t *ra = &r->high_low_container;
    uint64_t s = 0;
    for (int32_t i = 0; i < ra->size; i++) {
        uint8_t t = ra->typecodes[i];
        const void *c = unwrap_shared(ra->containers[i], t);
        s += host_container_card(c, t);
    }
    return s;
}

bool rb200_bitmap_validate(const roaring_bitmap_t *r, const char **reason) {
    static const char *why = "";
    const roaring_array_t *ra = &r->high_low_container;
#define BAD(msg) do { why = msg; if (reason) *reason = why; return false; } while (0)
    if (ra->size < 0 || ra->size > 65536) BAD("size out of range");
    if (ra->allocation_size < ra->size) BAD("allocation smaller than size");
    for (int32_t i = 0; i < ra->size; i++) {
        if (i > 0 && ra->keys[i] <= ra->keys[i - 1]) BAD("keys not strictly increasing");
        uint8_t t = ra->typecodes[i];
        const void *c = unwrap_shared(ra->containers[i], t);
        if (!c) BAD("null container");
        if (t == T_ARRAY) {
            const array_container_t *a = (const array_container_t *)c;
            if (a->cardinality < 1 || a->cardinality > MAX_ARRAY) BAD("array cardinality out of range");
            if (a->capacity < a->cardinality) BAD("array capacity too small");
            for (int32_t k = 1; k < a->cardinality; k++)
                if (a->array[k] <= a->array[k - 1]) BAD("array not sorted/unique");
        } else if (t == T_BITSET) {
            const bitset_container_t *b = (const bitset_container_t *)c;
            uint32_t s = 0;
            for (int k = 0; k < 1024; k++) s += (uint32_t)__builtin_popcountll(b->words[k]);
            if ((int32_t)s != b->cardinality) BAD("bitset cardinality field wrong");
            if (s <= (uint32_t)MAX_ARRAY) BAD("bitset with cardinality <= 4096");
        } else if (t == T_RUN) {
            const run_container_t *rc = (const run_container_t *)c;
            if (rc->n_runs < 1) BAD("empty run container");
            if (rc->capacity < rc->n_runs) BAD("run capacity too small");
            for (int32_t k = 0; k < rc->n_runs; k++) {
                uint32_t s = rc->runs[k].value, e = s + rc->runs[k].length;
                if (e > 65535) BAD("run overflows");
                if (k > 0) {
                    uint32_t pe = (uint32_t)rc->runs[k - 1].value + rc->runs[k - 1].length;
                    if (s <= pe + 1) BAD("runs overlap or are adjacent");
                }
            }
        } else {
            BAD("unknown typecode");
        }
    }
#undef BAD
    if (reason) *reason = "";
    return true;
}

// ---- portable format ------------------------------------------------------------------
size_t rb200_bitmap_portable_size_in_bytes(const roaring_bitmap_t *r) {
    const roaring_array_t *ra = &r->high_low_container;
    bool hasrun = false;
    size_t payload = 0;
    for (int32_t i = 0; i < ra->size; i++) {
        uint8_t t = ra->typecodes[i];
        const void *c = unwrap_shared(ra->containers[i], t);
        if (t == T_RUN) {
            hasrun = true;
            payload += 2 + 4 * (size_t)((const run_container_t *)c)->n_runs;
        } else if (t == T_ARRAY) {
            payload += 2 * (size_t)((const array_container_t *)c)->cardinality;
        } else {
            payload += BITSET_BYTES;
        }
    }
    const size_t n = (size_t)ra->size;
    size_t hdr;
    if (hasrun) hdr = 4 + (n + 7) / 8 + (ra->size < NO_OFFSET_THRESHOLD ? 4 * n : 8 * n);
    else hdr = 8 + 8 * n;
    return hdr + payload;
}

size_t rb200_bitmap_portable_serialize(const roaring_bitmap_t *r, char *buf) {
    const roaring_array_t *ra = &r->high_low_container;
    const size_t n = (size_t)ra->size;
    bool hasrun = false;
    for (int32_t i = 0; i < ra->size; i++) {
        uint8_t t = ra->typecodes[i];
        unwrap_shared(ra->containers[i], t);
        hasrun |= (t == T_RUN);
    }
    uint8_t *p = (uint8_t *)buf;
    uint32_t start;
    if (hasrun) {
        const uint32_t cookie = SERIAL_COOKIE | ((uint32_t)(ra->size - 1) << 16);
        memcpy(p, &cookie, 4);
        p += 4;
        const size_t s = (n + 7) / 8;
        memset(p, 0, s);
        for (int32_t i = 0; i < ra->size; i++) {
            uint8_t t = ra->typecodes[i];
            unwrap_shared(ra->containers[i], t);
            if (t == T_RUN) p[i / 8] |= (uint8_t)(1 << (i % 8));
        }
        p += s;
        start = (uint32_t)(4 + s + (ra->size < NO_OFFSET_THRESHOLD ? 4 * n : 8 * n));
    } else {
        const uint32_t cookie = SERIAL_COOKIE_NO_RUN, sz = (uint32_t)ra->size;
        memcpy(p, &cookie, 4);
        memcpy(p + 4, &sz, 4);
        p += 8;
        start = (uint32_t)(8 + 8 * n);
    }
    for (int32_t i = 0; i < ra->size; i++) {
        uint8_t t = ra->typecodes[i];
        const void *c = unwrap_shared(ra->containers[i], t);
        const uint16_t key = ra->keys[i], cm1 = (uint16_t)(host_container_card(c, t) - 1);
        memcpy(p, &key, 2);
        memcpy(p + 2, &cm1, 2);
        p += 4;
    }
    if (!hasrun || ra->size >= NO_OFFSET_THRESHOLD) {
        uint32_t off = start;
        for (int32_t i = 0; i < ra->size; i++) {
            memcpy(p, &off, 4);
            p += 4;
            uint8_t t = ra->typecodes[i];
            const void *c = unwrap_shared(ra->containers[i], t);
            off += t == T_BITSET ? (uint32_t)BITSET_BYTES
                   : t == T_ARRAY ? 2u * (uint32_t)((const array_container_t *)c)->cardinality
                                  : 2u + 4u * (uint32_t)((const run_container_t *)c)->n_runs;
        }
    }
    for (int32_t i = 0; i < ra->size; i++) {
        uint8_t t = ra->typecodes[i];
        const void *c = unwrap_shared(ra->containers[i], t);
        if (t == T_BITSET) {
            memcpy(p, ((const bitset_container_t *)c)->words, BITSET_BYTES);
            p += BITSET_BYTES;
        } else if (t == T_ARRAY) {
            const array_container_t *a = (const array_container_t *)c;
            memcpy(p, a->array, 2 * (size_t)a->cardinality);
            p += 2 * (size_t)a->cardinality;
        } else {
            const run_container_t *rc = (const run_container_t *)c;
            const uint16_t nr = (uint16_t)rc->n_runs;
            memcpy(p, &nr, 2);
            memcpy(p + 2, rc->runs, 4 * (size_t)rc->n_runs);
            p += 2 + 4 * (size_t)rc->n_runs;
        }
    }
    return (size_t)(p - (uint8_t *)buf);
}

}  // extern "C"

namespace {

// Parsed view of one portable-serialized bitmap (no allocation): per container key, type,
// cardinality, length and a pointer to the stored payload inside the buffer.
struct PView {
    int32_t size = 0;
    std::vector<uint16_t> key;
    std::vector<uint8_t> type;
    std::vector<uint32_t> card, len;
    std::vector<const uint8_t *> ptr;
};

bool parse_portable(const uint8_t *buf, size_t len, PView &v) {
    if (len < 4) return false;
    uint32_t cookie;
    memcpy(&cookie, buf, 4);
    size_t pos = 4;
    int32_t size;
    const uint8_t *runflags = nullptr;
    bool hasrun = false;
    if ((cookie & 0xFFFF) == SERIAL_COOKIE) {
        size = (int32_t)(cookie >> 16) + 1;
        hasrun = true;
        runflags = buf + pos;
        pos += (size_t)(size + 7) / 8;
    } else if (cookie == SERIAL_COOKIE_NO_RUN) {
        if (len < 8) return false;
        uint32_t s;
        memcpy(&s, buf + 4, 4);
        size = (int32_t)s;
        pos = 8;
    } else {
        return false;
    }
    if (size < 0 || size > 65536) return false;
    if (pos + 4 * (size_t)size > len) return false;
    const uint8_t *kc = buf + pos;
    pos += 4 * (size_t)size;
    if (!hasrun || size >= NO_OFFSET_THRESHOLD) pos += 4 * (size_t)size;
    v.size = size;
    v.key.resize(size);
    v.type.resize(size);
    v.card.resize(size);
    v.len.resize(size);
    v.ptr.resize(size);
    for (int32_t i = 0; i < size; i++) {
        uint16_t key, cm1;
        memcpy(&key, kc + 4 * i, 2);
        memcpy(&cm1, kc + 4 * i + 2, 2);
        if (i > 0 && key <= v.key[i - 1]) return false;
        const uint32_t card = (uint32_t)cm1 + 1;
        v.key[i] = key;
        v.card[i] = card;
        const bool isrun = hasrun && ((runflags[i / 8] >> (i % 8)) & 1);
        if (isrun) {
            if (pos + 2 > len) return false;
            uint16_t nr;
            memcpy(&nr, buf + pos, 2);
            pos += 2;
            if (pos + 4 * (size_t)nr > len) return false;
            v.type[i] = T_RUN;
            v.len[i] = nr;
            v.ptr[i] = buf + pos;
            pos += 4 * (size_t)nr;
        } else if (card > (uint32_t)MAX_ARRAY) {
            if (pos + BITSET_BYTES > len) return false;
            v.type[i] = T_BITSET;
            v.len[i] = 1024;
            v.ptr[i] = buf + pos;
            pos += BITSET_BYTES;
        } else {
            if (pos + 2 * (size_t)card > len) return false;
            v.type[i] = T_ARRAY;
            v.len[i] = card;
            v.ptr[i] = buf + pos;
            pos += 2 * (size_t)card;
        }
    }
    return true;
}

}  // namespace

extern "C" roaring_bitmap_t *rb200_bitmap_portable_deserialize_safe(const char *buf, size_t maxbytes) {
    PView v;
    if (!parse_portable((const uint8_t *)buf, maxbytes, v)) return nullptr;
    roaring_bitmap_t *r = bitmap_alloc(v.size);
    if (!r) return nullptr;
    roaring_array_t *ra = &r->high_low_container;
    for (int32_t i = 0; i < v.size; i++) {
        void *c = container_from_payload(v.type[i], v.card[i], v.len[i], v.ptr[i]);
        if (!c) {
            bitmap_free_host(r);
            return nullptr;
        }
        ra->containers[i] = c;
        ra->keys[i] = v.key[i];
        ra->typecodes[i] = v.type[i];
        ra->size = i + 1;
    }
    return r;
}

// =================================================================== upload
namespace {

// Source of containers for packing: either host bitmaps or parsed portable buffers.
struct PackSrc {
    const roaring_bitmap_t *const *bms = nullptr;
    const std::vector<PView> *views = nullptr;
    size_t n = 0;
};

rb200_set *upload_impl(const PackSrc &src) {
    if (!ctx_init()) return nullptr;
    const size_t nb = src.n;
    // pass 1: sizes
    uint64_t nc = 0, slab = 0;
    for (size_t b = 0; b < nb; b++) {
        if (src.bms) {
            const roaring_array_t *ra = &src.bms[b]->high_low_container;
            nc += (uint64_t)ra->size;
            for (int32_t i = 0; i < ra->size; i++) {
                uint8_t t = ra->typecodes[i];
                const void *c = unwrap_shared(ra->containers[i], t);
                uint32_t len = t == T_BITSET ? 1024u
                               : t == T_ARRAY ? (uint32_t)((const array_container_t *)c)->cardinality
                                              : (uint32_t)((const run_container_t *)c)->n_runs;
                slab += round16(stored_bytes(t, len));
            }
        } else {
            const PView &v = (*src.views)[b];
            nc += (uint64_t)v.size;
            for (int32_t i = 0; i < v.size; i++) slab += round16(stored_bytes(v.type[i], v.len[i]));
        }
    }
    rb200_set *s = set_new((uint32_t)nb, nc, slab);
    if (!s) return nullptr;
    s->n_containers = nc;
    s->slab_used = slab;
    // pass 2: directory into one pinned block, payload streamed through two pinned chunks
    uint8_t *hd = (uint8_t *)pin_alloc(s->L.total);
    const size_t CH = (size_t)32 << 20;
    uint8_t *chunk[2] = {(uint8_t *)pin_alloc(CH), (uint8_t *)pin_alloc(CH)};
    cudaEvent_t cev[2];
    bool ok = hd && chunk[0] && chunk[1];
    for (int k = 0; k < 2; k++) cudaEventCreateWithFlags(&cev[k], cudaEventDisableTiming);
    bool cev_used[2] = {false, false};
    if (ok) {
        uint32_t *bm_beg = (uint32_t *)(hd + s->L.o_beg), *bm_cnt = (uint32_t *)(hd + s->L.o_cnt);
        uint64_t *bm_card = (uint64_t *)(hd + s->L.o_bcard);
        uint16_t *c_key = (uint16_t *)(hd + s->L.o_key);
        uint8_t *c_type = hd + s->L.o_type;
        uint32_t *c_card = (uint32_t *)(hd + s->L.o_card), *c_len = (uint32_t *)(hd + s->L.o_len);
        uint64_t *c_off = (uint64_t *)(hd + s->L.o_off);
        uint32_t *c_src = (uint32_t *)(hd + s->L.o_src);
        if (src.bms) s->h_ptr_all = std::make_shared<std::vector<const void *>>(nc);
        uint64_t ci = 0, off = 0, chunk_base = 0;
        int cur = 0;
        size_t used = 0;
        auto flush = [&]() -> bool {
            if (used) {
                if (cudaMemcpyAsync(s->d_slab + chunk_base, chunk[cur], used, cudaMemcpyHostToDevice,
                                    g.stream) != cudaSuccess) return false;
                cudaEventRecord(cev[cur], g.stream);
                cev_used[cur] = true;
            }
            chunk_base += used;
            used = 0;
            cur ^= 1;
            if (cev_used[cur]) cudaEventSynchronize(cev[cur]);
            return true;
        };
        for (size_t b = 0; b < nb && ok; b++) {
            const roaring_array_t *ra = src.bms ? &src.bms[b]->high_low_container : nullptr;
            const PView *pv = src.views ? &(*src.views)[b] : nullptr;
            const int32_t size = ra ? ra->size : pv->size;
            bm_beg[b] = (uint32_t)ci;
            bm_cnt[b] = (uint32_t)size;
            s->h_cnt[b] = (uint32_t)size;
            s->h_flags[b] = ra ? (ra->flags & FLAG_COW) : 0;
            uint64_t bcard = 0, bbytes = 0, bebytes = 0;
            for (int32_t i = 0; i < size; i++, ci++) {
                uint8_t t;
                uint32_t card, len;
                const uint8_t *p;
                uint16_t key;
                bool was_shared = false;
                if (ra) {
                    t = ra->typecodes[i];
                    was_shared = t == T_SHARED;
                    const void *c = unwrap_shared(ra->containers[i], t);
                    key = ra->keys[i];
                    card = host_container_card(c, t);
                    if (t == T_BITSET) {
                        len = 1024;
                        p = (const uint8_t *)((const bitset_container_t *)c)->words;
                        if (((const bitset_container_t *)c)->cardinality < 0) {  // lazy state
                            card |= CARD_UNKNOWN;
                            s->lazy = true;
                        }
                    }
                    else if (t == T_ARRAY) { len = card; p = (const uint8_t *)((const array_container_t *)c)->array; }
                    else {
                        len = (uint32_t)((const run_container_t *)c)->n_runs;
                        p = (const uint8_t *)((const run_container_t *)c)->runs;
                        if (4 * (uint64_t)len > BITSET_BYTES) s->lazy = true;  // only lazy unions leave such runs
                    }
                } else {
                    t = pv->type[i];
                    key = pv->key[i];
                    len = pv->len[i];
                    p = pv->ptr[i];
                    if (t == T_RUN) {
                        card = 0;
                        for (uint32_t k = 0; k < len; k++) {
                            uint16_t l;
                            memcpy(&l, p + 4 * k + 2, 2);
                            card += (uint32_t)l + 1;
                        }
                    } else {
                        card = pv->card[i];
                    }
                }
                const uint32_t sb = stored_bytes(t, len), sb16 = round16(sb);
                if (used + sb16 > CH) ok = flush();
                memcpy(chunk[cur] + used, p, sb);
                if (sb16 > sb) memset(chunk[cur] + used + sb, 0, sb16 - sb);
                used += sb16;
                c_key[ci] = key;
                c_type[ci] = t;
                c_card[ci] = card;
                c_len[ci] = len;
                c_off[ci] = off;
                c_src[ci] = was_shared ? SRC_SHARED : SRC_NONE;
                if (s->h_ptr_all) (*s->h_ptr_all)[ci] = p;
                off += sb16;
                bcard += card & CARD_MASK;
                bbytes += sb16;
                bebytes += effective_bytes(t, len, card & CARD_MASK);
                s->portable_bytes += portable_bytes(t, len);
            }
            bm_card[b] = bcard;
            s->h_bytes[b] = bbytes;
            s->h_ebytes[b] = bebytes;
        }
        if (ok) ok = flush();
        if (ok && cudaMemcpyAsync(s->d_dir, hd, s->L.total, cudaMemcpyHostToDevice, g.stream) != cudaSuccess)
            ok = false;
        if (cudaStreamSynchronize(g.stream) != cudaSuccess) ok = false;
    }
    for (int k = 0; k < 2; k++) cudaEventDestroy(cev[k]);
    pin_free(hd, s->L.total);
    pin_free(chunk[0], CH);
    pin_free(chunk[1], CH);
    if (!ok) {
        if (t_err.empty()) t_err = "upload failed";
        set_delete(s);
        return nullptr;
    }
    return s;
}

}  // namespace

extern "C" {

rb200_set_t *rb200_set_upload(const roaring_bitmap_t *const *bitmaps, size_t n) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    PackSrc src;
    src.bms = bitmaps;
    src.n = n;
    return upload_impl(src);
}

// Portable-serialized inputs are parsed ON THE DEVICE (src/roaring_array.c:633-813 restated as
// k_deser_dir / k_deser_copy): the host only reads each blob's cookie (to size the directory) and
// streams the raw bytes through pinned staging chunks; no per-container host work.
static rb200_set *upload_blobs_impl(const char *const *bufs, const size_t *lens, size_t n, bool frozen);
rb200_set_t *rb200_set_upload_serialized(const char *const *bufs, const size_t *lens, size_t n) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return upload_blobs_impl(bufs, lens, n, false);
}
// The same for the FROZEN format (roaring_bitmap_frozen_serialize output, src/roaring.c:3180-3456);
// the blobs need no particular alignment here (frozen_view's 32-byte rule is about in-place use).
rb200_set_t *rb200_set_upload_frozen(const char *const *bufs, const size_t *lens, size_t n) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return upload_blobs_impl(bufs, lens, n, true);
}
static rb200_set *upload_blobs_impl(const char *const *bufs, const size_t *lens, size_t n, bool frozen) {
    if (!ctx_init()) return nullptr;
    if (n > 0xffffffffull) { t_err = "too many bitmaps"; return nullptr; }
    // pass 1 (host): container count of every blob from its cookie; staging offsets
    uint64_t nc = 0, raw_total = 0, slab_total = 0;
    std::vector<uint32_t> cnt(n);
    for (size_t i = 0; i < n; i++) {
        uint32_t cookie = 0, size = 0;
        bool ok = lens[i] >= 4;
        if (ok && frozen) {
            memcpy(&cookie, bufs[i] + lens[i] - 4, 4);   // the header is the LAST word
            size = cookie >> 15;
            ok = (cookie & 0x7FFF) == 13766 /* FROZEN_COOKIE */ && 5ull * size + 4 <= lens[i];
        } else if (ok) {
            memcpy(&cookie, bufs[i], 4);
            if ((cookie & 0xFFFF) == SERIAL_COOKIE) size = (cookie >> 16) + 1;
            else if (cookie == SERIAL_COOKIE_NO_RUN && lens[i] >= 8) memcpy(&size, bufs[i] + 4, 4);
            else ok = false;
        }
        if (!ok || size > 65536 || 4ull * size > lens[i]) {
            t_err = std::string(frozen ? "malformed frozen bitmap at index " : "malformed portable bitmap at index ") + std::to_string(i);
            return nullptr;
        }
        cnt[i] = size;
        nc += size;
        raw_total += (lens[i] + 15) & ~(uint64_t)15;
        slab_total += ((lens[i] + 15) & ~(uint64_t)15) + 16ull * size;   // payload <= blob bytes, + 16-byte padding per container
    }
    rb200_set *s = set_new((uint32_t)n, nc, slab_total + 16);
    if (!s) return nullptr;
    s->n_containers = nc;
    s->slab_used = slab_total;
    // per-bitmap tables: [roff | rlen | slab_base] for the kernels, bm_beg / bm_cnt into the directory
    const size_t tb = 24 * (n ? n : 1);
    uint64_t *h_tab = (uint64_t *)pin_alloc(tb), *d_tab = (uint64_t *)dev_alloc(tb);
    uint32_t *h_bc = (uint32_t *)pin_alloc(8 * (n ? n : 1));
    uint8_t *d_raw = (uint8_t *)dev_alloc(raw_total ? raw_total : 16);
    uint64_t *d_src = (uint64_t *)dev_alloc(8 * (nc ? nc : 1));
    const size_t CH = (size_t)32 << 20;
    uint8_t *chunk[2] = {(uint8_t *)pin_alloc(CH), (uint8_t *)pin_alloc(CH)};
    cudaEvent_t cev[2] = {nullptr, nullptr};
    bool cev_used[2] = {false, false};
    bool ok = h_tab && d_tab && h_bc && d_raw && d_src && chunk[0] && chunk[1];
    for (int k = 0; k < 2 && ok; k++) ok = cudaEventCreateWithFlags(&cev[k], cudaEventDisableTiming) == cudaSuccess;
    if (ok) {
        uint64_t ro = 0, so = 0, cb = 0;
        for (size_t i = 0; i < n; i++) {
            h_tab[i] = ro;
            h_tab[n + i] = lens[i];
            h_tab[2 * n + i] = so;
            h_bc[i] = (uint32_t)cb;
            h_bc[n + i] = cnt[i];
            s->h_cnt[i] = cnt[i];
            s->h_bytes[i] = lens[i] + 16ull * cnt[i];
            s->h_ebytes[i] = (uint64_t)cnt[i] * BITSET_BYTES + lens[i];   // replaced by the device's figures (ensure_mirrors)
            const uint64_t hdr = ((cnt[i] && (((uint8_t)bufs[i][0] | ((uint8_t)bufs[i][1] << 8)) == SERIAL_COOKIE))
                                     ? 4 + (cnt[i] + 7) / 8 + (cnt[i] < (uint32_t)NO_OFFSET_THRESHOLD ? 4ull : 8ull) * cnt[i]
                                     : 8 + 8ull * cnt[i]);
            s->portable_bytes += frozen ? lens[i] - 4 - 5ull * cnt[i] + 0 : (lens[i] > hdr ? lens[i] - hdr : 0);
            ro += (lens[i] + 15) & ~(uint64_t)15;
            so += ((lens[i] + 15) & ~(uint64_t)15) + 16ull * cnt[i];
            cb += cnt[i];
        }
        ok = cudaMemcpyAsync(d_tab, h_tab, tb, cudaMemcpyHostToDevice, g.stream) == cudaSuccess &&
             (n == 0 ||
              (cudaMemcpyAsync(s->d_dir + s->L.o_beg, h_bc, 4 * n, cudaMemcpyHostToDevice, g.stream) == cudaSuccess &&
               cudaMemcpyAsync(s->d_dir + s->L.o_cnt, h_bc + n, 4 * n, cudaMemcpyHostToDevice, g.stream) == cudaSuccess));
        // raw bytes as one stream through the two pinned chunks
        int cur = 0;
        size_t used = 0;
        uint64_t base = 0;
        auto flush = [&]() -> bool {
            if (used) {
                if (cudaMemcpyAsync(d_raw + base, chunk[cur], used, cudaMemcpyHostToDevice, g.stream) != cudaSuccess)
                    return false;
                cudaEventRecord(cev[cur], g.stream);
                cev_used[cur] = true;
            }
            base += used;
            used = 0;
            cur ^= 1;
            if (cev_used[cur]) cudaEventSynchronize(cev[cur]);
            return true;
        };
        for (size_t i = 0; i < n && ok; i++) {
            size_t done = 0;
            const size_t padded = (lens[i] + 15) & ~(size_t)15;
            while (done < padded && ok) {
                if (used == CH) ok = flush();
                const size_t room = CH - used, want = padded - done;
                const size_t take = room < want ? room : want;
                const size_t real = done < lens[i] ? std::min(take, lens[i] - done) : 0;
                if (real) memcpy(chunk[cur] + used, bufs[i] + done, real);
                if (take > real) memset(chunk[cur] + used + real, 0, take - real);
                used += take;
                done += take;
            }
        }
        if (ok) ok = flush();
    }
    if (ok) {
        ok = stats_reset();
        if (frozen)
            launch_deserialize_frozen(d_raw, d_tab, d_tab + n, d_tab + 2 * n, (uint32_t)n, nc, s->out(), d_src,
                                      g.d_stats, g.stream);
        else
            launch_deserialize(d_raw, d_tab, d_tab + n, d_tab + 2 * n, (uint32_t)n, nc, s->out(), d_src, g.d_stats,
                               g.stream);
        ok = ok && stats_fetch();
        cudaError_t e = cudaStreamSynchronize(g.stream);
        if (e != cudaSuccess || (e = cudaGetLastError()) != cudaSuccess) {
            t_err = std::string("deserialize: ") + cudaGetErrorString(e);
            ok = false;
        }
        if (ok && g.h_stats->error == 4u) {
            t_err = "malformed serialized bitmap: invalid container contents (a run ends past 65535, runs "
                    "overlap or are out of order, or array values are not strictly increasing)";
            ok = false;
        } else if (ok && g.h_stats->error) {
            t_err = std::string(frozen ? "malformed frozen bitmap at index " : "malformed portable bitmap at index ") +
                    std::to_string((uint64_t)n - g.h_stats->nk);
            ok = false;
        }
    } else {
        cudaStreamSynchronize(g.stream);
    }
    if (ok) s->mirrors_pending = n > 0;   // exact per-bitmap bytes / effective bytes: k_deser_bitmap_cards wrote them
    for (int k = 0; k < 2; k++) if (cev[k]) cudaEventDestroy(cev[k]);
    pin_free(chunk[0], CH);
    pin_free(chunk[1], CH);
    pin_free(h_tab, tb);
    pin_free(h_bc, 8 * (n ? n : 1));
    dev_free(d_tab, tb);
    dev_free(d_raw, raw_total ? raw_total : 16);
    dev_free(d_src, 8 * (nc ? nc : 1));
    if (!ok) {
        if (t_err.empty()) t_err = "upload_serialized failed";
        set_delete(s);
        return nullptr;
    }
    return s;
}

// Declare that the host bitmaps this set was uploaded from stay alive (and unmodified) for as long
// as results derived from it are downloaded: pass-through containers of OR / XOR / ANDNOT results
// are then rebuilt from the caller's own memory instead of crossing PCIe a second time.
int rb200_set_bind_host(rb200_set_t *s, int enable) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (enable && !s->h_ptr_all) { t_err = "bind_host: set was not uploaded from host bitmaps"; return -1; }
    s->h_ptr = enable ? s->h_ptr_all : nullptr;
    return 0;
}

void rb200_set_free(rb200_set_t *s) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    set_delete(s);
}
size_t rb200_set_count(const rb200_set_t *s) { return s->n_bitmaps; }
// Counters of the batch op that produced `s` (waits for it if it is still in flight): device time
// of the whole op and of its compute kernel (CUDA events on the library stream), algorithmic bytes.
int rb200_set_op_stats(const rb200_set_t *s, float *device_ms, float *compute_ms, uint64_t *algorithmic_bytes) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!resolve(s)) return -1;
    if (device_ms) *device_ms = s->ms;
    if (compute_ms) *compute_ms = s->compute_ms;
    if (algorithmic_bytes) *algorithmic_bytes = s->algo_bytes;
    return 0;
}
uint64_t rb200_set_container_count(const rb200_set_t *s) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    resolve(s);
    return s->n_containers;
}
uint64_t rb200_set_payload_bytes(const rb200_set_t *s) { return s->portable_bytes; }

}  // extern "C"

// =================================================================== batched pairwise ops
namespace {

// Host mirrors of a batch result (containers / cardinality per bitmap) are fetched lazily: a
// result that is only measured, chained on the device or downloaded never pays this D2H.
bool ensure_mirrors(const rb200_set *cs) {
    rb200_set *s = const_cast<rb200_set *>(cs);
    if (!resolve(cs)) return false;
    if (!s->mirrors_pending) return true;
    const size_t nb = s->n_bitmaps;
    // one copy: [cnt | bcard | bbytes | bebytes], all written by the kernel that produced the set
    const size_t bytes = (s->L.o_bebytes - s->L.o_cnt) + 8 * nb;
    uint8_t *h = (uint8_t *)pin_alloc(bytes);
    if (!h) return false;
    bool ok = cudaMemcpyAsync(h, s->d_dir + s->L.o_cnt, bytes, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
              cudaStreamSynchronize(g.stream) == cudaSuccess;
    if (ok) {
        const uint32_t *cnt = (const uint32_t *)h;
        const uint64_t *card = (const uint64_t *)(h + (s->L.o_bcard - s->L.o_cnt));
        const uint64_t *bb = (const uint64_t *)(h + (s->L.o_bbytes - s->L.o_cnt));
        const uint64_t *be = (const uint64_t *)(h + (s->L.o_bebytes - s->L.o_cnt));
        s->h_card.assign(card, card + nb);
        for (size_t p = 0; p < nb; p++) {
            s->h_cnt[p] = cnt[p];
            s->h_bytes[p] = bb[p];    // exact stored bytes (16-byte rounded slots) of this bitmap
            s->h_ebytes[p] = be[p];   // what a later op on it can produce at most (see PairBuf::build)
        }
        s->mirrors_pending = false;
    } else {
        t_err = "fetching result directory failed";
    }
    pin_free(h, bytes);
    return ok;
}

struct ItemsBuf {
    uint8_t *block = nullptr;
    size_t bytes = 0;
    Items it;
    // with_desc: cell descriptors (k_compute_items); with_order: batches with at least order_min item
    // slots also get them sorted by class
    bool alloc(uint64_t W, bool with_desc, bool with_order) {
        size_t o = 0;
        const size_t o_off = o; o += al256(8 * W);
        const size_t o_desc = o; if (with_desc) o += al256(32 * W);
        const size_t o_dcls = o; if (with_order) o += al256(32 * W);
        const size_t o_cls = o; if (with_order) o += al256(W);
        const size_t o_ca = o; o += al256(4 * W);
        const size_t o_cb = o; o += al256(4 * W);
        const size_t o_ocard = o; o += al256(4 * W);
        const size_t o_olen = o; o += al256(4 * W);
        const size_t o_key = o; o += al256(2 * W);
        const size_t o_kind = o; o += al256(W);
        const size_t o_otype = o; o += al256(W);
        bytes = o ? o : 256;
        block = (uint8_t *)dev_alloc(bytes);
        if (!block) return false;
        it.slot_off = (uint64_t *)(block + o_off);
        it.desc = with_desc ? (uint4 *)(block + o_desc) : nullptr;
        it.desc_cls = with_order ? (uint4 *)(block + o_dcls) : nullptr;
        it.cls = with_order ? block + o_cls : nullptr;
        it.ca = (uint32_t *)(block + o_ca);
        it.cb = (uint32_t *)(block + o_cb);
        it.ocard = (uint32_t *)(block + o_ocard);
        it.olen = (uint32_t *)(block + o_olen);
        it.key = (uint16_t *)(block + o_key);
        it.kind = block + o_kind;
        it.otype = block + o_otype;
        return true;
    }
    void release() { dev_free(block, bytes); block = nullptr; }
};

// pair lists + item offsets: one pinned staging block, one H2D copy
struct PairBuf {
    uint8_t *h = nullptr, *d = nullptr;
    size_t bytes = 0;
    uint32_t *d_ia = nullptr, *d_ib = nullptr;
    uint64_t *d_off = nullptr;
    uint64_t W = 0, slab_bound = 0;
    // op: OP_* of the batch (OP_AND also for the cardinality-only sweeps, which need no slab)
    // flip: B is the range bitmap of rb200_batch_flip (every container ONE run)
    bool build(const rb200_set *A, const rb200_set *B, const uint32_t *ia, const uint32_t *ib,
               size_t np, int op, bool lazy = false, bool flip = false) {
        if (!ensure_mirrors(A) || !ensure_mirrors(B)) return false;
        if (np > 0xffffffffull) { t_err = "too many pairs in one batch (2^32 - 1 at most)"; return false; }
        const size_t o_off = 0, o_ia = al256(8 * (np + 1)), o_ib = o_ia + al256(4 * np);
        bytes = o_ib + al256(4 * np);
        h = (uint8_t *)pin_alloc(bytes);
        d = (uint8_t *)dev_alloc(bytes);
        if (!h || !d) return false;
        uint64_t *off = (uint64_t *)(h + o_off);
        uint32_t *hia = (uint32_t *)(h + o_ia), *hib = (uint32_t *)(h + o_ib);
        uint64_t w = 0, sb = 0;
        for (size_t p = 0; p < np; p++) {
            const uint32_t a = ia[p], b = ib[p];
            if (a >= A->n_bitmaps || b >= B->n_bitmaps) {
                t_err = "pair index out of range";
                return false;
            }
            hia[p] = a;
            hib[p] = b;
            off[p] = w;
            const uint32_t na = A->h_cnt[a], nb = B->h_cnt[b];
            w += (uint64_t)na + nb;
            // Upper bound of the result slab of this pair, from the per-bitmap "effective bytes" E
            // (sum over containers of max(stored, min(8192, 2 * card)), 16-byte rounded): every
            // result container — computed or passed through — is an array, a bitset or a run no
            // larger than either, so it fits min(8192, 2 * card_result); card_result <= cA + cB
            // (OR, XOR), <= min(cA, cB) (AND), <= cA (ANDNOT).  slot_bound() obeys the same limits.
            const uint64_t EA = A->h_ebytes[a], EB = B->h_ebytes[b];
            if (flip) {
                // the slots k_plan_pairs reserves: a copy of A's container (<= its effective bytes),
                // a copy of a one-run range container (16), a matched cell (slot_bound_lazy with
                // nB = 1: <= 8 KiB + 16 + twice A's stored bytes).  EB counts 8 KiB for every key
                // the range covers, which for a range over the whole universe is 512 MiB per pair.
                const uint64_t m = na < nb ? na : nb;
                sb += 2 * EA + 16 * (uint64_t)nb + m * (uint64_t)(BITSET_BYTES + 16) + 512;
            } else if (lazy) {
                // lazy array x run unions stay runs (4 bytes per input value / run), flips add 8 KiB per key
                const uint64_t m = na < nb ? na : nb;
                sb += 3 * (EA + EB) + m * (uint64_t)BITSET_BYTES + 512;
            } else if (op == OP_AND) {
                sb += (EA < EB ? EA : EB) + 64;
            } else if (op == OP_ANDNOT) {
                sb += EA + 64;
            } else {
                sb += EA + EB + 64;
            }
        }
        off[np] = w;
        // item ids, directory positions of the result and the order list are 32-bit on the device
        if (w > 0xffffffffull) { t_err = "batch too large: more than 2^32 - 1 container slots, split the pair list"; return false; }
        W = w;
        slab_bound = sb;
        d_off = (uint64_t *)(d + o_off);
        d_ia = (uint32_t *)(d + o_ia);
        d_ib = (uint32_t *)(d + o_ib);
        return cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, g.stream) == cudaSuccess;
    }
    void release() {
        pin_free(h, bytes);
        dev_free(d, bytes);
        h = d = nullptr;
    }
};

bool stats_reset() {
    return cudaMemsetAsync(g.d_stats, 0, sizeof(OpStats), g.stream) == cudaSuccess;
}
bool stats_fetch() {
    if (cudaMemcpyAsync(g.h_stats, g.d_stats, sizeof(OpStats), cudaMemcpyDeviceToHost, g.stream) != cudaSuccess)
        return false;
    return true;
}

bool reject_lazy(const rb200_set *s, const char *what) {
    if (!s->lazy) return false;
    t_err = std::string(what) + ": the set is in a lazy state, call rb200_set_repair_after_lazy first";
    return true;
}

rb200_set *batch_op_impl(int op, const rb200_set *A, const rb200_set *B, const uint32_t *ia,
                         const uint32_t *ib, size_t np, int rules = 0) {
    if (!ctx_init()) return nullptr;
    if (op < 0 || op > 3) { t_err = "bad op"; return nullptr; }
    if (rules & RULES_LAZY) {
        if (op != OP_OR && op != OP_XOR) { t_err = "lazy rules exist for OR and XOR only"; return nullptr; }
        if (op == OP_XOR && (rules & (RULES_CONV | RULES_NOFULL))) { t_err = "bad lazy flags for XOR"; return nullptr; }
        if ((rules & RULES_FLIP) && op != OP_XOR) { t_err = "bad flags"; return nullptr; }
    } else {
        if (rules & ~RULES_INPLACE) { t_err = "bad flags"; return nullptr; }
        if (reject_lazy(A, "batch op") || reject_lazy(B, "batch op")) return nullptr;
    }
    if (np > 0xffffffffull) { t_err = "too many pairs"; return nullptr; }
    PairBuf pb;
    ItemsBuf ib_;
    rb200_set *R = nullptr;
    bool ok = pb.build(A, B, ia, ib, np, op, (rules & RULES_LAZY) != 0, (rules & RULES_FLIP) != 0);
    // class-ordered tickets pay one more small kernel: only for batches that fill the GPU
    static const uint64_t order_min = []() { const char *e = getenv("RB200_ORDER_MIN"); return e ? (uint64_t)atoll(e) : 16384ull; }();
    // (tried in round 2: ONE launch with a CTA per pair doing plan -> cells -> finalize for small batches —
    //  the 199-pair successive sweep took more device time per call: a pair's cells serialise on
    //  its 8 warps while the three-kernel path spreads them over the GPU)
    if (ok) ok = ib_.alloc(pb.W, true, pb.W >= order_min);
    if (ok) {
        R = set_new((uint32_t)np, pb.W, pb.slab_bound);
        ok = R != nullptr;
    }
    if (ok) {
        for (int k = 0; k < 4; k++) R->ev[k] = ev_get();
        R->pstats = (OpStats *)pin_alloc(sizeof(OpStats));
        ok = R->pstats && R->ev[0] && R->ev[1] && R->ev[2] && R->ev[3];
    }
    if (ok) {
        cudaEventRecord(R->ev[0], g.stream);
        ok = stats_reset();
        const SetView va = A->view(), vb = B->view();
        launch_plan_pairs(va, vb, pb.d_ia, pb.d_ib, pb.d_off, (uint32_t)np, op, false, rules, ib_.it,
                          g.d_stats, g.stream);
        launch_order_items(ib_.it, pb.W, g.d_stats, g.stream);
        cudaEventRecord(R->ev[1], g.stream);
        // pass-through tickets: one item per lane, fewer lanes when the operands' containers are big
        // (32 x 8 KiB on one warp would be the tail of the launch)
        const uint64_t n_cont = A->n_containers + B->n_containers;
        const uint64_t avg_b = n_cont ? (A->slab_used + B->slab_used) / n_cont : 4096;
        // (on the real-data suite 4-32 items per ticket are within noise of each other, 1 item is
        //  clearly slower — RB200_COPY_TICKET overrides)
        static const int ct_env = []() { const char *e = getenv("RB200_COPY_TICKET"); return e ? std::min(32, std::max(1, atoi(e))) : 0; }();
        const int copy_ticket = ct_env ? ct_env : avg_b <= 256 ? 32 : avg_b <= 2048 ? 16 : 8;
        launch_compute_items(va, vb, ib_.it, pb.W, op, R->d_slab, R->slab_cap, g.d_stats, rules, copy_ticket, g.stream);
        cudaEventRecord(R->ev[2], g.stream);
        launch_finalize_pairs(va, vb, ib_.it, pb.d_off, (uint32_t)np, R->out(), g.d_stats, g.stream);
        ok = ok && cudaMemcpyAsync(R->pstats, g.d_stats, sizeof(OpStats), cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        cudaEventRecord(R->ev[3], g.stream);
        // no synchronisation here: the counters are taken over by resolve() on first use
        R->pending = true;
        R->staging = pb.h;            // the pinned pair list must outlive its H2D copy
        R->staging_bytes = pb.bytes;
        pb.h = nullptr;
        R->parentA = A->h_ptr;
        R->parentB = B->h_ptr;
        R->portable_bytes = 0;
        R->mirrors_pending = np > 0;  // h_cnt / h_bytes / h_card: see ensure_mirrors()
        R->lazy = (rules & RULES_LAZY) != 0 && !(rules & RULES_FLIP);
        for (size_t p = 0; p < np; p++) R->h_flags[p] = (A->h_flags[ia[p]] | B->h_flags[ib[p]]) & FLAG_COW;
        g.last_op = R;
    }
    pb.release();     // device buffers: stream-ordered reuse
    ib_.release();
    if (!ok) {
        if (t_err.empty()) t_err = "batch op: enqueue failed";
        set_delete(R);
        return nullptr;
    }
    return R;
}

}  // namespace

extern "C" {

rb200_set_t *rb200_batch_op(int op, const rb200_set_t *A, const rb200_set_t *B, const uint32_t *ia,
                            const uint32_t *ib, size_t npairs) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return batch_op_impl(op, A, B, ia, ib, npairs);
}

rb200_set_t *rb200_batch_op_ex(int op, int flags, const rb200_set_t *A, const rb200_set_t *B,
                               const uint32_t *ia, const uint32_t *ib, size_t npairs) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return batch_op_impl(op, A, B, ia, ib, npairs, flags & (RULES_INPLACE | RULES_LAZY | RULES_CONV | RULES_NOFULL));
}

int rb200_batch_and_cardinality(const rb200_set_t *A, const rb200_set_t *B, const uint32_t *ia,
                                const uint32_t *ib, size_t np, uint64_t *out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    if (np == 0) return 0;
    if (reject_lazy(A, "and_cardinality") || reject_lazy(B, "and_cardinality")) return -1;
    PairBuf pb;
    ItemsBuf ib_;
    uint64_t *d_out = nullptr, *h_out = nullptr;
    bool ok = pb.build(A, B, ia, ib, np, OP_AND);
    if (ok) ok = ib_.alloc(pb.W, false, false);
    if (ok) { d_out = (uint64_t *)dev_alloc(8 * np); h_out = (uint64_t *)pin_alloc(8 * np); ok = d_out && h_out; }
    if (ok) {
        cudaEventRecord(g.ev0, g.stream);
        ok = stats_reset();
        const SetView va = A->view(), vb = B->view();
        launch_plan_pairs(va, vb, pb.d_ia, pb.d_ib, pb.d_off, (uint32_t)np, OP_AND, true, 0, ib_.it,
                          g.d_stats, g.stream);
        cudaEventRecord(g.evk0, g.stream);
        launch_card_items(va, vb, ib_.it, pb.W, g.d_stats, g.stream);
        cudaEventRecord(g.evk1, g.stream);
        launch_finalize_cards(ib_.it, pb.d_off, (uint32_t)np, d_out, g.stream);
        cudaEventRecord(g.ev1, g.stream);
        ok = ok && cudaMemcpyAsync(h_out, d_out, 8 * np, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        cudaError_t e = cudaStreamSynchronize(g.stream);
        if (e != cudaSuccess) { t_err = std::string("and_cardinality: ") + cudaGetErrorString(e); ok = false; }
        if (ok && (e = cudaGetLastError()) != cudaSuccess) { t_err = std::string("and_cardinality launch: ") + cudaGetErrorString(e); ok = false; }
    }
    if (ok) {
        memcpy(out, h_out, 8 * np);
        g.last_op = nullptr;  // the rb200_last_* getters now describe this (synchronous) op
        cudaEventElapsedTime(&g.last_ms, g.ev0, g.ev1);
        cudaEventElapsedTime(&g.last_compute_ms, g.evk0, g.evk1);
    }
    dev_free(d_out, 8 * np);
    pin_free(h_out, 8 * np);
    pb.release();
    ib_.release();
    return ok ? 0 : -1;
}

// Sharded form: after k_or_many2 the per-key cardinalities of [span_lo, span_hi] are all-reduced
// across the communicator ON THE DEVICE (one ncclAllReduce on the library stream), then that
// span alone (4 * K bytes) is read back.
struct ShardArgs {
    rb200_comm *comm;
    uint32_t span_lo, span_hi;
    uint32_t *card_span;   // host, span_hi - span_lo + 1 entries (may be null)
    uint64_t *total_card;  // host (may be null)
};
static float g_last_collective_ms = 0.f;

static rb200_set *or_many_impl(const rb200_set_t *S, const uint32_t *idx, size_t n, uint32_t key_lo,
                               uint32_t key_hi, uint32_t *card_per_key, const ShardArgs *sh) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return nullptr;
    if (key_hi > 65535) key_hi = 65535;
    uint32_t span_n = 0;
    if (sh) {
        if (sh->span_hi > 65535 || sh->span_lo > sh->span_hi) { t_err = "or_many_sharded: bad key span"; return nullptr; }
        span_n = sh->span_hi - sh->span_lo + 1;
    }
    const bool want_ck = card_per_key != nullptr || sh != nullptr;
    if (reject_lazy(S, "or_many")) return nullptr;
    if (!ensure_mirrors(S)) return nullptr;
    if (idx == nullptr) n = S->n_bitmaps;
    // the index (rb200_many2.cu) holds input positions, per-key segments and counts in 32 bits; its
    // entry buffer is sized for every container of the inputs (the host has no per-bitmap keys to
    // count only those of [key_lo, key_hi]), so the container limit covers them all
    if (n > 0xffffffffu) { t_err = "or_many: more than 2^32 - 1 inputs"; return nullptr; }
    uint64_t tot = 0;
    for (size_t i = 0; i < n; i++) {
        const uint32_t b = idx ? idx[i] : (uint32_t)i;
        if (b >= S->n_bitmaps) { t_err = "or_many: index out of range"; return nullptr; }
        tot += S->h_cnt[b];
    }
    if (tot > 0xffffffffu) { t_err = "or_many: the inputs carry more than 2^32 - 1 containers (every key counts, whatever the key range)"; return nullptr; }
    uint64_t maxk = key_lo <= key_hi ? (uint64_t)key_hi - key_lo + 1 : 0;
    if (tot < maxk) maxk = tot;
    rb200_set *R = set_new(1, maxk, maxk * BITSET_BYTES);
    if (!R) return nullptr;
    uint32_t *d_idx = nullptr, *h_idx = nullptr;
    bool ok = true;
    if (idx && n) {
        d_idx = (uint32_t *)dev_alloc(4 * n);
        h_idx = (uint32_t *)pin_alloc(4 * n);
        ok = d_idx && h_idx;
        if (ok) {
            memcpy(h_idx, idx, 4 * n);
            ok = cudaMemcpyAsync(d_idx, h_idx, 4 * n, cudaMemcpyHostToDevice, g.stream) == cudaSuccess;
        }
    }
    uint32_t *h_ck = nullptr;
    cudaEvent_t evc0 = nullptr, evc1 = nullptr;
    if (ok && want_ck) { h_ck = (uint32_t *)pin_alloc(65536 * 4); ok = h_ck != nullptr; }
    if (ok && sh) { evc0 = ev_get(); evc1 = ev_get(); ok = evc0 && evc1; }
    // index: entries + work-unit table from the device pool
    uint64_t tot_kib = 0;
    for (size_t i = 0; i < n; i++) tot_kib += (S->h_bytes[idx ? idx[i] : i] >> 10) + 1;
    const uint64_t max_units = std::max<uint64_t>(1, std::min<uint64_t>(tot, std::min<uint64_t>(65536, tot) + tot_kib / 32 + 1));
    // key-window index build: per-(window, chunk of 256 bitmaps) key counts when there are several chunks
    const uint64_t m2_chunks = (n + 255) / 256;
    const size_t tab_bytes = m2_chunks > 1 && m2_chunks <= M2W_MAX_CHUNKS ? (size_t)2048 * m2_chunks * 32 * 4 : 0;
    const size_t e_bytes = al256(16 * tot) + al256(4 * max_units) + al256(tab_bytes);
    uint8_t *d_index = nullptr;
    if (ok) { d_index = (uint8_t *)dev_alloc(e_bytes); ok = d_index != nullptr; }
    if (ok) {
        cudaEventRecord(g.ev0, g.stream);
        ok = stats_reset();
        const SetView vs = S->view();
        Many2Index ix;
        ix.key_cu = (unsigned long long *)g.d_m2_tables;          // [0, 2): zeroed per call
        ix.w_shift = m2_weight_shift(n);
        ix.key_fill = g.d_m2_tables + 2 * 65536;                  // [2, 3): zeroed per call
        ix.key_count = g.d_m2_tables + 3 * 65536;
        ix.key_start = g.d_m2_tables + 4 * 65536;
        ix.key_slices = g.d_m2_tables + 5 * 65536;
        ix.key_scratch = g.d_m2_tables + 6 * 65536;
        ix.unit_first = g.d_m2_tables + 7 * 65536;
        ix.fold_first = (unsigned long long *)(g.d_m2_tables + 8 * 65536);
        ix.fold_second = (unsigned long long *)(g.d_m2_tables + 10 * 65536);
        ix.fold_F = g.d_m2_tables + 12 * 65536;
        ix.fold_L = g.d_m2_tables + 13 * 65536;
        ix.keys = g.d_keys;
        ix.ent = (uint4 *)d_index;
        ix.unit_ki = (uint32_t *)(d_index + al256(16 * tot));
        // operand staging by TMA bulk copies pays off when the containers are mostly bitsets
        // (RB200_OR_MANY_TMA=0/1 forces the choice)
        static const int tma_env = []() { const char *e = getenv("RB200_OR_MANY_TMA"); return e ? atoi(e) : -1; }();
        const bool use_tma = tma_env >= 0 ? tma_env != 0 : (tot > 0 && tot_kib / tot >= 7);   // measured: 6 KiB average (config 3, d = 0.1) is already faster direct
        // index build: key windows + shared-memory counting when the directories are long (a window
        // costs one directory search per input), one L2 atomic per container otherwise
        // (RB200_OR_MANY_INDEX=window / atomic forces the choice)
        static const int win_env = []() { const char *e = getenv("RB200_OR_MANY_INDEX"); return !e ? -1 : !strcmp(e, "window") ? 1 : 0; }();
        const bool window_index = m2_chunks <= M2W_MAX_CHUNKS && n > 0 && (win_env >= 0 ? win_env != 0 : (tot >= 64 * (uint64_t)n));
        cudaMemsetAsync(g.d_m2_tables, 0, 3 * 65536 * sizeof(uint32_t), g.stream);
        if (want_ck) cudaMemsetAsync(g.d_cardkey, 0, 65536 * 4, g.stream);
        launch_or_many2(vs, d_idx, (uint32_t)n, key_lo, key_hi, ix, (uint32_t)max_units,
                        g.d_m2_scratch, g.d_m2_tickets, M2_SCRATCH_SLOTS, R->out(), want_ck ? g.d_cardkey : nullptr,
                        g.d_stats, g.sms, g.stream, g.evk0, use_tma, window_index,
                        (uint32_t *)(d_index + al256(16 * tot) + al256(4 * max_units)));
    }
    if (ok) {
        cudaEventRecord(g.evk1, g.stream);
        if (sh) {  // the ONE collective of the path: per-key cardinalities, summed over the ranks, on the device
            cudaEventRecord(evc0, g.stream);
            ok = ok && comm_allreduce_sum(sh->comm, g.d_cardkey + sh->span_lo, span_n, false, g.stream, t_err);
            cudaEventRecord(evc1, g.stream);
        }
        cudaEventRecord(g.ev1, g.stream);
        ok = ok && stats_fetch();
        if (card_per_key)
            ok = ok && cudaMemcpyAsync(h_ck, g.d_cardkey, 65536 * 4, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        else if (sh)
            ok = ok && cudaMemcpyAsync(h_ck, g.d_cardkey + sh->span_lo, 4ull * span_n, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        cudaError_t e = cudaStreamSynchronize(g.stream);
        if (e != cudaSuccess) { t_err = std::string("or_many: ") + cudaGetErrorString(e); ok = false; }
        if (ok && (e = cudaGetLastError()) != cudaSuccess) { t_err = std::string("or_many launch: ") + cudaGetErrorString(e); ok = false; }
    }
    if (ok) {
        g.last_op = nullptr;  // the rb200_last_* getters now describe this (synchronous) op
        cudaEventElapsedTime(&g.last_ms, g.ev0, g.ev1);
        cudaEventElapsedTime(&g.last_compute_ms, g.evk0, g.evk1);
        const uint32_t nk = g.h_stats->nk;
        R->n_containers = nk;
        R->slab_used = (uint64_t)nk * BITSET_BYTES;
        R->h_cnt[0] = nk;
        R->h_bytes[0] = (uint64_t)nk * BITSET_BYTES;
        R->h_ebytes[0] = (uint64_t)nk * BITSET_BYTES;
        uint8_t fl = 0;
        // roaring_bitmap_lazy_or propagates COW from the inputs (roaring.c:2523)
        for (size_t i = 0; i < n; i++) fl |= S->h_flags[idx ? idx[i] : i];
        R->h_flags[0] = fl & FLAG_COW;
        if (card_per_key)
            for (int k = 0; k < 65536; k++) card_per_key[k] += h_ck[k];
        if (sh) {
            const uint32_t *span = card_per_key ? h_ck + sh->span_lo : h_ck;
            uint64_t tot = 0;
            for (uint32_t k = 0; k < span_n; k++) tot += span[k];
            if (sh->card_span) memcpy(sh->card_span, span, 4ull * span_n);
            if (sh->total_card) *sh->total_card = tot;
            cudaEventElapsedTime(&g_last_collective_ms, evc0, evc1);
        }
        // algorithmic bytes (SURVEY.md §8d): all input containers in range + outputs; the
        // output term is added by the caller-visible stat only when the set is downloaded,
        // here we account inputs exactly from the host mirrors when the whole key space is used.
        uint64_t inb = 0;
        if (key_lo == 0 && key_hi == 65535 && idx == nullptr) inb = S->portable_bytes;
        g.last_algo_bytes = inb;
    }
    dev_free(d_idx, 4 * n);
    dev_free(d_index, e_bytes);
    pin_free(h_idx, 4 * n);
    pin_free(h_ck, 65536 * 4);
    ev_put(evc0);
    ev_put(evc1);
    if (!ok) {
        if (t_err.empty()) t_err = "or_many failed";
        set_delete(R);
        return nullptr;
    }
    return R;
}

rb200_set_t *rb200_or_many_keyrange(const rb200_set_t *S, const uint32_t *idx, size_t n,
                                    uint32_t key_lo, uint32_t key_hi, uint32_t *card_per_key) {
    return or_many_impl(S, idx, n, key_lo, key_hi, card_per_key, nullptr);
}

rb200_set_t *rb200_or_many(const rb200_set_t *S, const uint32_t *idx, size_t n) {
    return or_many_impl(S, idx, n, 0, 65535, nullptr, nullptr);
}

// Key-sharded roaring_bitmap_or_many (SURVEY.md §8(e)): this rank reduces the keys [key_lo, key_hi]
// of its resident set (which normally holds only those keys, rb200_set_upload_serialized_keyrange),
// then the ranks exchange ONE all-reduce(sum) of the per-key result cardinalities over the key
// span [span_lo, span_hi] every rank agreed on (rb200_plan_key_ranges).
rb200_set_t *rb200_or_many_sharded(const rb200_set_t *S, const uint32_t *idx, size_t n, uint32_t key_lo,
                                   uint32_t key_hi, uint32_t span_lo, uint32_t span_hi, rb200_comm_t *comm,
                                   uint32_t *card_span, uint64_t *total_card) {
    ShardArgs sh{comm, span_lo, span_hi, card_span, total_card};
    return or_many_impl(S, idx, n, key_lo, key_hi, nullptr, &sh);
}
float rb200_last_collective_ms(void) { return g_last_collective_ms; }

// *d_acc (device, u64) += sum of the cardinalities of every bitmap of the set, on the library stream
// (a checksum that stays on the device until the caller reduces / reads it).
int rb200_set_add_cardinality_device(const rb200_set_t *s, uint64_t *d_acc) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    if (s->failed) { t_err = "the operation that produced this set failed"; return -1; }
    launch_sum_cardinalities((const uint64_t *)(s->d_dir + s->L.o_bcard), s->n_bitmaps, d_acc, g.stream);
    return 0;
}
// in-place all-reduce(sum) of `count` u64 words in device memory on the library stream
int rb200_comm_allreduce_u64(rb200_comm_t *comm, uint64_t *d_buf, size_t count) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    return comm_allreduce_sum(comm, d_buf, count, true, g.stream, t_err) ? 0 : -1;
}

// roaring_bitmap_xor_many (src/roaring.c:795-809) over S[idx[0..n)] (idx == NULL: all, in order).
rb200_set_t *rb200_xor_many(const rb200_set_t *S, const uint32_t *idx, size_t n) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return nullptr;
    if (reject_lazy(S, "xor_many")) return nullptr;
    if (!ensure_mirrors(S)) return nullptr;
    if (idx == nullptr) n = S->n_bitmaps;
    uint64_t tot = 0;
    for (size_t i = 0; i < n; i++) {
        const uint32_t b = idx ? idx[i] : (uint32_t)i;
        if (b >= S->n_bitmaps) { t_err = "xor_many: index out of range"; return nullptr; }
        tot += S->h_cnt[b];
    }
    const uint64_t maxk = std::min<uint64_t>(65536, tot);
    rb200_set *R = set_new(1, maxk, maxk * BITSET_BYTES);
    if (!R) return nullptr;
    uint32_t *d_idx = nullptr, *h_idx = nullptr;
    uint8_t *t_type = (uint8_t *)dev_alloc(maxk);
    uint32_t *t_card = (uint32_t *)dev_alloc(4 * maxk), *t_len = (uint32_t *)dev_alloc(4 * maxk);
    bool ok = t_type && t_card && t_len;
    if (ok && idx && n) {
        d_idx = (uint32_t *)dev_alloc(4 * n);
        h_idx = (uint32_t *)pin_alloc(4 * n);
        ok = d_idx && h_idx;
        if (ok) {
            memcpy(h_idx, idx, 4 * n);
            ok = cudaMemcpyAsync(d_idx, h_idx, 4 * n, cudaMemcpyHostToDevice, g.stream) == cudaSuccess;
        }
    }
    if (ok) {
        cudaEventRecord(g.ev0, g.stream);
        ok = stats_reset();
        const SetView vs = S->view();
        launch_many_mark(vs, d_idx, (uint32_t)n, 0, 65535, g.d_flags, g.stream);
        launch_many_compact(g.d_flags, g.d_keys, g.d_stats, g.stream);
        cudaEventRecord(g.evk0, g.stream);
        launch_xor_many(vs, d_idx, (uint32_t)n, g.d_keys, t_type, t_card, t_len, R->out(), g.d_stats,
                        g.sms, g.stream);
        cudaEventRecord(g.evk1, g.stream);
        cudaEventRecord(g.ev1, g.stream);
        ok = ok && stats_fetch();
        cudaError_t e = cudaStreamSynchronize(g.stream);
        if (e != cudaSuccess) { t_err = std::string("xor_many: ") + cudaGetErrorString(e); ok = false; }
        if (ok && (e = cudaGetLastError()) != cudaSuccess) { t_err = std::string("xor_many launch: ") + cudaGetErrorString(e); ok = false; }
    }
    if (ok) {
        g.last_op = nullptr;  // the rb200_last_* getters now describe this (synchronous) op
        cudaEventElapsedTime(&g.last_ms, g.ev0, g.ev1);
        cudaEventElapsedTime(&g.last_compute_ms, g.evk0, g.evk1);
        const uint32_t live = (uint32_t)g.h_stats->dir_cursor;
        R->n_containers = live;
        R->slab_used = (uint64_t)g.h_stats->nk * BITSET_BYTES;
        R->h_cnt[0] = live;
        R->h_bytes[0] = (uint64_t)live * BITSET_BYTES;
        R->h_ebytes[0] = (uint64_t)live * BITSET_BYTES;
        uint8_t fl = 0;
        for (size_t i = 0; i < n; i++) fl |= S->h_flags[idx ? idx[i] : i];
        R->h_flags[0] = fl & FLAG_COW;
        g.last_algo_bytes = (idx == nullptr) ? S->portable_bytes : 0;
    }
    dev_free(d_idx, 4 * n);
    pin_free(h_idx, 4 * n);
    dev_free(t_type, maxk);
    dev_free(t_card, 4 * maxk);
    dev_free(t_len, 4 * maxk);
    if (!ok) {
        set_delete(R);
        return nullptr;
    }
    return R;
}

int rb200_set_cardinalities(const rb200_set_t *s, uint64_t *out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    const size_t nb = s->n_bitmaps;
    if (!nb) return 0;
    if (!ensure_mirrors(s)) return -1;
    if (s->h_card.size() == nb) {  // cached by the op that produced this set
        memcpy(out, s->h_card.data(), 8 * nb);
        return 0;
    }
    uint64_t *h = (uint64_t *)pin_alloc(8 * nb);
    if (!h) return -1;
    // bm_card is maintained by upload / finalize / or_many
    bool ok = cudaMemcpyAsync(h, s->d_dir + s->L.o_bcard, 8 * nb, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
    ok = ok && cudaStreamSynchronize(g.stream) == cudaSuccess;
    if (ok) memcpy(out, h, 8 * nb);
    else t_err = "set_cardinalities: copy failed";
    pin_free(h, 8 * nb);
    return ok ? 0 : -1;
}

}  // extern "C"

// =================================================================== download
namespace {

bool ensure_mirror(rb200_set *s) {
    if (!resolve(s)) return false;
    if (s->m_dir) return true;
    s->m_dir = (uint8_t *)pin_alloc(s->L.total);
    s->m_slab = (uint8_t *)pin_alloc(s->slab_used);
    if (!s->m_dir || !s->m_slab) return false;
    bool ok = cudaMemcpyAsync(s->m_dir, s->d_dir, s->L.total, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
    if (s->slab_used)
        ok = ok && cudaMemcpyAsync(s->m_slab, s->d_slab, s->slab_used, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
    ok = ok && cudaStreamSynchronize(g.stream) == cudaSuccess;
    if (!ok) t_err = "download: copy failed";
    g.last_download_bytes = s->L.total + s->slab_used;
    return ok;
}

roaring_bitmap_t *build_bitmap(const rb200_set *s, size_t i, const uint8_t *slab = nullptr, uint64_t bias = 0) {
    if (!slab) slab = s->m_slab;
    const uint32_t *c_src = (const uint32_t *)(s->m_dir + s->L.o_src);
    const std::vector<const void *> *tabA = s->parentA.get(), *tabB = s->parentB.get();
    const uint32_t *bm_beg = (const uint32_t *)(s->m_dir + s->L.o_beg);
    const uint32_t *bm_cnt = (const uint32_t *)(s->m_dir + s->L.o_cnt);
    const uint16_t *c_key = (const uint16_t *)(s->m_dir + s->L.o_key);
    const uint8_t *c_type = s->m_dir + s->L.o_type;
    const uint32_t *c_card = (const uint32_t *)(s->m_dir + s->L.o_card);
    const uint32_t *c_len = (const uint32_t *)(s->m_dir + s->L.o_len);
    const uint64_t *c_off = (const uint64_t *)(s->m_dir + s->L.o_off);
    const uint32_t beg = bm_beg[i], cnt = bm_cnt[i];
    roaring_bitmap_t *r = bitmap_alloc((int32_t)cnt);
    if (!r) return nullptr;
    roaring_array_t *ra = &r->high_low_container;
    ra->flags = s->h_flags[i] & FLAG_COW;  // roaring.c:738,890
    for (uint32_t k = 0; k < cnt; k++) {
        const uint32_t c = beg + k;
        const uint8_t *pay = slab + (c_off[c] - bias);
        if (tabA || tabB) {  // pass-through container elided from the download: copy from the input
            const uint32_t sr = c_src[c];
            if (sr != SRC_NONE) {  // elided only when THAT parent is host-bound (same mask as k_pack_*)
                const std::vector<const void *> *tab = (sr & SRC_B) ? tabB : tabA;
                if (tab) pay = (const uint8_t *)(*tab)[sr & ~SRC_B];
            }
        }
        void *hc = container_from_payload(c_type[c], c_card[c], c_len[c], pay);
        if (!hc) {
            bitmap_free_host(r);
            return nullptr;
        }
        ra->containers[k] = hc;
        ra->keys[k] = c_key[c];
        ra->typecodes[k] = c_type[c];
        ra->size = (int32_t)k + 1;
    }
    return r;
}

}  // namespace

extern "C" {

}  // extern "C" (reopened below)

namespace {

// Persistent host worker pool (materialisation / bulk free).  run(fn, T) executes fn() on T
// threads (the caller is one of them); fn pulls its own work from a shared atomic counter.
void bind_to_local_cpus();

class Pool {
   public:
    void run(const std::function<void()> &fn, unsigned T) {
        if (T <= 1) { fn(); return; }
        std::lock_guard<std::mutex> one_run(run_mu_);  // callers: API threads and the downloader
        std::unique_lock<std::mutex> lk(mu_);
        while (workers_.size() < T - 1) workers_.emplace_back([this]() { bind_to_local_cpus(); loop(); });
        fn_ = &fn;
        want_ = T - 1;
        started_ = 0;
        running_ = 0;
        gen_++;
        lk.unlock();
        cv_.notify_all();
        fn();
        lk.lock();
        done_cv_.wait(lk, [this]() { return started_ == want_ && running_ == 0; });
        fn_ = nullptr;
    }

   private:
    void loop() {
        uint64_t seen = 0;
        for (;;) {
            std::unique_lock<std::mutex> lk(mu_);
            cv_.wait(lk, [&]() { return gen_ != seen && fn_ != nullptr && started_ < want_; });
            seen = gen_;
            started_++;
            running_++;
            const std::function<void()> *f = fn_;
            lk.unlock();
            (*f)();
            lk.lock();
            running_--;
            if (started_ == want_ && running_ == 0) done_cv_.notify_all();
        }
    }
    std::mutex mu_, run_mu_;
    std::condition_variable cv_, done_cv_;
    std::vector<std::thread> workers_;
    const std::function<void()> *fn_ = nullptr;
    unsigned want_ = 0, started_ = 0, running_ = 0;
    uint64_t gen_ = 0;
};
Pool &pool() {
    static Pool *p = new Pool();  // intentionally leaked: workers are detached for process life
    return *p;
}
// CPUs local to the GPU's PCIe root (sysfs local_cpulist); empty when unknown.
std::vector<int> &local_cpus() {
    // function-local static: initialised once, thread-safe (API threads, pool workers and the
    // downloader may all get here first)
    static std::vector<int> cpus = []() {
        std::vector<int> v;
        char bus[32] = {0};
        if (cudaDeviceGetPCIBusId(bus, sizeof(bus), g.device) != cudaSuccess) return v;
        for (char *c = bus; *c; c++) *c = (char)tolower(*c);
        std::string path = std::string("/sys/bus/pci/devices/") + bus + "/local_cpulist";
        FILE *f = fopen(path.c_str(), "r");
        if (!f) return v;
        char line[1024] = {0};
        if (fgets(line, sizeof(line), f)) {
            char *save = nullptr;
            for (char *tok = strtok_r(line, ",\n", &save); tok; tok = strtok_r(nullptr, ",\n", &save)) {
                int lo = 0, hi = 0;
                if (sscanf(tok, "%d-%d", &lo, &hi) == 2) { for (int c = lo; c <= hi; c++) v.push_back(c); }
                else if (sscanf(tok, "%d", &lo) == 1) v.push_back(lo);
            }
        }
        fclose(f);
        return v;
    }();
    return cpus;
}
// Move the calling thread onto the GPU-local CPUs; *saved receives the previous mask.
bool enter_local_cpus(cpu_set_t *saved) {
    if (getenv("RB200_NO_NUMA")) return false;
    const std::vector<int> &cpus = local_cpus();
    if (cpus.empty()) return false;
    if (pthread_getaffinity_np(pthread_self(), sizeof(*saved), saved) != 0) return false;
    cpu_set_t set;
    CPU_ZERO(&set);
    for (int c : cpus) if (c < CPU_SETSIZE) CPU_SET(c, &set);
    return pthread_setaffinity_np(pthread_self(), sizeof(set), &set) == 0;
}
void bind_to_local_cpus() {
    const std::vector<int> &cpus = local_cpus();
    if (cpus.empty()) return;
    cpu_set_t set;
    CPU_ZERO(&set);
    for (int c : cpus) if (c < CPU_SETSIZE) CPU_SET(c, &set);
    pthread_setaffinity_np(pthread_self(), sizeof(set), &set);
}
// Host worker threads for materialisation.  On a two-socket host the stream is PCIe bound well
// before all cores are busy, and threads on the remote socket slow it down (remote-socket traffic
// on the pinned staging buffers), so the default is 24 threads bound to the CPUs of the GPU's
// NUMA node.  RB200_HOST_THREADS overrides.
unsigned host_workers() {
    static unsigned T = 0;
    if (!T) {
        const char *e = getenv("RB200_HOST_THREADS");
        const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
        // several ranks on one node (torchrun exports LOCAL_WORLD_SIZE) share the host cores
        const char *lw = getenv("LOCAL_WORLD_SIZE");
        const unsigned local_world = lw && atoi(lw) > 0 ? (unsigned)atoi(lw) : 1u;
        T = e ? (unsigned)atoi(e) : std::min(24u, std::max(2u, hw / (2 * local_world)));
        if (T > 256) T = 256;
        if (T < 1) T = 1;
    }
    return T;
}

}  // namespace

// Streaming download: results leave the device chunk by chunk while the caller consumes (and
// frees) the previous chunk, so host memory stays bounded and D2H overlaps materialisation.
struct rb200_download_stream {
    rb200_set *P = nullptr;        // packed copy (device)
    size_t nb = 0;
    uint64_t *h_ob = nullptr;      // [off(nb+1) | beg(nb+1)] pinned
    std::vector<size_t> chunk_end; // bitmap index closing each chunk
    uint8_t *hbuf[2] = {nullptr, nullptr};
    size_t hbuf_bytes = 0;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    size_t next_copy = 0, next_build = 0;
    uint64_t total_bytes = 0;
};

namespace {

bool stream_enqueue(rb200_download_stream *st) {
    if (st->next_copy >= st->chunk_end.size()) return true;
    const size_t k = st->next_copy;
    const size_t p0 = k ? st->chunk_end[k - 1] : 0, p1 = st->chunk_end[k];
    const uint64_t b0 = st->h_ob[p0], b1 = st->h_ob[p1];
    if (b1 > b0 && cudaMemcpyAsync(st->hbuf[k & 1], st->P->d_slab + b0, b1 - b0, cudaMemcpyDeviceToHost,
                                   g.stream) != cudaSuccess)
        return false;
    cudaEventRecord(st->ev[k & 1], g.stream);
    st->next_copy++;
    return true;
}

void stream_free(rb200_download_stream *st, bool sync = true) {
    if (!st) return;
    if (sync) cudaStreamSynchronize(g.stream);
    for (int k = 0; k < 2; k++) {
        if (st->ev[k]) cudaEventDestroy(st->ev[k]);
        pin_free(st->hbuf[k], st->hbuf_bytes);
    }
    if (st->P) {
        pin_free(st->P->m_dir, st->P->L.total);
        st->P->m_dir = st->P->m_slab = nullptr;
        set_delete(st->P);
    }
    pin_free(st->h_ob, 16 * (st->nb + 1));
    delete st;
}

}  // namespace

extern "C" {

static rb200_download_stream *download_begin_impl(const rb200_set *s, size_t chunk_bitmaps, bool defer);
rb200_download_stream_t *rb200_download_begin(const rb200_set_t *s, size_t chunk_bitmaps) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return download_begin_impl(s, chunk_bitmaps, false);
}
// defer: pack only; the caller owns the staging ring and enqueues the copies itself
static rb200_download_stream *download_begin_impl(const rb200_set *s, size_t chunk_bitmaps, bool defer) {
    if (!ctx_init()) return nullptr;
    if (!resolve(s)) return nullptr;
    const size_t nb = s->n_bitmaps;
    rb200_download_stream *st = new rb200_download_stream();
    st->nb = nb;
    if (nb == 0) return st;
    if (chunk_bitmaps == 0) chunk_bitmaps = 1024;
    uint64_t *d_bytes = (uint64_t *)dev_alloc(8 * nb), *d_off = (uint64_t *)dev_alloc(8 * (nb + 1)),
             *d_beg = (uint64_t *)dev_alloc(8 * (nb + 1));
    uint32_t *d_cnt = (uint32_t *)dev_alloc(4 * nb);
    st->h_ob = (uint64_t *)pin_alloc(16 * (nb + 1));
    bool ok = d_bytes && d_off && d_beg && d_cnt && st->h_ob;
    if (ok) {
        const int elide = (s->parentA ? 1 : 0) | (s->parentB ? 2 : 0);
        launch_pack(s->view(), (uint32_t)nb, elide, d_bytes, d_cnt, d_off, d_beg, g.stream);
        ok = cudaMemcpyAsync(st->h_ob, d_off, 8 * (nb + 1), cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaMemcpyAsync(st->h_ob + nb + 1, d_beg, 8 * (nb + 1), cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaStreamSynchronize(g.stream) == cudaSuccess;
    }
    const uint64_t *h_off = st->h_ob, *h_beg = st->h_ob ? st->h_ob + nb + 1 : nullptr;
    if (ok) {
        st->P = set_new((uint32_t)nb, h_beg[nb], h_off[nb]);
        ok = st->P != nullptr;
    }
    if (ok) {
        rb200_set *P = st->P;
        P->n_containers = h_beg[nb];
        P->slab_used = h_off[nb];
        P->h_flags = s->h_flags;
        P->parentA = s->parentA;
        P->parentB = s->parentB;
        launch_pack_copy(s->view(), (uint32_t)nb, (s->parentA ? 1 : 0) | (s->parentB ? 2 : 0), d_off, d_beg,
                         P->out(), g.stream);
        P->m_dir = (uint8_t *)pin_alloc(P->L.total);
        ok = P->m_dir != nullptr &&
             cudaMemcpyAsync(P->m_dir, P->d_dir, P->L.total, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        // chunks: at most chunk_bitmaps bitmaps and ~64 MB of payload each
        const uint64_t CAP = (uint64_t)64 << 20;
        uint64_t maxb = 0;
        size_t p0 = 0;
        while (p0 < nb) {
            size_t p1 = p0 + 1;
            while (p1 < nb && p1 - p0 < chunk_bitmaps && h_off[p1 + 1] - h_off[p0] <= CAP) p1++;
            st->chunk_end.push_back(p1);
            maxb = std::max(maxb, h_off[p1] - h_off[p0]);
            p0 = p1;
        }
        st->hbuf_bytes = maxb;
        for (int k = 0; k < 2 && ok && !defer; k++) {
            st->hbuf[k] = (uint8_t *)pin_alloc(maxb);
            ok = st->hbuf[k] != nullptr && cudaEventCreateWithFlags(&st->ev[k], cudaEventDisableTiming) == cudaSuccess;
        }
        st->total_bytes = P->L.total + P->slab_used;
        g.last_download_bytes = st->total_bytes;
        if (!defer) ok = ok && stream_enqueue(st) && stream_enqueue(st);
    }
    dev_free(d_bytes, 8 * nb);
    dev_free(d_off, 8 * (nb + 1));
    dev_free(d_beg, 8 * (nb + 1));
    dev_free(d_cnt, 4 * nb);
    if (!ok) {
        if (t_err.empty()) t_err = "download_begin failed";
        stream_free(st);
        return nullptr;
    }
    return st;
}

size_t rb200_download_chunk_capacity(const rb200_download_stream_t *st) {
    size_t m = 0, p0 = 0;
    for (size_t e : st->chunk_end) { m = std::max(m, e - p0); p0 = e; }
    return m;
}

// Materialise the next chunk into out[] (capacity >= rb200_download_chunk_capacity); returns the
// number of bitmaps produced, 0 at the end of the stream, (size_t)-1 on error.
size_t rb200_download_next(rb200_download_stream_t *st, roaring_bitmap_t **out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (st->next_build >= st->chunk_end.size()) return 0;
    const size_t k = st->next_build;
    const size_t p0 = k ? st->chunk_end[k - 1] : 0, p1 = st->chunk_end[k];
    if (cudaEventSynchronize(st->ev[k & 1]) != cudaSuccess) { t_err = "download_next: copy failed"; return (size_t)-1; }
    const uint8_t *buf = st->hbuf[k & 1];
    const uint64_t bias = st->h_ob[p0];
    const size_t n = p1 - p0;
    std::atomic<size_t> next(0);
    std::atomic<int> failed(0);
    const rb200_set *P = st->P;
    std::function<void()> work = [&]() {
        for (;;) {
            const size_t i0 = next.fetch_add(8);
            if (i0 >= n) break;
            const size_t i1 = std::min(n, i0 + 8);
            for (size_t i = i0; i < i1; i++) {
                out[i] = build_bitmap(P, p0 + i, buf, bias);
                if (!out[i]) failed = 1;
            }
        }
    };
    // threads scaled to the work of this chunk: waking 64 workers for a few hundred tiny
    // bitmaps costs more than it saves
    const uint64_t chunk_bytes = st->h_ob[p1] - st->h_ob[p0];
    const uint64_t chunk_conts = st->h_ob[st->nb + 1 + p1] - st->h_ob[st->nb + 1 + p0];
    uint64_t want = (chunk_bytes + 256 * chunk_conts + 512 * n) / (192 << 10) + 1;
    unsigned T = host_workers();
    if (want < T) T = (unsigned)want;
    if ((size_t)T * 8 > n) T = (unsigned)((n + 7) / 8);
    pool().run(work, T);
    st->next_build++;
    if (!stream_enqueue(st)) failed = 1;  // refill the buffer we just drained
    if (failed) {
        for (size_t i = 0; i < n; i++) { bitmap_free_host(out[i]); out[i] = nullptr; }
        t_err = "download_next: host allocation or copy failed";
        return (size_t)-1;
    }
    return n;
}

void rb200_download_end(rb200_download_stream_t *st) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    stream_free(st);
}

// Visitor form of the streaming download: every bitmap of the set is materialised as a host
// roaring_bitmap_t (reference layout), handed to `fn` ON A WORKER THREAD, and freed right after
// unless fn returns non-zero (then the callee owns it).  Building, consuming and freeing a result
// on the same thread is what the reference's own loops do (create, use, roaring_bitmap_free —
// microbenchmarks/bench.cpp:85-96): the allocator recycles hot blocks instead of touching
// gigabytes of fresh memory.  Returns 0 on success.
int rb200_download_foreach(const rb200_set_t *s, rb200_visit_fn fn, void *ctx) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    const auto t_enter = std::chrono::steady_clock::now();
    rb200_download_stream *st = rb200_download_begin(s, 4096);
    if (!st) return -1;
    std::atomic<int> failed(0);
    const bool trace = getenv("RB200_TRACE") != nullptr;
    double t_wait = 0, t_build = 0;
    const auto t_begin = std::chrono::steady_clock::now();
    auto ms_since = [](std::chrono::steady_clock::time_point t) {
        return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count();
    };
    const double t_pack = ms_since(t_enter);
    while (st->next_build < st->chunk_end.size()) {
        const size_t k = st->next_build;
        const size_t p0 = k ? st->chunk_end[k - 1] : 0, p1 = st->chunk_end[k];
        const auto t0 = std::chrono::steady_clock::now();
        if (cudaEventSynchronize(st->ev[k & 1]) != cudaSuccess) { failed = 1; break; }
        t_wait += ms_since(t0);
        const auto t1 = std::chrono::steady_clock::now();
        const uint8_t *buf = st->hbuf[k & 1];
        const uint64_t bias = st->h_ob[p0];
        const size_t n = p1 - p0;
        std::atomic<size_t> next(0);
        const rb200_set *P = st->P;
        std::function<void()> work = [&]() {
            for (;;) {
                const size_t i0 = next.fetch_add(8);
                if (i0 >= n) break;
                const size_t i1 = std::min(n, i0 + 8);
                for (size_t i = i0; i < i1; i++) {
                    roaring_bitmap_t *bm = build_bitmap(P, p0 + i, buf, bias);
                    if (!bm) { failed = 1; continue; }
                    if (fn(p0 + i, bm, ctx) == 0) bitmap_free_host(bm);
                }
            }
        };
        const uint64_t chunk_bytes = st->h_ob[p1] - st->h_ob[p0];
        const uint64_t chunk_conts = st->h_ob[st->nb + 1 + p1] - st->h_ob[st->nb + 1 + p0];
        uint64_t want = (chunk_bytes + 256 * chunk_conts + 512 * n) / (128 << 10) + 1;
        unsigned T = host_workers();
        if (want < T) T = (unsigned)want;
        if ((size_t)T * 8 > n) T = (unsigned)((n + 7) / 8);
        pool().run(work, T);
        t_build += ms_since(t1);
        st->next_build++;
        if (!stream_enqueue(st)) { failed = 1; break; }
    }
    if (trace)
        fprintf(stderr, "rb200 foreach: %zu bitmaps %zu chunks %.1f MB | pack %.2f ms, copy-wait %.2f ms, build %.2f ms, loop %.2f ms\n",
                st->nb, st->chunk_end.size(), st->total_bytes / 1e6, t_pack, t_wait, t_build, ms_since(t_begin));
    stream_free(st);
    if (failed) {
        if (t_err.empty()) t_err = "download_foreach: host allocation or copy failed";
        return -1;
    }
    return 0;
}

// Visitor download of SEVERAL result sets as one pipelined stream: every set is packed on the
// device first, then all their chunks cross PCIe back to back through one staging ring while the
// workers materialise the previous chunk — the copy engine never idles between sets, and the
// builds of small / host-bound sets hide behind the transfers of the large ones.  fn receives a
// running index (set 0's bitmaps first).  Returns 0 on success.
int rb200_download_foreach_many(const rb200_set_t *const *sets, size_t nsets, rb200_visit_fn fn, void *ctx) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    std::vector<rb200_download_stream *> sts(nsets, nullptr);
    struct Ref { size_t set; size_t k; };
    std::vector<Ref> order;
    std::vector<size_t> first_index(nsets, 0);
    size_t ring_bytes = 0, running = 0;
    uint64_t total = 0;
    bool ok = true;
    for (size_t i = 0; i < nsets && ok; i++) {
        sts[i] = download_begin_impl(sets[i], 4096, true);
        ok = sts[i] != nullptr;
        if (!ok) break;
        first_index[i] = running;
        running += sts[i]->nb;
        ring_bytes = std::max(ring_bytes, sts[i]->hbuf_bytes);
        total += sts[i]->total_bytes;
        for (size_t k = 0; k < sts[i]->chunk_end.size(); k++) order.push_back(Ref{i, k});
    }
    // staging ring: RING buffers, so the copy engine can run up to RING-1 chunks ahead of the
    // builders (chunks alternate between copy-bound and build-bound; 2 buffers stall either side)
    constexpr int RING = 4;
    uint8_t *ring[RING] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t rev[RING] = {nullptr, nullptr, nullptr, nullptr};
    for (int k = 0; k < RING && ok; k++) {
        ring[k] = (uint8_t *)pin_alloc(ring_bytes ? ring_bytes : 16);
        ok = ring[k] != nullptr && cudaEventCreateWithFlags(&rev[k], cudaEventDisableTiming) == cudaSuccess;
    }
    auto enqueue = [&](size_t gidx) -> bool {
        if (gidx >= order.size()) return true;
        const rb200_download_stream *st = sts[order[gidx].set];
        const size_t k = order[gidx].k;
        const size_t p0 = k ? st->chunk_end[k - 1] : 0, p1 = st->chunk_end[k];
        const uint64_t b0 = st->h_ob[p0], b1 = st->h_ob[p1];
        if (b1 > b0 && cudaMemcpyAsync(ring[gidx % RING], st->P->d_slab + b0, b1 - b0, cudaMemcpyDeviceToHost,
                                       g.stream) != cudaSuccess)
            return false;
        return cudaEventRecord(rev[gidx % RING], g.stream) == cudaSuccess;
    };
    std::atomic<int> failed(0);
    const bool trace = getenv("RB200_TRACE") != nullptr;
    double t_wait = 0, t_build = 0;
    auto ms_since = [](std::chrono::steady_clock::time_point t) {
        return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count();
    };
    const auto t_begin = std::chrono::steady_clock::now();
    for (int k = 0; k < RING && ok; k++) ok = enqueue((size_t)k);
    for (size_t gidx = 0; gidx < order.size() && ok; gidx++) {
        const rb200_download_stream *st = sts[order[gidx].set];
        const size_t k = order[gidx].k, base_index = first_index[order[gidx].set];
        const size_t p0 = k ? st->chunk_end[k - 1] : 0, p1 = st->chunk_end[k];
        const auto t0 = std::chrono::steady_clock::now();
        if (cudaEventSynchronize(rev[gidx % RING]) != cudaSuccess) { ok = false; break; }
        t_wait += ms_since(t0);
        const auto t1 = std::chrono::steady_clock::now();
        const uint8_t *buf = ring[gidx % RING];
        const uint64_t bias = st->h_ob[p0];
        const size_t n = p1 - p0;
        std::atomic<size_t> next(0);
        const rb200_set *P = st->P;
        std::function<void()> work = [&]() {
            for (;;) {
                const size_t i0 = next.fetch_add(8);
                if (i0 >= n) break;
                const size_t i1 = std::min(n, i0 + 8);
                for (size_t i = i0; i < i1; i++) {
                    roaring_bitmap_t *bm = build_bitmap(P, p0 + i, buf, bias);
                    if (!bm) { failed = 1; continue; }
                    if (fn(base_index + p0 + i, bm, ctx) == 0) bitmap_free_host(bm);
                }
            }
        };
        const uint64_t chunk_bytes = st->h_ob[p1] - st->h_ob[p0];
        const uint64_t chunk_conts = st->h_ob[st->nb + 1 + p1] - st->h_ob[st->nb + 1 + p0];
        uint64_t want = (chunk_bytes + 256 * chunk_conts + 512 * n) / (128 << 10) + 1;
        unsigned T = host_workers();
        if (want < T) T = (unsigned)want;
        if ((size_t)T * 8 > n) T = (unsigned)((n + 7) / 8);
        pool().run(work, T);
        t_build += ms_since(t1);
        ok = enqueue(gidx + RING);
    }
    if (trace)
        fprintf(stderr, "rb200 foreach_many: %zu sets %zu chunks %.1f MB | copy-wait %.2f ms, build %.2f ms, loop %.2f ms\n",
                nsets, order.size(), total / 1e6, t_wait, t_build, ms_since(t_begin));
    cudaStreamSynchronize(g.stream);
    for (int k = 0; k < RING; k++) {
        if (rev[k]) cudaEventDestroy(rev[k]);
        pin_free(ring[k], ring_bytes ? ring_bytes : 16);
    }
    for (auto st : sts) if (st) stream_free(st);
    g.last_download_bytes = total;
    if (!ok || failed) {
        if (t_err.empty()) t_err = "download_foreach_many: host allocation or copy failed";
        return -1;
    }
    return 0;
}

}  // extern "C"

// ---- asynchronous visitor download ---------------------------------------------------------
// rb200_download_foreach_async packs the set on the caller's thread (device kernels on the library
// stream) and hands the packed copy to ONE background downloader thread, which owns a second CUDA
// stream and a 4-deep pinned staging ring: chunks of all queued sets cross PCIe back to back while
// the worker pool materialises the previous chunk — and while the caller goes on uploading and
// launching the next ops.  rb200_download_wait drains the queue.
namespace {
struct DlJob {
    rb200_download_stream *st = nullptr;
    rb200_visit_fn fn = nullptr;
    void *ctx = nullptr;
    cudaEvent_t ready = nullptr;  // recorded on the library stream after the pack
    size_t next_copy = 0, built = 0;
};
struct Downloader {
    std::mutex mu;
    std::condition_variable cv, idle_cv;
    std::deque<DlJob *> q;
    size_t active = 0;  // jobs queued or in progress
    bool started = false;
    int failed = 0;
    std::string err;
    uint64_t bytes = 0;
    void loop();
};
Downloader &dl() {
    static Downloader *d = new Downloader();  // leaked on purpose: the thread lives as long as the process
    return *d;
}

void Downloader::loop() {
    cudaSetDevice(g.device);
    bind_to_local_cpus();
    constexpr int RING = 4;
    cudaStream_t stream = nullptr;
    cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
    uint8_t *ring[RING] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t rev[RING];
    for (int k = 0; k < RING; k++) cudaEventCreateWithFlags(&rev[k], cudaEventDisableTiming);
    size_t ring_bytes = 0;
    struct Flight { DlJob *job; size_t k; int slot; };
    std::deque<Flight> inflight;
    std::deque<DlJob *> jobs;  // taken from q, not yet fully enqueued
    uint64_t nslot = 0;
    auto fail = [&](const char *why) {
        std::lock_guard<std::mutex> lk(mu);
        failed = 1;
        if (err.empty()) err = why;
    };
    auto finish = [&](DlJob *j) {
        cudaEventDestroy(j->ready);
        stream_free(j->st, false);
        delete j;
        std::lock_guard<std::mutex> lk(mu);
        if (--active == 0) idle_cv.notify_all();
    };
    for (;;) {
        {
            std::unique_lock<std::mutex> lk(mu);
            if (jobs.empty() && inflight.empty()) cv.wait(lk, [&]() { return !q.empty(); });
            while (!q.empty()) { jobs.push_back(q.front()); q.pop_front(); }
        }
        // keep the copy engine up to RING chunks ahead
        while ((int)inflight.size() < RING && !jobs.empty()) {
            DlJob *j = jobs.front();
            const rb200_download_stream *st = j->st;
            if (st->chunk_end.empty()) { jobs.pop_front(); finish(j); continue; }
            if (st->hbuf_bytes > ring_bytes) {  // grow the ring (only with nothing in flight)
                if (!inflight.empty()) break;
                for (int k = 0; k < RING; k++) { pin_free(ring[k], ring_bytes); ring[k] = (uint8_t *)pin_alloc(st->hbuf_bytes); }
                ring_bytes = st->hbuf_bytes;
                if (!ring[0] || !ring[1] || !ring[2] || !ring[3]) { fail("downloader: pinned allocation failed"); ring_bytes = 0; }
            }
            const size_t k = j->next_copy;
            if (k == 0) cudaStreamWaitEvent(stream, j->ready, 0);
            const size_t p0 = k ? st->chunk_end[k - 1] : 0, p1 = st->chunk_end[k];
            const uint64_t b0 = st->h_ob[p0], b1 = st->h_ob[p1];
            const int slot = (int)(nslot++ % RING);
            if (ring_bytes && b1 > b0 &&
                cudaMemcpyAsync(ring[slot], st->P->d_slab + b0, b1 - b0, cudaMemcpyDeviceToHost, stream) != cudaSuccess)
                fail("downloader: D2H copy failed");
            cudaEventRecord(rev[slot], stream);
            inflight.push_back(Flight{j, k, slot});
            if (++j->next_copy == st->chunk_end.size()) jobs.pop_front();
        }
        if (inflight.empty()) continue;
        const Flight f = inflight.front();
        inflight.pop_front();
        if (cudaEventSynchronize(rev[f.slot]) != cudaSuccess) fail("downloader: copy failed");
        const rb200_download_stream *st = f.job->st;
        const size_t p0 = f.k ? st->chunk_end[f.k - 1] : 0, p1 = st->chunk_end[f.k];
        if (ring_bytes) {
            const uint8_t *buf = ring[f.slot];
            const uint64_t bias = st->h_ob[p0];
            const size_t n = p1 - p0;
            std::atomic<size_t> next(0);
            std::atomic<int> bad(0);
            const rb200_set *P = st->P;
            const rb200_visit_fn fn = f.job->fn;
            void *ctx = f.job->ctx;
            std::function<void()> work = [&]() {
                for (;;) {
                    const size_t i0 = next.fetch_add(8);
                    if (i0 >= n) break;
                    const size_t i1 = std::min(n, i0 + 8);
                    for (size_t i = i0; i < i1; i++) {
                        roaring_bitmap_t *bm = build_bitmap(P, p0 + i, buf, bias);
                        if (!bm) { bad = 1; continue; }
                        if (fn(p0 + i, bm, ctx) == 0) bitmap_free_host(bm);
                    }
                }
            };
            const uint64_t chunk_bytes = st->h_ob[p1] - st->h_ob[p0];
            const uint64_t chunk_conts = st->h_ob[st->nb + 1 + p1] - st->h_ob[st->nb + 1 + p0];
            uint64_t want = (chunk_bytes + 256 * chunk_conts + 512 * n) / (128 << 10) + 1;
            unsigned T = host_workers();
            if (want < T) T = (unsigned)want;
            if ((size_t)T * 8 > n) T = (unsigned)((n + 7) / 8);
            pool().run(work, T);
            if (bad) fail("downloader: host allocation failed");
        }
        if (++f.job->built == st->chunk_end.size()) finish(f.job);
    }
}
}  // namespace

extern "C" {

// Enqueue the visitor download of `s` and return at once (the set may be freed right away: the
// job owns a packed device copy).  fn runs on worker threads with the index of the bitmap in `s`.
int rb200_download_foreach_async(const rb200_set_t *s, rb200_visit_fn fn, void *ctx) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    DlJob *j = new DlJob();
    j->st = download_begin_impl(s, 4096, true);
    if (!j->st) { delete j; return -1; }
    j->fn = fn;
    j->ctx = ctx;
    if (cudaEventCreateWithFlags(&j->ready, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventRecord(j->ready, g.stream) != cudaSuccess) {
        t_err = "download_foreach_async: event failed";
        stream_free(j->st);
        delete j;
        return -1;
    }
    Downloader &d = dl();
    {
        std::lock_guard<std::mutex> dk(d.mu);
        d.bytes += j->st->total_bytes;
        d.active++;
        d.q.push_back(j);
        if (!d.started) {
            d.started = true;
            std::thread([&d]() { d.loop(); }).detach();
        }
    }
    d.cv.notify_one();
    return 0;
}

// Wait for every queued download; 0 on success.  rb200_last_download_bytes() then reports the
// bytes that crossed PCIe since the previous wait.
int rb200_download_wait(void) {
    Downloader &d = dl();
    std::unique_lock<std::mutex> dk(d.mu);
    d.idle_cv.wait(dk, [&]() { return d.active == 0; });
    const int failed = d.failed;
    const std::string why = d.err;
    g.last_download_bytes = d.bytes;
    d.bytes = 0;
    d.failed = 0;
    d.err.clear();
    dk.unlock();
    if (failed) {
        std::lock_guard<std::recursive_mutex> lk(g.mu);
        t_err = why.empty() ? "asynchronous download failed" : why;
        return -1;
    }
    return 0;
}

// A ready-made visitor: *(uint64_t*)ctx += cardinality(bitmap) (atomic); the bitmap is released.
int rb200_visit_sum_cardinality(size_t index, roaring_bitmap_t *bm, void *ctx) {
    (void)index;
    __atomic_fetch_add((uint64_t *)ctx, rb200_bitmap_get_cardinality(bm), __ATOMIC_RELAXED);
    return 0;
}

roaring_bitmap_t *rb200_set_download(const rb200_set_t *cs, size_t i) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    rb200_set *s = const_cast<rb200_set *>(cs);
    if (i >= s->n_bitmaps) { t_err = "download: index out of range"; return nullptr; }
    if (!ensure_mirror(s)) return nullptr;
    return build_bitmap(s, i);
}

// Download every bitmap of a set as host roaring_bitmap_t (reference layout).
// Pipeline: (1) device-side pack — directory in bitmap order, payload contiguous in bitmap
// order, no slot slack; (2) D2H of the payload in ~32 MB chunks of whole bitmaps into pinned
// memory, one event per chunk; (3) host threads build the bitmaps of a chunk (per-container
// roaring_malloc + memcpy, the ownership contract of src/containers/containers.c:58-77) as soon
// as its event fires, while later chunks are still crossing PCIe.
int rb200_set_download_all(const rb200_set_t *cs, roaring_bitmap_t **out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    const rb200_set *s = cs;
    const size_t nb = s->n_bitmaps;
    if (nb == 0) return 0;
    const bool trace = getenv("RB200_TRACE") != nullptr;
    auto now = []() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t_start = now();
    double t_packed = 0, t_copies = 0, t_built = 0;
    // ---- (1) pack
    uint64_t *d_bytes = (uint64_t *)dev_alloc(8 * nb), *d_off = (uint64_t *)dev_alloc(8 * (nb + 1)),
             *d_beg = (uint64_t *)dev_alloc(8 * (nb + 1));
    uint32_t *d_cnt = (uint32_t *)dev_alloc(4 * nb);
    uint64_t *h_ob = (uint64_t *)pin_alloc(16 * (nb + 1));
    rb200_set *P = nullptr;
    uint8_t *hp = nullptr;
    size_t hp_bytes = 0;
    std::vector<cudaEvent_t> evs;
    bool ok = d_bytes && d_off && d_beg && d_cnt && h_ob;
    if (ok) {
        const int elide = (s->parentA ? 1 : 0) | (s->parentB ? 2 : 0);
        launch_pack(s->view(), (uint32_t)nb, elide, d_bytes, d_cnt, d_off, d_beg, g.stream);
        ok = cudaMemcpyAsync(h_ob, d_off, 8 * (nb + 1), cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaMemcpyAsync(h_ob + nb + 1, d_beg, 8 * (nb + 1), cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaStreamSynchronize(g.stream) == cudaSuccess;
    }
    const uint64_t *h_off = h_ob, *h_beg = h_ob ? h_ob + nb + 1 : nullptr;
    t_packed = now();
    if (ok) {
        P = set_new((uint32_t)nb, h_beg[nb], h_off[nb]);
        ok = P != nullptr;
    }
    if (ok) {
        P->n_containers = h_beg[nb];
        P->slab_used = h_off[nb];
        P->h_flags = s->h_flags;
        P->parentA = s->parentA;
        P->parentB = s->parentB;
        launch_pack_copy(s->view(), (uint32_t)nb, (s->parentA ? 1 : 0) | (s->parentB ? 2 : 0), d_off, d_beg,
                         P->out(), g.stream);
        // ---- (2) directory, then payload chunks
        P->m_dir = (uint8_t *)pin_alloc(P->L.total);
        hp_bytes = P->slab_used;
        hp = (uint8_t *)pin_alloc(hp_bytes);
        ok = P->m_dir && hp;
    }
    std::vector<size_t> chunk_end;  // bitmap index (exclusive) closing each chunk
    if (ok) {
        P->m_slab = hp;
        ok = cudaMemcpyAsync(P->m_dir, P->d_dir, P->L.total, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        const uint64_t CH = (uint64_t)32 << 20;
        size_t p0 = 0;
        while (ok && p0 < nb) {
            size_t p1 = p0 + 1;
            while (p1 < nb && h_off[p1 + 1] - h_off[p0] <= CH) p1++;
            const uint64_t b0 = h_off[p0], b1 = h_off[p1];
            if (b1 > b0)
                ok = cudaMemcpyAsync(hp + b0, P->d_slab + b0, b1 - b0, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
            cudaEvent_t ev;
            ok = ok && cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) == cudaSuccess;
            if (ok) {
                cudaEventRecord(ev, g.stream);
                evs.push_back(ev);
                chunk_end.push_back(p1);
            }
            p0 = p1;
        }
    }
    t_copies = now();
    // ---- (3) host threads
    if (ok) {
        std::atomic<size_t> next(0);
        std::atomic<int> failed(0);
        const size_t BLK = 16;
        unsigned T = std::thread::hardware_concurrency();
        if (T > 48) T = 48;
        if (T < 1) T = 1;
        if ((size_t)T * BLK > nb) T = (unsigned)((nb + BLK - 1) / BLK);
        const int dev = g.device;
        auto work = [&]() {
            cudaSetDevice(dev);
            size_t cur = 0, done_upto = 0;  // chunks [0, done_upto) are known complete
            for (;;) {
                const size_t i0 = next.fetch_add(BLK);
                if (i0 >= nb) break;
                const size_t i1 = std::min(nb, i0 + BLK);
                while (cur + 1 < chunk_end.size() && chunk_end[cur] < i1) cur++;
                // the chunk holding bitmap i1-1 (and every earlier one: same stream) must be done
                if (cur >= done_upto) {
                    if (cudaEventSynchronize(evs[cur]) != cudaSuccess) { failed = 1; break; }
                    done_upto = cur + 1;
                }
                for (size_t i = i0; i < i1; i++) {
                    out[i] = build_bitmap(P, i);
                    if (!out[i]) failed = 1;
                }
            }
        };
        std::vector<std::thread> th;
        for (unsigned t = 1; t < T; t++) th.emplace_back(work);
        work();
        for (auto &t : th) t.join();
        t_built = now();
        if (cudaStreamSynchronize(g.stream) != cudaSuccess) failed = 1;
        if (failed) {
            for (size_t i = 0; i < nb; i++) { bitmap_free_host(out[i]); out[i] = nullptr; }
            t_err = "download: host allocation or copy failed";
            ok = false;
        }
        g.last_download_bytes = P->L.total + P->slab_used;
    } else {
        cudaStreamSynchronize(g.stream);
        if (t_err.empty()) t_err = "download: packing failed";
    }
    if (trace)
        fprintf(stderr, "[rb200] download_all nb=%zu bytes=%.1f MB: measure+scan %.2f ms, alloc+enqueue %.2f ms, "
                        "copy+build %.2f ms, total %.2f ms (chunks %zu)\n",
                nb, P ? (P->L.total + P->slab_used) / 1e6 : 0.0, t_packed - t_start, t_copies - t_packed,
                t_built - t_copies, now() - t_start, evs.size());
    for (auto ev : evs) cudaEventDestroy(ev);
    if (P) {
        pin_free(P->m_dir, P->L.total);
        P->m_dir = nullptr;
        P->m_slab = nullptr;
        set_delete(P);
    }
    pin_free(hp, hp_bytes);
    pin_free(h_ob, 16 * (nb + 1));
    dev_free(d_bytes, 8 * nb);
    dev_free(d_off, 8 * (nb + 1));
    dev_free(d_beg, 8 * (nb + 1));
    dev_free(d_cnt, 4 * nb);
    return ok ? 0 : -1;
}

// roaring_bitmap_run_optimize (mode 1) / roaring_bitmap_remove_run_compression (mode 0) applied
// to every bitmap of a set on the device; returns a new resident set (same bitmaps, same keys).
static rb200_set *convert_impl(const rb200_set *S, int mode);
rb200_set_t *rb200_set_run_optimize(const rb200_set_t *S, int mode) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (reject_lazy(S, "run_optimize")) return nullptr;
    return convert_impl(S, mode ? 1 : 0);
}
// roaring_bitmap_repair_after_lazy (src/roaring.c:2845) on every bitmap of a set produced by lazy
// ops: bitsets are recounted (<= 4096 values -> array), runs go through the efficient-container
// rule, arrays stay.  Returns a new, ordinary (non-lazy) set.
rb200_set_t *rb200_set_repair_after_lazy(const rb200_set_t *S) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return convert_impl(S, 2);
}
static rb200_set *convert_impl(const rb200_set *S, int mode) {
    if (!ctx_init()) return nullptr;
    if (!resolve(S)) return nullptr;
    const uint64_t nc = S->n_containers;
    // mode 1 never grows a container by more than its 16-byte padding; mode 0 may expand runs
    const uint64_t bound = S->slab_used + 16 * nc + (mode == 0 ? nc * (uint64_t)BITSET_BYTES : 0) + 512;
    rb200_set *R = set_new(S->n_bitmaps, nc, bound);
    if (!R) return nullptr;
    bool ok = stats_reset();
    launch_run_optimize(S->view(), S->n_bitmaps, nc, mode, R->out(), g.d_stats, g.stream);
    ok = ok && stats_fetch();
    cudaError_t e = cudaStreamSynchronize(g.stream);
    if (e != cudaSuccess || (e = cudaGetLastError()) != cudaSuccess) {
        t_err = std::string("run_optimize: ") + cudaGetErrorString(e);
        ok = false;
    }
    if (!ok) { set_delete(R); return nullptr; }
    R->n_containers = nc;
    R->slab_used = g.h_stats->slab_cursor;
    R->h_flags = S->h_flags;
    if (!ensure_mirrors(S)) { set_delete(R); return nullptr; }
    R->h_cnt = S->h_cnt;
    for (size_t b = 0; b < R->n_bitmaps; b++) {
        R->h_bytes[b] = (uint64_t)R->h_cnt[b] * BITSET_BYTES;
        R->h_ebytes[b] = std::max<uint64_t>(R->h_bytes[b], S->h_ebytes[b]);
    }
    return R;
}

// roaring_bitmap_to_uint32_array for every bitmap of a set: *vals (pinned host memory owned by the
// library) holds all values; bitmap i = vals[off[i] .. off[i+1]).  Release with rb200_values_free.
int rb200_set_to_uint32(const rb200_set_t *S, uint32_t **vals, uint64_t **off_out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    if (!resolve(S)) return -1;
    const size_t nb = S->n_bitmaps;
    const uint64_t nc = S->n_containers;
    *vals = nullptr;
    *off_out = (uint64_t *)malloc(8 * (nb + 1));
    if (!*off_out) return -1;
    (*off_out)[0] = 0;
    if (nb == 0) return 0;
    uint64_t *d_bv = (uint64_t *)dev_alloc(8 * nb), *d_off = (uint64_t *)dev_alloc(8 * (nb + 1)),
             *d_dummy = (uint64_t *)dev_alloc(8 * (nb + 1)), *d_cstart = (uint64_t *)dev_alloc(8 * nc);
    uint32_t *d_zero = (uint32_t *)dev_alloc(4 * nb), *d_cbm = (uint32_t *)dev_alloc(4 * nc);
    uint64_t *h_off = (uint64_t *)pin_alloc(8 * (nb + 1));
    uint32_t *d_vals = nullptr, *h_vals = nullptr;
    uint64_t total = 0;
    bool ok = d_bv && d_off && d_dummy && d_cstart && d_zero && d_cbm && h_off;
    if (ok) {
        launch_values_measure(S->view(), (uint32_t)nb, d_bv, d_zero, d_cstart, d_cbm, g.stream);
        launch_pack_scan(d_bv, d_zero, (uint32_t)nb, d_off, d_dummy, g.stream);
        ok = cudaMemcpyAsync(h_off, d_off, 8 * (nb + 1), cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaStreamSynchronize(g.stream) == cudaSuccess;
    }
    if (ok) {
        total = h_off[nb];
        memcpy(*off_out, h_off, 8 * (nb + 1));
        d_vals = (uint32_t *)dev_alloc(4 * total);
        h_vals = (uint32_t *)pin_alloc(4 * total);
        ok = d_vals && h_vals;
    }
    if (ok) {
        launch_values_write(S->view(), (uint32_t)nb, d_off, d_cstart, d_cbm, nc, d_vals, g.stream);
        ok = cudaMemcpyAsync(h_vals, d_vals, 4 * total, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaStreamSynchronize(g.stream) == cudaSuccess && cudaGetLastError() == cudaSuccess;
    }
    dev_free(d_bv, 8 * nb);
    dev_free(d_off, 8 * (nb + 1));
    dev_free(d_dummy, 8 * (nb + 1));
    dev_free(d_cstart, 8 * nc);
    dev_free(d_zero, 4 * nb);
    dev_free(d_cbm, 4 * nc);
    dev_free(d_vals, 4 * total);
    pin_free(h_off, 8 * (nb + 1));
    if (!ok) {
        pin_free(h_vals, 4 * total);
        if (t_err.empty()) t_err = "set_to_uint32 failed";
        return -1;
    }
    *vals = h_vals;
    g_serialized_sizes[(uint8_t *)h_vals] = 4 * total;
    return 0;
}

void rb200_values_free(uint32_t *vals, uint64_t *off) { rb200_serialized_free((char *)vals, off, nullptr); }

// Device-side portable serialization of every bitmap of a set + one D2H copy.
// *buf is pinned host memory owned by the library (release with rb200_serialized_free);
// blob i = *buf + (*off)[i], (*len)[i] bytes, byte-identical to roaring_bitmap_portable_serialize.
static int serialize_impl(const rb200_set *s, char **buf, uint64_t **off_out, uint64_t **len_out, bool frozen);
int rb200_set_serialize(const rb200_set_t *s, char **buf, uint64_t **off_out, uint64_t **len_out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return serialize_impl(s, buf, off_out, len_out, false);
}
// Device-side roaring_bitmap_frozen_serialize (src/roaring.c:3246-3330) of every bitmap of the set:
// blob starts are 32-byte aligned inside *buf, so roaring_bitmap_frozen_view works on them in place.
int rb200_set_serialize_frozen(const rb200_set_t *s, char **buf, uint64_t **off_out, uint64_t **len_out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return serialize_impl(s, buf, off_out, len_out, true);
}
static int serialize_impl(const rb200_set *s, char **buf, uint64_t **off_out, uint64_t **len_out, bool frozen) {
    if (!ctx_init()) return -1;
    if (!resolve(s)) return -1;
    if (reject_lazy(s, "serialize")) return -1;
    const size_t nb = s->n_bitmaps;
    *buf = nullptr;
    *off_out = (uint64_t *)malloc(8 * (nb + 1));
    *len_out = (uint64_t *)malloc(8 * (nb + 1));
    if (!*off_out || !*len_out) return -1;
    (*off_out)[0] = 0;
    if (nb == 0) return 0;
    uint64_t *d_sz = (uint64_t *)dev_alloc(8 * nb), *d_off = (uint64_t *)dev_alloc(8 * (nb + 1)),
             *d_dummy = (uint64_t *)dev_alloc(8 * (nb + 1));
    uint32_t *d_exact = (uint32_t *)dev_alloc(4 * nb), *d_hasrun = (uint32_t *)dev_alloc(4 * nb);
    uint8_t *h_meta = (uint8_t *)pin_alloc(8 * (nb + 1) + 4 * nb);
    uint8_t *d_blob = nullptr, *h_blob = nullptr;
    uint64_t total = 0;
    bool ok = d_sz && d_off && d_dummy && d_exact && d_hasrun && h_meta;
    if (ok) {
        const SetView v = s->view();
        if (frozen) launch_frozen_measure(v, (uint32_t)nb, d_sz, d_exact, d_hasrun, g.stream);
        else launch_serialize_measure(v, (uint32_t)nb, d_sz, d_exact, d_hasrun, g.stream);
        launch_pack_scan(d_sz, d_hasrun, (uint32_t)nb, d_off, d_dummy, g.stream);
        ok = cudaMemcpyAsync(h_meta, d_off, 8 * (nb + 1), cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaMemcpyAsync(h_meta + 8 * (nb + 1), d_exact, 4 * nb, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaStreamSynchronize(g.stream) == cudaSuccess;
    }
    if (ok) {
        const uint64_t *h_off = (const uint64_t *)h_meta;
        const uint32_t *h_exact = (const uint32_t *)(h_meta + 8 * (nb + 1));
        total = h_off[nb];
        for (size_t i = 0; i < nb; i++) { (*off_out)[i] = h_off[i]; (*len_out)[i] = h_exact[i]; }
        (*off_out)[nb] = total;
        d_blob = (uint8_t *)dev_alloc(total);
        h_blob = (uint8_t *)pin_alloc(total);
        ok = d_blob && h_blob;
    }
    if (ok) {
        if (frozen) {
            uint64_t *d_cdst = (uint64_t *)dev_alloc(8 * (s->n_containers ? s->n_containers : 1));
            ok = d_cdst != nullptr;
            if (ok) launch_frozen_write(s->view(), (uint32_t)nb, s->n_containers, d_off, d_blob, d_cdst, g.stream);
            dev_free(d_cdst, 8 * (s->n_containers ? s->n_containers : 1));  // stream-ordered reuse only
        } else {
            launch_serialize_write(s->view(), (uint32_t)nb, d_off, d_hasrun, d_blob, g.stream);
        }
        ok = cudaMemcpyAsync(h_blob, d_blob, total, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaStreamSynchronize(g.stream) == cudaSuccess && cudaGetLastError() == cudaSuccess;
    }
    g.last_download_bytes = total;
    dev_free(d_sz, 8 * nb);
    dev_free(d_off, 8 * (nb + 1));
    dev_free(d_dummy, 8 * (nb + 1));
    dev_free(d_exact, 4 * nb);
    dev_free(d_hasrun, 4 * nb);
    dev_free(d_blob, total);
    pin_free(h_meta, 8 * (nb + 1) + 4 * nb);
    if (!ok) {
        pin_free(h_blob, total);
        free(*off_out);
        free(*len_out);
        *off_out = *len_out = nullptr;
        if (t_err.empty()) t_err = "set_serialize failed";
        return -1;
    }
    *buf = (char *)h_blob;
    g_serialized_sizes[h_blob] = total;
    return 0;
}

void rb200_serialized_free(char *buf, uint64_t *off, uint64_t *len) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (buf) {
        auto it = g_serialized_sizes.find((uint8_t *)buf);
        if (it != g_serialized_sizes.end()) {
            pin_free(buf, it->second);
            g_serialized_sizes.erase(it);
        }
    }
    free(off);
    free(len);
}

// Free many host bitmaps (results of rb200_set_download_all) with several threads.
void rb200_bitmaps_free(roaring_bitmap_t **bms, size_t n) {
    unsigned T = host_workers();
    if (n < 64 || T <= 1) {
        for (size_t i = 0; i < n; i++) bitmap_free_host(bms[i]);
        return;
    }
    std::atomic<size_t> next(0);
    std::function<void()> work = [&]() {
        for (;;) {
            const size_t i0 = next.fetch_add(8);
            if (i0 >= n) break;
            const size_t i1 = std::min(n, i0 + 8);
            for (size_t i = i0; i < i1; i++) bitmap_free_host(bms[i]);
        }
    };
    if ((size_t)T * 8 > n) T = (unsigned)((n + 7) / 8);
    pool().run(work, T);
}

int rb200_batch_op_host(int op, const roaring_bitmap_t *const *a, const roaring_bitmap_t *const *b,
                        size_t np, roaring_bitmap_t **out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    // upload a[] and b[] as ONE set (2*np bitmaps) so there is a single H2D stream
    std::vector<const roaring_bitmap_t *> all(2 * np);
    std::vector<uint32_t> ia(np), ib(np);
    for (size_t p = 0; p < np; p++) {
        all[p] = a[p];
        all[np + p] = b[p];
        ia[p] = (uint32_t)p;
        ib[p] = (uint32_t)(np + p);
    }
    rb200_set *S = rb200_set_upload(all.data(), all.size());
    if (!S) return -1;
    rb200_set_bind_host(S, 1);  // the inputs outlive this call
    rb200_set *R = batch_op_impl(op, S, S, ia.data(), ib.data(), np);
    int rc = -1;
    if (R) {
        rc = rb200_set_download_all(R, out);
        set_delete(R);
    }
    set_delete(S);
    return rc;
}

}  // extern "C"
namespace rb200 {
void set_error(const std::string &msg) { t_err = msg; }
void parallel_for(size_t n, const std::function<void(size_t)> &fn) {
    if (n == 0) return;
    unsigned T = host_workers();
    if (T <= 1 || n < 2) {
        for (size_t i = 0; i < n; i++) fn(i);
        return;
    }
    if ((size_t)T > n) T = (unsigned)n;
    std::atomic<size_t> next(0);
    std::function<void()> work = [&]() {
        for (;;) {
            const size_t i = next.fetch_add(1);
            if (i >= n) break;
            fn(i);
        }
    };
    pool().run(work, T);
}
}  // namespace rb200
extern "C" {

// =================================================================== drop-in entry points
// Entry points whose reference signature has no error channel (bool / void): a device failure is
// reported on stderr (and aborts under RB200_STRICT=1) instead of passing for an answer.
static void dropin_failed(const char *fn) {
    fprintf(stderr, "libroaring_b200: %s failed: %s\n", fn, t_err.empty() ? "unknown error" : t_err.c_str());
    const char *e = getenv("RB200_STRICT");
    if (e && e[0] == '1') abort();
}
// One small pair in ONE launch (rb200_fused.cu).  Returns 1: *out holds the result; 0: the pair
// does not qualify (too many containers / bytes) — use the batched path; -1: failure (t_err).
static int pair_fused(int op, const roaring_bitmap_t *r1, const roaring_bitmap_t *r2, int rules,
                      roaring_bitmap_t **out) {
    static const bool off = []() { const char *e = getenv("RB200_NO_FUSED"); return e && e[0] == '1'; }();
    if (off || !ctx_init()) return off ? 0 : -1;
    const roaring_array_t *ra[2] = {&r1->high_low_container, &r2->high_low_container};
    const uint32_t na = (uint32_t)ra[0]->size, nb = (uint32_t)ra[1]->size, n = na + nb;
    if (n > FUSED_MAX_ITEMS) return 0;
    // layout of the packed block
    FusedHdr hdr;
    memset(&hdr, 0, sizeof(hdr));
    hdr.na = na;
    hdr.nb = nb;
    size_t o = sizeof(FusedHdr);
    hdr.o_key = (uint32_t)o; o += (2 * (size_t)n + 15) & ~(size_t)15;
    hdr.o_type = (uint32_t)o; o += ((size_t)n + 15) & ~(size_t)15;
    hdr.o_shared = (uint32_t)o; o += ((size_t)n + 15) & ~(size_t)15;
    hdr.o_card = (uint32_t)o; o += (4 * (size_t)n + 15) & ~(size_t)15;
    hdr.o_len = (uint32_t)o; o += (4 * (size_t)n + 15) & ~(size_t)15;
    hdr.o_off = (uint32_t)o; o += (4 * (size_t)n + 15) & ~(size_t)15;
    uint8_t *h = g.h_fused_in;
    uint16_t *c_key = (uint16_t *)(h + hdr.o_key);
    uint8_t *c_type = h + hdr.o_type, *c_shared = h + hdr.o_shared;
    uint32_t *c_card = (uint32_t *)(h + hdr.o_card), *c_len = (uint32_t *)(h + hdr.o_len), *c_off = (uint32_t *)(h + hdr.o_off);
    uint64_t E[2] = {0, 0};
    uint32_t ci = 0;
    for (int side = 0; side < 2; side++) {
        for (int32_t i = 0; i < ra[side]->size; i++, ci++) {
            uint8_t t = ra[side]->typecodes[i];
            const bool was_shared = t == T_SHARED;
            const void *c = unwrap_shared(ra[side]->containers[i], t);
            uint32_t card = host_container_card(c, t), len;
            const uint8_t *p;
            if (t == T_BITSET) {
                len = 1024;
                p = (const uint8_t *)((const bitset_container_t *)c)->words;
                if (((const bitset_container_t *)c)->cardinality < 0) return 0;   // lazy state: batched path
            } else if (t == T_ARRAY) {
                len = card;
                p = (const uint8_t *)((const array_container_t *)c)->array;
            } else {
                len = (uint32_t)((const run_container_t *)c)->n_runs;
                p = (const uint8_t *)((const run_container_t *)c)->runs;
            }
            const uint32_t sb = stored_bytes(t, len), sb16 = round16(sb);
            if (o + sb16 > FUSED_IN_BYTES) return 0;
            memcpy(h + o, p, sb);
            if (sb16 > sb) memset(h + o + sb, 0, sb16 - sb);
            c_key[ci] = ra[side]->keys[i];
            c_type[ci] = t;
            c_shared[ci] = was_shared ? 1 : 0;
            c_card[ci] = card;
            c_len[ci] = len;
            c_off[ci] = (uint32_t)o;
            o += sb16;
            E[side] += effective_bytes(t, len, card);
        }
    }
    // the result slots must fit the mapped block (same bound as PairBuf::build)
    const uint64_t need = FUSED_OUT_PAYLOAD + (op == OP_AND ? std::min(E[0], E[1]) : op == OP_ANDNOT ? E[0] : E[0] + E[1]);
    if (need > FUSED_OUT_BYTES) return 0;
    memcpy(h, &hdr, sizeof(hdr));
    const uint32_t seq = ++g.fused_seq ? g.fused_seq : ++g.fused_seq;
    FusedOutHdr *oh = (FusedOutHdr *)g.h_fused_out;
    if (cudaMemcpyAsync(g.d_fused_in, h, o, cudaMemcpyHostToDevice, g.stream) != cudaSuccess ||
        !launch_pair_fused(op, g.d_fused_in, g.d_fused_out, FUSED_OUT_BYTES, rules, seq, g.stream)) {
        t_err = std::string("fused pair: ") + cudaGetErrorString(cudaGetLastError());
        return -1;
    }
    // wait for the sequence word in mapped memory (the kernel writes it last, after a system fence);
    // a short spin, then the ordinary stream synchronisation
    bool seen = false;
    for (int spin = 0; spin < 20000 && !seen; spin++) {
        seen = oh->seq == seq;
        if (!seen) __builtin_ia32_pause();
    }
    if (!seen) {
        const cudaError_t e = cudaStreamSynchronize(g.stream);
        if (e != cudaSuccess || oh->seq != seq) {
            t_err = std::string("fused pair: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "result never arrived");
            return -1;
        }
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    if (oh->error == 2) return 0;   // slots did not fit after all: batched path
    if (oh->error) { t_err = "fused pair: internal: result slot bound exceeded"; return -1; }
    const uint32_t no = oh->n_out;
    roaring_bitmap_t *r = bitmap_alloc((int32_t)no);
    if (!r) { t_err = "out of host memory"; return -1; }
    roaring_array_t *rr = &r->high_low_container;
    rr->flags = (ra[0]->flags | ra[1]->flags) & FLAG_COW;   // roaring.c:738, 890
    const uint8_t *ob = g.h_fused_out;
    const uint16_t *o_key = (const uint16_t *)(ob + FUSED_OUT_KEY);
    const uint8_t *o_type = ob + FUSED_OUT_TYPE;
    const uint32_t *o_card = (const uint32_t *)(ob + FUSED_OUT_CARD), *o_len = (const uint32_t *)(ob + FUSED_OUT_LEN),
                   *o_off = (const uint32_t *)(ob + FUSED_OUT_OFF);
    for (uint32_t k = 0; k < no; k++) {
        void *hc = container_from_payload(o_type[k], o_card[k], o_len[k], ob + o_off[k]);
        if (!hc) { bitmap_free_host(r); t_err = "out of host memory"; return -1; }
        rr->containers[k] = hc;
        rr->keys[k] = o_key[k];
        rr->typecodes[k] = o_type[k];
        rr->size = (int32_t)k + 1;
    }
    *out = r;
    return 1;
}

static roaring_bitmap_t *dropin_pair(int op, const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    roaring_bitmap_t *out = nullptr;
    {
        std::lock_guard<std::recursive_mutex> lk(g.mu);
        const int f = pair_fused(op, r1, r2, 0, &out);
        if (f == 1) return out;
        if (f < 0) return nullptr;
    }
    if (rb200_batch_op_host(op, &r1, &r2, 1, &out) != 0) return nullptr;
    return out;
}

roaring_bitmap_t *roaring_bitmap_and(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    return dropin_pair(OP_AND, r1, r2);
}
roaring_bitmap_t *roaring_bitmap_or(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    return dropin_pair(OP_OR, r1, r2);
}
roaring_bitmap_t *roaring_bitmap_xor(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    return dropin_pair(OP_XOR, r1, r2);
}
roaring_bitmap_t *roaring_bitmap_andnot(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    return dropin_pair(OP_ANDNOT, r1, r2);
}

roaring_bitmap_t *roaring_bitmap_or_many(size_t number, const roaring_bitmap_t **rs) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    rb200_set *S = rb200_set_upload(rs, number);
    if (!S) return nullptr;
    rb200_set *R = rb200_or_many(S, nullptr, number);
    roaring_bitmap_t *out = nullptr;
    if (R) {
        out = rb200_set_download(R, 0);
        set_delete(R);
    }
    set_delete(S);
    return out;
}

// In-place twins (src/roaring.c:812 and_inplace, :1063 or_inplace, :1200 xor_inplace, :1342
// andnot_inplace): the result is computed on the device with the in-place type rules and then
// swapped into x1 (its old containers and directory are released, its flags kept).
// replace x1's directory and containers by those of `out` (consumed); x1 keeps its flags
static void swap_into(roaring_bitmap_t *x1, roaring_bitmap_t *out);
static void dropin_inplace(int op, roaring_bitmap_t *x1, const roaring_bitmap_t *x2, int rules = RULES_INPLACE) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (rules == RULES_INPLACE) {   // (the lazy in-place twins take the batched path)
        roaring_bitmap_t *fo = nullptr;
        const int f = pair_fused(op, x1, x2, RULES_INPLACE, &fo);
        if (f == 1) { swap_into(x1, fo); return; }
        if (f < 0) { dropin_failed("roaring_bitmap_*_inplace"); return; }
    }
    const roaring_bitmap_t *both[2] = {x1, x2};
    rb200_set *S = rb200_set_upload(both, 2);
    if (!S) { dropin_failed("roaring_bitmap_*_inplace"); return; }
    rb200_set_bind_host(S, 1);
    const uint32_t ia = 0, ib = 1;
    rb200_set *R = batch_op_impl(op, S, S, &ia, &ib, 1, rules);
    roaring_bitmap_t *out = R ? rb200_set_download(R, 0) : nullptr;
    set_delete(R);
    set_delete(S);
    if (!out) { dropin_failed("roaring_bitmap_*_inplace"); return; }  // x1 is left untouched
    swap_into(x1, out);
}
static void swap_into(roaring_bitmap_t *x1, roaring_bitmap_t *out) {
    roaring_array_t *ra = &x1->high_low_container, *rn = &out->high_low_container;
    const uint8_t flags = ra->flags;
    if (!(flags & FLAG_FROZEN)) {
        for (int32_t i = 0; i < ra->size; i++) container_free_host(ra->containers[i], ra->typecodes[i]);
        h_free(ra->containers);
    }
    *ra = *rn;
    ra->flags = flags;
    h_free(out);
}
void roaring_bitmap_and_inplace(roaring_bitmap_t *x1, const roaring_bitmap_t *x2) {
    if (x1 == x2) return;  // roaring.c:814
    dropin_inplace(OP_AND, x1, x2);
}
void roaring_bitmap_or_inplace(roaring_bitmap_t *x1, const roaring_bitmap_t *x2) { dropin_inplace(OP_OR, x1, x2); }
void roaring_bitmap_xor_inplace(roaring_bitmap_t *x1, const roaring_bitmap_t *x2) { dropin_inplace(OP_XOR, x1, x2); }
void roaring_bitmap_andnot_inplace(roaring_bitmap_t *x1, const roaring_bitmap_t *x2) { dropin_inplace(OP_ANDNOT, x1, x2); }

roaring_bitmap_t *roaring_bitmap_xor_many(size_t number, const roaring_bitmap_t **rs) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    rb200_set *S = rb200_set_upload(rs, number);
    if (!S) return nullptr;
    rb200_set *R = rb200_xor_many(S, nullptr, number);
    roaring_bitmap_t *out = nullptr;
    if (R) {
        out = rb200_set_download(R, 0);
        set_delete(R);
    }
    set_delete(S);
    return out;
}

uint64_t roaring_bitmap_and_cardinality(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    const roaring_bitmap_t *both[2] = {r1, r2};
    rb200_set *S = rb200_set_upload(both, 2);
    if (!S) return UINT64_MAX;
    const uint32_t ia = 0, ib = 1;
    uint64_t out = UINT64_MAX;
    if (rb200_batch_and_cardinality(S, S, &ia, &ib, 1, &out) != 0) out = UINT64_MAX;
    set_delete(S);
    return out;
}

// src/roaring.c:3078-3107: inclusion-exclusion on and_cardinality + the two cardinalities
uint64_t roaring_bitmap_or_cardinality(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    const uint64_t c1 = rb200_bitmap_get_cardinality(r1), c2 = rb200_bitmap_get_cardinality(r2);
    const uint64_t inter = roaring_bitmap_and_cardinality(r1, r2);
    return inter == UINT64_MAX ? UINT64_MAX : c1 + c2 - inter;
}
uint64_t roaring_bitmap_andnot_cardinality(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    const uint64_t c1 = rb200_bitmap_get_cardinality(r1);
    const uint64_t inter = roaring_bitmap_and_cardinality(r1, r2);
    return inter == UINT64_MAX ? UINT64_MAX : c1 - inter;
}
uint64_t roaring_bitmap_xor_cardinality(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    const uint64_t c1 = rb200_bitmap_get_cardinality(r1), c2 = rb200_bitmap_get_cardinality(r2);
    const uint64_t inter = roaring_bitmap_and_cardinality(r1, r2);
    return inter == UINT64_MAX ? UINT64_MAX : c1 + c2 - 2 * inter;
}
double roaring_bitmap_jaccard_index(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    const uint64_t c1 = rb200_bitmap_get_cardinality(r1), c2 = rb200_bitmap_get_cardinality(r2);
    const uint64_t inter = roaring_bitmap_and_cardinality(r1, r2);
    if (inter == UINT64_MAX) return std::numeric_limits<double>::quiet_NaN();  // device failure: rb200_last_error()
    return (double)inter / (double)(c1 + c2 - inter);
}
bool roaring_bitmap_intersect(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    const uint64_t inter = roaring_bitmap_and_cardinality(r1, r2);
    if (inter == UINT64_MAX) dropin_failed("roaring_bitmap_intersect");
    return inter != 0 && inter != UINT64_MAX;
}

// ---- equality / subset relations (src/roaring.c:2128-2200, 3172; cells mixed_equal.c,
// mixed_subset.c): A == B  <=>  |A| = |B| = |A and B|;  A subset of B  <=>  |A and B| = |A|.
// One k_card_items sweep over the pair list + the per-bitmap cardinalities already on the device.
// out[k]: bit 0 = equals, bit 1 = is_subset(a, b), bit 2 = is_strict_subset(a, b).
int rb200_batch_relations(const rb200_set_t *A, const rb200_set_t *B, const uint32_t *ia,
                          const uint32_t *ib, size_t np, uint8_t *out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (np == 0) return 0;
    std::vector<uint64_t> inter(np), ca(A->n_bitmaps), cb(B->n_bitmaps);
    if (rb200_batch_and_cardinality(A, B, ia, ib, np, inter.data()) != 0) return -1;
    if (rb200_set_cardinalities(A, ca.data()) != 0 || rb200_set_cardinalities(B, cb.data()) != 0) return -1;
    for (size_t k = 0; k < np; k++) {
        const uint64_t a = ca[ia[k]], b = cb[ib[k]], x = inter[k];
        const bool sub = x == a;
        out[k] = (uint8_t)((sub && a == b ? 1 : 0) | (sub ? 2 : 0) | (sub && b > a ? 4 : 0));
    }
    return 0;
}
static int dropin_relation(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    const roaring_bitmap_t *both[2] = {r1, r2};
    rb200_set *S = rb200_set_upload(both, 2);
    if (!S) { dropin_failed("roaring_bitmap_equals / is_subset / is_strict_subset"); return -1; }
    const uint32_t ia = 0, ib = 1;
    uint8_t out = 0;
    const int rc = rb200_batch_relations(S, S, &ia, &ib, 1, &out);
    set_delete(S);
    if (rc != 0) dropin_failed("roaring_bitmap_equals / is_subset / is_strict_subset");
    return rc != 0 ? -1 : out;
}
bool roaring_bitmap_equals(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    const int r = dropin_relation(r1, r2);
    return r > 0 && (r & 1);
}
bool roaring_bitmap_is_subset(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    const int r = dropin_relation(r1, r2);
    return r > 0 && (r & 2);
}
bool roaring_bitmap_is_strict_subset(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    const int r = dropin_relation(r1, r2);
    return r > 0 && (r & 4);
}

// ---- negation: roaring_bitmap_flip (src/roaring.c:2289-2349) ------------------------------------
// result[k] = S[idx[k]] with [range_start, range_end) negated.  The range is materialised as ONE
// tiny bitmap of run containers (one {lo, hi-lo} run per key it touches) and every flip is a
// symmetric difference with it under the negation type rules (RULES_FLIP), batched like any op.
rb200_set_t *rb200_batch_flip(const rb200_set_t *S, const uint32_t *idx, size_t n, uint64_t range_start,
                              uint64_t range_end) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return nullptr;
    if (reject_lazy(S, "flip")) return nullptr;
    if (idx == nullptr) n = S->n_bitmaps;
    std::vector<uint32_t> ia(n), ib(n, 0);
    for (size_t i = 0; i < n; i++) ia[i] = idx ? idx[i] : (uint32_t)i;
    std::vector<uint8_t> blob;
    // roaring.c:2292 (open range empty / start past the 32-bit universe) and :2303 (the CLOSED
    // range, after the reference's truncation of both ends to 32 bits, is empty): plain copy
    const bool noop = range_start >= range_end || range_start > (uint64_t)UINT32_MAX + 1 ||
                      (uint32_t)range_start > (uint32_t)(range_end - 1);
    if (noop) {  // copy: symmetric difference with the empty bitmap
        const uint32_t hdr[2] = {SERIAL_COOKIE_NO_RUN, 0};
        blob.assign((const uint8_t *)hdr, (const uint8_t *)hdr + 8);
    } else {
        const uint32_t first = (uint32_t)range_start, last = (uint32_t)(range_end - 1);
        const uint32_t hb0 = first >> 16, hb1 = last >> 16, nk = hb1 - hb0 + 1;
        const size_t nfb = (nk + 7) / 8, hdr = 4 + nfb + 4 * (size_t)nk + (nk >= (uint32_t)NO_OFFSET_THRESHOLD ? 4 * (size_t)nk : 0);
        blob.assign(hdr + 6 * (size_t)nk, 0);
        const uint32_t cookie = SERIAL_COOKIE | ((nk - 1) << 16);
        memcpy(blob.data(), &cookie, 4);
        memset(blob.data() + 4, 0xFF, nfb);  // every container is a run
        if (nk & 7) blob[4 + nfb - 1] = (uint8_t)((1u << (nk & 7)) - 1);
        uint8_t *kc = blob.data() + 4 + nfb, *offs = kc + 4 * (size_t)nk, *pay = blob.data() + hdr;
        for (uint32_t k = 0; k < nk; k++) {
            const uint32_t hb = hb0 + k, lo = hb == hb0 ? (first & 0xFFFF) : 0, hi = hb == hb1 ? (last & 0xFFFF) : 0xFFFF;
            const uint16_t key = (uint16_t)hb, cm1 = (uint16_t)(hi - lo), one = 1, v0 = (uint16_t)lo;
            memcpy(kc + 4 * (size_t)k, &key, 2);
            memcpy(kc + 4 * (size_t)k + 2, &cm1, 2);
            if (nk >= (uint32_t)NO_OFFSET_THRESHOLD) {
                const uint32_t o = (uint32_t)(hdr + 6 * (size_t)k);
                memcpy(offs + 4 * (size_t)k, &o, 4);
            }
            memcpy(pay + 6 * (size_t)k, &one, 2);
            memcpy(pay + 6 * (size_t)k + 2, &v0, 2);
            memcpy(pay + 6 * (size_t)k + 4, &cm1, 2);
        }
    }
    const char *bp = (const char *)blob.data();
    const size_t bl = blob.size();
    rb200_set *Rg = upload_blobs_impl(&bp, &bl, 1, false);
    if (!Rg) return nullptr;
    rb200_set *R = batch_op_impl(OP_XOR, S, Rg, ia.data(), ib.data(), n, noop ? 0 : (RULES_LAZY | RULES_FLIP));
    set_delete(Rg);
    return R;
}
roaring_bitmap_t *roaring_bitmap_flip(const roaring_bitmap_t *r1, uint64_t range_start, uint64_t range_end) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    const roaring_bitmap_t *one[1] = {r1};
    rb200_set *S = rb200_set_upload(one, 1);
    if (!S) return nullptr;
    rb200_set_bind_host(S, 1);
    rb200_set *R = rb200_batch_flip(S, nullptr, 1, range_start, range_end);
    roaring_bitmap_t *out = R ? rb200_set_download(R, 0) : nullptr;
    set_delete(R);
    set_delete(S);
    return out;
}
void roaring_bitmap_flip_inplace(roaring_bitmap_t *r1, uint64_t range_start, uint64_t range_end) {
    if (range_start >= range_end || range_start > (uint64_t)UINT32_MAX + 1) return;  // roaring.c:2353
    if ((uint32_t)range_start > (uint32_t)(range_end - 1)) return;                    // roaring.c:2364
    roaring_bitmap_t *out = roaring_bitmap_flip(r1, range_start, range_end);
    if (!out) dropin_failed("roaring_bitmap_flip_inplace");
    if (out) {
        std::lock_guard<std::recursive_mutex> lk(g.mu);
        swap_into(r1, out);
    }
}

// ---- 64-bit bitmaps through their portable format (src/roaring64.c) -------------------------
// roaring64_bitmap_{and,or,xor,andnot} (roaring64.c:1332, 1541, 1663, 1809) apply the same
// container cells to equal high-48-bit keys; the 64-bit portable format (roaring64.c:2262-2395)
// stores one ordinary 32-bit portable bitmap per high-32 "bucket".  Here every bucket of every
// input becomes one bitmap of ONE resident set, matching buckets of a pair become one pair of the
// batched kernel (unmatched ones are paired with an empty bitmap = pass-through), and the result
// buckets are serialized on the device and stitched back into 64-bit blobs.
namespace {
struct R64Bucket { uint32_t high; const char *ptr; size_t len; };
// length of the 32-bit portable bitmap starting at buf (0 = malformed); header walk only
size_t portable_length(const uint8_t *buf, size_t maxlen) {
    if (maxlen < 4) return 0;
    uint32_t cookie;
    memcpy(&cookie, buf, 4);
    size_t pos = 4, size;
    const uint8_t *runflags = nullptr;
    if ((cookie & 0xFFFF) == SERIAL_COOKIE) {
        size = (cookie >> 16) + 1;
        runflags = buf + 4;
        pos += (size + 7) / 8;
    } else if (cookie == SERIAL_COOKIE_NO_RUN && maxlen >= 8) {
        uint32_t sz;
        memcpy(&sz, buf + 4, 4);
        size = sz;
        pos = 8;
    } else {
        return 0;
    }
    if (size > 65536 || pos + 4 * size > maxlen) return 0;
    const uint8_t *kc = buf + pos;
    pos += 4 * size;
    if (!runflags || size >= (size_t)NO_OFFSET_THRESHOLD) pos += 4 * size;
    for (size_t i = 0; i < size; i++) {
        uint16_t cm1;
        memcpy(&cm1, kc + 4 * i + 2, 2);
        if (runflags && ((runflags[i / 8] >> (i % 8)) & 1)) {
            if (pos + 2 > maxlen) return 0;
            uint16_t nr;
            memcpy(&nr, buf + pos, 2);
            pos += 2 + 4 * (size_t)nr;
        } else {
            pos += (uint32_t)cm1 + 1 > (uint32_t)MAX_ARRAY ? (size_t)BITSET_BYTES : 2 * ((size_t)cm1 + 1);
        }
        if (pos > maxlen) return 0;
    }
    return pos;
}
bool parse_r64(const char *buf, size_t len, std::vector<R64Bucket> &out) {
    out.clear();
    if (len < 8) return false;
    uint64_t n;
    memcpy(&n, buf, 8);
    if (n > UINT32_MAX) return false;
    size_t pos = 8;
    for (uint64_t i = 0; i < n; i++) {
        if (pos + 4 > len) return false;
        R64Bucket b;
        memcpy(&b.high, buf + pos, 4);
        pos += 4;
        if (i && b.high <= out.back().high) return false;
        b.ptr = buf + pos;
        b.len = portable_length((const uint8_t *)buf + pos, len - pos);
        if (!b.len) return false;
        pos += b.len;
        out.push_back(b);
    }
    return true;
}
struct R64Plan {
    rb200_set *S = nullptr;                 // every bucket of every input + one empty bitmap (last)
    std::vector<uint32_t> pa, pb, high;     // bucket pairs and their high-32 value
    std::vector<size_t> first;              // per 64-bit pair: its bucket pairs are [first[p], first[p+1])
};
// op < 0: cardinality planning (matched buckets only)
bool plan_r64(int op, const char *const *a, const size_t *alen, size_t na, const char *const *b,
              const size_t *blen, size_t nb, const uint32_t *ia, const uint32_t *ib, size_t np, R64Plan &P) {
    std::vector<std::vector<R64Bucket>> A(na), B(nb);
    std::vector<size_t> baseA(na), baseB(nb);
    std::vector<const char *> ptrs;
    std::vector<size_t> lens;
    for (size_t i = 0; i < na; i++) {
        if (!parse_r64(a[i], alen[i], A[i])) { t_err = "malformed 64-bit portable bitmap (left) at index " + std::to_string(i); return false; }
        baseA[i] = ptrs.size();
        for (auto &x : A[i]) { ptrs.push_back(x.ptr); lens.push_back(x.len); }
    }
    for (size_t i = 0; i < nb; i++) {
        if (!parse_r64(b[i], blen[i], B[i])) { t_err = "malformed 64-bit portable bitmap (right) at index " + std::to_string(i); return false; }
        baseB[i] = ptrs.size();
        for (auto &x : B[i]) { ptrs.push_back(x.ptr); lens.push_back(x.len); }
    }
    static const uint32_t empty_blob[2] = {SERIAL_COOKIE_NO_RUN, 0};
    const uint32_t EMPTY = (uint32_t)ptrs.size();
    ptrs.push_back((const char *)empty_blob);
    lens.push_back(8);
    P.first.assign(1, 0);
    for (size_t p = 0; p < np; p++) {
        if (ia[p] >= na || ib[p] >= nb) { t_err = "pair index out of range"; return false; }
        const auto &x = A[ia[p]], &y = B[ib[p]];
        size_t i = 0, j = 0;
        while (i < x.size() || j < y.size()) {
            const bool only1 = j >= y.size() || (i < x.size() && x[i].high < y[j].high);
            const bool only2 = !only1 && (i >= x.size() || y[j].high < x[i].high);
            const bool keep = only1 ? (op == OP_OR || op == OP_XOR || op == OP_ANDNOT)
                              : only2 ? (op == OP_OR || op == OP_XOR) : true;
            if (keep) {
                P.pa.push_back(only2 ? EMPTY : (uint32_t)(baseA[ia[p]] + i));
                P.pb.push_back(only1 ? EMPTY : (uint32_t)(baseB[ib[p]] + j));
                P.high.push_back(only2 ? y[j].high : x[i].high);
            }
            if (!only2) i++;
            if (!only1) j++;
        }
        P.first.push_back(P.pa.size());
    }
    P.S = upload_blobs_impl(ptrs.data(), lens.data(), ptrs.size(), false);
    return P.S != nullptr;
}
}  // namespace

// result[k] = roaring64 op of (a[ia[k]], b[ib[k]]), all in the 64-bit portable format.  *out is
// pinned memory owned by the library (blob k at *out + (*off)[k], (*len)[k] bytes); release with
// rb200_serialized_free.
int rb200_r64_batch_op_serialized(int op, const char *const *a, const size_t *alen, size_t na,
                                  const char *const *b, const size_t *blen, size_t nb, const uint32_t *ia,
                                  const uint32_t *ib, size_t np, char **out, uint64_t **off_out, uint64_t **len_out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    if (op < 0 || op > 3) { t_err = "bad op"; return -1; }
    *out = nullptr;
    *off_out = *len_out = nullptr;
    R64Plan P;
    if (!plan_r64(op, a, alen, na, b, blen, nb, ia, ib, np, P)) return -1;
    rb200_set *R = batch_op_impl(op, P.S, P.S, P.pa.data(), P.pb.data(), P.pa.size());
    char *sbuf = nullptr;
    uint64_t *soff = nullptr, *slen = nullptr;
    int rc = R ? serialize_impl(R, &sbuf, &soff, &slen, false) : -1;
    set_delete(R);
    set_delete(P.S);
    if (rc != 0) return -1;
    // stitch: u64 bucket count, then per non-empty bucket u32 high32 + 32-bit blob
    uint64_t *off = (uint64_t *)malloc(8 * (np + 1)), *len = (uint64_t *)malloc(8 * (np + 1));
    uint64_t total = 0;
    auto empty_bucket = [&](size_t q) {
        uint32_t w[2];
        if (slen[q] != 8) return false;
        memcpy(w, sbuf + soff[q], 8);
        return w[0] == SERIAL_COOKIE_NO_RUN && w[1] == 0;
    };
    if (off && len) {
        for (size_t p = 0; p < np; p++) {
            uint64_t sz = 8;
            for (size_t q = P.first[p]; q < P.first[p + 1]; q++)
                if (!empty_bucket(q)) sz += 4 + slen[q];
            off[p] = total;
            len[p] = sz;
            total += (sz + 15) & ~(uint64_t)15;
        }
        off[np] = total;
    }
    uint8_t *dst = (off && len) ? (uint8_t *)pin_alloc(total ? total : 16) : nullptr;
    if (dst) {
        for (size_t p = 0; p < np; p++) {
            uint8_t *o = dst + off[p];
            uint64_t kept = 0;
            size_t pos = 8;
            for (size_t q = P.first[p]; q < P.first[p + 1]; q++) {
                if (empty_bucket(q)) continue;
                memcpy(o + pos, &P.high[q], 4);
                memcpy(o + pos + 4, sbuf + soff[q], slen[q]);
                pos += 4 + slen[q];
                kept++;
            }
            memcpy(o, &kept, 8);
        }
        g_serialized_sizes[dst] = total ? total : 16;
    }
    rb200_serialized_free(sbuf, soff, slen);
    if (!dst) {
        free(off);
        free(len);
        t_err = "r64 batch op: host allocation failed";
        return -1;
    }
    *out = (char *)dst;
    *off_out = off;
    *len_out = len;
    return 0;
}

// out[k] = roaring64_bitmap_and_cardinality(a[ia[k]], b[ib[k]]) (roaring64.c:1375)
int rb200_r64_batch_and_cardinality_serialized(const char *const *a, const size_t *alen, size_t na,
                                               const char *const *b, const size_t *blen, size_t nb,
                                               const uint32_t *ia, const uint32_t *ib, size_t np, uint64_t *out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    R64Plan P;
    if (!plan_r64(OP_AND, a, alen, na, b, blen, nb, ia, ib, np, P)) return -1;
    std::vector<uint64_t> c(P.pa.size());
    const int rc = P.pa.empty() ? 0 : rb200_batch_and_cardinality(P.S, P.S, P.pa.data(), P.pb.data(), P.pa.size(), c.data());
    set_delete(P.S);
    if (rc != 0) return -1;
    for (size_t p = 0; p < np; p++) {
        uint64_t s = 0;
        for (size_t q = P.first[p]; q < P.first[p + 1]; q++) s += c[q];
        out[p] = s;
    }
    return 0;
}

// ---- in-memory roaring64_bitmap_t (include/roaring/roaring64.h:423-522; src/roaring64.c:1332-1895)
// The 64-bit bitmap is an ART of (high-48 key -> container) owned by the reference library; its
// layout is private to that library (src/art/art.c), so the binding goes through the two format
// functions the reference exports for exactly this purpose: the operands are written with the
// HOST APPLICATION's roaring64_bitmap_portable_serialize (resolved with dlsym in the running
// process — the reference must be loaded, or nobody could have built a roaring64_bitmap_t), the
// container grid runs on the device (rb200_r64_batch_op_serialized), and the result bytes become
// a roaring64_bitmap_t again through roaring64_bitmap_portable_deserialize_safe.  Results are
// byte-identical to the reference's (tests/test_gpu_r64.py).
namespace {
struct R64Api {
    size_t (*size)(const roaring64_bitmap_t *) = nullptr;
    size_t (*ser)(const roaring64_bitmap_t *, char *) = nullptr;
    roaring64_bitmap_t *(*deser)(const char *, size_t) = nullptr;
    uint64_t (*card)(const roaring64_bitmap_t *) = nullptr;
    bool ok() {
        if (size && ser && deser && card) return true;   // looked up lazily: the host library may load later
        size = (decltype(size))dlsym(RTLD_DEFAULT, "roaring64_bitmap_portable_size_in_bytes");
        ser = (decltype(ser))dlsym(RTLD_DEFAULT, "roaring64_bitmap_portable_serialize");
        deser = (decltype(deser))dlsym(RTLD_DEFAULT, "roaring64_bitmap_portable_deserialize_safe");
        card = (decltype(card))dlsym(RTLD_DEFAULT, "roaring64_bitmap_get_cardinality");
        if (size && ser && deser && card) return true;
        t_err = "roaring64: the host CRoaring library (roaring64_bitmap_portable_serialize / _deserialize_safe) "
                "is not loaded in this process";
        return false;
    }
} g_r64;

// serialize n distinct in-memory bitmaps (in parallel) into owned buffers
bool r64_serialize_all(const roaring64_bitmap_t *const *bms, size_t n, std::vector<std::vector<char>> &bufs) {
    bufs.resize(n);
    std::atomic<bool> ok(true);
    rb200::parallel_for(n, [&](size_t i) {
        const size_t sz = g_r64.size(bms[i]);
        bufs[i].resize(sz ? sz : 1);
        if (g_r64.ser(bms[i], bufs[i].data()) != sz) ok = false;
    });
    if (!ok) t_err = "roaring64: serialization of an operand failed";
    return ok;
}
}  // namespace

// out[k] = roaring64_bitmap_{and,or,xor,andnot}(a[k], b[k]) for npairs in-memory 64-bit bitmaps of the
// host application's CRoaring; out[k] is a fresh roaring64_bitmap_t the caller frees with
// roaring64_bitmap_free.  0 on success.
int rb200_r64_batch_op(int op, const roaring64_bitmap_t *const *a, const roaring64_bitmap_t *const *b,
                       size_t npairs, roaring64_bitmap_t **out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!g_r64.ok()) return -1;
    if (npairs == 0) return 0;
    std::vector<std::vector<char>> sa, sb;
    if (!r64_serialize_all(a, npairs, sa) || !r64_serialize_all(b, npairs, sb)) return -1;
    std::vector<const char *> pa(npairs), pb(npairs);
    std::vector<size_t> la(npairs), lb(npairs);
    std::vector<uint32_t> ia(npairs), ib(npairs);
    for (size_t k = 0; k < npairs; k++) {
        pa[k] = sa[k].data(); la[k] = g_r64.size(a[k]);
        pb[k] = sb[k].data(); lb[k] = g_r64.size(b[k]);
        ia[k] = ib[k] = (uint32_t)k;
    }
    char *blob = nullptr;
    uint64_t *off = nullptr, *len = nullptr;
    if (rb200_r64_batch_op_serialized(op, pa.data(), la.data(), npairs, pb.data(), lb.data(), npairs, ia.data(),
                                      ib.data(), npairs, &blob, &off, &len) != 0)
        return -1;
    std::atomic<bool> ok(true);
    rb200::parallel_for(npairs, [&](size_t k) {
        out[k] = g_r64.deser(blob + off[k], (size_t)len[k]);
        if (!out[k]) ok = false;
    });
    rb200_serialized_free(blob, off, len);
    if (!ok) {
        // all or nothing: the results that were built go back to the host library
        auto r64_free = (void (*)(roaring64_bitmap_t *))dlsym(RTLD_DEFAULT, "roaring64_bitmap_free");
        for (size_t k = 0; k < npairs; k++) {
            if (out[k] && r64_free) r64_free(out[k]);
            out[k] = nullptr;
        }
        t_err = "roaring64: the host library refused a result blob";
        return -1;
    }
    return 0;
}

int rb200_r64_batch_and_cardinality(const roaring64_bitmap_t *const *a, const roaring64_bitmap_t *const *b,
                                    size_t npairs, uint64_t *out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!g_r64.ok()) return -1;
    if (npairs == 0) return 0;
    std::vector<std::vector<char>> sa, sb;
    if (!r64_serialize_all(a, npairs, sa) || !r64_serialize_all(b, npairs, sb)) return -1;
    std::vector<const char *> pa(npairs), pb(npairs);
    std::vector<size_t> la(npairs), lb(npairs);
    std::vector<uint32_t> ia(npairs), ib(npairs);
    for (size_t k = 0; k < npairs; k++) {
        pa[k] = sa[k].data(); la[k] = g_r64.size(a[k]);
        pb[k] = sb[k].data(); lb[k] = g_r64.size(b[k]);
        ia[k] = ib[k] = (uint32_t)k;
    }
    return rb200_r64_batch_and_cardinality_serialized(pa.data(), la.data(), npairs, pb.data(), lb.data(), npairs,
                                                      ia.data(), ib.data(), npairs, out);
}

// drop-in symbols, include/roaring/roaring64.h:423-522
static roaring64_bitmap_t *r64_dropin(int op, const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2) {
    roaring64_bitmap_t *out = nullptr;
    return rb200_r64_batch_op(op, &r1, &r2, 1, &out) == 0 ? out : nullptr;
}
roaring64_bitmap_t *roaring64_bitmap_and(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2) { return r64_dropin(OP_AND, r1, r2); }
roaring64_bitmap_t *roaring64_bitmap_or(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2) { return r64_dropin(OP_OR, r1, r2); }
roaring64_bitmap_t *roaring64_bitmap_xor(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2) { return r64_dropin(OP_XOR, r1, r2); }
roaring64_bitmap_t *roaring64_bitmap_andnot(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2) { return r64_dropin(OP_ANDNOT, r1, r2); }
uint64_t roaring64_bitmap_and_cardinality(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2) {
    uint64_t c = UINT64_MAX;
    if (rb200_r64_batch_and_cardinality(&r1, &r2, 1, &c) != 0) return UINT64_MAX;
    return c;
}
// roaring64.c:1411-1437, 1600-1622...: inclusion-exclusion on and_cardinality
uint64_t roaring64_bitmap_or_cardinality(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2) {
    const uint64_t i = roaring64_bitmap_and_cardinality(r1, r2);
    return i == UINT64_MAX ? i : g_r64.card(r1) + g_r64.card(r2) - i;
}
uint64_t roaring64_bitmap_xor_cardinality(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2) {
    const uint64_t i = roaring64_bitmap_and_cardinality(r1, r2);
    return i == UINT64_MAX ? i : g_r64.card(r1) + g_r64.card(r2) - 2 * i;
}
uint64_t roaring64_bitmap_andnot_cardinality(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2) {
    const uint64_t i = roaring64_bitmap_and_cardinality(r1, r2);
    return i == UINT64_MAX ? i : g_r64.card(r1) - i;
}
double roaring64_bitmap_jaccard_index(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2) {
    const uint64_t i = roaring64_bitmap_and_cardinality(r1, r2);
    if (i == UINT64_MAX) return std::numeric_limits<double>::quiet_NaN();
    return (double)i / (double)(g_r64.card(r1) + g_r64.card(r2) - i);
}
bool roaring64_bitmap_intersect(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2) {
    const uint64_t i = roaring64_bitmap_and_cardinality(r1, r2);
    if (i == UINT64_MAX) dropin_failed("roaring64_bitmap_intersect");
    return i != 0 && i != UINT64_MAX;
}

// ---- public lazy API (include/roaring/roaring.h:932-977) ------------------------------------
// The lazy state lives in ordinary host bitmaps exactly as the reference leaves it (bitsets with
// cardinality -1, unconverted runs), so the reference's own functions accept what we return.
static roaring_bitmap_t *dropin_lazy_pair(int op, const roaring_bitmap_t *r1, const roaring_bitmap_t *r2, int rules) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    const roaring_bitmap_t *both[2] = {r1, r2};
    rb200_set *S = rb200_set_upload(both, 2);
    if (!S) return nullptr;
    rb200_set_bind_host(S, 1);
    const uint32_t ia = 0, ib = 1;
    rb200_set *R = batch_op_impl(op, S, S, &ia, &ib, 1, rules);
    roaring_bitmap_t *out = R ? rb200_set_download(R, 0) : nullptr;
    set_delete(R);
    set_delete(S);
    return out;
}
roaring_bitmap_t *roaring_bitmap_lazy_or(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2, const bool bitsetconversion) {
    return dropin_lazy_pair(OP_OR, r1, r2, RULES_LAZY | (bitsetconversion ? RULES_CONV : 0));
}
void roaring_bitmap_lazy_or_inplace(roaring_bitmap_t *r1, const roaring_bitmap_t *r2, const bool bitsetconversion) {
    dropin_inplace(OP_OR, r1, r2, RULES_LAZY | RULES_INPLACE | (bitsetconversion ? RULES_CONV : 0));
}
roaring_bitmap_t *roaring_bitmap_lazy_xor(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    return dropin_lazy_pair(OP_XOR, r1, r2, RULES_LAZY);
}
void roaring_bitmap_lazy_xor_inplace(roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    dropin_inplace(OP_XOR, r1, r2, RULES_LAZY | RULES_INPLACE);
}
void roaring_bitmap_repair_after_lazy(roaring_bitmap_t *r1) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    const roaring_bitmap_t *one[1] = {r1};
    rb200_set *S = rb200_set_upload(one, 1);
    if (!S) { dropin_failed("roaring_bitmap_repair_after_lazy"); return; }
    rb200_set *R = rb200_set_repair_after_lazy(S);
    roaring_bitmap_t *out = R ? rb200_set_download(R, 0) : nullptr;
    set_delete(R);
    set_delete(S);
    if (out) swap_into(r1, out);
    else dropin_failed("roaring_bitmap_repair_after_lazy");
}

// ---- roaring_bitmap_or_many_heap (src/roaring_priority_queue.c:200-250) ------------------------
// The reference orders pairwise LAZY unions with a binary min-heap keyed by
// roaring_bitmap_portable_size_in_bytes; the result TYPES depend on that order, so the same heap
// (same sift loops, same tie behaviour) is replayed here and every union runs on the device:
// lazy_or (both inputs), lazy_or_inplace (one temporary) or lazy_or_from_lazy_inputs (two).
namespace {
struct HeapEl {
    uint64_t size;
    bool temp;
    rb200_set *set;
    uint32_t index;
};
void heap_down(std::vector<HeapEl> &e, uint32_t n, uint32_t i) {  // percolate_down :46-66
    const uint32_t half = n >> 1;
    const HeapEl cur = e[i];
    while (i < half) {
        uint32_t child = 2 * i + 1;
        if (child + 1 < n && e[child + 1].size < e[child].size) child++;
        if (!(e[child].size < cur.size)) break;
        e[i] = e[child];
        i = child;
    }
    e[i] = cur;
}
void heap_push(std::vector<HeapEl> &e, uint32_t &n, const HeapEl &t) {  // pq_add :31-42
    uint32_t i = n++;
    while (i > 0) {
        const uint32_t parent = (i - 1) >> 1;
        if (!(t.size < e[parent].size)) break;
        e[i] = e[parent];
        i = parent;
    }
    e[i] = t;
}
HeapEl heap_pop(std::vector<HeapEl> &e, uint32_t &n) {  // pq_poll :84-95
    const HeapEl top = e[0];
    if (n > 1) {
        e[0] = e[--n];
        heap_down(e, n, 0);
    } else {
        --n;
    }
    return top;
}
// portable sizes (header + containers) of every bitmap of a set, lazy state included
bool portable_sizes(const rb200_set *S, std::vector<uint32_t> &out) {
    if (!resolve(S)) return false;
    const size_t nb = S->n_bitmaps;
    out.assign(nb, 0);
    if (!nb) return true;
    uint64_t *d16 = (uint64_t *)dev_alloc(8 * nb);
    uint32_t *dex = (uint32_t *)dev_alloc(4 * nb), *dhr = (uint32_t *)dev_alloc(4 * nb);
    uint32_t *h = (uint32_t *)pin_alloc(4 * nb);
    bool ok = d16 && dex && dhr && h;
    if (ok) {
        launch_serialize_measure(S->view(), (uint32_t)nb, d16, dex, dhr, g.stream);
        ok = cudaMemcpyAsync(h, dex, 4 * nb, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaStreamSynchronize(g.stream) == cudaSuccess;
        if (ok) out.assign(h, h + nb);
    }
    dev_free(d16, 8 * nb);
    dev_free(dex, 4 * nb);
    dev_free(dhr, 4 * nb);
    pin_free(h, 4 * nb);
    if (!ok && t_err.empty()) t_err = "portable_sizes failed";
    return ok;
}
}  // namespace

rb200_set_t *rb200_or_many_heap(const rb200_set_t *S, const uint32_t *idx, size_t n) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return nullptr;
    if (reject_lazy(S, "or_many_heap")) return nullptr;
    if (idx == nullptr) n = S->n_bitmaps;
    for (size_t i = 0; i < n; i++)
        if (idx && idx[i] >= S->n_bitmaps) { t_err = "or_many_heap: index out of range"; return nullptr; }
    if (n == 0) return rb200_or_many(S, idx, 0);
    if (n == 1) {  // roaring_bitmap_copy: union with an empty bitmap = pass-through of every container
        roaring_bitmap_t *e = bitmap_alloc(0);
        if (!e) return nullptr;
        const roaring_bitmap_t *one[1] = {e};
        rb200_set *E = rb200_set_upload(one, 1);
        bitmap_free_host(e);
        if (!E) return nullptr;
        const uint32_t a = idx ? idx[0] : 0u, z = 0;
        rb200_set *R = batch_op_impl(OP_OR, S, E, &a, &z, 1, 0);
        set_delete(E);
        return R;
    }
    std::vector<uint32_t> sz;
    if (!portable_sizes(S, sz)) return nullptr;
    std::vector<HeapEl> e(n);
    for (size_t i = 0; i < n; i++) {
        const uint32_t b = idx ? idx[i] : (uint32_t)i;
        e[i] = HeapEl{sz[b], false, const_cast<rb200_set *>(S), b};
    }
    uint32_t cnt = (uint32_t)n;
    for (int32_t i = (int32_t)(cnt >> 1); i >= 0; i--) heap_down(e, cnt, (uint32_t)i);  // create_pq :68-82
    bool ok = true;
    while (cnt > 1 && ok) {
        const HeapEl a = heap_pop(e, cnt), b = heap_pop(e, cnt);
        rb200_set *R;
        if (a.temp && b.temp)
            R = batch_op_impl(OP_OR, a.set, b.set, &a.index, &b.index, 1, RULES_LAZY | RULES_INPLACE | RULES_NOFULL);
        else if (b.temp)  // roaring_bitmap_lazy_or_inplace(x2, x1, false)
            R = batch_op_impl(OP_OR, b.set, a.set, &b.index, &a.index, 1, RULES_LAZY | RULES_INPLACE);
        else if (a.temp)
            R = batch_op_impl(OP_OR, a.set, b.set, &a.index, &b.index, 1, RULES_LAZY | RULES_INPLACE);
        else
            R = batch_op_impl(OP_OR, a.set, b.set, &a.index, &b.index, 1, RULES_LAZY);
        if (a.temp) set_delete(a.set);
        if (b.temp) set_delete(b.set);
        if (!R || !resolve(R)) { set_delete(R); ok = false; break; }
        heap_push(e, cnt, HeapEl{R->out_portable, true, R, 0});  // size measured by k_finalize_pairs
    }
    if (!ok) {
        for (uint32_t i = 0; i < cnt; i++) if (e[i].temp) set_delete(e[i].set);
        return nullptr;
    }
    const HeapEl top = heap_pop(e, cnt);
    rb200_set *out = convert_impl(top.set, 2);  // roaring_bitmap_repair_after_lazy
    set_delete(top.set);
    return out;
}

roaring_bitmap_t *roaring_bitmap_or_many_heap(uint32_t number, const roaring_bitmap_t **rs) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    rb200_set *S = rb200_set_upload(rs, number);
    if (!S) return nullptr;
    rb200_set *R = rb200_or_many_heap(S, nullptr, number);
    roaring_bitmap_t *out = R ? rb200_set_download(R, 0) : nullptr;
    set_delete(R);
    set_delete(S);
    return out;
}

}  // extern "C"
