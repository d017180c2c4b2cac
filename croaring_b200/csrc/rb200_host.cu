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
#include <numeric>
#include <string>
#include <type_traits>
#include <vector>

#pragma GCC visibility push(default)
#include "../../include/roaring_b200.h"
#pragma GCC visibility pop
#include "rb200_common.h"
#include "rb200_device.cuh"
#include "rb200_internal.h"
#include "rb200_portable.h"

using namespace rb200;

// ------------------------------------------------------------------ reference-compatible structs
namespace {

struct array_container_t { int32_t cardinality; int32_t capacity; uint16_t *array; };   // array.h:46-50
struct bitset_container_t { int32_t cardinality; uint64_t *words; };                     // bitset.h:45-48
struct rle16_t { uint16_t value, length; };                                              // run.h:48-51
struct run_container_t { int32_t n_runs; int32_t capacity; rle16_t *runs; };            // run.h:69-73
struct shared_container_t { void *container; uint8_t typecode; uint32_t counter; };      // containers.h:71-75

constexpr uint8_t FLAG_COW = 1, FLAG_FROZEN = 2;  // roaring_types.h:46-49
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
    // pair-list uploads (PairBuf): enqueued as soon as the host has built the list, ahead of the
    // library stream's queue, which waits for them through an event instead of holding the copy
    // between two chained launches
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, evk0 = nullptr, evk1 = nullptr;
    OpStats *d_stats = nullptr;
    OpStats *h_stats = nullptr;  // pinned
    // counters of the deferred ops (DeferredCall): zero between ops without a memset on the stream —
    // the op's k_finalize_pairs hands them to the result's pinned block and zeroes them, and every
    // kernel of the next op touches them only after it has waited for its predecessors
    OpStats *d_dstats = nullptr;
    uint32_t *d_flags = nullptr;   // 65536 key flags (xor_many)
    uint16_t *d_keys = nullptr;    // 65536 compacted keys
    uint32_t *d_cardkey = nullptr; // 65536 per-key cardinalities
    // or_many (rb200_many2.cu): per-key tables + split-key scratch (kept zeroed)
    uint32_t *d_m2_tables = nullptr;   // 14 x 65536 u32: key_cu(2) | fill | count | units16 | fill | start | slices | scratch | unit_first | fold_first(2) | fold_second(2) | fold_F | fold_L
    uint32_t *d_m2_scratch = nullptr, *d_m2_tickets = nullptr;
    // single-pair fused path (rb200_fused.cu): packed operands (pinned + device), mapped result block
    uint8_t *h_fused_in = nullptr, *d_fused_in = nullptr, *h_fused_out = nullptr, *d_fused_out = nullptr;
    uint32_t fused_seq = 0;
    std::multimap<size_t, void *> dpool, hpool;
    // device blocks the copy stream writes into: a block comes back here only once nothing queued
    // can still read it (CopyBlock), so a copy into it never has to wait for the library stream
    std::multimap<size_t, void *> cpool;
    std::mutex alloc_mu;  // dpool / hpool are also used by the background downloader thread
    uint64_t dev_in_use = 0;  // bytes of device blocks handed out by dev_alloc and not returned (under alloc_mu)
    uint64_t last_algo_bytes = 0;
    float last_ms = 0.f, last_compute_ms = 0.f;
    uint64_t last_download_bytes = 0;
    uint64_t last_out_portable = 0;  // portable bytes of the last batch's results (all pairs)
    std::vector<cudaEvent_t> evpool, evpool_nt;  // timing / completion-only events recycled between ops (under alloc_mu)
    struct rb200_set *last_op = nullptr;  // result of the most recent batch op (counters may be pending)
} g;
// rb200_last_error() is per calling thread: concurrent callers do not read each other's failures
thread_local std::string t_err;

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
    CK(cudaStreamCreateWithFlags(&g.copy_stream, cudaStreamNonBlocking));
    CK(cudaEventCreate(&g.ev0));
    CK(cudaEventCreate(&g.ev1));
    CK(cudaEventCreate(&g.evk0));
    CK(cudaEventCreate(&g.evk1));
    CK(cudaMalloc(&g.d_stats, sizeof(OpStats)));
    CK(cudaMalloc(&g.d_dstats, sizeof(OpStats)));
    CK(cudaMemset(g.d_dstats, 0, sizeof(OpStats)));
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
    CK(cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, g.device));
    g_halloc.look();  // resolve the host allocator once, before any worker thread exists
    g.inited = true;
    return true;
}

void *dev_alloc(size_t n, std::multimap<size_t, void *> &pool = g.dpool) {
    std::lock_guard<std::mutex> alk(g.alloc_mu);
    if (n == 0) n = 1;
    const size_t b = bucket(n);
    auto it = pool.find(b);
    if (it != pool.end()) {
        void *p = it->second;
        pool.erase(it);
        g.dev_in_use += b;
        return p;
    }
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, b);
    if (e != cudaSuccess) {
        // drop the cache and retry once; the failure is reported through t_err, so it must not stay
        // behind as the runtime's last error for the next launch check to find
        (void)cudaGetLastError();
        for (auto *q : {&g.dpool, &g.cpool}) {
            for (auto &kv : *q) cudaFree(kv.second);
            q->clear();
        }
        e = cudaMalloc(&p, b);
        if (e != cudaSuccess) {
            (void)cudaGetLastError();
            t_err = std::string("cudaMalloc: ") + cudaGetErrorString(e);
            return nullptr;
        }
    }
    g.dev_in_use += b;
    return p;
}
// RB200_POISON_POOL=1 (read when the library loads): every block is zero-filled as it goes back to its
// pool, so a kernel or copy that still reads a released block sees zeros instead of the old bytes, and
// a lifetime bug shows up as wrong results (zeroed counts and offsets keep stale reads inside their
// buffers).  Off by default: no fill, no other change.
const bool g_poison = []() {
    const char *e = getenv("RB200_POISON_POOL");
    const bool on = e && e[0] == '1';
    if (on) fprintf(stderr, "libroaring_b200: pool poisoning on\n");
    return on;
}();

void dev_free(void *p, size_t n, std::multimap<size_t, void *> &pool = g.dpool) {
    if (!p) return;
    if (n == 0) n = 1;
    // ordered after every reader, which was queued before the release: the library stream for the
    // device pool, the copy stream (the next writer of the block) for the copy pool
    if (g_poison && cudaMemsetAsync(p, 0, bucket(n), &pool == &g.cpool ? g.copy_stream : g.stream) != cudaSuccess)
        (void)cudaGetLastError();
    std::lock_guard<std::mutex> alk(g.alloc_mu);
    pool.insert({bucket(n), p});
    g.dev_in_use -= bucket(n);
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
    if (n == 0) n = 1;
    if (g_poison) memset(p, 0, bucket(n));   // pinned blocks come back only when nothing is in flight
    std::lock_guard<std::mutex> alk(g.alloc_mu);
    g.hpool.insert({bucket(n), p});
}

// Owner of one block of the device pool, of the copy stream's device pool or of the pinned pool: it
// keeps the byte size it asked for, so the block goes back under the size class it came from.  A
// device block may be released as soon as the work using it is enqueued (stream-ordered reuse on the
// library stream); a copy-stream block or a pinned block only once nothing that reads or writes it
// can still be in flight.
enum PoolKind { POOL_PINNED, POOL_DEVICE, POOL_COPY };
template <typename T, PoolKind Kind>
class PoolBlock {
   public:
    PoolBlock() = default;
    explicit PoolBlock(size_t count) { reset(count); }
    PoolBlock(PoolBlock &&o) noexcept : p_(o.p_), bytes_(o.bytes_) { o.p_ = nullptr, o.bytes_ = 0; }
    PoolBlock &operator=(PoolBlock &&o) noexcept {
        if (this != &o) {
            reset();
            std::swap(p_, o.p_);
            std::swap(bytes_, o.bytes_);
        }
        return *this;
    }
    ~PoolBlock() { reset(); }
    // A block of `count` elements (at least one byte) in place of the current one; false: out of
    // memory (t_err says so) and the owner is empty.
    bool reset(size_t count) {
        reset();
        const size_t b = count ? sizeof(T) * count : 1;
        p_ = (T *)(Kind == POOL_PINNED ? pin_alloc(b) : dev_alloc(b, Kind == POOL_COPY ? g.cpool : g.dpool));
        bytes_ = p_ ? b : 0;
        return p_ != nullptr;
    }
    void reset() {
        if (p_) Kind == POOL_PINNED ? pin_free(p_, bytes_) : dev_free(p_, bytes_, Kind == POOL_COPY ? g.cpool : g.dpool);
        p_ = nullptr;
        bytes_ = 0;
    }
    T *get() const { return p_; }
    size_t bytes() const { return bytes_; }
    explicit operator bool() const { return p_ != nullptr; }

   private:
    T *p_ = nullptr;
    size_t bytes_ = 0;
};
template <typename T> using DevBlock = PoolBlock<T, POOL_DEVICE>;
template <typename T> using PinBlock = PoolBlock<T, POOL_PINNED>;
template <typename T> using CopyBlock = PoolBlock<T, POOL_COPY>;

std::map<uint8_t *, PinBlock<uint8_t>> g_serialized;  // pinned blobs handed out, until rb200_serialized_free

// What a serialization hands out: off (n + 1 entries) and len (optional) from malloc, and the
// pinned blob.  They belong to this object until hand_out(), so a failed call leaves nothing behind.
struct HostArrays {
    uint64_t *off = nullptr, *len = nullptr;
    PinBlock<uint8_t> blob;
    HostArrays() = default;
    HostArrays(const HostArrays &) = delete;
    ~HostArrays() {
        free(off);
        free(len);
    }
    bool alloc(size_t n, bool with_len) {
        off = (uint64_t *)malloc(8 * (n + 1));
        if (with_len) len = (uint64_t *)malloc(8 * (n + 1));
        if (!off || (with_len && !len)) return false;
        off[0] = 0;
        return true;
    }
    // Everything to the caller (*buf = NULL without a blob); the blob is released by
    // rb200_serialized_free.  Returns 0, the status of a successful call.
    template <typename T>
    int hand_out(T **buf, uint64_t **off_out, uint64_t **len_out) {
        uint8_t *p = blob.get();
        if (p) g_serialized.emplace(p, std::move(blob));
        *buf = (T *)p;
        *off_out = off;
        off = nullptr;
        if (len_out) *len_out = len;
        len = nullptr;
        return 0;
    }
};

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

// A set's payload slab.  Held by the set and by every batch result whose pass-through containers
// point into it (rb200_set::held): it goes back to the pool when the last holder is freed.
// Reuse is stream-ordered like every pool block: whatever read it was queued before the release.
struct Slab {
    DevBlock<uint8_t> block;
    uint8_t *p;
    size_t cap;
    explicit Slab(size_t cap_) : block(cap_), p(block.get()), cap(cap_) {}
};

// Owning handles of sets: a temporary set goes back when its handle leaves scope, and release()
// hands a set to the caller.
struct SetFree { void operator()(rb200_set *s) const; };
struct Set64Free { void operator()(rb200_set64 *s) const; };
using SetPtr = std::unique_ptr<rb200_set, SetFree>;
using Set64Ptr = std::unique_ptr<rb200_set64, Set64Free>;

}  // namespace

struct rb200_set {
    uint32_t n_bitmaps = 0;
    uint64_t dir_cap = 0;      // directory entries allocated
    uint64_t n_containers = 0; // directory entries in use
    uint64_t slab_cap = 0, slab_used = 0;
    // sum of container_size_in_bytes: set by the uploads and builders that know it (portable_known),
    // otherwise computed from the directory on first request (payload_bytes_of)
    uint64_t portable_bytes = 0;
    bool portable_known = false;
    DirLayout L;
    DevBlock<uint8_t> d_dir;    // one block
    uint8_t *d_slab = nullptr;  // own payload slab (owned through `slab`)
    uint8_t *d_base = nullptr;  // payload base of the view: d_slab, or below it for a batch result that shares
    std::shared_ptr<Slab> slab;
    // the slabs of the operands (A, B) this batch result shares pass-through containers with; c_off
    // is relative to d_base, the lowest of d_slab and the operands' bases.  An operand that shares
    // itself is copied from instead, so holds never chain: a result keeps at most its two operands'
    // own slabs alive, and a fold that frees its previous accumulator runs in bounded memory.
    std::shared_ptr<Slab> held[2];
    bool sharing() const { return held[0] || held[1]; }
    std::vector<uint32_t> h_cnt;    // host mirror: containers per bitmap
    std::vector<uint64_t> h_card;   // host mirror: cardinality per bitmap (empty = not cached)
    bool mirrors_pending = false;   // batch results: h_cnt / h_bytes / h_card are fetched on first use
    bool lazy = false;              // produced by a lazy op: needs rb200_set_repair_after_lazy
    // Deferred counters of the batch op that produced this set: the op returns as soon as its
    // kernels and the D2H copy of its counters are queued; resolve() waits for them on first use,
    // so consecutive batch calls pipeline on the stream without a host round trip.
    bool pending = false, failed = false;
    PinBlock<OpStats> pstats;
    PinBlock<uint8_t> staging;                  // pair list of the op (alive until it ran)
    CopyBlock<uint8_t> staging_dev;             // its device copy (alive until the op ran)
    cudaEvent_t done = nullptr;                 // the op's end (completion only: its times are in pstats)
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
    // host copy of the directory (pinned) and, for a set packed for download, of its payload
    PinBlock<uint8_t> m_dir, m_slab;
    SetPtr mirror;                  // rb200_set_download: this set packed, directory and payload on the host
    // exclusive scan of the directory's cardinalities (n_containers + 1 entries), built by the first
    // rank / get_index / select query (ensure_cum); a set never changes after the op that made it
    DevBlock<uint64_t> c_cum;

    SetView view() const {
        const uint8_t *d = d_dir.get();
        SetView v;
        v.bm_beg = (const uint32_t *)(d + L.o_beg);
        v.bm_cnt = (const uint32_t *)(d + L.o_cnt);
        v.c_key = (const uint16_t *)(d + L.o_key);
        v.c_type = (const uint8_t *)(d + L.o_type);
        v.c_card = (const uint32_t *)(d + L.o_card);
        v.c_len = (const uint32_t *)(d + L.o_len);
        v.c_off = (const uint64_t *)(d + L.o_off);
        v.c_src = (const uint32_t *)(d + L.o_src);
        v.payload = d_base;
        return v;
    }
    SetOut out() {
        uint8_t *d = d_dir.get();
        SetOut v;
        v.bm_beg = (uint32_t *)(d + L.o_beg);
        v.bm_cnt = (uint32_t *)(d + L.o_cnt);
        v.bm_card = (uint64_t *)(d + L.o_bcard);
        v.bm_bytes = (uint64_t *)(d + L.o_bbytes);
        v.bm_ebytes = (uint64_t *)(d + L.o_bebytes);
        v.c_key = (uint16_t *)(d + L.o_key);
        v.c_type = (uint8_t *)(d + L.o_type);
        v.c_card = (uint32_t *)(d + L.o_card);
        v.c_len = (uint32_t *)(d + L.o_len);
        v.c_off = (uint64_t *)(d + L.o_off);
        v.c_src = (uint32_t *)(d + L.o_src);
        v.payload = d_slab;
        return v;
    }
};

namespace {

// mirrors = false: h_cnt / h_bytes / h_ebytes stay empty, for a batch result whose first
// ensure_mirrors() fills them from the device (a result that is only measured, chained on the device or
// downloaded never needs them)
SetPtr set_new(uint32_t nb, uint64_t dir_cap, uint64_t slab_cap, bool mirrors = true) {
    SetPtr s(new rb200_set());
    s->n_bitmaps = nb;
    s->dir_cap = dir_cap;
    s->slab_cap = slab_cap;
    s->L.compute(nb, dir_cap);
    if (!s->d_dir.reset(s->L.total)) return nullptr;
    s->slab = std::make_shared<Slab>(slab_cap);
    if (!s->slab->p) return nullptr;
    s->d_slab = s->d_base = s->slab->p;
    if (mirrors) {
        s->h_cnt.assign(nb, 0);
        s->h_bytes.assign(nb, 0);
        s->h_ebytes.assign(nb, 0);
    }
    s->h_flags.assign(nb, 0);
    return s;
}

// timing = false: an event that only marks completion (cudaEventDisableTiming).  Recorded between two
// programmatic launches it keeps them chained; a timing event makes the second wait for the first.
cudaEvent_t ev_get(bool timing = true) {
    std::vector<cudaEvent_t> &pool = timing ? g.evpool : g.evpool_nt;
    {
        std::lock_guard<std::mutex> alk(g.alloc_mu);
        if (!pool.empty()) {
            cudaEvent_t e = pool.back();
            pool.pop_back();
            return e;
        }
    }
    cudaEvent_t e = nullptr;
    cudaEventCreateWithFlags(&e, timing ? cudaEventDefault : cudaEventDisableTiming);
    return e;
}
void ev_put(cudaEvent_t e, bool timing = true) {
    if (!e) return;
    std::lock_guard<std::mutex> alk(g.alloc_mu);
    (timing ? g.evpool : g.evpool_nt).push_back(e);
}

// Host bytes -> one device buffer as a stream through two pinned chunks on the library stream: the
// copy of one chunk overlaps the memcpy into the other.  put() appends (src == nullptr: zeros),
// flush() sends the rest.  The chunks go back to the pool when the stager is destroyed, so it must
// outlive a synchronisation of the stream after the last flush.
struct H2DStager {
    static constexpr size_t CH = (size_t)32 << 20;
    uint8_t *dst;
    PinBlock<uint8_t> chunk[2];
    cudaEvent_t cev[2] = {nullptr, nullptr};
    bool cev_used[2] = {false, false};
    bool ok;
    int cur = 0;
    size_t used = 0;
    uint64_t base = 0;
    explicit H2DStager(uint8_t *d) : dst(d), chunk{PinBlock<uint8_t>(CH), PinBlock<uint8_t>(CH)} {
        ok = chunk[0] && chunk[1];
        for (int k = 0; k < 2 && ok; k++) ok = cudaEventCreateWithFlags(&cev[k], cudaEventDisableTiming) == cudaSuccess;
    }
    ~H2DStager() {
        for (int k = 0; k < 2; k++) if (cev[k]) cudaEventDestroy(cev[k]);
    }
    bool flush() {
        if (used) {
            if (cudaMemcpyAsync(dst + base, chunk[cur].get(), used, cudaMemcpyHostToDevice, g.stream) != cudaSuccess)
                return false;
            cudaEventRecord(cev[cur], g.stream);
            cev_used[cur] = true;
        }
        base += used;
        used = 0;
        cur ^= 1;
        if (cev_used[cur]) cudaEventSynchronize(cev[cur]);
        return true;
    }
    bool put(const void *src, size_t n) {
        const uint8_t *p = (const uint8_t *)src;
        while (n) {
            if (used == CH && !flush()) return false;
            const size_t take = std::min(CH - used, n);
            if (p) {
                memcpy(chunk[cur].get() + used, p, take);
                p += take;
            } else {
                memset(chunk[cur].get() + used, 0, take);
            }
            used += take;
            n -= take;
        }
        return true;
    }
};

// The ending of a call that waits for its device work before it returns.  begin() records the op's
// start event (a timed call) and resets the stats; kernels_begin() / kernels_end() / end() mark the
// timed brackets; finish(ok) fetches the stats, waits for the stream and checks for a launch error,
// and a timed call then becomes what the rb200_last_* getters describe.  A call that returns before
// finish() still waits for the stream, here in the destructor: declared after the pinned blocks the
// stream may still be copying, the helper is destroyed, and the stream drained, before they go back
// to the pool.  `what` / `launch_what` head t_err for a failed wait / launch (no message if null).
class SyncCall {
   public:
    explicit SyncCall(const char *what = nullptr, const char *launch_what = nullptr, bool timed = false)
        : what_(what), launch_what_(launch_what ? launch_what : what), timed_(timed) {}
    SyncCall(const SyncCall &) = delete;
    ~SyncCall() { if (!finished_) cudaStreamSynchronize(g.stream); }
    bool begin() {
        if (timed_) cudaEventRecord(g.ev0, g.stream);
        return stats_reset();
    }
    void kernels_begin() { cudaEventRecord(g.evk0, g.stream); }
    void kernels_end() { cudaEventRecord(g.evk1, g.stream); }
    void end() { cudaEventRecord(g.ev1, g.stream); }
    bool finish(bool ok, bool fetch_stats = true) {
        finished_ = true;
        if (fetch_stats) ok = ok && stats_fetch();
        cudaError_t e = cudaStreamSynchronize(g.stream);
        const bool waited = e == cudaSuccess;
        if (waited) e = cudaGetLastError();
        if (e != cudaSuccess) {
            if (what_ && (!waited || ok)) t_err = std::string(waited ? launch_what_ : what_) + ": " + cudaGetErrorString(e);
            ok = false;
        }
        if (ok && timed_) {
            g.last_op = nullptr;  // the rb200_last_* getters now describe this (synchronous) op
            cudaEventElapsedTime(&g.last_ms, g.ev0, g.ev1);
            cudaEventElapsedTime(&g.last_compute_ms, g.evk0, g.evk1);
        }
        return ok;
    }

   private:
    const char *what_, *launch_what_;
    bool timed_, finished_ = false;
};

// The ending of a batch op that returns as soon as its work is queued: its counters are taken over
// by resolve() on first use, so consecutive ops pipeline on the stream without a host round trip.
// begin() gives the result R an event and pinned counters (zero until the op's k_finalize_pairs
// writes them through deliver()); the op's kernels count and time themselves in g.d_dstats (see
// OpStats::t_begin); finish(ok) records the op's end and hands R over, pending, with the staging
// block its kernels or copies read.  No memset, copy or timing event sits between the op's kernels
// and those of the ops before and after it, so their launches stay chained (launch_kernel_chained).
// A failed call returns NULL (R is freed by its owner) after waiting for the stream and zeroing the
// counters it may have left behind.  `what` heads the default t_err.
class DeferredCall {
   public:
    // staging_dev: a device block the copy stream filled for the op's kernels, held like staging
    DeferredCall(const char *what, SetPtr &R, PinBlock<uint8_t> &staging, CopyBlock<uint8_t> *staging_dev = nullptr)
        : what_(what), R_(R), staging_(staging), staging_dev_(staging_dev) {}
    DeferredCall(const DeferredCall &) = delete;
    bool begin() {
        R_->done = ev_get(false);
        if (!R_->pstats.reset(1) || !R_->done) return false;
        memset(R_->pstats.get(), 0, sizeof(OpStats));
        return cudaHostGetDevicePointer((void **)&deliver_, R_->pstats.get(), 0) == cudaSuccess;
    }
    OpStats *deliver() const { return deliver_; }
    rb200_set *finish(bool ok) {
        if (ok) ok = cudaEventRecord(R_->done, g.stream) == cudaSuccess;
        if (!ok) {
            if (t_err.empty()) t_err = std::string(what_) + ": enqueue failed";
            // a chain cut short leaves its counters in g.d_dstats: zero them for the next op
            if (deliver_) cudaMemsetAsync(g.d_dstats, 0, sizeof(OpStats), g.stream);
            if (staging_ || deliver_) cudaStreamSynchronize(g.stream);
            return nullptr;
        }
        R_->pending = true;
        R_->staging = std::move(staging_);
        if (staging_dev_) R_->staging_dev = std::move(*staging_dev_);
        R_->mirrors_pending = R_->n_bitmaps > 0;  // h_cnt / h_bytes / h_card: see ensure_mirrors()
        g.last_op = R_.get();
        return R_.release();
    }

   private:
    const char *what_;
    SetPtr &R_;
    PinBlock<uint8_t> &staging_;
    CopyBlock<uint8_t> *staging_dev_;
    OpStats *deliver_ = nullptr;   // R's pinned counters, device address
};

// The batch op that produced s has run (or was never enqueued): its events, counters and pair list
// go back to the pools.
void retire_op(rb200_set *s) {
    ev_put(s->done, false);
    s->done = nullptr;
    s->pstats.reset();
    s->staging.reset();
    s->staging_dev.reset();
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
    const OpStats &st = *s->pstats.get();
    cudaError_t e = cudaEventSynchronize(s->done);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) {
        t_err = std::string("batch op: ") + cudaGetErrorString(e);
        s->failed = true;
    } else if (st.error) {
        t_err = st.error == 2 ? "internal: result slab bound exceeded" : "internal: result slot bound exceeded";
        s->failed = true;
    } else {
        s->ms = st.t_end > st.t_begin ? (float)((st.t_end - st.t_begin) * 1e-6) : 0.f;
        s->compute_ms = st.t_cells1 > st.t_cells0 ? (float)((st.t_cells1 - st.t_cells0) * 1e-6) : 0.f;
        s->algo_bytes = st.algo_bytes;
        s->out_portable = st.out_portable;
        s->n_containers = st.dir_cursor;
        s->slab_used = st.slab_cursor;
        for (int k = 0; k < 2; k++)   // an operand none of whose containers was shared is not held
            if (!st.shared_used[k]) s->held[k].reset();
        if (s->n_bitmaps == 1 && !s->sharing()) {  // a single result: its mirrors are the op's counters, no extra D2H
            s->h_cnt.assign(1, (uint32_t)s->n_containers);
            s->h_bytes.assign(1, s->slab_used);
            s->h_ebytes.assign(1, std::max<uint64_t>(s->slab_used, s->n_containers * (uint64_t)BITSET_BYTES));
            s->mirrors_pending = false;
        }
    }
    retire_op(s);
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
    retire_op(s);                // (only needed if the enqueue failed half way)
    if (g.last_op == s) g.last_op = nullptr;
    delete s;  // the slabs return to the pool unless a result still points into them
}
void SetFree::operator()(rb200_set *s) const { set_delete(s); }

// container_size_in_bytes summed over the set's containers, waiting for the op that produced it.  A set
// made by an op is summed from its directory (types and lengths, one D2H) on the first request and
// keeps the sum: a set never changes after the op that made it.  0 with t_err set if the set failed.
uint64_t payload_bytes_of(const rb200_set *cs) {
    rb200_set *s = const_cast<rb200_set *>(cs);
    if (!resolve(s)) return 0;
    if (s->portable_known) return s->portable_bytes;
    const size_t nc = s->n_containers;
    PinBlock<uint8_t> h(5 * nc);
    const bool ok = h && (nc == 0 ||
                          (cudaMemcpyAsync(h.get(), s->d_dir.get() + s->L.o_type, nc, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
                           cudaMemcpyAsync(h.get() + nc, s->d_dir.get() + s->L.o_len, 4 * nc, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
                           cudaStreamSynchronize(g.stream) == cudaSuccess));
    if (!ok) {
        t_err = "fetching the set's directory failed";
        return 0;
    }
    const uint8_t *type = h.get();
    uint64_t sum = 0;
    for (size_t c = 0; c < nc; c++) {
        uint32_t len;
        memcpy(&len, h.get() + nc + 4 * c, 4);
        sum += portable_bytes(type[c], len);
    }
    s->portable_bytes = sum;
    s->portable_known = true;
    return sum;
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

// Container i of a host bitmap, SHARED unwrapped (*was_shared tells whether it was), payload in the
// slab's layout.  A lazy bitset (cardinality field negative, bitset.h:42) has CARD_UNKNOWN set.
inline PortableEntry entry_of(const roaring_array_t *ra, int32_t i, bool *was_shared = nullptr) {
    uint8_t t = ra->typecodes[i];
    if (was_shared) *was_shared = t == T_SHARED;
    const void *c = unwrap_shared(ra->containers[i], t);
    PortableEntry e;
    e.key = ra->keys[i];
    e.type = t;
    e.card = host_container_card(c, t);
    if (t == T_BITSET) {
        e.len = 1024;
        e.payload = (const uint8_t *)((const bitset_container_t *)c)->words;
        if (((const bitset_container_t *)c)->cardinality < 0) e.card |= CARD_UNKNOWN;
    } else if (t == T_ARRAY) {
        e.len = e.card;
        e.payload = (const uint8_t *)((const array_container_t *)c)->array;
    } else {
        e.len = (uint32_t)((const run_container_t *)c)->n_runs;
        e.payload = (const uint8_t *)((const run_container_t *)c)->runs;
    }
    return e;
}

}  // namespace

// =================================================================== C ABI: helpers
extern "C" {

const char *rb200_last_error(void) { return t_err.c_str(); }
uint64_t rb200_kernel_launches(void) { return g_launches; }
uint64_t rb200_device_bytes_in_use(void) {
    std::lock_guard<std::mutex> alk(g.alloc_mu);
    return g.dev_in_use;
}
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
    for (int32_t i = 0; i < ra->size; i++) s += entry_of(ra, i).card & CARD_MASK;
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
    return portable_size((uint32_t)ra->size, [ra](uint32_t i) { return entry_of(ra, (int32_t)i); });
}

size_t rb200_bitmap_portable_serialize(const roaring_bitmap_t *r, char *buf) {
    const roaring_array_t *ra = &r->high_low_container;
    return write_portable((uint8_t *)buf, (uint32_t)ra->size, [ra](uint32_t i) { return entry_of(ra, (int32_t)i); });
}

roaring_bitmap_t *rb200_bitmap_portable_deserialize_safe(const char *buf, size_t maxbytes) {
    std::vector<PortableEntry> c;
    if (!walk_portable((const uint8_t *)buf, maxbytes, [&c](const PortableEntry &e) { c.push_back(e); })) return nullptr;
    roaring_bitmap_t *r = bitmap_alloc((int32_t)c.size());
    if (!r) return nullptr;
    roaring_array_t *ra = &r->high_low_container;
    for (const PortableEntry &e : c) {
        void *hc = container_from_payload(e.type, e.card, e.len, e.payload);
        if (!hc) {
            bitmap_free_host(r);
            return nullptr;
        }
        ra->containers[ra->size] = hc;
        ra->keys[ra->size] = e.key;
        ra->typecodes[ra->size] = e.type;
        ra->size++;
    }
    return r;
}

}  // extern "C"

// =================================================================== upload
namespace {

rb200_set *upload_impl(const roaring_bitmap_t *const *bms, size_t nb) {
    if (!ctx_init()) return nullptr;
    // pass 1: sizes
    uint64_t nc = 0, slab = 0;
    for (size_t b = 0; b < nb; b++) {
        const roaring_array_t *ra = &bms[b]->high_low_container;
        nc += (uint64_t)ra->size;
        for (int32_t i = 0; i < ra->size; i++) {
            uint8_t t = ra->typecodes[i];
            const void *c = unwrap_shared(ra->containers[i], t);
            uint32_t len = t == T_BITSET ? 1024u
                           : t == T_ARRAY ? (uint32_t)((const array_container_t *)c)->cardinality
                                          : (uint32_t)((const run_container_t *)c)->n_runs;
            slab += round16(stored_bytes(t, len));
        }
    }
    SetPtr s = set_new((uint32_t)nb, nc, slab);
    if (!s) return nullptr;
    s->n_containers = nc;
    s->slab_used = slab;
    // pass 2: directory into one pinned block, payload streamed through two pinned chunks
    PinBlock<uint8_t> dir(s->L.total);
    H2DStager stage(s->d_slab);
    bool ok = dir && stage.ok;
    if (ok) {
        uint8_t *hd = dir.get();
        uint32_t *bm_beg = (uint32_t *)(hd + s->L.o_beg), *bm_cnt = (uint32_t *)(hd + s->L.o_cnt);
        uint64_t *bm_card = (uint64_t *)(hd + s->L.o_bcard);
        uint16_t *c_key = (uint16_t *)(hd + s->L.o_key);
        uint8_t *c_type = hd + s->L.o_type;
        uint32_t *c_card = (uint32_t *)(hd + s->L.o_card), *c_len = (uint32_t *)(hd + s->L.o_len);
        uint64_t *c_off = (uint64_t *)(hd + s->L.o_off);
        uint32_t *c_src = (uint32_t *)(hd + s->L.o_src);
        s->h_ptr_all = std::make_shared<std::vector<const void *>>(nc);
        uint64_t ci = 0, off = 0;
        for (size_t b = 0; b < nb && ok; b++) {
            const roaring_array_t *ra = &bms[b]->high_low_container;
            bm_beg[b] = (uint32_t)ci;
            bm_cnt[b] = (uint32_t)ra->size;
            s->h_cnt[b] = (uint32_t)ra->size;
            s->h_flags[b] = ra->flags & FLAG_COW;
            uint64_t bcard = 0, bbytes = 0, bebytes = 0;
            for (int32_t i = 0; i < ra->size; i++, ci++) {
                bool was_shared;
                const PortableEntry e = entry_of(ra, i, &was_shared);
                if (e.card & CARD_UNKNOWN) s->lazy = true;
                if (e.type == T_RUN && 4 * (uint64_t)e.len > BITSET_BYTES) s->lazy = true;  // only lazy unions leave such runs
                const uint32_t sb = stored_bytes(e.type, e.len), sb16 = round16(sb);
                ok = ok && stage.put(e.payload, sb) && stage.put(nullptr, sb16 - sb);
                c_key[ci] = e.key;
                c_type[ci] = e.type;
                c_card[ci] = e.card;
                c_len[ci] = e.len;
                c_off[ci] = off;
                c_src[ci] = was_shared ? SRC_SHARED : SRC_NONE;
                (*s->h_ptr_all)[ci] = e.payload;
                off += sb16;
                bcard += e.card & CARD_MASK;
                bbytes += sb16;
                bebytes += effective_bytes(e.type, e.len, e.card & CARD_MASK);
                s->portable_bytes += portable_bytes(e.type, e.len);
            }
            bm_card[b] = bcard;
            s->h_bytes[b] = bbytes;
            s->h_ebytes[b] = bebytes;
        }
        s->portable_known = true;
        ok = ok && stage.flush() &&
             cudaMemcpyAsync(s->d_dir.get(), hd, s->L.total, cudaMemcpyHostToDevice, g.stream) == cudaSuccess;
        if (cudaStreamSynchronize(g.stream) != cudaSuccess) ok = false;
    }
    if (!ok) {
        if (t_err.empty()) t_err = "upload failed";
        return nullptr;
    }
    return s.release();
}

}  // namespace

extern "C" {

rb200_set_t *rb200_set_upload(const roaring_bitmap_t *const *bitmaps, size_t n) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return upload_impl(bitmaps, n);
}

// Portable-serialized inputs are parsed ON THE DEVICE (src/roaring_array.c:633-813 restated as
// k_deser_dir / k_deser_copy): the host only reads each blob's cookie (to size the directory) and
// streams the raw bytes through pinned staging chunks; no per-container host work.
static rb200_set *upload_blobs_impl(const char *const *bufs, const size_t *lens, size_t n, bool frozen,
                                    size_t *bad_blob = nullptr);
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
// A malformed blob is named in t_err and, when bad_blob is given, its index is stored there.
static rb200_set *upload_blobs_impl(const char *const *bufs, const size_t *lens, size_t n, bool frozen,
                                    size_t *bad_blob) {
    const char *what = frozen ? "malformed frozen bitmap at index " : "malformed portable bitmap at index ";
    if (!ctx_init()) return nullptr;
    if (n > 0xffffffffull) { t_err = "too many bitmaps"; return nullptr; }
    // pass 1 (host): container count of every blob from its cookie; staging offsets
    uint64_t nc = 0, raw_total = 0, slab_total = 0, payload = 0;
    std::vector<uint32_t> cnt(n);
    for (size_t i = 0; i < n; i++) {
        uint32_t size = 0;
        bool hasrun = false, ok;
        if (frozen) {
            uint32_t cookie = 0;
            ok = lens[i] >= 4;
            if (ok) memcpy(&cookie, bufs[i] + lens[i] - 4, 4);   // the header is the LAST word
            size = cookie >> 15;
            ok = ok && (cookie & 0x7FFF) == FROZEN_COOKIE && 5ull * size + 4 <= lens[i] && size <= 65536;
        } else {
            ok = portable_count((const uint8_t *)bufs[i], lens[i], size, hasrun);
        }
        if (!ok) {
            t_err = what + std::to_string(i);
            if (bad_blob) *bad_blob = i;
            return nullptr;
        }
        cnt[i] = size;
        nc += size;
        raw_total += (lens[i] + 15) & ~(uint64_t)15;
        slab_total += ((lens[i] + 15) & ~(uint64_t)15) + 16ull * size;   // payload <= blob bytes, + 16-byte padding per container
        const uint64_t hdr = frozen ? 4 + 5ull * size : portable_header_bytes(size, hasrun);
        payload += lens[i] > hdr ? lens[i] - hdr : 0;
    }
    SetPtr s = set_new((uint32_t)n, nc, slab_total + 16);
    if (!s) return nullptr;
    s->n_containers = nc;
    s->slab_used = slab_total;
    // a portable blob's payload is its containers' container_size_in_bytes; a frozen blob stores run
    // containers without their 2-byte run count, so its sum is taken from the directory when asked
    s->portable_bytes = payload;
    s->portable_known = !frozen;
    // per-bitmap tables: [roff | rlen | slab_base] for the kernels, bm_beg / bm_cnt into the directory
    PinBlock<uint64_t> tab(3 * n);
    PinBlock<uint32_t> bc(2 * n);
    DevBlock<uint64_t> d_tab(3 * n), d_src(nc);
    DevBlock<uint8_t> d_raw(raw_total);
    H2DStager stage(d_raw.get());
    SyncCall call("deserialize");
    bool ok = tab && d_tab && bc && d_raw && d_src && stage.ok;
    if (ok) {
        uint64_t *h_tab = tab.get();
        uint32_t *h_bc = bc.get();
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
            ro += (lens[i] + 15) & ~(uint64_t)15;
            so += ((lens[i] + 15) & ~(uint64_t)15) + 16ull * cnt[i];
            cb += cnt[i];
        }
        ok = cudaMemcpyAsync(d_tab.get(), h_tab, d_tab.bytes(), cudaMemcpyHostToDevice, g.stream) == cudaSuccess &&
             (n == 0 ||
              (cudaMemcpyAsync(s->d_dir.get() + s->L.o_beg, h_bc, 4 * n, cudaMemcpyHostToDevice, g.stream) == cudaSuccess &&
               cudaMemcpyAsync(s->d_dir.get() + s->L.o_cnt, h_bc + n, 4 * n, cudaMemcpyHostToDevice, g.stream) == cudaSuccess));
        // raw bytes as one stream through the two pinned chunks
        for (size_t i = 0; i < n && ok; i++)
            ok = stage.put(bufs[i], lens[i]) && stage.put(nullptr, ((lens[i] + 15) & ~(size_t)15) - lens[i]);
        if (ok) ok = stage.flush();
    }
    if (ok) {
        ok = call.begin();
        const uint64_t *t = d_tab.get();
        if (frozen)
            launch_deserialize_frozen(d_raw.get(), t, t + n, t + 2 * n, (uint32_t)n, nc, s->out(), d_src.get(),
                                      g.d_stats, g.stream);
        else
            launch_deserialize(d_raw.get(), t, t + n, t + 2 * n, (uint32_t)n, nc, s->out(), d_src.get(), g.d_stats,
                               g.stream);
        ok = call.finish(ok);
        if (ok && g.h_stats->error) {   // 3: structure (k_deser_dir / k_frozen_parse_dir), 4: contents (k_deser_copy)
            const size_t bad = (size_t)n - g.h_stats->nk;
            t_err = what + std::to_string(bad);
            if (g.h_stats->error == 4u)
                t_err += ": invalid container contents (the reference's validator refuses them: runs that are "
                         "empty, end past 65535, overlap, touch or are out of order; an array above 4096 values "
                         "or not strictly increasing; a bitset whose cardinality is not its popcount or is 4096 "
                         "or less)";
            if (bad_blob) *bad_blob = bad;
            ok = false;
        }
    }
    if (!ok) {
        if (t_err.empty()) t_err = "upload_serialized failed";
        return nullptr;
    }
    s->mirrors_pending = n > 0;   // exact per-bitmap bytes / effective bytes: k_deser_bitmap_cards wrote them
    return s.release();
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
uint64_t rb200_set_payload_bytes(const rb200_set_t *s) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return payload_bytes_of(s);
}

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
    PinBlock<uint8_t> hb(bytes);
    if (!hb) return false;
    const uint8_t *h = hb.get();
    const bool ok = cudaMemcpyAsync(hb.get(), s->d_dir.get() + s->L.o_cnt, bytes, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
                    cudaStreamSynchronize(g.stream) == cudaSuccess;
    if (ok) {
        const uint32_t *cnt = (const uint32_t *)h;
        const uint64_t *card = (const uint64_t *)(h + (s->L.o_bcard - s->L.o_cnt));
        const uint64_t *bb = (const uint64_t *)(h + (s->L.o_bbytes - s->L.o_cnt));
        const uint64_t *be = (const uint64_t *)(h + (s->L.o_bebytes - s->L.o_cnt));
        s->h_card.assign(card, card + nb);
        s->h_cnt.assign(cnt, cnt + nb);
        s->h_bytes.assign(bb, bb + nb);    // exact stored bytes (16-byte rounded slots) of each bitmap
        s->h_ebytes.assign(be, be + nb);   // what a later op on it can produce at most (see PairBuf::build)
        s->mirrors_pending = false;
    } else {
        t_err = "fetching result directory failed";
    }
    return ok;
}

struct ItemsBuf {
    DevBlock<uint8_t> mem;
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
        if (!mem.reset(o ? o : 256)) return false;
        uint8_t *block = mem.get();
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
};

#ifdef RB200_HOST_TIMING
// Host time of every batch_op_impl call, split by phase (tools/time_host_call.py reads it through
// rb200_host_timing_take).  Only the timing variant of the library carries it.
enum { HT_CHECKS, HT_STAGING, HT_PAIRS, HT_COPY, HT_ITEMS, HT_SET_NEW, HT_BEGIN, HT_LAUNCH, HT_FINISH, HT_N };
struct HostTiming {
    double last = 0, entry = 0, copied = 0, ph[HT_N] = {};
    std::vector<double> rec;   // per call: entry, copy enqueued (CLOCK_MONOTONIC s), HT_N phase durations (s)
};
HostTiming g_ht;
double ht_now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
void ht_mark(int k) {
    const double t = ht_now();
    g_ht.ph[k] += t - g_ht.last;
    g_ht.last = t;
    if (k == HT_COPY) g_ht.copied = t;
}
void ht_enter() {
    g_ht = HostTiming{0, 0, 0, {}, std::move(g_ht.rec)};
    g_ht.entry = g_ht.last = ht_now();
}
void ht_leave() {
    ht_mark(HT_FINISH);
    g_ht.rec.push_back(g_ht.entry);
    g_ht.rec.push_back(g_ht.copied);
    g_ht.rec.insert(g_ht.rec.end(), g_ht.ph, g_ht.ph + HT_N);
}
#define HT_MARK(k) ht_mark(k)
#else
#define HT_MARK(k) ((void)0)
#endif

// pair lists + item offsets: one pinned staging block, one H2D copy on the copy stream, which the
// library stream waits for.  The copy starts as soon as the list is built instead of behind the
// kernels already queued, and no copy sits between two chained launches.  The device block comes
// from the copy stream's pool and stays with the caller (a batch result: until its op has run), so
// the copy never overwrites what a queued kernel still reads.
// (tried: k_plan_pairs reading the staging block through its mapped address instead, which keeps the
//  copy off the stream — its scattered 4- and 8-byte reads over PCIe made the kernel 2-3x slower)
struct PairBuf {
    PinBlock<uint8_t> h;
    CopyBlock<uint8_t> d;
    uint32_t *d_ia = nullptr, *d_ib = nullptr;
    uint64_t *d_off = nullptr;
    uint64_t W = 0;
    // result slab bound for the sharing mode `share` of build() (bit 0: A's pass-through containers
    // shared, bit 1: B's), and the bound when everything is copied
    uint64_t slab_bound = 0, slab_bound_copy = 0;
    bool cow = false;   // some selected bitmap of A or B carries the COW flag
    // op: OP_* of the batch (OP_AND also for the cardinality-only sweeps, which need no slab)
    // rules: RULES_* of the batch; with RULES_FLIP, B is the range bitmap of rb200_batch_flip (every
    // container ONE run)
    bool build(const rb200_set *A, const rb200_set *B, const uint32_t *ia, const uint32_t *ib,
               size_t np, int op, int rules = 0, int share = 0) {
        if (!ensure_mirrors(A) || !ensure_mirrors(B)) return false;
        if (np > 0xffffffffull) { t_err = "too many pairs in one batch (2^32 - 1 at most)"; return false; }
        const size_t o_off = 0, o_ia = al256(8 * (np + 1)), o_ib = o_ia + al256(4 * np);
        const size_t bytes = o_ib + al256(4 * np);
        HT_MARK(HT_CHECKS);
        if (!h.reset(bytes) || !d.reset(bytes)) return false;
        HT_MARK(HT_STAGING);
        Lists L{(uint64_t *)(h.get() + o_off), (uint32_t *)(h.get() + o_ia), (uint32_t *)(h.get() + o_ib)};
        const Side a = side(A), b = side(B);
        const bool andnot = op == OP_ANDNOT;
        bool ok;
        if (rules & RULES_FLIP) ok = pairs<Bound::Flip>(a, b, ia, ib, np, andnot, share, L);
        else if (rules & RULES_LAZY) ok = pairs<Bound::Lazy>(a, b, ia, ib, np, andnot, share, L);
        else if (op == OP_AND) ok = pairs<Bound::And>(a, b, ia, ib, np, andnot, share, L);
        else if (rules & RULES_KEEP_RUN) ok = pairs<Bound::KeepRun>(a, b, ia, ib, np, andnot, share, L);
        else ok = pairs<Bound::Plain>(a, b, ia, ib, np, andnot, share, L);
        if (!ok) return false;
        // item ids, directory positions of the result and the order list are 32-bit on the device
        if (W > 0xffffffffull) { t_err = "batch too large: more than 2^32 - 1 container slots, split the pair list"; return false; }
        if (!share) slab_bound = slab_bound_copy;
        d_off = (uint64_t *)(d.get() + o_off);
        d_ia = (uint32_t *)(d.get() + o_ia);
        d_ib = (uint32_t *)(d.get() + o_ib);
        HT_MARK(HT_PAIRS);
        ok = cudaMemcpyAsync(d.get(), h.get(), bytes, cudaMemcpyHostToDevice, g.copy_stream) == cudaSuccess;
        if (ok) {
            // completion only: the wait binds to this record, so the event can go back to the pool at once
            cudaEvent_t ev = ev_get(false);
            ok = ev && cudaEventRecord(ev, g.copy_stream) == cudaSuccess && cudaStreamWaitEvent(g.stream, ev, 0) == cudaSuccess;
            ev_put(ev, false);
            if (!ok) {
                cudaStreamSynchronize(g.copy_stream);   // h and d are released with nothing in flight
                t_err = "pair list upload failed";
            }
        }
        HT_MARK(HT_COPY);
        return ok;
    }

   private:
    // The slab bound rule of a batch (see pairs()): each has its own instance of the pair loop, so the
    // loop branches on neither the op nor its rules.
    enum class Bound { Flip, Lazy, And, KeepRun, Plain };
    // an operand's host mirrors (current: ensure_mirrors) as the pair loop reads them
    struct Side {
        const uint32_t *cnt;
        const uint64_t *ebytes;
        const uint8_t *flags;
        uint64_t n;
    };
    static Side side(const rb200_set *S) { return {S->h_cnt.data(), S->h_ebytes.data(), S->h_flags.data(), S->n_bitmaps}; }
    // the staging block's item offsets (np + 1) and pair lists
    struct Lists {
        uint64_t *off;
        uint32_t *ia, *ib;
    };
    // One pass over the pairs: checks both indices, writes the pair lists and item offsets, and sums
    // the items W, the slab bounds and the COW flags.
    template <Bound R>
    bool pairs(const Side A, const Side B, const uint32_t *ia, const uint32_t *ib, size_t np, bool andnot,
               int share, const Lists L) {
        // 1 where a side's pass-through containers are copied into the result's own slab
        const uint64_t ownA = share & 1 ? 0 : 1, ownB = share & 2 || andnot ? 0 : 1, withB = andnot ? 0 : 1;
        uint64_t *__restrict off = L.off;
        uint32_t *__restrict hia = L.ia, *__restrict hib = L.ib;
        uint64_t w = 0, sb = 0, sbs = 0;
        uint8_t flags = 0;
        for (size_t p = 0; p < np; p++) {
            const uint32_t a = ia[p], b = ib[p];
            if (a >= A.n || b >= B.n) {
                t_err = "pair index out of range";
                return false;
            }
            hia[p] = a;
            hib[p] = b;
            flags |= A.flags[a] | B.flags[b];
            off[p] = w;
            const uint32_t na = A.cnt[a], nb = B.cnt[b];
            w += (uint64_t)na + nb;
            // Upper bound of the result slab of this pair, from the per-bitmap "effective bytes" E
            // (sum over containers of max(stored, min(8192, 2 * card)), 16-byte rounded): every
            // result container — computed or passed through — is an array, a bitset or a run no
            // larger than either, so it fits min(8192, 2 * card_result); card_result <= cA + cB
            // (OR, XOR), <= min(cA, cB) (AND), <= cA (ANDNOT).  slot_bound() obeys the same limits.
            const uint64_t EA = A.ebytes[a], EB = B.ebytes[b], m = na < nb ? na : nb;
            if constexpr (R == Bound::Flip) {
                // the slots k_plan_pairs reserves: a copy of A's container (<= its effective bytes),
                // a copy of a one-run range container (16), a matched cell (slot_bound_lazy with
                // nB = 1: <= 8 KiB + 16 + twice A's stored bytes).  EB counts 8 KiB for every key
                // the range covers, which for a range over the whole universe is 512 MiB per pair.
                sb += 2 * EA + 16 * (uint64_t)nb + m * (uint64_t)(BITSET_BYTES + 16) + 512;
            } else if constexpr (R == Bound::Lazy) {
                // lazy array x run unions stay runs (4 bytes per input value / run), flips add 8 KiB per key
                sb += 3 * (EA + EB) + m * (uint64_t)BITSET_BYTES + 512;
            } else if constexpr (R == Bound::And) {
                sb += (EA < EB ? EA : EB) + 64;
            } else {
                // KeepRun (add_many / remove_many): a cell with a run on the left takes
                // slot_bound_keep_run, min(128 KiB, 4 (lA + cB)) <= A's container's bytes + min(128 KiB,
                // 4 cB), and the last term is at most 16 x the effective bytes of B's container (2 cB up
                // to 4096 values, 8 KiB above).  Every other slot is bounded as for the op itself.
                const uint64_t E = R == Bound::KeepRun ? EA + 16 * EB : EA + withB * EB;
                sb += E + 64;
                // shared pass-through containers take no slot: the result's own containers are the
                // copied side's and cells of matched keys, at most min(na, nb) of them, each <= 8 KiB
                // (KeepRun: <= 128 KiB)
                const uint64_t own = ownA * EA + ownB * EB + m * (uint64_t)(R == Bound::KeepRun ? 131072 : BITSET_BYTES);
                sbs += (own < E ? own : E) + 64;
            }
        }
        off[np] = w;
        W = w;
        slab_bound_copy = sb;
        slab_bound = sbs;   // used when share != 0 (build())
        cow = (flags & FLAG_COW) != 0;
        return true;
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

// the message of a selection whose entry idx[k] = v is out of range of a set of `count` bitmaps
void index_error(const char *what, size_t k, uint32_t v, uint64_t count) {
    t_err = std::string(what) + ": index out of range: idx[" + std::to_string(k) + "] = " + std::to_string(v) +
            ", the set holds " + std::to_string(count) + " bitmaps";
}

// idx[0..n) of a selection of a set of `count` bitmaps: n < 2^32 (checked before idx is read) and
// every entry in range; `what` heads t_err.
bool check_indices(const char *what, const uint32_t *idx, size_t n, uint64_t count) {
    if (n > 0xffffffffull) { t_err = std::string(what) + ": more than 2^32 - 1 bitmaps selected"; return false; }
    for (size_t k = 0; k < n; k++) {
        if (idx[k] >= count) {
            index_error(what, k, idx[k], count);
            return false;
        }
    }
    return true;
}

// The bitmaps S[idx[0..n)] an entry point works on; idx == NULL selects every bitmap of S in order.
// Set: rb200_set, or rb200_set64 for the checks and indices alone.
template <typename Set>
struct SelectionOf {
    const Set *S;
    const uint32_t *idx;
    size_t n;
    // Refuse a selection the device must never see, before any device call; `what` heads t_err.
    // n is checked before idx is read, and becomes the set's size when idx is NULL.
    bool check(const char *what) {
        if (!S) { t_err = std::string(what) + ": S is NULL"; return false; }
        uint64_t count;
        if constexpr (std::is_same<Set, rb200_set>::value) {
            if (reject_lazy(S, what)) return false;
            count = S->n_bitmaps;
        } else {
            count = S->n;   // a 64-bit set is never lazy
        }
        if (!idx) { n = count; return true; }
        return check_indices(what, idx, n, count);
    }
    uint32_t operator[](size_t k) const { return idx ? idx[k] : (uint32_t)k; }
    bool all() const { return idx == nullptr; }
    // containers of the selected bitmaps (S's mirrors must be current)
    uint64_t containers() const {
        uint64_t t = 0;
        for (size_t k = 0; k < n; k++) t += S->h_cnt[(*this)[k]];
        return t;
    }
    uint8_t cow(size_t k) const { return S->h_flags[(*this)[k]] & FLAG_COW; }
    // whether the selected flags differ, which is when a fold's flag depends on its order
    bool cow_mixed() const {
        for (size_t k = 1; k < n; k++) if (cow(k) != cow(0)) return true;
        return false;
    }
    // The COW flag of the lazy fold roaring_bitmap_or_many / xor_many (roaring.c:775-809) of the
    // selection.  lazy_<op>(x0, x1) returns a copy of a non-empty operand next to an empty one and
    // takes both flags otherwise (:2509-2523, 2684-2697); a later step keeps the flag, unless it
    // overwrites an empty accumulator with a non-empty input (:2609-2610, 2772-2773).
    // acc_empty(k): the fold of inputs [0, k) is empty, for k >= 2.
    template <typename F> uint8_t fold_cow(F acc_empty) const {
        if (n < 2) return n ? cow(0) : 0;
        const auto empty = [&](size_t k) { return S->h_cnt[(*this)[k]] == 0; };
        uint8_t f = empty(0) ? cow(1) : empty(1) ? cow(0) : cow(0) | cow(1);
        for (size_t k = 2; k < n; k++)
            if (!empty(k) && acc_empty(k)) f = cow(k);
        return f;
    }
    // idx on the device through the pinned block h, which must outlive the copy; d stays NULL for
    // all(), which the kernels read as the identity
    bool to_device(DevBlock<uint32_t> &d, PinBlock<uint32_t> &h) const {
        if (!idx || !n) return true;
        if (!d.reset(n) || !h.reset(n)) return false;
        memcpy(h.get(), idx, 4 * n);
        return cudaMemcpyAsync(d.get(), h.get(), 4 * n, cudaMemcpyHostToDevice, g.stream) == cudaSuccess;
    }
};
using Selection = SelectionOf<rb200_set>;

// Host fields of a one-bitmap result of `containers` bitset slots (or_many, xor_many).
void fill_single_result(rb200_set *R, uint32_t containers, uint64_t slab_used, uint8_t cow) {
    R->n_containers = containers;
    R->slab_used = slab_used;
    R->h_cnt[0] = containers;
    R->h_bytes[0] = R->h_ebytes[0] = (uint64_t)containers * BITSET_BYTES;
    R->h_flags[0] = cow;
}

// The COW flag the reference gives x1 op x2 under `rules`, from the operands' flags and whether they
// are empty (hold no container).
// - A union or xor with an empty operand is a copy of the other (roaring.c:882-886, 1126-1130,
//   2515-2519, 2689-2693), and so is an andnot with an empty x2 (:1286).  Other results take both
//   flags (:738, 890, 1283, 1290).
// - The in-place twins keep x1's flag, unless a union or xor overwrites an empty x1 with a non-empty
//   x2 (roaring_bitmap_overwrite, :1072, 1210, 2610, 2773).  So do flips (:2307) and the updates of
//   add_many / remove_many, which modify x1.
// - lazy_or_from_lazy_inputs (RULES_NOFULL, roaring_priority_queue.c:99-111) returns its non-empty
//   operand next to an empty one, and otherwise a new bitmap without the flag.
uint8_t result_cow(int op, int rules, uint8_t fa, uint8_t fb, bool emptyA, bool emptyB) {
    fa &= FLAG_COW;
    fb &= FLAG_COW;
    const bool unite = op == OP_OR || op == OP_XOR;
    if (rules & (RULES_FLIP | RULES_KEEP_RUN)) return fa;
    if (rules & RULES_NOFULL) return emptyA ? fb : emptyB ? fa : 0;
    if (rules & RULES_INPLACE) return unite && emptyA && !emptyB ? fb : fa;
    if (unite) return emptyA ? fb : emptyB ? fa : fa | fb;
    return op == OP_ANDNOT && emptyB && !emptyA ? fa : fa | fb;
}

// Let R point into A's payload (onA) and / or B's (onB): R holds their slabs and its payload base
// moves to the lowest of its own slab and their bases.  false (nothing changed) when the span from
// that base to the end of the highest slab would not fit the 44 bits of a cell descriptor's offsets.
bool share_operands(rb200_set *R, const rb200_set *A, const rb200_set *B, bool onA, bool onB, PassShare &sh) {
    uintptr_t lo = (uintptr_t)R->d_slab, hi = lo + R->slab_cap;
    for (const rb200_set *P : {onA ? A : nullptr, onB ? B : nullptr}) {
        if (!P) continue;
        lo = std::min(lo, (uintptr_t)P->d_base);
        hi = std::max(hi, (uintptr_t)P->slab->p + P->slab->cap);
    }
    if (hi - lo >= (1ull << 44)) return false;
    if (onA) R->held[0] = A->slab;
    if (onB) R->held[1] = B->slab;
    R->d_base = (uint8_t *)lo;
    sh.onA = onA;
    sh.onB = onB;
    sh.dA = onA ? (uint64_t)((uintptr_t)A->d_base - lo) : 0;
    sh.dB = onB ? (uint64_t)((uintptr_t)B->d_base - lo) : 0;
    sh.bias = (uint64_t)((uintptr_t)R->d_slab - lo);
    return true;
}

// Payload bytes a set stores (16-byte rounded slots), wherever they live; its mirrors must be current.
uint64_t stored_bytes_total(const rb200_set *s) {
    return s->sharing() ? std::accumulate(s->h_bytes.begin(), s->h_bytes.end(), (uint64_t)0) : s->slab_used;
}

rb200_set *batch_op_impl(int op, const rb200_set *A, const rb200_set *B, const uint32_t *ia,
                         const uint32_t *ib, size_t np, int rules = 0) {
#ifdef RB200_HOST_TIMING
    ht_enter();
    struct Leave { ~Leave() { ht_leave(); } } leave;
#endif
    if (!ctx_init()) return nullptr;
    if (op < 0 || op > 3) { t_err = "bad op"; return nullptr; }
    if (rules & RULES_LAZY) {
        if (op != OP_OR && op != OP_XOR) { t_err = "lazy rules exist for OR and XOR only"; return nullptr; }
        if (op == OP_XOR && (rules & (RULES_CONV | RULES_NOFULL))) { t_err = "bad lazy flags for XOR"; return nullptr; }
        if ((rules & RULES_FLIP) && op != OP_XOR) { t_err = "bad flags"; return nullptr; }
    } else {
        if (rules & ~(RULES_INPLACE | RULES_KEEP_RUN)) { t_err = "bad flags"; return nullptr; }
        if ((rules & RULES_KEEP_RUN) && ((op != OP_OR && op != OP_ANDNOT) || (rules & RULES_INPLACE))) {
            t_err = "bad flags";
            return nullptr;
        }
        if (reject_lazy(A, "batch op") || reject_lazy(B, "batch op")) return nullptr;
    }
    if (np > 0xffffffffull) { t_err = "too many pairs"; return nullptr; }
    PairBuf pb;
    ItemsBuf ib_;
    SetPtr R;
    // Non-lazy ops share the unmatched containers of their operands instead of copying them: the
    // result points into the operands' slabs (the reference shares them too when copy-on-write is on,
    // roaring.c:918-922; no batch op ever writes into an operand).  Lazy ops and flips keep copying,
    // and so does every op from an operand that shares containers itself (see rb200_set::held).
    // (ensure_mirrors: an operand's holds are settled when its op's counters are read)
    if (!ensure_mirrors(A) || !ensure_mirrors(B)) return nullptr;
    const bool can_share = !(rules & RULES_LAZY) && op != OP_AND && np > 0;
    const bool onA = can_share && !A->sharing(), onB = can_share && op != OP_ANDNOT && !B->sharing();
    bool ok = pb.build(A, B, ia, ib, np, op, rules, (onA ? 1 : 0) | (onB ? 2 : 0));
    // class-ordered tickets pay one more small kernel: only for batches that fill the GPU
    static const uint64_t order_min = []() { const char *e = getenv("RB200_ORDER_MIN"); return e ? (uint64_t)atoll(e) : 16384ull; }();
    // (tried in round 2: ONE launch with a CTA per pair doing plan -> cells -> finalize for small batches —
    //  the 199-pair successive sweep took more device time per call: a pair's cells serialise on
    //  its 8 warps while the three-kernel path spreads them over the GPU)
    if (ok) ok = ib_.alloc(pb.W, true, pb.W >= order_min);
    HT_MARK(HT_ITEMS);
    PassShare sh = {false, false, 0, 0, 0};
    if (ok) {
        R = set_new((uint32_t)np, pb.W, pb.slab_bound, false);
        if (R && (onA || onB) && !share_operands(R.get(), A, B, onA, onB, sh)) {
            R.reset();   // out of the offsets' reach: copy everything into a slab sized for it
            R = set_new((uint32_t)np, pb.W, pb.slab_bound_copy, false);
        }
        ok = R != nullptr;
    }
    HT_MARK(HT_SET_NEW);
    DeferredCall call("batch op", R, pb.h, &pb.d);
    if (ok) ok = call.begin();
    HT_MARK(HT_BEGIN);
    if (ok) {
        const SetView va = A->view(), vb = B->view();
        launch_plan_pairs(va, vb, pb.d_ia, pb.d_ib, pb.d_off, (uint32_t)np, op, false, rules, sh, ib_.it,
                          g.d_dstats, g.stream);
        launch_order_items(ib_.it, pb.W, g.d_dstats, g.stream);
        // pass-through tickets: one item per lane, fewer lanes when the operands' containers are big
        // (32 x 8 KiB on one warp would be the tail of the launch)
        const uint64_t n_cont = A->n_containers + B->n_containers;
        const uint64_t avg_b = n_cont ? (stored_bytes_total(A) + stored_bytes_total(B)) / n_cont : 4096;
        // (on the real-data suite 4-32 items per ticket are within noise of each other, 1 item is
        //  clearly slower — RB200_COPY_TICKET overrides)
        static const int ct_env = []() { const char *e = getenv("RB200_COPY_TICKET"); return e ? std::min(32, std::max(1, atoi(e))) : 0; }();
        const int copy_ticket = ct_env ? ct_env : avg_b <= 256 ? 32 : avg_b <= 2048 ? 16 : 8;
        launch_compute_items(va, vb, ib_.it, pb.W, op, R->d_slab, R->slab_cap, g.d_dstats, rules, copy_ticket, g.stream);
        launch_finalize_pairs(va, vb, ib_.it, pb.d_off, (uint32_t)np, sh, R->out(), g.d_dstats, call.deliver(),
                              g.stream);
        R->parentA = A->h_ptr;
        R->parentB = B->h_ptr;
        R->lazy = (rules & RULES_LAZY) != 0 && !(rules & RULES_FLIP);
        // without a COW operand every result flag is 0, as set_new left them (result_cow of two zero
        // flags); the per-pair rules cost more host time than a small batch call takes on the device
        if (pb.cow)
            for (size_t p = 0; p < np; p++)
                R->h_flags[p] = result_cow(op, rules, A->h_flags[ia[p]], B->h_flags[ib[p]], A->h_cnt[ia[p]] == 0,
                                           B->h_cnt[ib[p]] == 0);
    }
    HT_MARK(HT_LAUNCH);
    // the device buffers go back when pb / ib_ leave scope: stream-ordered reuse
    return call.finish(ok);
}

}  // namespace

extern "C" {

#ifdef RB200_HOST_TIMING
// Copies up to `cap` doubles of the recorded calls (2 + HT_N per call, see HostTiming) to `out` and
// forgets them; returns the number of doubles recorded (out == NULL: just count).
__attribute__((visibility("default"))) size_t rb200_host_timing_take(double *out, size_t cap) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    const size_t n = g_ht.rec.size();
    if (out) {
        std::copy(g_ht.rec.begin(), g_ht.rec.begin() + std::min(n, cap), out);
        g_ht.rec.clear();
    }
    return n;
}
#endif

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
    DevBlock<uint64_t> d_out;
    PinBlock<uint64_t> h_out;
    SyncCall call("and_cardinality", "and_cardinality launch", true);
    bool ok = pb.build(A, B, ia, ib, np, OP_AND) && ib_.alloc(pb.W, false, false) && d_out.reset(np) && h_out.reset(np);
    if (ok) {
        ok = call.begin();
        const SetView va = A->view(), vb = B->view();
        launch_plan_pairs(va, vb, pb.d_ia, pb.d_ib, pb.d_off, (uint32_t)np, OP_AND, true, 0, PassShare{false, false, 0, 0, 0}, ib_.it,
                          g.d_stats, g.stream);
        call.kernels_begin();
        launch_card_items(va, vb, ib_.it, pb.W, g.d_stats, g.stream);
        call.kernels_end();
        launch_finalize_cards(ib_.it, pb.d_off, (uint32_t)np, d_out.get(), g.stream);
        call.end();
        ok = ok && cudaMemcpyAsync(h_out.get(), d_out.get(), 8 * np, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        ok = call.finish(ok, false);
    }
    if (ok) memcpy(out, h_out.get(), 8 * np);
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
    Selection sel{S, idx, n};
    if (!sel.check("or_many") || !ctx_init()) return nullptr;
    n = sel.n;
    if (key_hi > 65535) key_hi = 65535;
    uint32_t span_n = 0;
    if (sh) {
        if (sh->span_hi > 65535 || sh->span_lo > sh->span_hi) { t_err = "or_many_sharded: bad key span"; return nullptr; }
        span_n = sh->span_hi - sh->span_lo + 1;
    }
    const bool want_ck = card_per_key != nullptr || sh != nullptr;
    if (!ensure_mirrors(S)) return nullptr;
    // the index (rb200_many2.cu) holds input positions, per-key segments and counts in 32 bits; its
    // entry buffer is sized for every container of the inputs (the host has no per-bitmap keys to
    // count only those of [key_lo, key_hi]), so the container limit covers them all
    const uint64_t tot = sel.containers();
    if (tot > 0xffffffffu) { t_err = "or_many: the inputs carry more than 2^32 - 1 containers (every key counts, whatever the key range)"; return nullptr; }
    uint64_t maxk = key_lo <= key_hi ? (uint64_t)key_hi - key_lo + 1 : 0;
    if (tot < maxk) maxk = tot;
    SetPtr R = set_new(1, maxk, maxk * BITSET_BYTES);
    if (!R) return nullptr;
    DevBlock<uint32_t> d_idx;
    PinBlock<uint32_t> h_idx, ck;
    DevBlock<uint8_t> d_index;
    SyncCall call("or_many", "or_many launch", true);
    bool ok = sel.to_device(d_idx, h_idx);
    cudaEvent_t evc0 = nullptr, evc1 = nullptr;
    if (ok && want_ck) ok = ck.reset(65536);
    if (ok && sh) { evc0 = ev_get(); evc1 = ev_get(); ok = evc0 && evc1; }
    // index: entries + work-unit table from the device pool
    uint64_t tot_kib = 0;
    for (size_t i = 0; i < n; i++) tot_kib += (S->h_bytes[sel[i]] >> 10) + 1;
    const uint64_t max_units = std::max<uint64_t>(1, std::min<uint64_t>(tot, std::min<uint64_t>(65536, tot) + tot_kib / 32 + 1));
    // key-window index build: per-(window, chunk of 256 bitmaps) key counts when there are several chunks
    const uint64_t m2_chunks = (n + 255) / 256;
    const size_t tab_bytes = m2_chunks > 1 && m2_chunks <= M2W_MAX_CHUNKS ? (size_t)2048 * m2_chunks * 32 * 4 : 0;
    if (ok) ok = d_index.reset(al256(16 * tot) + al256(4 * max_units) + al256(tab_bytes));
    if (ok) {
        ok = call.begin();
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
        ix.ent = (uint4 *)d_index.get();
        ix.unit_ki = (uint32_t *)(d_index.get() + al256(16 * tot));
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
        launch_or_many2(vs, d_idx.get(), (uint32_t)n, key_lo, key_hi, ix, (uint32_t)max_units,
                        g.d_m2_scratch, g.d_m2_tickets, M2_SCRATCH_SLOTS, R->out(), want_ck ? g.d_cardkey : nullptr,
                        g.d_stats, g.stream, g.evk0, use_tma, window_index,
                        (uint32_t *)(d_index.get() + al256(16 * tot) + al256(4 * max_units)));
    }
    if (ok) {
        call.kernels_end();
        if (sh) {  // the ONE collective of the path: per-key cardinalities, summed over the ranks, on the device
            cudaEventRecord(evc0, g.stream);
            ok = ok && comm_allreduce_sum(sh->comm, g.d_cardkey + sh->span_lo, span_n, false, g.stream, t_err);
            cudaEventRecord(evc1, g.stream);
        }
        call.end();
        if (card_per_key)
            ok = ok && cudaMemcpyAsync(ck.get(), g.d_cardkey, 65536 * 4, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        else if (sh)
            ok = ok && cudaMemcpyAsync(ck.get(), g.d_cardkey + sh->span_lo, 4ull * span_n, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        ok = call.finish(ok);
    }
    if (ok) {
        const uint32_t *h_ck = ck.get();
        const uint32_t nk = g.h_stats->nk;
        size_t first = 0;   // the first non-empty input: a union is empty until it
        while (first < n && S->h_cnt[sel[first]] == 0) first++;
        fill_single_result(R.get(), nk, (uint64_t)nk * BITSET_BYTES, sel.fold_cow([&](size_t k) { return k <= first; }));
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
        if (key_lo == 0 && key_hi == 65535 && sel.all()) inb = payload_bytes_of(S);
        g.last_algo_bytes = inb;
    }
    ev_put(evc0);
    ev_put(evc1);
    if (!ok) {
        if (t_err.empty()) t_err = "or_many failed";
        return nullptr;
    }
    return R.release();
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
    launch_sum_cardinalities((const uint64_t *)(s->d_dir.get() + s->L.o_bcard), s->n_bitmaps, d_acc, g.stream);
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
    Selection sel{S, idx, n};
    if (!sel.check("xor_many") || !ctx_init() || !ensure_mirrors(S)) return nullptr;
    const uint64_t maxk = std::min<uint64_t>(65536, sel.containers());
    SetPtr R = set_new(1, maxk, maxk * BITSET_BYTES);
    if (!R) return nullptr;
    DevBlock<uint32_t> d_idx;
    PinBlock<uint32_t> h_idx;
    DevBlock<uint8_t> t_type(maxk);
    DevBlock<uint32_t> t_card(maxk), t_len(maxk);
    SyncCall call("xor_many", "xor_many launch", true);
    bool ok = t_type && t_card && t_len && sel.to_device(d_idx, h_idx);
    // Copy-on-write inputs only: their COW bits per position (the kernel's SHARED accumulators), and
    // when the flags are mixed, where each key's accumulator turns live or empty (the result's flag).
    bool any_cow = false;
    for (size_t k = 0; k < sel.n && !any_cow; k++) any_cow = sel.cow(k) != 0;
    const bool mixed = sel.cow_mixed();
    DevBlock<uint8_t> d_cow;
    PinBlock<uint8_t> h_cow;
    DevBlock<int32_t> d_live;
    PinBlock<int32_t> h_live;
    if (ok && any_cow) {
        ok = d_cow.reset(sel.n) && h_cow.reset(sel.n);
        for (size_t k = 0; ok && k < sel.n; k++) h_cow.get()[k] = sel.cow(k);
        ok = ok && cudaMemcpyAsync(d_cow.get(), h_cow.get(), sel.n, cudaMemcpyHostToDevice, g.stream) == cudaSuccess;
    }
    if (ok && mixed)
        ok = d_live.reset(sel.n) && h_live.reset(sel.n) &&
             cudaMemsetAsync(d_live.get(), 0, 4 * sel.n, g.stream) == cudaSuccess;
    if (ok) {
        ok = call.begin();
        const SetView vs = S->view();
        launch_many_mark(vs, d_idx.get(), (uint32_t)sel.n, 0, 65535, g.d_flags, g.stream);
        launch_many_compact(g.d_flags, g.d_keys, g.d_stats, g.stream);
        call.kernels_begin();
        launch_xor_many(vs, d_idx.get(), (uint32_t)sel.n, g.d_keys, d_cow.get(), d_live.get(), t_type.get(), t_card.get(),
                        t_len.get(), R->out(), g.d_stats, g.stream);
        call.kernels_end();
        call.end();
        if (mixed)
            ok = ok && cudaMemcpyAsync(h_live.get(), d_live.get(), 4 * sel.n, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        ok = call.finish(ok);
    }
    if (ok) {
        // live keys after input k: the prefix sums of the kernel's +1 / -1 per position
        std::vector<int64_t> live_after(mixed ? sel.n : 0);
        int64_t live = 0;
        for (size_t k = 0; k < live_after.size(); k++) live_after[k] = live += h_live.get()[k];
        const uint8_t cow = mixed ? sel.fold_cow([&](size_t k) { return live_after[k - 1] == 0; }) : sel.n ? sel.cow(0) : 0;
        fill_single_result(R.get(), (uint32_t)g.h_stats->dir_cursor, (uint64_t)g.h_stats->nk * BITSET_BYTES, cow);
        g.last_algo_bytes = sel.all() ? payload_bytes_of(S) : 0;
    }
    return ok ? R.release() : nullptr;
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
    PinBlock<uint64_t> h(nb);
    if (!h) return -1;
    // bm_card is maintained by upload / finalize / or_many
    bool ok = cudaMemcpyAsync(h.get(), s->d_dir.get() + s->L.o_bcard, 8 * nb, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
    ok = ok && cudaStreamSynchronize(g.stream) == cudaSuccess;
    if (ok) memcpy(out, h.get(), 8 * nb);
    else t_err = "set_cardinalities: copy failed";
    return ok ? 0 : -1;
}

}  // extern "C"

// =================================================================== download
namespace {

roaring_bitmap_t *build_bitmap(const rb200_set *s, size_t i, const uint8_t *slab = nullptr, uint64_t bias = 0) {
    if (!slab) slab = s->m_slab.get();
    const uint8_t *m_dir = s->m_dir.get();
    const uint32_t *c_src = (const uint32_t *)(m_dir + s->L.o_src);
    const std::vector<const void *> *tabA = s->parentA.get(), *tabB = s->parentB.get();
    const uint32_t *bm_beg = (const uint32_t *)(m_dir + s->L.o_beg);
    const uint32_t *bm_cnt = (const uint32_t *)(m_dir + s->L.o_cnt);
    const uint16_t *c_key = (const uint16_t *)(m_dir + s->L.o_key);
    const uint8_t *c_type = m_dir + s->L.o_type;
    const uint32_t *c_card = (const uint32_t *)(m_dir + s->L.o_card);
    const uint32_t *c_len = (const uint32_t *)(m_dir + s->L.o_len);
    const uint64_t *c_off = (const uint64_t *)(m_dir + s->L.o_off);
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

// Persistent host worker pool.  run(fn, T) executes fn() on T threads (the caller is one of them);
// fn pulls its own work from a shared atomic counter.  A run started on a thread that is already
// inside a run of the same pool (one of its workers, or the caller during its run) executes fn()
// inline: waiting for the pool there would wait for itself.
//
// Lock order, outermost first: a run of visitor_pool(), g.mu, a run of pool().  Visitors run only
// on visitor_pool(), whose runs start with g.mu released, so a visitor may call any entry point;
// jobs on pool() (materialisation into arrays, bulk frees) never call out of the library, so a
// thread holding g.mu only ever waits for work that finishes on its own.
void bind_to_local_cpus();

class Pool {
   public:
    // The pool whose run the calling thread is inside, or null.
    static const Pool *current() { return in_run_; }
    void run(const std::function<void()> &fn, unsigned T) {
        const Pool *outer = in_run_;
        in_run_ = this;
        if (T <= 1 || outer == this) {
            fn();
            in_run_ = outer;
            return;
        }
        std::lock_guard<std::mutex> one_run(run_mu_);  // callers: API threads and the downloader
        std::unique_lock<std::mutex> lk(mu_);
        while (workers_.size() < T - 1)
            workers_.emplace_back([this]() {
                in_run_ = this;   // everything a worker executes is part of a run of this pool
                bind_to_local_cpus();
                loop();
            });
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
        in_run_ = outer;
    }

   private:
    static thread_local const Pool *in_run_;
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
thread_local const Pool *Pool::in_run_ = nullptr;
Pool &pool() {
    static Pool *p = new Pool();  // intentionally leaked: workers are detached for process life
    return *p;
}
// The threads that run visitors (rb200_visit_fn): synchronous and asynchronous visitor downloads.
Pool &visitor_pool() {
    static Pool *p = new Pool();  // leaked like pool()
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

// fn(i) for every i in [0, n) on up to T threads of `on`, which claim the indices in blocks of blk.
void pool_for(size_t n, unsigned T, size_t blk, const std::function<void(size_t)> &fn, Pool &on = pool()) {
    if ((size_t)T * blk > n) T = (unsigned)((n + blk - 1) / blk);
    std::atomic<size_t> next(0);
    std::function<void()> work = [&]() {
        for (size_t i0; (i0 = next.fetch_add(blk)) < n;)
            for (size_t i = i0, i1 = std::min(n, i0 + blk); i < i1; i++) fn(i);
    };
    on.run(work, T);
}

// Every bulk download takes the same three steps: pack_for_download() lays the set out for the
// trip (on the library stream), a Ring of pinned slots brings the payload over chunk by chunk, and
// materialise() builds the bitmaps of each staged chunk on the worker pool while the next chunks
// are still crossing PCIe.

// A set packed for download: directory in bitmap order, mirrored in pinned memory; payload
// contiguous in bitmap order with no slot slack (device), cut into chunks of whole bitmaps.
// Every copy out of P must have landed before a Packed is destroyed.
struct Packed {
    SetPtr P;
    size_t nb = 0;
    PinBlock<uint64_t> ob;          // [payload offset (nb+1) | first container (nb+1)]
    std::vector<size_t> chunk_end;  // bitmap index closing each chunk
    uint64_t max_chunk = 0;         // payload bytes of the largest chunk
    uint64_t bytes = 0;             // directory + payload: what crosses PCIe
    const uint64_t *h_ob() const { return ob.get(); }
    size_t begin(size_t k) const { return k ? chunk_end[k - 1] : 0; }
};

using Clock = std::chrono::steady_clock;
double ms_since(Clock::time_point t) { return std::chrono::duration<double, std::milli>(Clock::now() - t).count(); }

// What a download moved and where its time went: report() sets rb200_last_download_bytes and
// prints the RB200_TRACE line.
struct DlStats {
    const char *path;
    size_t sets = 0, bitmaps = 0, chunks = 0;
    uint64_t bytes = 0;
    double pack = 0, wait = 0, build = 0;  // ms
    Clock::time_point t0 = Clock::now();
    explicit DlStats(const char *p) : path(p) {}
    void add(const DlStats &o) {
        if (o.sets && !sets) t0 = o.t0;
        sets += o.sets, bitmaps += o.bitmaps, chunks += o.chunks, bytes += o.bytes;
        pack += o.pack, wait += o.wait, build += o.build;
    }
    void report() const {
        g.last_download_bytes = bytes;
        if (getenv("RB200_TRACE"))
            fprintf(stderr, "rb200 %s: %zu sets %zu bitmaps %zu chunks %.1f MB | pack %.2f ms, copy-wait %.2f ms, "
                            "build %.2f ms, total %.2f ms\n",
                    path, sets, bitmaps, chunks, bytes / 1e6, pack, wait, build, ms_since(t0));
    }
};

// Pack s for download on the library stream: chunks of at most chunk_bitmaps bitmaps and ~64 MB of
// payload.  The directory copy is only enqueued; it lands before any chunk copied after it on the
// library stream (the background downloader orders its stream after the pack with an event).
std::unique_ptr<Packed> pack_for_download(const rb200_set *s, size_t chunk_bitmaps, DlStats &stats) {
    const auto t = Clock::now();
    if (!resolve(s)) return nullptr;
    std::unique_ptr<Packed> pk(new Packed());
    const size_t nb = pk->nb = s->n_bitmaps;
    bool ok = true;
    if (nb) {
        if (chunk_bitmaps == 0) chunk_bitmaps = 1024;
        DevBlock<uint64_t> d_bytes(nb), d_off(nb + 1), d_beg(nb + 1);
        DevBlock<uint32_t> d_cnt(nb);
        ok = d_bytes && d_off && d_beg && d_cnt && pk->ob.reset(2 * (nb + 1));
        const int elide = (s->parentA ? 1 : 0) | (s->parentB ? 2 : 0);
        uint64_t *h_off = pk->ob.get(), *h_beg = ok ? h_off + nb + 1 : nullptr;
        if (ok) {
            launch_pack(s->view(), (uint32_t)nb, elide, d_bytes.get(), d_cnt.get(), d_off.get(), d_beg.get(), g.stream);
            ok = cudaMemcpyAsync(h_off, d_off.get(), 8 * (nb + 1), cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
                 cudaMemcpyAsync(h_beg, d_beg.get(), 8 * (nb + 1), cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
                 cudaStreamSynchronize(g.stream) == cudaSuccess;
        }
        if (ok) {
            pk->P = set_new((uint32_t)nb, h_beg[nb], h_off[nb]);
            ok = pk->P != nullptr;
        }
        if (ok) {
            rb200_set *P = pk->P.get();
            P->n_containers = h_beg[nb];
            P->slab_used = h_off[nb];
            P->h_flags = s->h_flags;
            P->parentA = s->parentA;
            P->parentB = s->parentB;
            launch_pack_copy(s->view(), (uint32_t)nb, elide, d_off.get(), d_beg.get(), P->out(), g.stream);
            ok = P->m_dir.reset(P->L.total) &&
                 cudaMemcpyAsync(P->m_dir.get(), P->d_dir.get(), P->L.total, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
            const uint64_t CAP = (uint64_t)64 << 20;
            for (size_t p0 = 0, p1; p0 < nb; p0 = p1) {
                p1 = p0 + 1;
                while (p1 < nb && p1 - p0 < chunk_bitmaps && h_off[p1 + 1] - h_off[p0] <= CAP) p1++;
                pk->chunk_end.push_back(p1);
                pk->max_chunk = std::max(pk->max_chunk, h_off[p1] - h_off[p0]);
            }
            pk->bytes = P->L.total + P->slab_used;
        }
    }
    if (!ok) {
        cudaStreamSynchronize(g.stream);  // before ~Packed recycles what the copies write
        if (t_err.empty()) t_err = "download: packing failed";
        return nullptr;
    }
    stats.sets++, stats.bitmaps += nb, stats.chunks += pk->chunk_end.size(), stats.bytes += pk->bytes;
    stats.pack += ms_since(t);
    return pk;
}

// Host copy of a whole set for rb200_set_download, made on first use: the set packed on the device
// (a batch result's pass-through containers can live in its operands' slabs), then the packed
// payload copied to pinned memory.  build_bitmap() reads it.
const rb200_set *ensure_mirror(rb200_set *s) {
    if (s->mirror) return s->mirror.get();
    DlStats stats("download");
    std::unique_ptr<Packed> pk = pack_for_download(s, 0, stats);
    if (!pk) return nullptr;
    rb200_set *P = pk->P.get();
    bool ok = P->m_slab.reset(P->slab_used);
    if (ok && P->slab_used)
        ok = cudaMemcpyAsync(P->m_slab.get(), P->d_slab, P->slab_used, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
    ok = cudaStreamSynchronize(g.stream) == cudaSuccess && ok;   // (also the directory copy of the pack)
    if (!ok) {
        t_err = "download: copy failed";
        return nullptr;
    }
    P->d_dir.reset();   // the copies have landed: only the pinned host copies are kept
    P->slab.reset();
    P->d_slab = P->d_base = nullptr;
    s->mirror = std::move(pk->P);
    stats.report();
    return P;
}

// Pinned staging slots that D2H copies of chunks fill in turn, so the copy engine can run up to
// slots-1 chunks ahead of the builders.  Chunks alternate between copy-bound and build-bound, so
// download_sets() and the background downloader use 4 slots: 2 stall one side or the other.
class Ring {
   public:
    explicit Ring(size_t slots) : buf_(slots), ev_(slots, nullptr) {
        for (auto &e : ev_) e = ev_get();
    }
    ~Ring() {  // nothing may be in flight
        for (cudaEvent_t e : ev_) ev_put(e);
    }
    uint64_t capacity() const { return bytes_; }
    bool idle() const { return issued_ == waited_; }
    bool full() const { return issued_ - waited_ == buf_.size(); }
    // Slots of at least `bytes`; the ring only grows while idle().
    bool reserve(uint64_t bytes) {
        bytes = std::max<uint64_t>(bytes, 1);
        if (bytes <= bytes_) return true;
        for (auto &b : buf_) b.reset();
        bytes_ = 0;
        for (auto &b : buf_)
            if (!b.reset(bytes)) {
                for (auto &c : buf_) c.reset();
                return false;
            }
        bytes_ = bytes;
        return true;
    }
    // Copy chunk k of pk into the next slot on `stream` (the ring must not be full()).
    bool enqueue(const Packed &pk, size_t k, cudaStream_t stream) {
        const size_t slot = issued_++ % buf_.size();
        const uint64_t b0 = pk.h_ob()[pk.begin(k)], b1 = pk.h_ob()[pk.chunk_end[k]];
        const bool ok = b1 == b0 || cudaMemcpyAsync(buf_[slot].get(), pk.P->d_slab + b0, b1 - b0,
                                                    cudaMemcpyDeviceToHost, stream) == cudaSuccess;
        return cudaEventRecord(ev_[slot], stream) == cudaSuccess && ok;
    }
    // Wait for the oldest copy in flight; its slot, or nullptr if the copy failed.
    const uint8_t *wait() {
        const size_t slot = waited_++ % buf_.size();
        return cudaEventSynchronize(ev_[slot]) == cudaSuccess ? buf_[slot].get() : nullptr;
    }

   private:
    std::vector<PinBlock<uint8_t>> buf_;
    std::vector<cudaEvent_t> ev_;
    uint64_t bytes_ = 0;
    size_t issued_ = 0, waited_ = 0;
};

// Where materialise() puts each bitmap: out[i] (i counted from the chunk's first bitmap), or
// fn(base + index in the set, bitmap, ctx), which keeps the bitmap by returning non-zero.
struct Sink {
    roaring_bitmap_t **out;
    rb200_visit_fn fn;
    void *ctx;
    size_t base;
};

// Build the bitmaps of chunk k of pk from its staged payload `buf`: on pool() into out[], on
// visitor_pool() for a visitor (the caller must not hold g.mu then, see Pool).  Each visited bitmap
// is built, visited and freed on one thread.  False if one failed (its out[] slot is then null).
bool materialise(const Packed &pk, size_t k, const uint8_t *buf, const Sink &sink) {
    const size_t p0 = pk.begin(k), p1 = pk.chunk_end[k], n = p1 - p0;
    const uint64_t *off = pk.h_ob(), *beg = off + pk.nb + 1;
    // threads scaled to the work of the chunk: waking every worker for a few hundred tiny bitmaps
    // costs more than it saves
    const uint64_t want = (off[p1] - off[p0] + 256 * (beg[p1] - beg[p0]) + 512 * n) / (128 << 10) + 1;
    std::atomic<int> failed(0);
    pool_for(n, (unsigned)std::min<uint64_t>(want, host_workers()), 8, [&](size_t i) {
        roaring_bitmap_t *bm = build_bitmap(pk.P.get(), p0 + i, buf, off[p0]);
        if (!bm) failed = 1;
        if (sink.out) sink.out[i] = bm;
        else if (bm && sink.fn(sink.base + p0 + i, bm, sink.ctx) == 0) bitmap_free_host(bm);
    }, sink.out ? pool() : visitor_pool());
    return !failed;
}

// Wait for the ring's oldest copy, chunk k of pk, and materialise it.
bool drain(Ring &ring, const Packed &pk, size_t k, const Sink &sink, DlStats &stats) {
    auto t = Clock::now();
    const uint8_t *buf = ring.wait();
    stats.wait += ms_since(t);
    t = Clock::now();
    const bool ok = buf && materialise(pk, k, buf, sink);
    stats.build += ms_since(t);
    return ok;
}

// Every chunk of the packed sets, in order, through one 4-slot ring on the library stream: into
// out[] (indexed over all the sets) or to the visitor (index running on across the sets).  The
// caller holds g.mu through lk; it is released while a chunk is visited, so the visitor may call
// back into the library (the ring and the packed sets belong to this call alone).
bool download_sets(const std::vector<std::unique_ptr<Packed>> &pks, roaring_bitmap_t **out, rb200_visit_fn fn,
                   void *ctx, DlStats &stats, std::unique_lock<std::recursive_mutex> &lk) {
    struct Ref { const Packed *pk; size_t k, base; };
    std::vector<Ref> order;
    uint64_t slot_bytes = 0;
    size_t base = 0;
    for (const auto &pk : pks) {
        for (size_t k = 0; k < pk->chunk_end.size(); k++) order.push_back(Ref{pk.get(), k, base});
        base += pk->nb;
        slot_bytes = std::max(slot_bytes, pk->max_chunk);
    }
    Ring ring(4);
    bool ok = ring.reserve(slot_bytes);
    size_t copied = 0;
    for (size_t c = 0; c < order.size() && ok; c++) {
        for (; ok && copied < order.size() && !ring.full(); copied++)
            ok = ring.enqueue(*order[copied].pk, order[copied].k, g.stream);
        const Ref &r = order[c];
        const Sink sink = out ? Sink{out + r.base + r.pk->begin(r.k), nullptr, nullptr, 0} : Sink{nullptr, fn, ctx, r.base};
        if (!out) lk.unlock();
        ok = ok && drain(ring, *r.pk, r.k, sink, stats);
        if (!out) lk.lock();
    }
    cudaStreamSynchronize(g.stream);
    return ok;
}

}  // namespace

// Streaming download: results leave the device chunk by chunk while the caller consumes (and
// frees) the previous chunk, so host memory stays bounded and D2H overlaps materialisation.
struct rb200_download_stream {
    std::unique_ptr<Packed> pk;
    Ring ring{2};
    DlStats stats{"download_stream"};
    size_t next_copy = 0, next_build = 0;
};

namespace {

// Keep every slot of the stream's ring busy.
bool stream_refill(rb200_download_stream *st) {
    for (; st->next_copy < st->pk->chunk_end.size() && !st->ring.full(); st->next_copy++)
        if (!st->ring.enqueue(*st->pk, st->next_copy, g.stream)) return false;
    return true;
}

}  // namespace

extern "C" {

rb200_download_stream_t *rb200_download_begin(const rb200_set_t *s, size_t chunk_bitmaps) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return nullptr;
    rb200_download_stream *st = new rb200_download_stream();
    st->pk = pack_for_download(s, chunk_bitmaps, st->stats);
    if (st->pk && st->ring.reserve(st->pk->max_chunk) && stream_refill(st)) return st;
    if (t_err.empty()) t_err = "download_begin failed";
    cudaStreamSynchronize(g.stream);
    delete st;
    return nullptr;
}

size_t rb200_download_chunk_capacity(const rb200_download_stream_t *st) {
    size_t m = 0;
    for (size_t k = 0; k < st->pk->chunk_end.size(); k++) m = std::max(m, st->pk->chunk_end[k] - st->pk->begin(k));
    return m;
}

// Materialise the next chunk into out[] (capacity >= rb200_download_chunk_capacity); returns the
// number of bitmaps produced, 0 at the end of the stream, (size_t)-1 on error.
size_t rb200_download_next(rb200_download_stream_t *st, roaring_bitmap_t **out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (st->next_build >= st->pk->chunk_end.size()) return 0;
    const size_t k = st->next_build++;
    const size_t n = st->pk->chunk_end[k] - st->pk->begin(k);
    std::fill(out, out + n, nullptr);
    if (!drain(st->ring, *st->pk, k, Sink{out, nullptr, nullptr, 0}, st->stats) || !stream_refill(st)) {
        for (size_t i = 0; i < n; i++) { bitmap_free_host(out[i]); out[i] = nullptr; }
        t_err = "download_next: host allocation or copy failed";
        return (size_t)-1;
    }
    return n;
}

void rb200_download_end(rb200_download_stream_t *st) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!st) return;
    cudaStreamSynchronize(g.stream);
    st->stats.report();
    delete st;
}

// Visitor download of SEVERAL result sets as one pipelined stream: every set is packed on the
// device first, then all their chunks cross PCIe back to back through one staging ring while the
// workers materialise the previous chunk — the copy engine never idles between sets, and the
// builds of small / host-bound sets hide behind the transfers of the large ones.  fn receives a
// running index (set 0's bitmaps first).  Returns 0 on success.
int rb200_download_foreach_many(const rb200_set_t *const *sets, size_t nsets, rb200_visit_fn fn, void *ctx) {
    std::unique_lock<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    DlStats stats("foreach_many");
    std::vector<std::unique_ptr<Packed>> pks;
    bool ok = true;
    for (size_t i = 0; i < nsets && ok; i++) {
        pks.push_back(pack_for_download(sets[i], 4096, stats));
        ok = pks.back() != nullptr;
    }
    ok = ok && download_sets(pks, nullptr, fn, ctx, stats, lk);
    stats.report();
    if (!ok) {
        if (t_err.empty()) t_err = "download_foreach: host allocation or copy failed";
        return -1;
    }
    return 0;
}

// Visitor form of the streaming download: every bitmap of the set is materialised as a host
// roaring_bitmap_t (reference layout), handed to `fn` ON A WORKER THREAD, and freed right after
// unless fn returns non-zero (then the callee owns it).  Building, consuming and freeing a result
// on the same thread is what the reference's own loops do (create, use, roaring_bitmap_free —
// microbenchmarks/bench.cpp:85-96): the allocator recycles hot blocks instead of touching
// gigabytes of fresh memory.  Returns 0 on success.
int rb200_download_foreach(const rb200_set_t *s, rb200_visit_fn fn, void *ctx) {
    return rb200_download_foreach_many(&s, 1, fn, ctx);
}

}  // extern "C"

// ---- asynchronous visitor download ---------------------------------------------------------
// rb200_download_foreach_async packs the set on the caller's thread (device kernels on the library
// stream) and hands the packed copy to ONE background downloader thread, which owns a second CUDA
// stream and a 4-slot Ring: chunks of all queued sets cross PCIe back to back while the worker
// pool materialises the previous chunk — and while the caller goes on uploading and launching the
// next ops.  rb200_download_wait drains the queue.
namespace {
struct DlJob {
    std::unique_ptr<Packed> pk;
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
    DlStats stats{"foreach_async"};  // since the previous rb200_download_wait
    void loop();
};
Downloader &dl() {
    static Downloader *d = new Downloader();  // leaked on purpose: the thread lives as long as the process
    return *d;
}

void Downloader::loop() {
    cudaSetDevice(g.device);
    bind_to_local_cpus();
    cudaStream_t stream = nullptr;
    cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
    Ring ring(4);
    std::deque<std::pair<DlJob *, size_t>> inflight;  // (job, chunk) in ring order
    std::deque<DlJob *> jobs;                         // taken from q, not yet fully enqueued
    auto fail = [&](const char *why) {
        std::lock_guard<std::mutex> lk(mu);
        failed = 1;
        if (err.empty()) err = why;
    };
    auto finish = [&](DlJob *j) {
        cudaEventDestroy(j->ready);
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
        while (!ring.full() && !jobs.empty()) {
            DlJob *j = jobs.front();
            const Packed &pk = *j->pk;
            if (pk.chunk_end.empty()) { jobs.pop_front(); finish(j); continue; }
            if (pk.max_chunk > ring.capacity()) {
                if (!ring.idle()) break;
                if (!ring.reserve(pk.max_chunk)) fail("downloader: pinned allocation failed");
            }
            if (j->next_copy == 0) cudaStreamWaitEvent(stream, j->ready, 0);
            if (!ring.enqueue(pk, j->next_copy, stream)) fail("downloader: D2H copy failed");
            inflight.emplace_back(j, j->next_copy);
            if (++j->next_copy == pk.chunk_end.size()) jobs.pop_front();
        }
        if (inflight.empty()) continue;
        DlJob *j = inflight.front().first;
        const size_t k = inflight.front().second;
        inflight.pop_front();
        DlStats t(nullptr);
        if (!drain(ring, *j->pk, k, Sink{nullptr, j->fn, j->ctx, 0}, t)) fail("downloader: copy or host allocation failed");
        {
            std::lock_guard<std::mutex> lk(mu);
            stats.add(t);
        }
        if (++j->built == j->pk->chunk_end.size()) finish(j);
    }
}
}  // namespace

extern "C" {

// Enqueue the visitor download of `s` and return at once (the set may be freed right away: the
// job owns a packed device copy).  fn runs on worker threads with the index of the bitmap in `s`.
int rb200_download_foreach_async(const rb200_set_t *s, rb200_visit_fn fn, void *ctx) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    DlStats t(nullptr);
    DlJob *j = new DlJob();
    j->pk = pack_for_download(s, 4096, t);
    if (!j->pk) { delete j; return -1; }
    j->fn = fn;
    j->ctx = ctx;
    if (cudaEventCreateWithFlags(&j->ready, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventRecord(j->ready, g.stream) != cudaSuccess) {
        t_err = "download_foreach_async: event failed";
        cudaStreamSynchronize(g.stream);
        delete j;
        return -1;
    }
    Downloader &d = dl();
    {
        std::lock_guard<std::mutex> dk(d.mu);
        d.stats.add(t);
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
    if (Pool::current() == &visitor_pool()) {   // the download running this visitor may be among them
        t_err = "download_wait: not allowed in a visitor";
        return -1;
    }
    Downloader &d = dl();
    std::unique_lock<std::mutex> dk(d.mu);
    d.idle_cv.wait(dk, [&]() { return d.active == 0; });
    const int failed = d.failed;
    const std::string why = d.err;
    d.stats.report();
    d.stats = DlStats("foreach_async");
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
    const rb200_set *m = ensure_mirror(s);
    return m ? build_bitmap(m, i) : nullptr;
}

// Download every bitmap of a set as host roaring_bitmap_t (reference layout): pack, then the
// chunks of the packed set through a 4-slot ring, each materialised into out[] as it lands.
int rb200_set_download_all(const rb200_set_t *s, roaring_bitmap_t **out) {
    std::unique_lock<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    DlStats stats("download_all");
    std::vector<std::unique_ptr<Packed>> pks;
    pks.push_back(pack_for_download(s, 4096, stats));
    if (!pks[0]) return -1;
    std::fill(out, out + pks[0]->nb, nullptr);
    const bool ok = download_sets(pks, out, nullptr, nullptr, stats, lk);
    stats.report();
    if (!ok) {
        for (size_t i = 0; i < pks[0]->nb; i++) { bitmap_free_host(out[i]); out[i] = nullptr; }
        t_err = "download: host allocation or copy failed";
        return -1;
    }
    return 0;
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
    if (!ensure_mirrors(S)) return nullptr;
    const uint64_t nc = S->n_containers;
    // mode 1 never grows a container by more than its 16-byte padding; mode 0 may expand runs
    const uint64_t bound = stored_bytes_total(S) + 16 * nc + (mode == 0 ? nc * (uint64_t)BITSET_BYTES : 0) + 512;
    SetPtr R = set_new(S->n_bitmaps, nc, bound);
    if (!R) return nullptr;
    SyncCall call("run_optimize");
    const bool ok = call.begin();
    launch_run_optimize(S->view(), S->n_bitmaps, nc, mode, R->out(), g.d_stats, g.stream);
    if (!call.finish(ok)) return nullptr;
    R->n_containers = nc;
    R->slab_used = g.h_stats->slab_cursor;
    R->h_flags = S->h_flags;
    R->h_cnt = S->h_cnt;
    for (size_t b = 0; b < R->n_bitmaps; b++) {
        R->h_bytes[b] = (uint64_t)R->h_cnt[b] * BITSET_BYTES;
        R->h_ebytes[b] = std::max<uint64_t>(R->h_bytes[b], S->h_ebytes[b]);
    }
    return R.release();
}

// roaring_bitmap_to_uint32_array for every bitmap of a set: *vals (pinned host memory owned by the
// library) holds all values; bitmap i = vals[off[i] .. off[i+1]).  Release with rb200_values_free.
int rb200_set_to_uint32(const rb200_set_t *S, uint32_t **vals, uint64_t **off_out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    *vals = nullptr;
    *off_out = nullptr;
    if (!ctx_init()) return -1;
    if (!resolve(S)) return -1;
    const size_t nb = S->n_bitmaps;
    const uint64_t nc = S->n_containers;
    HostArrays out;
    if (!out.alloc(nb, false)) return -1;
    if (nb == 0) return out.hand_out(vals, off_out, nullptr);
    DevBlock<uint64_t> d_bv(nb), d_off(nb + 1), d_cstart(nc);
    DevBlock<uint32_t> d_cbm(nc), d_vals;
    PinBlock<uint64_t> h_off(nb + 1);
    SyncCall call;
    uint64_t total = 0;
    bool ok = d_bv && d_off && d_cstart && d_cbm && h_off;
    if (ok) {
        launch_values_measure(S->view(), (uint32_t)nb, d_bv.get(), d_cstart.get(), d_cbm.get(), g.stream);
        launch_pack_scan(d_bv.get(), nullptr, (uint32_t)nb, d_off.get(), nullptr, g.stream);
        ok = cudaMemcpyAsync(h_off.get(), d_off.get(), 8 * (nb + 1), cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaStreamSynchronize(g.stream) == cudaSuccess;
    }
    if (ok) {
        total = h_off.get()[nb];
        memcpy(out.off, h_off.get(), 8 * (nb + 1));
        ok = d_vals.reset(total) && out.blob.reset(4 * total);
    }
    if (ok) {
        launch_values_write(S->view(), (uint32_t)nb, d_off.get(), d_cstart.get(), d_cbm.get(), nc, d_vals.get(), g.stream);
        ok = cudaMemcpyAsync(out.blob.get(), d_vals.get(), 4 * total, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        ok = call.finish(ok, false);
    }
    if (!ok) {
        if (t_err.empty()) t_err = "set_to_uint32 failed";
        return -1;
    }
    return out.hand_out(vals, off_out, nullptr);
}

void rb200_values_free(uint32_t *vals, uint64_t *off) { rb200_serialized_free((char *)vals, off, nullptr); }

extern "C++" {
// p is device (or managed) memory of the library's device
static bool device_memory(const char *what, const char *name, const void *p) {
    cudaPointerAttributes a = {};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        (void)cudaGetLastError();
        a.type = cudaMemoryTypeUnregistered;
    }
    if ((a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == g.device) return true;
    t_err = std::string(what) + ": " + name + " is not device memory of the library's device";
    return false;
}

// One list of values per bitmap, the argument of the set builders and of the add_many / remove_many
// updates: bitmap k < n takes vals[off[k] .. off[k + 1]).  vals and off are both host memory, or both
// device memory of the library's device (device: the *_device entry points read the values in place).
template <typename V>
struct ValueLists {
    const V *vals;
    const uint64_t *off;
    size_t n;
    bool device;
    const uint64_t *h_off = nullptr;   // after check(): the checked offsets on the host; null: presorted()
    uint64_t N = 0;                    // after check(): the number of values
    PinBlock<uint64_t> read_back;      // device offsets as check() read them

    ValueLists(const V *vals_, const uint64_t *off_, size_t n_, bool device_)
        : vals(vals_), off(off_), n(n_), device(device_) {}
    // Device offsets of N values in segments that are sorted already (the buckets of the 64-bit
    // builder): never checked, and never sorted again.
    static ValueLists presorted(const V *d_vals, const uint64_t *d_off, size_t n, uint64_t N) {
        ValueLists in(d_vals, d_off, n, true);
        in.N = N;
        return in;
    }

    // Refuse lists no kernel may read, then ready the library's device; host lists are refused before
    // any CUDA call.  n < 2^32; off not NULL, off[0] == 0, non-decreasing; vals not NULL unless there
    // are no values.  Device offsets are read back and checked here, and the builder uploads that
    // checked copy.  `what` names the entry point in t_err; `name`, if given, names it in the messages
    // about n and the offsets' values instead (set_from_uint32_device reports those as set_from_uint32).
    bool check(const char *what, const char *name = nullptr) {
        const std::string head = std::string(name ? name : what) + ": ";
        if (n > 0xffffffffull) {
            t_err = head + std::to_string((uint64_t)n) + " bitmaps, at most 2^32 - 1 fit in a set";
            return false;
        }
        if (!off) { t_err = std::string(what) + ": offsets are NULL"; return false; }
        h_off = off;
        if (device) {
            // a host pointer never reaches the read back or a kernel
            if (!ctx_init() || (vals && !device_memory(what, "vals", vals)) || !device_memory(what, "off", off) ||
                !read_back.reset(n + 1))
                return false;
            if (cudaMemcpyAsync(read_back.get(), off, 8 * (n + 1), cudaMemcpyDeviceToHost, g.stream) != cudaSuccess ||
                cudaStreamSynchronize(g.stream) != cudaSuccess) {
                (void)cudaGetLastError();
                t_err = std::string(what) + ": offsets are not readable device memory of the library's device";
                return false;
            }
            h_off = read_back.get();
        }
        if (h_off[0] != 0) {
            t_err = head + "offsets must start at 0 (off[0] = " + std::to_string(h_off[0]) + ")";
            return false;
        }
        for (size_t i = 0; i < n; i++)
            if (h_off[i + 1] < h_off[i]) {
                t_err = head + "offsets decrease at bitmap " + std::to_string((uint64_t)i) + " (off[" +
                        std::to_string((uint64_t)i) + "] = " + std::to_string(h_off[i]) + ", off[" +
                        std::to_string((uint64_t)i + 1) + "] = " + std::to_string(h_off[i + 1]) + ")";
                return false;
            }
        N = h_off[n];
        if (!vals && N) { t_err = std::string(what) + ": values are NULL"; return false; }
        return device || ctx_init();
    }
};

// Segmented sort of src (n segments: h_off on the host, d_off on the device) into `sorted`, a new device
// buffer of h_off[n] values; the input stays as it was.  cub sorts fewer than 2^31 values per call, so
// the segments go in chunks of that size; a segment too large for one call is sorted already (the
// measure pass refuses it otherwise) and is copied.  temp: the caller's scratch, grown here.
template <typename T>
static bool sort_segments(const T *src, const uint64_t *h_off, const uint64_t *d_off, size_t n, DevBlock<T> &sorted,
                          DevBlock<uint8_t> &temp) {
    struct Chunk { uint64_t s0, s1; bool copy; };
    std::vector<Chunk> chunks;
    const uint64_t LIM = (1ull << 31) - 1, N = h_off[n];
    for (uint64_t s0 = 0; s0 < n;) {
        uint64_t s1 = s0;
        while (s1 < n && h_off[s1 + 1] - h_off[s0] <= LIM && s1 - s0 < LIM - 1) s1++;
        if (s1 == s0) { chunks.push_back({s0, s0 + 1, true}); s0++; continue; }
        chunks.push_back({s0, s1, false});
        s0 = s1;
    }
    size_t sort_bytes = 0;
    uint64_t max_seg = 0;
    bool ok = true;
    for (const Chunk &c : chunks) {
        const uint64_t items = h_off[c.s1] - h_off[c.s0];
        if (c.copy || !items) continue;
        size_t b = 0;
        if (!build_sort_chunk(nullptr, &b, src, (T *)nullptr, nullptr, h_off[c.s0], items, (uint32_t)(c.s1 - c.s0),
                              nullptr, g.stream)) { ok = false; break; }
        sort_bytes = std::max(sort_bytes, b);
        max_seg = std::max(max_seg, c.s1 - c.s0);
    }
    if (ok && sort_bytes > temp.bytes()) ok = temp.reset(sort_bytes);
    DevBlock<int> rel;   // stream-ordered reuse only
    ok = ok && sorted.reset(N) && rel.reset(max_seg + 1);
    for (size_t k = 0; k < chunks.size() && ok; k++) {
        const Chunk &c = chunks[k];
        const uint64_t first = h_off[c.s0], items = h_off[c.s1] - first;
        if (!items) continue;
        if (c.copy) {
            ok = cudaMemcpyAsync(sorted.get() + first, src + first, sizeof(T) * items, cudaMemcpyDeviceToDevice,
                                 g.stream) == cudaSuccess;
        } else {
            size_t b = temp.bytes();
            ok = build_sort_chunk(temp.get(), &b, src, sorted.get(), d_off + c.s0, first, items, (uint32_t)(c.s1 - c.s0),
                                  rel.get(), g.stream);
        }
    }
    return ok;
}

// The first passes of the set builders (rb200_build.cu), the same for 32- and 64-bit values: the
// offsets and host values go to the device, then the measure pass counts per tile the starts of the
// containers (32-bit) or buckets (64-bit) and scans them, so the total is their count if every
// bitmap's values are sorted.  Unsorted bitmaps are sorted by segment and measured again.
template <typename V>
struct BuildInput {
    const char *what;         // the builder, in messages
    const ValueLists<V> &lists;   // checked by the entry point, or presorted
    size_t n;
    uint64_t N, ntiles;
    const uint64_t *h_off;    // checked host offsets; null: presorted device segments
    const uint64_t *offs = nullptr;   // the offsets on the device
    const V *src = nullptr;   // the values on the device, sorted once measure_sorted() returned true
    DevBlock<uint64_t> d_off, tcnt, tbase;
    DevBlock<V> vals, sorted;
    DevBlock<uint32_t> flag;
    DevBlock<uint8_t> temp;   // cub scratch, grown by grow_temp()
    PinBlock<uint64_t> meta;  // [count | unsorted flags | two words of the caller's]

    BuildInput(const char *what_, const ValueLists<V> &lists_)
        : what(what_), lists(lists_), n(lists_.n), N(lists_.N), ntiles(build_tile_count(lists_.N)), h_off(lists_.h_off) {}
    bool grow_temp(size_t b) { return b <= temp.bytes() || temp.reset(b); }

    // Offsets (the checked host copy uploaded, presorted ones in place) and values (host ones staged,
    // device ones in place) on the device; false: t_err says why.
    bool load() {
        const bool stage_vals = !lists.device;
        if (ntiles >= (1ull << 31) - 1) { t_err = std::string(what) + ": too many values for one call"; return false; }
        if (h_off && !d_off.reset(n + 1)) return false;
        if (stage_vals && !vals.reset(N)) return false;
        if (!tcnt.reset(ntiles + 1) || !tbase.reset(ntiles + 1) || !flag.reset(1) || !meta.reset(4)) return false;
        offs = h_off ? d_off.get() : lists.off;
        src = stage_vals ? vals.get() : lists.vals;
        if (h_off && cudaMemcpyAsync(d_off.get(), h_off, 8 * (n + 1), cudaMemcpyHostToDevice, g.stream) != cudaSuccess)
            return false;
        if (stage_vals && N) {
            H2DStager stage((uint8_t *)vals.get());
            const bool ok = stage.ok && stage.put(lists.vals, sizeof(V) * N) && stage.flush();
            return cudaStreamSynchronize(g.stream) == cudaSuccess && ok;   // the chunks are recycled after this
        }
        return true;
    }

    // launch(src) enqueues the measure kernel over the values; *count: containers (buckets).
    template <typename Launch>
    bool measure_sorted(Launch launch, uint64_t &count) {
        uint64_t *h = meta.get();
        auto measure = [&]() -> bool {
            size_t b = 0;
            if (!build_scan(nullptr, &b, tcnt.get(), tbase.get(), ntiles + 1, g.stream) || !grow_temp(b)) return false;
            launch(src);
            return build_scan(temp.get(), &b, tcnt.get(), tbase.get(), ntiles + 1, g.stream) &&
                   cudaMemcpyAsync(h, tbase.get() + ntiles, 8, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
                   cudaMemcpyAsync(h + 1, flag.get(), 4, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
                   cudaStreamSynchronize(g.stream) == cudaSuccess;
        };
        h[1] = 0;
        if (cudaMemsetAsync(flag.get(), 0, 4, g.stream) != cudaSuccess ||
            cudaMemsetAsync(tcnt.get() + ntiles, 0, 8, g.stream) != cudaSuccess || !measure())
            return false;
        const uint32_t unsorted = (uint32_t)h[1];
        if (unsorted && !h_off) {
            t_err = "internal: presorted segments are not sorted";
            return false;
        }
        if (unsorted & 2u) {
            t_err = std::string(what) + ": a bitmap of 2^31 values or more is not sorted; pass it sorted";
            return false;
        }
        if (unsorted) {
            bool ok = sort_segments(src, h_off, d_off.get(), n, sorted, temp);
            if (ok) {
                src = sorted.get();
                ok = measure();
            }
            if (!ok) {
                if (t_err.empty()) t_err = std::string(what) + ": segmented sort failed";
                return false;
            }
        }
        count = h[0];
        return true;
    }
};
}  // extern "C++"

// roaring_bitmap_of_ptr of every bitmap (rb200_build.cu) of checked or presorted value lists.  Host
// values are staged through pinned chunks, device values read in place.
static rb200_set *from_uint32_impl(const ValueLists<uint32_t> &lists) {
    BuildInput<uint32_t> in("set_from_uint32", lists);
    const size_t n = lists.n;
    const uint64_t N = in.N;
    SetPtr s;
    DevBlock<uint64_t> d_cpos, d_slot;
    SyncCall call("set_from_uint32");
    uint64_t nc = 0;
    bool ok = in.load() && in.measure_sorted([&](const uint32_t *src) {
        launch_build_measure(src, in.offs, (uint32_t)n, N, in.tcnt.get(), in.flag.get(), g.stream);
    }, nc);
    if (ok && nc > 0xffffffffull) { t_err = "set_from_uint32: more than 2^32 - 1 containers"; ok = false; }
    // every container stores at most 2 bytes per input value (an array 2 d <= 2 count, a bitset needs
    // d > 4096, so 8192 < 2 count) plus its 16-byte padding
    if (ok) ok = (s = set_new((uint32_t)n, nc, 2 * N + 16 * nc + 16)) != nullptr;
    if (ok && nc) {
        size_t b = 0;
        ok = d_cpos.reset(nc) && d_slot.reset(nc) && build_scan(nullptr, &b, d_slot.get(), s->out().c_off, nc, g.stream) &&
             in.grow_temp(b);
        if (ok) {
            launch_build_emit(in.src, in.offs, (uint32_t)n, N, in.tbase.get(), s->out().c_key, d_cpos.get(), g.stream);
            launch_build_slots(d_cpos.get(), nc, N, d_slot.get(), g.stream);
            b = in.temp.bytes();
            ok = build_scan(in.temp.get(), &b, d_slot.get(), s->out().c_off, nc, g.stream);
        }
    }
    if (ok) {
        ok = call.begin();
        if (n && !nc) ok = ok && cudaMemsetAsync(s->out().bm_cnt, 0, 4 * n, g.stream) == cudaSuccess &&
                           cudaMemsetAsync(s->out().bm_beg, 0, 4 * n, g.stream) == cudaSuccess;
        if (nc) launch_build_bitmaps(in.offs, (uint32_t)n, d_cpos.get(), nc, s->out().bm_beg, s->out().bm_cnt, g.stream);
        launch_build_write(in.src, d_cpos.get(), nc, N, s->out(), s->slab_cap, g.d_stats, g.stream);
        launch_bitmap_figures(s->out(), (uint32_t)n, g.d_stats, g.stream);
        ok = call.finish(ok);
        if (ok && g.h_stats->error) {
            t_err = "internal: result slab bound exceeded";
            ok = false;
        }
    }
    if (!ok) {
        if (t_err.empty()) t_err = "set_from_uint32 failed";
        return nullptr;
    }
    s->n_containers = nc;
    s->slab_used = g.h_stats->slab_cursor;
    s->portable_bytes = g.h_stats->payload_bytes;
    s->portable_known = true;
    s->mirrors_pending = n > 0;   // containers / bytes / effective bytes per bitmap: k_deser_bitmap_cards wrote them
    return s.release();
}

rb200_set_t *rb200_set_from_uint32(const uint32_t *vals, const uint64_t *off, size_t n) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    ValueLists<uint32_t> lists(vals, off, n, false);
    return lists.check("set_from_uint32") ? from_uint32_impl(lists) : nullptr;
}

rb200_set_t *rb200_set_from_uint32_device(const uint32_t *d_vals, const uint64_t *d_off, size_t n) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    ValueLists<uint32_t> lists(d_vals, d_off, n, true);
    return lists.check("set_from_uint32_device", "set_from_uint32") ? from_uint32_impl(lists) : nullptr;
}

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
    *buf = nullptr;
    *off_out = *len_out = nullptr;
    if (!ctx_init()) return -1;
    if (!resolve(s)) return -1;
    if (reject_lazy(s, "serialize")) return -1;
    const size_t nb = s->n_bitmaps;
    HostArrays out;
    if (!out.alloc(nb, true)) return -1;
    if (nb == 0) return out.hand_out(buf, off_out, len_out);
    DevBlock<uint64_t> d_sz(nb), d_off(nb + 1);
    DevBlock<uint32_t> d_exact(nb), d_hasrun(nb);
    DevBlock<uint8_t> d_blob;
    PinBlock<uint8_t> h_meta(8 * (nb + 1) + 4 * nb);
    SyncCall call;
    uint64_t total = 0;
    bool ok = d_sz && d_off && d_exact && d_hasrun && h_meta;
    if (ok) {
        const SetView v = s->view();
        if (frozen) launch_frozen_measure(v, (uint32_t)nb, d_sz.get(), d_exact.get(), d_hasrun.get(), g.stream);
        else launch_serialize_measure(v, (uint32_t)nb, d_sz.get(), d_exact.get(), d_hasrun.get(), g.stream);
        launch_pack_scan(d_sz.get(), nullptr, (uint32_t)nb, d_off.get(), nullptr, g.stream);
        ok = cudaMemcpyAsync(h_meta.get(), d_off.get(), 8 * (nb + 1), cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaMemcpyAsync(h_meta.get() + 8 * (nb + 1), d_exact.get(), 4 * nb, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaStreamSynchronize(g.stream) == cudaSuccess;
    }
    if (ok) {
        const uint64_t *h_off = (const uint64_t *)h_meta.get();
        const uint32_t *h_exact = (const uint32_t *)(h_meta.get() + 8 * (nb + 1));
        total = h_off[nb];
        for (size_t i = 0; i < nb; i++) { out.off[i] = h_off[i]; out.len[i] = h_exact[i]; }
        out.off[nb] = total;
        ok = d_blob.reset(total) && out.blob.reset(total);
    }
    if (ok) {
        if (frozen) {
            DevBlock<uint64_t> d_cdst(s->n_containers);   // released at once: stream-ordered reuse only
            ok = (bool)d_cdst;
            if (ok) launch_frozen_write(s->view(), (uint32_t)nb, s->n_containers, d_off.get(), d_blob.get(), d_cdst.get(), g.stream);
        } else {
            launch_serialize_write(s->view(), (uint32_t)nb, d_off.get(), d_hasrun.get(), d_blob.get(), g.stream);
        }
        ok = ok && cudaMemcpyAsync(out.blob.get(), d_blob.get(), total, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        ok = call.finish(ok, false);
    }
    g.last_download_bytes = total;
    if (!ok) {
        if (t_err.empty()) t_err = "set_serialize failed";
        return -1;
    }
    return out.hand_out(buf, off_out, len_out);
}

void rb200_serialized_free(char *buf, uint64_t *off, uint64_t *len) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (buf) g_serialized.erase((uint8_t *)buf);
    free(off);
    free(len);
}

// Free many host bitmaps (results of rb200_set_download_all) with several threads.
void rb200_bitmaps_free(roaring_bitmap_t **bms, size_t n) {
    pool_for(n, n < 64 ? 1 : host_workers(), 8, [&](size_t i) { bitmap_free_host(bms[i]); });
}

}  // extern "C"

namespace {
// Host bitmaps as a temporary set bound to them (rb200_set_bind_host): the callers below keep their
// inputs alive for the whole call, so a result's pass-through containers are rebuilt from the
// caller's memory instead of crossing PCIe again.
SetPtr upload_bound(const roaring_bitmap_t *const *bms, size_t n) {
    SetPtr S(rb200_set_upload(bms, n));
    if (S) rb200_set_bind_host(S.get(), 1);
    return S;
}
SetPtr upload_bound(std::initializer_list<const roaring_bitmap_t *> bms) { return upload_bound(bms.begin(), bms.size()); }

// r1 op r2 under `rules` on the batched path: the resident result, NULL on failure (t_err).
SetPtr pair_result(int op, const roaring_bitmap_t *r1, const roaring_bitmap_t *r2, int rules) {
    const SetPtr S = upload_bound({r1, r2});
    if (!S) return nullptr;
    const uint32_t ia = 0, ib = 1;
    return SetPtr(batch_op_impl(op, S.get(), S.get(), &ia, &ib, 1, rules));
}
}  // namespace

extern "C" {

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
    const SetPtr S = upload_bound(all.data(), all.size());
    if (!S) return -1;
    SetPtr R(batch_op_impl(op, S.get(), S.get(), ia.data(), ib.data(), np));
    return R ? rb200_set_download_all(R.get(), out) : -1;
}

}  // extern "C"
namespace rb200 {
void set_error(const std::string &msg) { t_err = msg; }
void parallel_for(size_t n, const std::function<void(size_t)> &fn) { pool_for(n, host_workers(), 1, fn); }
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
            bool was_shared;
            const PortableEntry e = entry_of(ra[side], i, &was_shared);
            if (e.card & CARD_UNKNOWN) return 0;   // lazy state: batched path
            const uint32_t sb = stored_bytes(e.type, e.len), sb16 = round16(sb);
            if (o + sb16 > FUSED_IN_BYTES) return 0;
            memcpy(h + o, e.payload, sb);
            if (sb16 > sb) memset(h + o + sb, 0, sb16 - sb);
            c_key[ci] = e.key;
            c_type[ci] = e.type;
            c_shared[ci] = was_shared ? 1 : 0;
            c_card[ci] = e.card;
            c_len[ci] = e.len;
            c_off[ci] = (uint32_t)o;
            o += sb16;
            E[side] += effective_bytes(e.type, e.len, e.card);
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
    rr->flags = result_cow(op, rules, ra[0]->flags, ra[1]->flags, ra[0]->size == 0, ra[1]->size == 0);
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
    const SetPtr S = upload_bound(rs, number);
    if (!S) return nullptr;
    SetPtr R(rb200_or_many(S.get(), nullptr, number));
    return R ? rb200_set_download(R.get(), 0) : nullptr;
}

// The end of an in-place call: the result `out` (consumed) replaces x1's directory and containers
// (the old ones are released); x1 takes the result's COW flag, which follows the in-place rules of
// result_cow, and keeps its other flags.  Without a result x1 is left untouched and the failure of
// `fn` is reported.
static void finish_inplace(roaring_bitmap_t *x1, roaring_bitmap_t *out, const char *fn) {
    if (!out) { dropin_failed(fn); return; }
    roaring_array_t *ra = &x1->high_low_container, *rn = &out->high_low_container;
    const uint8_t flags = ra->flags;
    if (!(flags & FLAG_FROZEN)) {
        for (int32_t i = 0; i < ra->size; i++) container_free_host(ra->containers[i], ra->typecodes[i]);
        h_free(ra->containers);
    }
    *ra = *rn;
    ra->flags = (flags & ~FLAG_COW) | (rn->flags & FLAG_COW);
    h_free(out);
}
// In-place twins (src/roaring.c:812 and_inplace, :1063 or_inplace, :1200 xor_inplace, :1342
// andnot_inplace): the result is computed on the device with the in-place type rules and then
// swapped into x1.
static void dropin_inplace(int op, roaring_bitmap_t *x1, const roaring_bitmap_t *x2, int rules = RULES_INPLACE) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    roaring_bitmap_t *out = nullptr;
    // (the lazy in-place twins take the batched path)
    const int f = rules == RULES_INPLACE ? pair_fused(op, x1, x2, RULES_INPLACE, &out) : 0;
    if (f == 0) {
        const SetPtr R = pair_result(op, x1, x2, rules);
        out = R ? rb200_set_download(R.get(), 0) : nullptr;
    }
    finish_inplace(x1, out, "roaring_bitmap_*_inplace");
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
    const SetPtr S = upload_bound(rs, number);
    if (!S) return nullptr;
    SetPtr R(rb200_xor_many(S.get(), nullptr, number));
    return R ? rb200_set_download(R.get(), 0) : nullptr;
}

uint64_t roaring_bitmap_and_cardinality(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    const SetPtr S = upload_bound({r1, r2});
    if (!S) return UINT64_MAX;
    const uint32_t ia = 0, ib = 1;
    uint64_t out = UINT64_MAX;
    if (rb200_batch_and_cardinality(S.get(), S.get(), &ia, &ib, 1, &out) != 0) out = UINT64_MAX;
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
    const SetPtr S = upload_bound({r1, r2});
    if (!S) { dropin_failed("roaring_bitmap_equals / is_subset / is_strict_subset"); return -1; }
    const uint32_t ia = 0, ib = 1;
    uint8_t out = 0;
    const int rc = rb200_batch_relations(S.get(), S.get(), &ia, &ib, 1, &out);
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

// ---- shift: roaring_bitmap_add_offset (src/roaring.c:2426-2507) ----------------------------------
// result[k] = S[idx[k]] with offsets[k] added to every value.  Every source container owns two item
// slots, its lo and its hi part (rb200_offset.cu); k_finalize_pairs compacts them into the result
// directory.  Key-aligned shifts (offset % 65536 == 0) share the operand's containers, or copy them
// when S shares containers itself (holds never chain, see rb200_set::held); one batch may mix both.
rb200_set_t *rb200_batch_add_offset(const rb200_set_t *S, const uint32_t *idx, size_t n, const int64_t *offsets) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!offsets) { t_err = "add_offset: offsets is NULL"; return nullptr; }
    Selection sel{S, idx, n};
    if (!sel.check("add_offset") || !ctx_init() || !ensure_mirrors(S)) return nullptr;
    n = sel.n;
    // item slots and the result slab, sized from the host mirrors before the launch.  A computed
    // container holds at most min(8192, 2 x its cardinality) bytes (offset_type: a run is kept only
    // when it is no larger, a bitset only above 4096 values), and its parts come from at most two
    // sources, each feeding at most two containers: 2 x the effective bytes of the operand, plus the
    // 16-byte rounding of every slot.  Copied key-aligned containers take their stored bytes.
    const size_t o_off = 0, o_idx = al256(8 * (n + 1)), o_ofs = o_idx + al256(4 * n), bytes = o_ofs + al256(8 * n);
    PinBlock<uint8_t> h(bytes);
    DevBlock<uint8_t> d(bytes);
    if (!h || !d) return nullptr;
    uint64_t *off = (uint64_t *)(h.get() + o_off);
    uint32_t *hidx = (uint32_t *)(h.get() + o_idx);
    int64_t *hofs = (int64_t *)(h.get() + o_ofs);
    uint64_t w = 0, sb = 64, sb_copy = 0;
    bool any_aligned = false;
    for (size_t p = 0; p < n; p++) {
        const uint32_t b = sel[p];
        hidx[p] = b;
        hofs[p] = offsets[p];
        off[p] = w;
        w += 2 * (uint64_t)S->h_cnt[b];
        if ((offsets[p] & 0xffff) == 0) {
            any_aligned = true;
            sb_copy += S->h_bytes[b];
        } else {
            sb += 2 * S->h_ebytes[b] + 32 * (uint64_t)S->h_cnt[b];
        }
    }
    off[n] = w;
    if (w > 0xffffffffull) { t_err = "add_offset: batch too large: more than 2^32 - 1 container slots, split it"; return nullptr; }
    const bool share = any_aligned && !S->sharing();
    SetPtr R = set_new((uint32_t)n, w, share ? sb : sb + sb_copy);
    PassShare sh = {false, false, 0, 0, 0};
    if (R && share && !share_operands(R.get(), S, S, true, false, sh)) {
        R.reset();   // out of the offsets' reach: copy everything into a slab sized for it
        R = set_new((uint32_t)n, w, sb + sb_copy);
    }
    ItemsBuf ib_;
    DevBlock<uint4> cell;
    DeferredCall call("add_offset", R, h);
    const bool ok = R && ib_.alloc(w, false, false) && cell.reset(w) && call.begin() &&
                    cudaMemcpyAsync(d.get(), h.get(), bytes, cudaMemcpyHostToDevice, g.stream) == cudaSuccess;
    if (ok) {
        const SetView vs = S->view();
        const uint64_t *d_off = (const uint64_t *)(d.get() + o_off);
        launch_offset_plan(vs, (const uint32_t *)(d.get() + o_idx), (const int64_t *)(d.get() + o_ofs), d_off,
                           (uint32_t)n, sh, ib_.it, cell.get(), R->slab_cap, g.d_dstats, g.stream);
        launch_offset_cells(vs, ib_.it, cell.get(), w, sh.bias, R->d_slab, g.d_dstats, g.stream);
        launch_finalize_pairs(vs, vs, ib_.it, d_off, (uint32_t)n, sh, R->out(), g.d_dstats, call.deliver(), g.stream);
        R->parentA = S->h_ptr;
        for (size_t p = 0; p < n; p++) R->h_flags[p] = S->h_flags[hidx[p]] & FLAG_COW;   // roaring.c:2449-2450
    }
    return call.finish(ok);
}

// ---- range updates: roaring_bitmap_add_range_closed / remove_range_closed (src/roaring.c:251, 302) --
// result[k] = S[idx[k]] with [mins[k], maxs[k]] added (add) or removed; mins[k] > maxs[k] changes
// nothing.  An add gives item k one slot per container of S[idx[k]] plus one per key of its range, a
// removal one per container (rb200_range.cu); k_finalize_pairs compacts them into the result
// directory.  Containers outside the range are shared with S, or copied when S shares containers
// itself (holds never chain, see rb200_set::held).  This is not a batch op with a range bitmap per item,
// as flip is: the type rules differ from OR / ANDNOT, and every key the range covers whole would cost
// a cell of its own.
extern "C++" {
namespace {
// keys of [lo, hi] (0 for an empty range)
uint64_t range_keys(uint32_t lo, uint32_t hi) { return lo <= hi ? (hi >> 16) - (lo >> 16) + 1 : 0; }

const char *range_too_large = ": batch too large: more than 2^32 - 1 container slots, split it";

rb200_set *range_impl(bool add, const std::string &what, const rb200_set *S, const uint32_t *idx, size_t n,
                      const uint32_t *mins, const uint32_t *maxs) {
    // the ranges of m items; an add whose range keys alone exceed the item slots a batch can address is
    // refused here (a full 32-bit range is 65536 keys per item).  With an idx, n is known before S is read.
    const auto ranges_ok = [&](size_t m) {
        if (m && (!mins || !maxs)) { t_err = what + ": min / max is NULL"; return false; }
        uint64_t keys = 0;
        for (size_t p = 0; add && p < m && keys <= 0xffffffffull; p++) keys += range_keys(mins[p], maxs[p]);
        if (keys > 0xffffffffull) { t_err = what + range_too_large; return false; }
        return true;
    };
    Selection sel{S, idx, n};
    if ((idx && !ranges_ok(n)) || !sel.check(what.c_str()) || (!idx && !ranges_ok(sel.n))) return nullptr;
    n = sel.n;
    if (!ctx_init() || !ensure_mirrors(S)) return nullptr;
    // item slots and the result slab, sized from the host mirrors before the launch: 8 KiB for each
    // of the at most two boundary cells (every result type is at most a bitset), 16 bytes for every
    // key an add writes whole (a full run, or a new key's container_range_of_ones), and the stored
    // bytes of S's containers when they are copied rather than shared.
    const size_t o_off = 0, o_idx = al256(8 * (n + 1)), o_min = o_idx + al256(4 * n), o_max = o_min + al256(4 * n),
                 bytes = o_max + al256(4 * n);
    PinBlock<uint8_t> h(bytes);
    DevBlock<uint8_t> d(bytes);
    if (!h || !d) return nullptr;
    uint64_t *off = (uint64_t *)(h.get() + o_off);
    uint32_t *hidx = (uint32_t *)(h.get() + o_idx), *hmin = (uint32_t *)(h.get() + o_min), *hmax = (uint32_t *)(h.get() + o_max);
    uint64_t w = 0, sb = 64, sb_copy = 0;
    for (size_t p = 0; p < n; p++) {
        const uint32_t b = sel[p];
        const uint64_t nk = range_keys(mins[p], maxs[p]);
        hidx[p] = b;
        hmin[p] = mins[p];
        hmax[p] = maxs[p];
        off[p] = w;
        w += S->h_cnt[b] + (add ? nk : 0);
        sb += (nk ? 2 * (uint64_t)BITSET_BYTES : 0) + (add ? 16 * nk : 0);
        sb_copy += S->h_bytes[b];
    }
    off[n] = w;
    if (w > 0xffffffffull) { t_err = what + range_too_large; return nullptr; }
    const bool share = !S->sharing();
    SetPtr R = set_new((uint32_t)n, w, share ? sb : sb + sb_copy);
    PassShare sh = {false, false, 0, 0, 0};
    if (R && share && !share_operands(R.get(), S, S, true, false, sh)) {
        R.reset();   // out of the offsets' reach: copy everything into a slab sized for it
        R = set_new((uint32_t)n, w, sb + sb_copy);
    }
    ItemsBuf ib_;
    DevBlock<uint4> cell;
    DeferredCall call(what.c_str(), R, h);
    const bool ok = R && ib_.alloc(w, false, false) && cell.reset(2 * n) && call.begin() &&
                    cudaMemcpyAsync(d.get(), h.get(), bytes, cudaMemcpyHostToDevice, g.stream) == cudaSuccess;
    if (ok) {
        const SetView vs = S->view();
        const uint64_t *d_off = (const uint64_t *)(d.get() + o_off);
        launch_range_plan(vs, (const uint32_t *)(d.get() + o_idx), (const uint32_t *)(d.get() + o_min),
                          (const uint32_t *)(d.get() + o_max), d_off, (uint32_t)n, add, sh, ib_.it, cell.get(),
                          R->d_slab, R->slab_cap, g.d_dstats, g.stream);
        launch_range_cells(vs, ib_.it, cell.get(), (uint32_t)n, add, sh.bias, R->d_slab, g.d_dstats, g.stream);
        launch_finalize_pairs(vs, vs, ib_.it, d_off, (uint32_t)n, sh, R->out(), g.d_dstats, call.deliver(), g.stream);
        R->parentA = S->h_ptr;
        for (size_t p = 0; p < n; p++) R->h_flags[p] = sel.cow(p);   // the reference updates S in place
    }
    return call.finish(ok);
}
}  // namespace
}  // extern "C++"

rb200_set_t *rb200_batch_add_range_closed(const rb200_set_t *S, const uint32_t *idx, size_t n, const uint32_t *min,
                                          const uint32_t *max) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return range_impl(true, "add_range_closed", S, idx, n, min, max);
}
rb200_set_t *rb200_batch_remove_range_closed(const rb200_set_t *S, const uint32_t *idx, size_t n, const uint32_t *min,
                                             const uint32_t *max) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return range_impl(false, "remove_range_closed", S, idx, n, min, max);
}

// ---- negation: roaring_bitmap_flip (src/roaring.c:2289-2349) ------------------------------------
// result[k] = S[idx[k]] with [range_start, range_end) negated.  The range is materialised as ONE
// tiny bitmap of run containers (one {lo, hi-lo} run per key it touches) and every flip is a
// symmetric difference with it under the negation type rules (RULES_FLIP), batched like any op.
rb200_set_t *rb200_batch_flip(const rb200_set_t *S, const uint32_t *idx, size_t n, uint64_t range_start,
                              uint64_t range_end) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    Selection sel{S, idx, n};
    if (!sel.check("flip") || !ctx_init()) return nullptr;
    std::vector<uint32_t> ia(sel.n), ib(sel.n, 0);
    for (size_t i = 0; i < sel.n; i++) ia[i] = sel[i];
    // roaring.c:2292 (open range empty / start past the 32-bit universe) and :2303 (the CLOSED
    // range, after the reference's truncation of both ends to 32 bits, is empty): plain copy, the
    // symmetric difference with the empty bitmap
    const bool noop = range_start >= range_end || range_start > (uint64_t)UINT32_MAX + 1 ||
                      (uint32_t)range_start > (uint32_t)(range_end - 1);
    const uint32_t first = (uint32_t)range_start, last = (uint32_t)(range_end - 1);
    const uint32_t hb0 = first >> 16, hb1 = last >> 16, nk = noop ? 0 : hb1 - hb0 + 1;
    std::vector<rle16_t> runs(nk);   // one run {lo, hi - lo} per key
    for (uint32_t k = 0; k < nk; k++) {
        const uint32_t hb = hb0 + k, lo = hb == hb0 ? (first & 0xFFFF) : 0, hi = hb == hb1 ? (last & 0xFFFF) : 0xFFFF;
        runs[k] = rle16_t{(uint16_t)lo, (uint16_t)(hi - lo)};
    }
    const auto range = [&](uint32_t k) {
        return PortableEntry{(uint16_t)(hb0 + k), T_RUN, runs[k].length + 1u, 1, (const uint8_t *)&runs[k]};
    };
    std::vector<uint8_t> blob(portable_size(nk, range));
    write_portable(blob.data(), nk, range);
    const char *bp = (const char *)blob.data();
    const size_t bl = blob.size();
    SetPtr Rg(upload_blobs_impl(&bp, &bl, 1, false));
    if (!Rg) return nullptr;
    rb200_set *R = batch_op_impl(OP_XOR, S, Rg.get(), ia.data(), ib.data(), sel.n, noop ? 0 : (RULES_LAZY | RULES_FLIP));
    // an empty range copies every bitmap with its flag (roaring.c:2293), an empty one included
    if (R && noop) for (size_t p = 0; p < sel.n; p++) R->h_flags[p] = sel.cow(p);
    return R;
}
// ---- point queries: roaring_bitmap_contains / rank / get_index / select (roaring.h:478, src/roaring.c:2862,
// 2916, 2974) ---------------------------------------------------------------------------------------
// out[k] = the answer of bitmap S[idx[k]] about vals[k], a warp per query (rb200_query.cu).  rank, get_index
// and select add the cardinalities of the containers before the answer's; they come from the set's c_cum,
// built once by the first such query.
namespace {
// The arguments of a query call other than its selection: the kind, then vals / out (NULL only if n == 0).
bool query_args(const char *what, int kind, size_t n, const void *vals, const void *out) {
    if (kind < Q_CONTAINS || kind > Q_SELECT) {
        t_err = std::string(what) + ": unknown query kind " + std::to_string(kind);
        return false;
    }
    if (n && !vals) { t_err = std::string(what) + ": vals are NULL"; return false; }
    if (n && !out) { t_err = std::string(what) + ": out is NULL"; return false; }
    return true;
}
// The set's c_cum on the library stream, unless it is there already.  A set without containers has
// none: every bitmap is empty and no query reads it.
bool ensure_cum(const rb200_set *cs) {
    rb200_set *s = const_cast<rb200_set *>(cs);
    const uint64_t nc = s->n_containers;
    if (s->c_cum || !nc) return true;
    if (nc >= 0x7fffffffull) { t_err = "query: more than 2^31 - 2 containers in the set"; return false; }
    DevBlock<uint64_t> cards(nc + 1), cum(nc + 1);
    DevBlock<uint8_t> temp;
    size_t tb = 0;
    if (!cards || !cum) return false;
    if (!build_scan(nullptr, &tb, cards.get(), cum.get(), nc + 1, g.stream) || !temp.reset(tb)) {
        if (t_err.empty()) t_err = "query: scan setup failed";
        return false;
    }
    launch_query_cards(s->view().c_card, nc, cards.get(), g.stream);
    if (!build_scan(temp.get(), &tb, cards.get(), cum.get(), nc + 1, g.stream)) {
        t_err = "query: scan launch failed";
        return false;
    }
    s->c_cum = std::move(cum);   // cards and temp go back to the pool: stream-ordered reuse
    return true;
}
bool query_enqueue(int kind, const rb200_set *S, const uint32_t *d_idx, size_t n, const uint32_t *d_vals,
                   int64_t *d_out, unsigned long long *d_bad) {
    if (kind != Q_CONTAINS && !ensure_cum(S)) return false;
    launch_query(kind, S->view(), S->c_cum.get(), S->n_bitmaps, d_idx, d_vals, (uint32_t)n, d_out, d_bad, g.stream);
    return true;
}
}  // namespace

int rb200_batch_query(int kind, const rb200_set_t *S, const uint32_t *idx, size_t n, const uint32_t *vals,
                      int64_t *out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    Selection sel{S, idx, n};
    if (!sel.check("query") || !query_args("query", kind, sel.n, vals, out)) return -1;   // before any CUDA call
    if (!ctx_init() || !ensure_mirrors(S)) return -1;   // a failed batch op fails here, not as data
    n = sel.n;
    if (!n) return 0;
    // one block each way: [first bad position | idx | vals] up, out down
    const size_t o_idx = al256(8), o_vals = o_idx + (sel.all() ? 0 : al256(4 * n)), o_out = o_vals + al256(4 * n);
    const size_t bytes = o_out + 8 * n;
    PinBlock<uint8_t> h(bytes);
    DevBlock<uint8_t> d(bytes);
    if (!h || !d) return -1;
    memset(h.get(), 0xff, 8);
    if (!sel.all()) memcpy(h.get() + o_idx, idx, 4 * n);
    memcpy(h.get() + o_vals, vals, 4 * n);
    SyncCall call("query", "query launch");
    bool ok = cudaMemcpyAsync(d.get(), h.get(), o_out, cudaMemcpyHostToDevice, g.stream) == cudaSuccess &&
              query_enqueue(kind, S, sel.all() ? nullptr : (const uint32_t *)(d.get() + o_idx), n,
                            (const uint32_t *)(d.get() + o_vals), (int64_t *)(d.get() + o_out),
                            (unsigned long long *)d.get()) &&
              cudaMemcpyAsync(h.get() + o_out, d.get() + o_out, 8 * n, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
    ok = call.finish(ok, false);
    if (ok) memcpy(out, h.get() + o_out, 8 * n);
    return ok ? 0 : -1;
}

int rb200_batch_query_device(int kind, const rb200_set_t *S, const uint32_t *d_idx, size_t n, const uint32_t *d_vals,
                             int64_t *d_out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    Selection sel{S, nullptr, n};
    if (!sel.check("query_device")) return -1;   // the entries of d_idx are checked by the kernel
    if (d_idx) {
        if (n > 0xffffffffull) { t_err = "query_device: more than 2^32 - 1 queries"; return -1; }
        sel.n = n;
    }
    n = sel.n;
    if (!query_args("query_device", kind, n, d_vals, d_out) || !ctx_init()) return -1;
    // a host pointer never reaches the kernel
    if (n && (!device_memory("query_device", "vals", d_vals) || !device_memory("query_device", "out", d_out) ||
              (d_idx && !device_memory("query_device", "idx", d_idx))))
        return -1;
    if (!ensure_mirrors(S)) return -1;
    if (!n) return 0;
    DevBlock<unsigned long long> d_bad(1);
    PinBlock<unsigned long long> h_bad(1);
    if (!d_bad || !h_bad) return -1;
    SyncCall call("query_device", "query_device launch");
    bool ok = cudaMemsetAsync(d_bad.get(), 0xff, 8, g.stream) == cudaSuccess &&
              query_enqueue(kind, S, d_idx, n, d_vals, d_out, d_bad.get()) &&
              cudaMemcpyAsync(h_bad.get(), d_bad.get(), 8, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
    ok = call.finish(ok, false);
    if (ok && *h_bad.get() != ~0ull) {   // the first out-of-range entry, reported as the host check does
        const uint64_t k = *h_bad.get();
        uint32_t v = 0;
        if (cudaMemcpyAsync(&v, d_idx + k, 4, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess)
            cudaStreamSynchronize(g.stream);
        index_error("query_device", k, v, S->n_bitmaps);
        ok = false;
    }
    return ok ? 0 : -1;
}

roaring_bitmap_t *roaring_bitmap_flip(const roaring_bitmap_t *r1, uint64_t range_start, uint64_t range_end) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    const SetPtr S = upload_bound({r1});
    if (!S) return nullptr;
    SetPtr R(rb200_batch_flip(S.get(), nullptr, 1, range_start, range_end));
    return R ? rb200_set_download(R.get(), 0) : nullptr;
}
void roaring_bitmap_flip_inplace(roaring_bitmap_t *r1, uint64_t range_start, uint64_t range_end) {
    if (range_start >= range_end || range_start > (uint64_t)UINT32_MAX + 1) return;  // roaring.c:2353
    if ((uint32_t)range_start > (uint32_t)(range_end - 1)) return;                    // roaring.c:2364
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    finish_inplace(r1, roaring_bitmap_flip(r1, range_start, range_end), "roaring_bitmap_flip_inplace");
}

// ---- 64-bit bitmaps resident on the device (src/roaring64.c) -------------------------------
// roaring64_bitmap_{and,or,xor,andnot} (roaring64.c:1332, 1541, 1663, 1809) apply the same container
// cells to equal high-48-bit keys, and the 64-bit portable format (roaring64.c:2262-2395) stores one
// ordinary 32-bit portable bitmap per high-32 "bucket".  So a resident set of 64-bit bitmaps is one
// ordinary set holding every bucket as a 32-bit bitmap (the inner set: every kernel, mirror and
// deferred counter of 32-bit sets applies to it) plus a bucket directory: per 64-bit bitmap its range
// of inner bitmaps, per bucket its high 32 bits.  The inner set always ends with one empty bitmap, the
// sentinel, in no 64-bit bitmap: a bucket without a partner in the other operand is paired with it.
// A result may hold empty buckets (x XOR x, AND of disjoint keys); they are never planned, counted or
// serialized, as the reference never keeps an empty container.
}  // extern "C"
struct rb200_set64 {
    SetPtr inner;
    uint32_t n = 0, nbuckets = 0;   // 64-bit bitmaps; inner bitmaps, the sentinel included
    PinBlock<uint32_t> h_dir;       // host mirror: [b_beg (n) | b_cnt (n) | high (nbuckets)]
    DevBlock<uint32_t> d_dir;       // the same in device memory (copied there when a kernel first needs it)
    bool dir_on_device = false;
    size_t dir_bytes = 0;
    // exclusive scan of the buckets' cardinalities (nbuckets + 1 entries), built by the first rank /
    // get_index / select query (ensure_bcum)
    DevBlock<uint64_t> b_cum;
    const uint32_t *b_beg() const { return h_dir.get(); }
    const uint32_t *b_cnt() const { return h_dir.get() + n; }
    const uint32_t *high() const { return h_dir.get() + 2 * (size_t)n; }
};
extern "C" {
namespace {
struct R64Bucket { uint32_t high; const char *ptr; size_t len; };
// The bucket headers of one 64-bit portable blob (roaring64.c:2440-2531); nullptr when they are
// well formed, else what is wrong.  The buckets' contents are checked by the device parse.
const char *parse_r64(const char *buf, size_t len, std::vector<R64Bucket> &out) {
    out.clear();
    if (len < 8 || !buf) return "shorter than its 8-byte bucket count";
    uint64_t n;
    memcpy(&n, buf, 8);
    if (n > UINT32_MAX) return "bucket count above 2^32 - 1";
    size_t pos = 8;
    for (uint64_t i = 0; i < n; i++) {
        if (pos + 4 > len) return "truncated: a bucket header runs past the end";
        R64Bucket b;
        memcpy(&b.high, buf + pos, 4);
        pos += 4;
        if (i && b.high <= out.back().high) return "the high 32 bits of the buckets are not strictly increasing";
        b.ptr = buf + pos;
        b.len = walk_portable((const uint8_t *)buf + pos, len - pos, [](const PortableEntry &) {});
        if (!b.len) return "a bucket runs past the end of the blob or is not a 32-bit portable bitmap";
        pos += b.len;
        out.push_back(b);
    }
    return nullptr;
}

void set64_delete(rb200_set64 *s) { delete s; }   // the inner set and both directories go back with it
void Set64Free::operator()(rb200_set64 *s) const { set64_delete(s); }
// A set of n 64-bit bitmaps over nbuckets inner bitmaps; the caller fills h_dir (or d_dir).
Set64Ptr set64_new(uint32_t n, uint32_t nbuckets) {
    Set64Ptr s(new rb200_set64());
    s->n = n;
    s->nbuckets = nbuckets;
    s->dir_bytes = 4 * (2 * (size_t)n + nbuckets);
    if (!s->h_dir.reset(2 * (size_t)n + nbuckets) || !s->d_dir.reset(2 * (size_t)n + nbuckets)) return nullptr;
    return s;
}
// The device copy of the directory, for the serialization kernels; a set that is only an operand
// (the per-call entry points' inputs) never pays this copy.  The caller synchronises the stream
// before h_dir can be released.
bool set64_dir_on_device(const rb200_set64 *cs) {
    rb200_set64 *s = const_cast<rb200_set64 *>(cs);
    if (s->dir_on_device) return true;
    if (cudaMemcpyAsync(s->d_dir.get(), s->h_dir.get(), s->dir_bytes, cudaMemcpyHostToDevice, g.stream) != cudaSuccess) {
        t_err = "set64: directory upload failed";
        return false;
    }
    s->dir_on_device = true;
    return true;
}

// Every bucket of every blob, then the sentinel, as ONE upload_blobs_impl batch (one H2D stream; the
// device parse checks each bucket fully).  The headers are walked first: malformed input is refused
// before any CUDA call.
rb200_set64 *set64_upload_impl(const char *const *bufs, const size_t *lens, size_t n) {
    if (n > 0xffffffffull) { t_err = "set64: more than 2^32 - 1 bitmaps"; return nullptr; }
    std::vector<R64Bucket> bk;
    std::vector<const char *> ptrs;
    std::vector<size_t> blens;
    std::vector<uint32_t> cnt(n), highs;
    for (size_t i = 0; i < n; i++) {
        if (const char *why = parse_r64(bufs[i], lens[i], bk)) {
            t_err = "malformed 64-bit portable bitmap at index " + std::to_string((uint64_t)i) + ": " + why;
            return nullptr;
        }
        cnt[i] = (uint32_t)bk.size();
        for (const R64Bucket &b : bk) {
            ptrs.push_back(b.ptr);
            blens.push_back(b.len);
            highs.push_back(b.high);
        }
        if (ptrs.size() >= 0xffffffffull) { t_err = "set64: more than 2^32 - 2 buckets"; return nullptr; }
    }
    uint8_t empty_blob[8];
    blens.push_back(write_portable(empty_blob, 0, [](uint32_t) { return PortableEntry{}; }));
    ptrs.push_back((const char *)empty_blob);
    highs.push_back(0);
    if (!ctx_init()) return nullptr;
    Set64Ptr s = set64_new((uint32_t)n, (uint32_t)ptrs.size());
    if (!s) return nullptr;
    uint32_t *beg = s->h_dir.get(), *bc = beg + n;
    for (size_t i = 0, b = 0; i < n; b += cnt[i], i++) {
        beg[i] = (uint32_t)b;
        bc[i] = cnt[i];
    }
    memcpy(beg + 2 * n, highs.data(), 4 * highs.size());
    size_t bad = SIZE_MAX;
    s->inner.reset(upload_blobs_impl(ptrs.data(), blens.data(), ptrs.size(), false, &bad));
    if (!s->inner && bad < ptrs.size() - 1) {   // the device refused a bucket: name its 64-bit bitmap
        const size_t i = std::upper_bound(beg, beg + n, (uint32_t)bad) - beg - 1;
        const size_t why = t_err.find(": ");
        t_err = "malformed 64-bit portable bitmap at index " + std::to_string((uint64_t)i) + ": the bucket of high 32 bits " +
                std::to_string(highs[bad]) + (why == std::string::npos ? std::string(" is malformed") : t_err.substr(why));
    }
    return s->inner ? s.release() : nullptr;
}

// Bucket pairs of result[p] = A[ia[p]] op B[ib[p]] from the host mirrors: the two high-32 lists
// merged, empty buckets skipped; a bucket without partner is paired with the other inner set's
// sentinel (OR, XOR, and ANDNOT's left side) or dropped (AND).  cnt[p]: bucket pairs of result p.
struct Plan64 { std::vector<uint32_t> pa, pb, high, cnt; };
bool plan64(int op, const rb200_set64 *A, const rb200_set64 *B, const uint32_t *ia, const uint32_t *ib, size_t np,
            Plan64 &P) {
    if (!ensure_mirrors(A->inner.get()) || !ensure_mirrors(B->inner.get())) return false;
    const uint32_t *ca = A->inner->h_cnt.data(), *cb = B->inner->h_cnt.data();
    const uint32_t *ha = A->high(), *hb = B->high();
    const uint32_t EA = A->nbuckets - 1, EB = B->nbuckets - 1;
    P.cnt.resize(np);
    for (size_t p = 0; p < np; p++) {
        if (ia[p] >= A->n || ib[p] >= B->n) { t_err = "pair index out of range"; return false; }
        uint32_t i = A->b_beg()[ia[p]], j = B->b_beg()[ib[p]];
        const uint32_t ie = i + A->b_cnt()[ia[p]], je = j + B->b_cnt()[ib[p]];
        const size_t first = P.pa.size();
        for (;;) {
            while (i < ie && !ca[i]) i++;
            while (j < je && !cb[j]) j++;
            if (i >= ie && j >= je) break;
            const bool only1 = j >= je || (i < ie && ha[i] < hb[j]);
            const bool only2 = !only1 && (i >= ie || hb[j] < ha[i]);
            const bool keep = only1 ? (op == OP_OR || op == OP_XOR || op == OP_ANDNOT)
                              : only2 ? (op == OP_OR || op == OP_XOR) : true;
            if (keep) {
                P.pa.push_back(only2 ? EA : i);
                P.pb.push_back(only1 ? EB : j);
                P.high.push_back(only2 ? hb[j] : ha[i]);
            }
            if (!only2) i++;
            if (!only1) j++;
        }
        P.cnt[p] = (uint32_t)(P.pa.size() - first);
        if (P.pa.size() >= 0xffffffffull) {   // + the result's sentinel must fit a 32-bit bitmap index
            t_err = "set64 batch: more than 2^32 - 2 bucket pairs, split the pair list";
            return false;
        }
    }
    return true;
}

rb200_set64 *batch_op64_impl(int op, const rb200_set64 *A, const rb200_set64 *B, const uint32_t *ia,
                             const uint32_t *ib, size_t np, int rules = 0) {
    if (!ctx_init()) return nullptr;
    if (op < 0 || op > 3) { t_err = "bad op"; return nullptr; }
    if (np > 0xffffffffull) { t_err = "too many pairs"; return nullptr; }
    Plan64 P;
    if (!plan64(op, A, B, ia, ib, np, P)) return nullptr;
    P.pa.push_back(A->nbuckets - 1);   // (sentinel, sentinel): the result's own sentinel
    P.pb.push_back(B->nbuckets - 1);
    P.high.push_back(0);
    Set64Ptr R = set64_new((uint32_t)np, (uint32_t)P.pa.size());
    if (!R) return nullptr;
    uint32_t *dir = R->h_dir.get();
    for (size_t p = 0, b = 0; p < np; b += P.cnt[p], p++) {
        dir[p] = (uint32_t)b;
        dir[np + p] = P.cnt[p];
    }
    memcpy(dir + 2 * np, P.high.data(), 4 * P.high.size());
    R->inner.reset(batch_op_impl(op, A->inner.get(), B->inner.get(), P.pa.data(), P.pb.data(), P.pa.size(), rules));
    return R->inner ? R.release() : nullptr;
}

int and_cardinality64_impl(const rb200_set64 *A, const rb200_set64 *B, const uint32_t *ia, const uint32_t *ib,
                           size_t np, uint64_t *out) {
    if (!ctx_init()) return -1;
    if (np == 0) return 0;
    Plan64 P;
    if (!plan64(OP_AND, A, B, ia, ib, np, P)) return -1;
    std::vector<uint64_t> c(P.pa.size());
    if (!P.pa.empty() &&
        rb200_batch_and_cardinality(A->inner.get(), B->inner.get(), P.pa.data(), P.pb.data(), P.pa.size(), c.data()) != 0)
        return -1;
    for (size_t p = 0, q = 0; p < np; p++) {
        uint64_t sum = 0;
        for (uint32_t k = 0; k < P.cnt[p]; k++) sum += c[q++];
        out[p] = sum;
    }
    return 0;
}

// Device-side roaring64_bitmap_portable_serialize of every 64-bit bitmap: the buckets' exact 32-bit
// sizes (k_ser_measure), the 64-bit blob sizes and their scan (k_r64_ser_sizes, k_pack_scan), one read
// back of the offsets, then the bucket counts, high words and bucket offsets (k_r64_ser_layout) and
// the buckets themselves (k_ser_write) into one buffer that leaves in one D2H.  Blob starts are
// 16-byte aligned; blob i = *buf + (*off)[i], (*len)[i] bytes.
int serialize64_impl(const rb200_set64 *s, char **buf, uint64_t **off_out, uint64_t **len_out) {
    *buf = nullptr;
    *off_out = *len_out = nullptr;
    if (!ctx_init()) return -1;
    if (!resolve(s->inner.get())) return -1;
    const size_t n = s->n, nb = s->nbuckets;
    HostArrays out;
    if (!out.alloc(n, true)) {
        t_err = "set64_serialize: host allocation failed";
        return -1;
    }
    if (n == 0) return out.hand_out(buf, off_out, len_out);
    const uint32_t *d_beg = s->d_dir.get(), *d_cnt = d_beg + n, *d_high = d_beg + 2 * n;
    DevBlock<uint64_t> d_sz(nb), d_boff(nb), d_s16(n), d_e64(n), d_off(n + 1);
    DevBlock<uint32_t> d_exact(nb), d_hasrun(nb);
    DevBlock<uint8_t> d_blob;
    PinBlock<uint64_t> h_meta(2 * n + 1);
    SyncCall call;
    uint64_t total = 0;
    const SetView v = s->inner->view();
    bool ok = d_sz && d_boff && d_exact && d_hasrun && d_s16 && d_e64 && d_off && h_meta &&
              set64_dir_on_device(s);
    if (ok) {
        launch_serialize_measure(v, (uint32_t)nb, d_sz.get(), d_exact.get(), d_hasrun.get(), g.stream);
        launch_r64_ser_sizes(d_beg, d_cnt, (uint32_t)n, v.bm_cnt, d_exact.get(), d_s16.get(), d_e64.get(), g.stream);
        launch_pack_scan(d_s16.get(), nullptr, (uint32_t)n, d_off.get(), nullptr, g.stream);
        ok = cudaMemcpyAsync(h_meta.get(), d_off.get(), 8 * (n + 1), cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaMemcpyAsync(h_meta.get() + n + 1, d_e64.get(), 8 * n, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess &&
             cudaStreamSynchronize(g.stream) == cudaSuccess;
    }
    if (ok) {
        total = h_meta.get()[n];
        memcpy(out.off, h_meta.get(), 8 * (n + 1));
        memcpy(out.len, h_meta.get() + n + 1, 8 * n);
        ok = d_blob.reset(total + 16) && out.blob.reset(total);   // + the scratch empty buckets write to
    }
    if (ok) {
        launch_r64_ser_layout(d_beg, d_cnt, d_high, (uint32_t)n, (uint32_t)nb, v.bm_cnt, d_exact.get(), d_off.get(),
                              d_boff.get(), d_blob.get(), g.stream);
        launch_serialize_write(v, (uint32_t)nb, d_boff.get(), d_hasrun.get(), d_blob.get(), g.stream);
        ok = cudaMemcpyAsync(out.blob.get(), d_blob.get(), total, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        ok = call.finish(ok, false);
    }
    g.last_download_bytes = total;
    if (!ok) {
        if (t_err.empty()) t_err = "set64_serialize failed";
        return -1;
    }
    return out.hand_out(buf, off_out, len_out);
}

// roaring64_bitmap_of_ptr of every bitmap (rb200_build.cu) of checked value lists: host values staged
// through pinned chunks, device values read in place.
rb200_set64 *from_uint64_impl(const ValueLists<uint64_t> &lists) {
    BuildInput<uint64_t> in("set64_from_uint64", lists);
    const size_t n = lists.n;
    const uint64_t N = in.N;
    Set64Ptr R;
    DevBlock<uint32_t> d_lo;
    DevBlock<uint64_t> d_bpos;
    SyncCall call;
    uint64_t nbk = 0;
    // bucket starts per tile, scanned: the total is the bucket count if the values are sorted
    bool ok = in.load() && in.measure_sorted([&](const uint64_t *src) {
        launch_build64_measure(src, in.offs, (uint32_t)n, N, in.tcnt.get(), in.flag.get(), g.stream);
    }, nbk);
    if (ok && nbk >= 0xffffffffull) { t_err = "set64_from_uint64: more than 2^32 - 2 buckets"; ok = false; }
    if (ok) ok = (R = set64_new((uint32_t)n, (uint32_t)(nbk + 1))) != nullptr;
    if (ok) {
        // bucket k of the inner set = the sorted low halves lo[b_pos[k] .. b_pos[k + 1]); the sentinel
        // is the empty segment [N, N)
        uint32_t *d_dir = R->d_dir.get(), *d_high = d_dir + 2 * n;
        uint64_t *h_meta = in.meta.get();
        h_meta[2] = h_meta[3] = N;
        ok = d_lo.reset(N) && d_bpos.reset(nbk + 2) &&
             cudaMemcpyAsync(d_bpos.get() + nbk, h_meta + 2, 16, cudaMemcpyHostToDevice, g.stream) == cudaSuccess &&
             cudaMemsetAsync(d_high + nbk, 0, 4, g.stream) == cudaSuccess;
        if (ok) {
            launch_build64_split(in.src, in.offs, (uint32_t)n, N, in.tbase.get(), d_lo.get(), d_bpos.get(), d_high, g.stream);
            launch_build_bitmaps(in.offs, (uint32_t)n, d_bpos.get(), nbk, d_dir, d_dir + n, g.stream);
            in.vals.reset();     // stream-ordered reuse: the inner build may take their memory
            in.sorted.reset();
            R->inner.reset(from_uint32_impl(ValueLists<uint32_t>::presorted(d_lo.get(), d_bpos.get(), nbk + 1, N)));
            ok = R->inner && cudaMemcpyAsync(R->h_dir.get(), d_dir, R->dir_bytes, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
            ok = call.finish(ok, false);
            R->dir_on_device = true;
        }
    }
    if (!ok) {
        if (t_err.empty()) t_err = "set64_from_uint64 failed";
        return nullptr;
    }
    return R.release();
}

// a[] then b[] as ONE resident set (one H2D); ib2 = ib shifted past a[]
rb200_set64 *r64_operands(const char *const *a, const size_t *alen, size_t na, const char *const *b,
                          const size_t *blen, size_t nb, const uint32_t *ia, const uint32_t *ib, size_t np,
                          std::vector<uint32_t> &ib2) {
    if (na + nb > 0xffffffffull) { t_err = "too many bitmaps"; return nullptr; }
    ib2.resize(np);
    for (size_t p = 0; p < np; p++) {
        if (ia[p] >= na || ib[p] >= nb) { t_err = "pair index out of range"; return nullptr; }
        ib2[p] = (uint32_t)(ib[p] + na);
    }
    std::vector<const char *> ptrs(a, a + na);
    std::vector<size_t> lens(alen, alen + na);
    ptrs.insert(ptrs.end(), b, b + nb);
    lens.insert(lens.end(), blen, blen + nb);
    return set64_upload_impl(ptrs.data(), lens.data(), ptrs.size());
}

// ---- updates: roaring_bitmap_add_many / remove_many (src/roaring.c:134, 696) and roaring64_bitmap_add_many /
// remove_many (roaring64.c:606, 950) ----------------------------------------------------------------
// result[k] = S[idx[k]] after adding (removing) the values vals[off[k] .. off[k+1]).  The values become
// a set V with roaring_bitmap_of_ptr's builder (from_uint32_impl, from_uint64_impl), and the update is
// the batch op (S[idx[k]], V[k]) under RULES_KEEP_RUN: OR to add, ANDNOT to remove
// (decide_type_keep_run).  The containers the values do not touch stay shared with S.  An added key
// that S lacks takes V's container, which the result holds like any operand's (rb200_set::held), so V
// is freed on return.  A 64-bit update is the same container_add / container_remove per 48-bit key, so
// the inner sets take the same batch op; plan64 keeps the buckets only V holds for OR and drops them
// for ANDNOT, and a bucket a removal empties stays an empty inner bitmap, which is never planned,
// counted or serialized.  device: vals / off are in device memory.
extern "C++" template <typename Set, typename V>
Set *update(int op, const char *what, const Set *S, const uint32_t *idx, size_t n, const V *vals,
            const uint64_t *off, bool device) {
    SelectionOf<Set> sel{S, idx, n};
    if (!sel.check(what)) return nullptr;
    ValueLists<V> lists(vals, off, sel.n, device);
    if (!lists.check(what)) return nullptr;
    std::vector<uint32_t> ia(sel.n), ib(sel.n);
    for (size_t k = 0; k < sel.n; k++) {
        ia[k] = sel[k];
        ib[k] = (uint32_t)k;
    }
    if constexpr (std::is_same<Set, rb200_set>::value) {
        const SetPtr W(from_uint32_impl(lists));
        return W ? batch_op_impl(op, S, W.get(), ia.data(), ib.data(), sel.n, RULES_KEEP_RUN) : nullptr;
    } else {
        const Set64Ptr W(from_uint64_impl(lists));
        return W ? batch_op64_impl(op, S, W.get(), ia.data(), ib.data(), sel.n, RULES_KEEP_RUN) : nullptr;
    }
}

// ---- range updates: roaring64_bitmap_add_range_closed / remove_range_closed (roaring64.c:651, 996) ------
// The same container_add_range / container_remove_range per 48-bit key, so one closed 32-bit range per
// bucket: [min_lo32, 2^32 - 1] on the first bucket of the span (or [min_lo32, max_lo32] when it is also
// the last), all of every middle bucket and [0, max_lo32] on the last.  The buckets are planned here as
// plan64 plans them: a bucket outside the span is a no-op item; an add makes an item of every bucket of
// its span, on the inner set's sentinel where S lacks it; a removal drops the middle buckets
// (roaring64.c:1017-1025).  ONE call of the 32-bit path over the inner set then updates every bucket, and
// a bucket a removal empties stays an empty inner bitmap, which is never planned, counted or serialized.
extern "C++" rb200_set64 *range64_impl(bool add, const std::string &what, const rb200_set64 *S, const uint32_t *idx,
                                       size_t n, const uint64_t *mins, const uint64_t *maxs) {
    // as range_impl: an add whose 48-bit range keys alone exceed the item slots of a batch is refused
    // before any device work (the keys also bound the buckets of the spans)
    const auto ranges_ok = [&](size_t m) {
        if (m && (!mins || !maxs)) { t_err = what + ": min / max is NULL"; return false; }
        uint64_t keys = 0;
        for (size_t p = 0; add && p < m && keys <= 0xffffffffull; p++)
            if (mins[p] <= maxs[p]) keys += (maxs[p] >> 16) - (mins[p] >> 16) + 1;
        if (keys > 0xffffffffull) { t_err = what + range_too_large; return false; }
        return true;
    };
    SelectionOf<rb200_set64> sel{S, idx, n};
    if ((idx && !ranges_ok(n)) || !sel.check(what.c_str()) || (!idx && !ranges_ok(sel.n))) return nullptr;
    n = sel.n;
    if (!ctx_init() || !ensure_mirrors(S->inner.get())) return nullptr;
    const uint32_t *cnt = S->inner->h_cnt.data(), *high = S->high(), E = S->nbuckets - 1;
    std::vector<uint32_t> ib, lo, hi, rhigh, rcnt(n);
    const auto item = [&](uint32_t bucket, uint32_t h, uint32_t l, uint32_t u) {
        ib.push_back(bucket);
        rhigh.push_back(h);
        lo.push_back(l);
        hi.push_back(u);
    };
    for (size_t p = 0; p < n; p++) {
        const uint32_t b = sel[p];
        uint32_t i = S->b_beg()[b];
        const uint32_t ie = i + S->b_cnt()[b];
        const size_t first = ib.size();
        const uint64_t mn = mins[p], mx = maxs[p];
        const bool live = mn <= mx;
        const uint32_t hmin = (uint32_t)(mn >> 32), hmax = (uint32_t)(mx >> 32);
        for (; i < ie && (!live || high[i] < hmin); i++)
            if (cnt[i]) item(i, high[i], 1, 0);
        if (live && add) {
            for (uint64_t h = hmin; h <= hmax; h++) {
                const bool has = i < ie && high[i] == h;
                item(has ? i : E, (uint32_t)h, h == hmin ? (uint32_t)mn : 0u, h == hmax ? (uint32_t)mx : 0xffffffffu);
                i += has;
            }
        } else if (live) {
            for (; i < ie && high[i] <= hmax; i++)
                if (cnt[i] && (high[i] == hmin || high[i] == hmax))
                    item(i, high[i], high[i] == hmin ? (uint32_t)mn : 0u, high[i] == hmax ? (uint32_t)mx : 0xffffffffu);
        }
        for (; i < ie; i++)
            if (cnt[i]) item(i, high[i], 1, 0);
        rcnt[p] = (uint32_t)(ib.size() - first);
        if (ib.size() >= 0xffffffffull) {   // + the result's sentinel must fit a 32-bit bitmap index
            t_err = what + ": more than 2^32 - 2 buckets, split the batch";
            return nullptr;
        }
    }
    item(E, 0, 1, 0);   // the result's own sentinel
    Set64Ptr R = set64_new((uint32_t)n, (uint32_t)ib.size());
    if (!R) return nullptr;
    uint32_t *dir = R->h_dir.get();
    for (size_t p = 0, b = 0; p < n; b += rcnt[p], p++) {
        dir[p] = (uint32_t)b;
        dir[n + p] = rcnt[p];
    }
    memcpy(dir + 2 * n, rhigh.data(), 4 * rhigh.size());
    R->inner.reset(range_impl(add, what, S->inner.get(), ib.data(), ib.size(), lo.data(), hi.data()));
    return R->inner ? R.release() : nullptr;
}

// ---- point queries: roaring64_bitmap_contains / rank / get_index / select (roaring64.c:682, 804, 827, 779) ----
// out[k] = the answer of 64-bit bitmap S[idx[k]] about vals[k], a warp per query (k_query64): the bucket of
// the value's high 32 bits (select: of the rank) in the bitmap's run of inner bitmaps, then the 32-bit answer
// in that inner bitmap.  rank, get_index and select add the cardinalities of the buckets before it; they
// come from the set's b_cum, built once by the first such query from the inner set's c_cum.

// The set's b_cum (and the inner c_cum) on the library stream, unless it is there already.
bool ensure_bcum(const rb200_set64 *cs) {
    rb200_set64 *s = const_cast<rb200_set64 *>(cs);
    if (s->b_cum) return true;
    if (!ensure_cum(s->inner.get())) return false;
    const uint64_t nb = s->nbuckets;
    if (nb >= 0x7fffffffull) { t_err = "set64_query: more than 2^31 - 2 buckets in the set"; return false; }
    DevBlock<uint64_t> cards(nb + 1), cum(nb + 1);
    DevBlock<uint8_t> temp;
    size_t tb = 0;
    if (!cards || !cum) return false;
    if (!build_scan(nullptr, &tb, cards.get(), cum.get(), nb + 1, g.stream) || !temp.reset(tb)) {
        if (t_err.empty()) t_err = "set64_query: scan setup failed";
        return false;
    }
    const SetView v = s->inner->view();
    launch_query64_cards(v.bm_beg, v.bm_cnt, s->inner->c_cum.get(), nb, cards.get(), g.stream);
    if (!build_scan(temp.get(), &tb, cards.get(), cum.get(), nb + 1, g.stream)) {
        t_err = "set64_query: scan launch failed";
        return false;
    }
    s->b_cum = std::move(cum);   // cards and temp go back to the pool: stream-ordered reuse
    return true;
}
bool query64_enqueue(int kind, const rb200_set64 *S, const uint32_t *d_idx, size_t n, const uint64_t *d_vals,
                     uint64_t *d_out, uint8_t *d_found, unsigned long long *d_bad) {
    // an uploaded set has only the host copy of its directory
    if (!set64_dir_on_device(S) || (kind != Q_CONTAINS && !ensure_bcum(S))) return false;
    const rb200_set *I = S->inner.get();
    const uint32_t *beg = S->d_dir.get(), *cnt = beg + S->n, *high = beg + 2 * (size_t)S->n;
    launch_query64(kind, I->view(), I->c_cum.get(), S->b_cum.get(), beg, cnt, high, S->n, d_idx, d_vals, (uint32_t)n,
                   d_out, d_found, d_bad, g.stream);
    return true;
}
}  // namespace

rb200_set64_t *rb200_set64_upload_serialized(const char *const *bufs, const size_t *lens, size_t n) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return set64_upload_impl(bufs, lens, n);
}
rb200_set64_t *rb200_set64_from_uint64(const uint64_t *vals, const uint64_t *off, size_t n) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    ValueLists<uint64_t> lists(vals, off, n, false);
    return lists.check("set64_from_uint64") ? from_uint64_impl(lists) : nullptr;
}
rb200_set64_t *rb200_set64_from_uint64_device(const uint64_t *d_vals, const uint64_t *d_off, size_t n) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    ValueLists<uint64_t> lists(d_vals, d_off, n, true);
    return lists.check("set64_from_uint64_device") ? from_uint64_impl(lists) : nullptr;
}
void rb200_set64_free(rb200_set64_t *s) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    set64_delete(s);
}
size_t rb200_set64_count(const rb200_set64_t *s) { return s->n; }
int rb200_set64_cardinalities(const rb200_set64_t *s, uint64_t *out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (s->n == 0) return 0;
    std::vector<uint64_t> c(s->nbuckets);
    if (rb200_set_cardinalities(s->inner.get(), c.data()) != 0) return -1;
    for (uint32_t i = 0; i < s->n; i++) {
        uint64_t sum = 0;
        for (uint32_t k = 0; k < s->b_cnt()[i]; k++) sum += c[s->b_beg()[i] + k];
        out[i] = sum;
    }
    return 0;
}
rb200_set64_t *rb200_set64_batch_op(int op, const rb200_set64_t *A, const rb200_set64_t *B, const uint32_t *ia,
                                    const uint32_t *ib, size_t npairs) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return batch_op64_impl(op, A, B, ia, ib, npairs);
}
int rb200_set64_batch_and_cardinality(const rb200_set64_t *A, const rb200_set64_t *B, const uint32_t *ia,
                                      const uint32_t *ib, size_t npairs, uint64_t *out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return and_cardinality64_impl(A, B, ia, ib, npairs, out);
}
rb200_set_t *rb200_batch_add_many(const rb200_set_t *S, const uint32_t *idx, size_t n, const uint32_t *vals,
                                  const uint64_t *off) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return update(OP_OR, "add_many", S, idx, n, vals, off, false);
}
rb200_set_t *rb200_batch_remove_many(const rb200_set_t *S, const uint32_t *idx, size_t n, const uint32_t *vals,
                                     const uint64_t *off) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return update(OP_ANDNOT, "remove_many", S, idx, n, vals, off, false);
}
rb200_set_t *rb200_batch_add_many_device(const rb200_set_t *S, const uint32_t *idx, size_t n, const uint32_t *d_vals,
                                         const uint64_t *d_off) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return update(OP_OR, "add_many_device", S, idx, n, d_vals, d_off, true);
}
rb200_set_t *rb200_batch_remove_many_device(const rb200_set_t *S, const uint32_t *idx, size_t n,
                                            const uint32_t *d_vals, const uint64_t *d_off) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return update(OP_ANDNOT, "remove_many_device", S, idx, n, d_vals, d_off, true);
}
rb200_set64_t *rb200_set64_batch_add_many(const rb200_set64_t *S, const uint32_t *idx, size_t n, const uint64_t *vals,
                                          const uint64_t *off) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return update(OP_OR, "set64_add_many", S, idx, n, vals, off, false);
}
rb200_set64_t *rb200_set64_batch_remove_many(const rb200_set64_t *S, const uint32_t *idx, size_t n,
                                             const uint64_t *vals, const uint64_t *off) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return update(OP_ANDNOT, "set64_remove_many", S, idx, n, vals, off, false);
}
rb200_set64_t *rb200_set64_batch_add_many_device(const rb200_set64_t *S, const uint32_t *idx, size_t n,
                                                 const uint64_t *d_vals, const uint64_t *d_off) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return update(OP_OR, "set64_add_many_device", S, idx, n, d_vals, d_off, true);
}
rb200_set64_t *rb200_set64_batch_remove_many_device(const rb200_set64_t *S, const uint32_t *idx, size_t n,
                                                    const uint64_t *d_vals, const uint64_t *d_off) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return update(OP_ANDNOT, "set64_remove_many_device", S, idx, n, d_vals, d_off, true);
}
rb200_set64_t *rb200_set64_batch_add_range_closed(const rb200_set64_t *S, const uint32_t *idx, size_t n,
                                                  const uint64_t *min, const uint64_t *max) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return range64_impl(true, "set64_add_range_closed", S, idx, n, min, max);
}
rb200_set64_t *rb200_set64_batch_remove_range_closed(const rb200_set64_t *S, const uint32_t *idx, size_t n,
                                                     const uint64_t *min, const uint64_t *max) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return range64_impl(false, "set64_remove_range_closed", S, idx, n, min, max);
}
rb200_set64_t *rb200_set64_run_optimize(const rb200_set64_t *S, int mode) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return nullptr;
    Set64Ptr R = set64_new(S->n, S->nbuckets);
    if (!R) return nullptr;
    memcpy(R->h_dir.get(), S->h_dir.get(), S->dir_bytes);
    R->inner.reset(convert_impl(S->inner.get(), mode ? 1 : 0));
    return R->inner ? R.release() : nullptr;
}
int rb200_set64_serialize(const rb200_set64_t *s, char **buf, uint64_t **off, uint64_t **len) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    return serialize64_impl(s, buf, off, len);
}

int rb200_set64_batch_query(int kind, const rb200_set64_t *S, const uint32_t *idx, size_t n, const uint64_t *vals,
                            uint64_t *out, uint8_t *found) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    SelectionOf<rb200_set64> sel{S, idx, n};
    if (!sel.check("set64_query") || !query_args("set64_query", kind, sel.n, vals, out)) return -1;   // before any CUDA call
    if (!ctx_init() || !ensure_mirrors(S->inner.get())) return -1;   // a failed batch op fails here, not as data
    n = sel.n;
    if (!n) return 0;
    // one block each way: [first bad position | idx | vals] up, [out | found] down
    const size_t o_idx = al256(8), o_vals = o_idx + (sel.all() ? 0 : al256(4 * n)), o_out = o_vals + al256(8 * n);
    const size_t o_found = o_out + 8 * n, bytes = o_found + n;
    PinBlock<uint8_t> h(bytes);
    DevBlock<uint8_t> d(bytes);
    if (!h || !d) return -1;
    memset(h.get(), 0xff, 8);
    if (!sel.all()) memcpy(h.get() + o_idx, idx, 4 * n);
    memcpy(h.get() + o_vals, vals, 8 * n);
    SyncCall call("set64_query", "set64_query launch");
    bool ok = cudaMemcpyAsync(d.get(), h.get(), o_out, cudaMemcpyHostToDevice, g.stream) == cudaSuccess &&
              query64_enqueue(kind, S, sel.all() ? nullptr : (const uint32_t *)(d.get() + o_idx), n,
                              (const uint64_t *)(d.get() + o_vals), (uint64_t *)(d.get() + o_out), d.get() + o_found,
                              (unsigned long long *)d.get()) &&
              cudaMemcpyAsync(h.get() + o_out, d.get() + o_out, 9 * n, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
    ok = call.finish(ok, false);
    if (ok) {
        memcpy(out, h.get() + o_out, 8 * n);
        if (found) memcpy(found, h.get() + o_found, n);
    }
    return ok ? 0 : -1;
}

int rb200_set64_batch_query_device(int kind, const rb200_set64_t *S, const uint32_t *d_idx, size_t n,
                                   const uint64_t *d_vals, uint64_t *d_out, uint8_t *d_found) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    SelectionOf<rb200_set64> sel{S, nullptr, n};
    if (!sel.check("set64_query_device")) return -1;   // the entries of d_idx are checked by the kernel
    if (d_idx) {
        if (n > 0xffffffffull) { t_err = "set64_query_device: more than 2^32 - 1 queries"; return -1; }
        sel.n = n;
    }
    n = sel.n;
    if (!query_args("set64_query_device", kind, n, d_vals, d_out) || !ctx_init()) return -1;
    // a host pointer never reaches the kernel
    const char *what = "set64_query_device";
    if (n && (!device_memory(what, "vals", d_vals) || !device_memory(what, "out", d_out) ||
              (d_idx && !device_memory(what, "idx", d_idx)) || (d_found && !device_memory(what, "found", d_found))))
        return -1;
    if (!ensure_mirrors(S->inner.get())) return -1;
    if (!n) return 0;
    DevBlock<unsigned long long> d_bad(1);
    PinBlock<unsigned long long> h_bad(1);
    if (!d_bad || !h_bad) return -1;
    SyncCall call(what, "set64_query_device launch");
    bool ok = cudaMemsetAsync(d_bad.get(), 0xff, 8, g.stream) == cudaSuccess &&
              query64_enqueue(kind, S, d_idx, n, d_vals, d_out, d_found, d_bad.get()) &&
              cudaMemcpyAsync(h_bad.get(), d_bad.get(), 8, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
    ok = call.finish(ok, false);
    if (ok && *h_bad.get() != ~0ull) {   // the first out-of-range entry, reported as the host check does
        const uint64_t k = *h_bad.get();
        uint32_t v = 0;
        if (cudaMemcpyAsync(&v, d_idx + k, 4, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess)
            cudaStreamSynchronize(g.stream);
        index_error(what, k, v, S->n);
        ok = false;
    }
    return ok ? 0 : -1;
}

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
    std::vector<uint32_t> ib2;
    Set64Ptr S(r64_operands(a, alen, na, b, blen, nb, ia, ib, np, ib2));
    if (!S) return -1;
    Set64Ptr R(batch_op64_impl(op, S.get(), S.get(), ia, ib2.data(), np));
    return R ? serialize64_impl(R.get(), out, off_out, len_out) : -1;
}

// out[k] = roaring64_bitmap_and_cardinality(a[ia[k]], b[ib[k]]) (roaring64.c:1375)
int rb200_r64_batch_and_cardinality_serialized(const char *const *a, const size_t *alen, size_t na,
                                               const char *const *b, const size_t *blen, size_t nb,
                                               const uint32_t *ia, const uint32_t *ib, size_t np, uint64_t *out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!ctx_init()) return -1;
    std::vector<uint32_t> ib2;
    Set64Ptr S(r64_operands(a, alen, na, b, blen, nb, ia, ib, np, ib2));
    if (!S) return -1;
    return and_cardinality64_impl(S.get(), S.get(), ia, ib2.data(), np, out);
}

// ---- in-memory roaring64_bitmap_t (include/roaring/roaring64.h:423-522; src/roaring64.c:1332-1895)
// The 64-bit bitmap is an ART of (high-48 key -> container) owned by the reference library; its
// layout is private to that library (src/art/art.c), so the binding goes through the two format
// functions the reference exports for exactly this purpose: the operands are written with the
// HOST APPLICATION's roaring64_bitmap_portable_serialize (resolved with dlsym in the running
// process — the reference must be loaded, or nobody could have built a roaring64_bitmap_t), the
// container grid runs on the device (a resident rb200_set64_t), and the result bytes become
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

// out[k] = the host library's deserialization of blob k (in parallel); all or nothing
bool r64_deserialize_all(const char *blob, const uint64_t *off, const uint64_t *len, size_t n,
                         roaring64_bitmap_t **out) {
    std::atomic<bool> ok(true);
    rb200::parallel_for(n, [&](size_t k) {
        out[k] = g_r64.deser(blob + off[k], (size_t)len[k]);
        if (!out[k]) ok = false;
    });
    if (ok) return true;
    // the results that were built go back to the host library
    auto r64_free = (void (*)(roaring64_bitmap_t *))dlsym(RTLD_DEFAULT, "roaring64_bitmap_free");
    for (size_t k = 0; k < n; k++) {
        if (out[k] && r64_free) r64_free(out[k]);
        out[k] = nullptr;
    }
    t_err = "roaring64: the host library refused a result blob";
    return false;
}

// The in-memory operands of rb200_r64_batch_*: a[k] and b[k] written by the host library, pair k
// made of a[k] and b[k].
struct R64Pairs {
    std::vector<std::vector<char>> sa, sb;
    std::vector<const char *> pa, pb;
    std::vector<size_t> la, lb;
    std::vector<uint32_t> idx;   // 0 .. npairs - 1, the pair list of either side
    bool build(const roaring64_bitmap_t *const *a, const roaring64_bitmap_t *const *b, size_t npairs) {
        if (!r64_serialize_all(a, npairs, sa) || !r64_serialize_all(b, npairs, sb)) return false;
        pa.resize(npairs), pb.resize(npairs), la.resize(npairs), lb.resize(npairs), idx.resize(npairs);
        for (size_t k = 0; k < npairs; k++) {
            pa[k] = sa[k].data(); la[k] = g_r64.size(a[k]);
            pb[k] = sb[k].data(); lb[k] = g_r64.size(b[k]);
            idx[k] = (uint32_t)k;
        }
        return true;
    }
};
}  // namespace

rb200_set64_t *rb200_set64_upload(const roaring64_bitmap_t *const *bitmaps, size_t n) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!g_r64.ok()) return nullptr;
    std::vector<std::vector<char>> bufs;
    if (!r64_serialize_all(bitmaps, n, bufs)) return nullptr;
    std::vector<const char *> ptrs(n);
    std::vector<size_t> lens(n);
    for (size_t i = 0; i < n; i++) {
        ptrs[i] = bufs[i].data();
        lens[i] = g_r64.size(bitmaps[i]);
    }
    return set64_upload_impl(ptrs.data(), lens.data(), n);
}

int rb200_set64_download_all(const rb200_set64_t *s, roaring64_bitmap_t **out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!g_r64.ok()) return -1;
    char *blob = nullptr;
    uint64_t *off = nullptr, *len = nullptr;
    if (serialize64_impl(s, &blob, &off, &len) != 0) return -1;
    const bool ok = r64_deserialize_all(blob, off, len, s->n, out);
    rb200_serialized_free(blob, off, len);
    return ok ? 0 : -1;
}

// out[k] = roaring64_bitmap_{and,or,xor,andnot}(a[k], b[k]) for npairs in-memory 64-bit bitmaps of the
// host application's CRoaring; out[k] is a fresh roaring64_bitmap_t the caller frees with
// roaring64_bitmap_free.  0 on success.
int rb200_r64_batch_op(int op, const roaring64_bitmap_t *const *a, const roaring64_bitmap_t *const *b,
                       size_t npairs, roaring64_bitmap_t **out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!g_r64.ok()) return -1;
    if (npairs == 0) return 0;
    R64Pairs P;
    if (!P.build(a, b, npairs)) return -1;
    char *blob = nullptr;
    uint64_t *off = nullptr, *len = nullptr;
    if (rb200_r64_batch_op_serialized(op, P.pa.data(), P.la.data(), npairs, P.pb.data(), P.lb.data(), npairs,
                                      P.idx.data(), P.idx.data(), npairs, &blob, &off, &len) != 0)
        return -1;
    const bool ok = r64_deserialize_all(blob, off, len, npairs, out);
    rb200_serialized_free(blob, off, len);
    return ok ? 0 : -1;
}

int rb200_r64_batch_and_cardinality(const roaring64_bitmap_t *const *a, const roaring64_bitmap_t *const *b,
                                    size_t npairs, uint64_t *out) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    if (!g_r64.ok()) return -1;
    if (npairs == 0) return 0;
    R64Pairs P;
    if (!P.build(a, b, npairs)) return -1;
    return rb200_r64_batch_and_cardinality_serialized(P.pa.data(), P.la.data(), npairs, P.pb.data(), P.lb.data(), npairs,
                                                      P.idx.data(), P.idx.data(), npairs, out);
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
roaring_bitmap_t *roaring_bitmap_lazy_or(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2, const bool bitsetconversion) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    const SetPtr R = pair_result(OP_OR, r1, r2, RULES_LAZY | (bitsetconversion ? RULES_CONV : 0));
    return R ? rb200_set_download(R.get(), 0) : nullptr;
}
void roaring_bitmap_lazy_or_inplace(roaring_bitmap_t *r1, const roaring_bitmap_t *r2, const bool bitsetconversion) {
    dropin_inplace(OP_OR, r1, r2, RULES_LAZY | RULES_INPLACE | (bitsetconversion ? RULES_CONV : 0));
}
roaring_bitmap_t *roaring_bitmap_lazy_xor(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    const SetPtr R = pair_result(OP_XOR, r1, r2, RULES_LAZY);
    return R ? rb200_set_download(R.get(), 0) : nullptr;
}
void roaring_bitmap_lazy_xor_inplace(roaring_bitmap_t *r1, const roaring_bitmap_t *r2) {
    dropin_inplace(OP_XOR, r1, r2, RULES_LAZY | RULES_INPLACE);
}
void roaring_bitmap_repair_after_lazy(roaring_bitmap_t *r1) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    const SetPtr S = upload_bound({r1});
    const SetPtr R(S ? rb200_set_repair_after_lazy(S.get()) : nullptr);
    finish_inplace(r1, R ? rb200_set_download(R.get(), 0) : nullptr, "roaring_bitmap_repair_after_lazy");
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
    DevBlock<uint64_t> d16(nb);
    DevBlock<uint32_t> dex(nb), dhr(nb);
    PinBlock<uint32_t> h(nb);
    SyncCall call;
    bool ok = d16 && dex && dhr && h;
    if (ok) {
        launch_serialize_measure(S->view(), (uint32_t)nb, d16.get(), dex.get(), dhr.get(), g.stream);
        ok = cudaMemcpyAsync(h.get(), dex.get(), 4 * nb, cudaMemcpyDeviceToHost, g.stream) == cudaSuccess;
        ok = call.finish(ok, false);
        if (ok) out.assign(h.get(), h.get() + nb);
    }
    if (!ok && t_err.empty()) t_err = "portable_sizes failed";
    return ok;
}
}  // namespace

rb200_set_t *rb200_or_many_heap(const rb200_set_t *S, const uint32_t *idx, size_t n) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    Selection sel{S, idx, n};
    if (!sel.check("or_many_heap") || !ctx_init()) return nullptr;
    if (sel.n == 0) return rb200_or_many(S, idx, 0);
    if (sel.n == 1) {  // roaring_bitmap_copy: union with an empty bitmap = pass-through of every container
        roaring_bitmap_t *e = bitmap_alloc(0);
        if (!e) return nullptr;
        const roaring_bitmap_t *one[1] = {e};
        SetPtr E(rb200_set_upload(one, 1));
        bitmap_free_host(e);
        if (!E) return nullptr;
        const uint32_t a = sel[0], z = 0;
        rb200_set *R = batch_op_impl(OP_OR, S, E.get(), &a, &z, 1, 0);
        if (R) R->h_flags[0] = sel.cow(0);   // the copy's flag, an empty input's included
        return R;
    }
    std::vector<uint32_t> sz;
    if (!portable_sizes(S, sz)) return nullptr;
    std::vector<HeapEl> e(sel.n);
    for (size_t i = 0; i < sel.n; i++) e[i] = HeapEl{sz[sel[i]], false, const_cast<rb200_set *>(S), sel[i]};
    uint32_t cnt = (uint32_t)sel.n;
    for (int32_t i = (int32_t)(cnt >> 1); i >= 0; i--) heap_down(e, cnt, (uint32_t)i);  // create_pq :68-82
    bool ok = true;
    while (cnt > 1 && ok) {
        const HeapEl a = heap_pop(e, cnt), b = heap_pop(e, cnt);
        const SetPtr a_temp(a.temp ? a.set : nullptr), b_temp(b.temp ? b.set : nullptr);  // consumed here
        SetPtr R;
        if (a.temp && b.temp)
            R.reset(batch_op_impl(OP_OR, a.set, b.set, &a.index, &b.index, 1, RULES_LAZY | RULES_INPLACE | RULES_NOFULL));
        else if (b.temp)  // roaring_bitmap_lazy_or_inplace(x2, x1, false)
            R.reset(batch_op_impl(OP_OR, b.set, a.set, &b.index, &a.index, 1, RULES_LAZY | RULES_INPLACE));
        else if (a.temp)
            R.reset(batch_op_impl(OP_OR, a.set, b.set, &a.index, &b.index, 1, RULES_LAZY | RULES_INPLACE));
        else
            R.reset(batch_op_impl(OP_OR, a.set, b.set, &a.index, &b.index, 1, RULES_LAZY));
        if (!R || !resolve(R.get())) { ok = false; break; }
        heap_push(e, cnt, HeapEl{R->out_portable, true, R.release(), 0});  // size measured by k_finalize_pairs
    }
    if (!ok) {
        for (uint32_t i = 0; i < cnt; i++) if (e[i].temp) SetFree()(e[i].set);
        return nullptr;
    }
    const SetPtr top(heap_pop(e, cnt).set);   // n >= 2: a temporary
    return convert_impl(top.get(), 2);        // roaring_bitmap_repair_after_lazy
}

roaring_bitmap_t *roaring_bitmap_or_many_heap(uint32_t number, const roaring_bitmap_t **rs) {
    std::lock_guard<std::recursive_mutex> lk(g.mu);
    const SetPtr S = upload_bound(rs, number);
    if (!S) return nullptr;
    SetPtr R(rb200_or_many_heap(S.get(), nullptr, number));
    return R ? rb200_set_download(R.get(), 0) : nullptr;
}

}  // extern "C"
