/*
 * roaring_b200.h — C ABI of the H100-native Roaring set-algebra engine (libroaring_b200.so).
 *
 * Plain C: only pointers, sizes and PODs cross this boundary; no torch / C++ / CUDA types.
 *
 * Part 1 (DROP-IN) exports, under the reference's own names, exactly the entry points of the
 * hot path of CRoaring 5.1.0 — the functions a caller / FFI binding of the reference binds
 * for set algebra.  Each declaration cites the reference declaration it replaces
 * (paths relative to the reference tree).  They take and return host `roaring_bitmap_t`
 * objects in the reference's memory layout, so every other reference function
 * (roaring_bitmap_free, _contains, _portable_serialize, iterators ...) keeps working on what
 * they return.  The work itself is done by sm_90a CUDA kernels; there is NO CPU fallback:
 * on a CUDA failure they return NULL / UINT64_MAX and rb200_last_error() says why.
 *
 * Part 2 (rb200_*) is the batched, device-resident form the GPU needs to be worth using:
 * upload a set of bitmaps once, run thousands of pairwise ops / an N-way union per launch,
 * keep results on the device, download only what the caller asks for.
 */
#ifndef ROARING_B200_H
#define ROARING_B200_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

/* The reference's own headers, when they are on the include path: its types are then used below,
 * whatever the order in which the application includes the two headers.  (The library itself is
 * built with RB200_BUILDING_LIBRARY: it never depends on an installed copy of the reference.) */
#if !defined(ROARING_H) && !defined(RB200_BUILDING_LIBRARY) && defined(__has_include)
#if __has_include(<roaring/roaring.h>)
#include <roaring/roaring.h>
#endif
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------
 * Layout-compatible types.  If the reference's headers are already included — or can be (they are
 * found on the include path) — we use theirs.
 * include/roaring/roaring_types.h:61-68 (roaring_array_t), include/roaring/roaring.h:39-41
 * (roaring_bitmap_t), containers/array.h:46-50, containers/bitset.h:45-48,
 * containers/run.h:48-51,69-73, containers/containers.h:48-51 (typecodes).
 * ------------------------------------------------------------------------------------- */
#ifndef ROARING_TYPES_H
typedef struct roaring_array_s {
    int32_t size;
    int32_t allocation_size;
    void **containers; /* base of ONE block [containers | keys | typecodes], roaring_array.c:55-66 */
    uint16_t *keys;
    uint8_t *typecodes;
    uint8_t flags; /* ROARING_FLAG_COW = 1, ROARING_FLAG_FROZEN = 2 (roaring_types.h:46-49) */
} roaring_array_t;
#endif
#ifndef ROARING_H
typedef struct roaring_bitmap_s {
    roaring_array_t high_low_container;
} roaring_bitmap_t;
#endif

/* ---------------------------------------------------------------------------------------
 * Part 1 — drop-in hot-path entry points (reference names, reference semantics).
 * ------------------------------------------------------------------------------------- */

/* include/roaring/roaring.h:225  (src/roaring.c:731) */
roaring_bitmap_t *roaring_bitmap_and(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
/* include/roaring/roaring.h:288  (src/roaring.c:877) */
roaring_bitmap_t *roaring_bitmap_or(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
/* include/roaring/roaring.h:320  (src/roaring.c:1121) */
roaring_bitmap_t *roaring_bitmap_xor(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
/* include/roaring/roaring.h:342  (src/roaring.c:1275) */
roaring_bitmap_t *roaring_bitmap_andnot(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
/* include/roaring/roaring.h:304  (src/roaring.c:775) */
roaring_bitmap_t *roaring_bitmap_or_many(size_t number, const roaring_bitmap_t **rs);
/* In-place twins, include/roaring/roaring.h:280,296,328,348 (src/roaring.c:812, 1063, 1200, 1342):
 * same cells with the in-place type rules (container_ior: a saturated bitset|bitset becomes the
 * full run, a full left container is kept as is); the result replaces the contents of r1. */
void roaring_bitmap_and_inplace(roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
void roaring_bitmap_or_inplace(roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
void roaring_bitmap_xor_inplace(roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
void roaring_bitmap_andnot_inplace(roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
/* include/roaring/roaring.h:334  (src/roaring.c:795) */
roaring_bitmap_t *roaring_bitmap_xor_many(size_t number, const roaring_bitmap_t **rs);
/* include/roaring/roaring.h:312  (src/roaring_priority_queue.c:200): pairwise lazy unions in the
 * order of the reference's size-keyed binary heap (the result TYPES depend on that order). */
roaring_bitmap_t *roaring_bitmap_or_many_heap(uint32_t number, const roaring_bitmap_t **rs);
/* Public lazy API, include/roaring/roaring.h:932-977 (src/roaring.c:2509, 2600, 2684, 2763, 2845).
 * The lazy state is kept in ordinary host bitmaps exactly as the reference keeps it (bitset
 * cardinality -1, unconverted runs), so these calls and the reference's own can be mixed. */
roaring_bitmap_t *roaring_bitmap_lazy_or(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2,
                                         const bool bitsetconversion);
void roaring_bitmap_lazy_or_inplace(roaring_bitmap_t *r1, const roaring_bitmap_t *r2,
                                    const bool bitsetconversion);
roaring_bitmap_t *roaring_bitmap_lazy_xor(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
void roaring_bitmap_lazy_xor_inplace(roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
void roaring_bitmap_repair_after_lazy(roaring_bitmap_t *r1);
/* include/roaring/roaring.h:986, 1004 (src/roaring.c:2289, 2351): negation of [range_start,
 * range_end) — the negation cells of mixed_negation.c as one more rule set of the pairwise kernel. */
roaring_bitmap_t *roaring_bitmap_flip(const roaring_bitmap_t *r1, uint64_t range_start, uint64_t range_end);
void roaring_bitmap_flip_inplace(roaring_bitmap_t *r1, uint64_t range_start, uint64_t range_end);
/* include/roaring/roaring.h:231  (src/roaring.c:3048) */
uint64_t roaring_bitmap_and_cardinality(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
/* include/roaring/roaring.h:258-271 (src/roaring.c:3086-3107): inclusion-exclusion on the above */
uint64_t roaring_bitmap_or_cardinality(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
uint64_t roaring_bitmap_andnot_cardinality(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
uint64_t roaring_bitmap_xor_cardinality(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
/* include/roaring/roaring.h:252  (src/roaring.c:3078) */
double roaring_bitmap_jaccard_index(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
/* include/roaring/roaring.h:237  (src/roaring.c:2998) */
bool roaring_bitmap_intersect(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
/* include/roaring/roaring.h:899, 905, 912 (src/roaring.c:2128, 2151, 3172): decided from
 * |r1 and r2|, |r1|, |r2| (same answers as the reference's early-exit container cells). */
bool roaring_bitmap_equals(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
bool roaring_bitmap_is_subset(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);
bool roaring_bitmap_is_strict_subset(const roaring_bitmap_t *r1, const roaring_bitmap_t *r2);

/* ---------------------------------------------------------------------------------------
 * Stand-alone helpers (our own implementations of the steps either side of the path, so the
 * library is usable without linking the reference; when the reference IS loaded in the
 * process its roaring_malloc/roaring_free hooks are used for every host allocation).
 * ------------------------------------------------------------------------------------- */

/* portable format: src/roaring_array.c:469-531 (write), :633-813 (read) */
roaring_bitmap_t *rb200_bitmap_portable_deserialize_safe(const char *buf, size_t maxbytes);
size_t rb200_bitmap_portable_size_in_bytes(const roaring_bitmap_t *r);
size_t rb200_bitmap_portable_serialize(const roaring_bitmap_t *r, char *buf);
/* src/roaring.c:552-560 */
void rb200_bitmap_free(roaring_bitmap_t *r);
/* src/roaring.c:1436 */
uint64_t rb200_bitmap_get_cardinality(const roaring_bitmap_t *r);
/* structural invariants of src/roaring.c:454-523; returns true when valid */
bool rb200_bitmap_validate(const roaring_bitmap_t *r, const char **reason);

/* ---------------------------------------------------------------------------------------
 * Part 2 — batched, device-resident API.
 * ------------------------------------------------------------------------------------- */
typedef struct rb200_set rb200_set_t; /* an ordered collection of bitmaps resident in HBM */

enum { RB200_AND = 0, RB200_OR = 1, RB200_XOR = 2, RB200_ANDNOT = 3 };

/* Context.  rb200_init is optional (first call initialises on the current device).
 * `cuda_stream` is a cudaStream_t passed as void*; NULL selects the library's own stream. */
int rb200_init(int device);
void rb200_set_stream(void *cuda_stream);
void rb200_synchronize(void);
const char *rb200_last_error(void);
/* number of kernels this library has launched since load (bench.py's gpu_launches) */
uint64_t rb200_kernel_launches(void);

/* Upload (H2D): pack n host bitmaps into one device-resident set (one contiguous copy). */
rb200_set_t *rb200_set_upload(const roaring_bitmap_t *const *bitmaps, size_t n);
/* Same from portable-serialized bytes ("identical serialized inputs"). */
rb200_set_t *rb200_set_upload_serialized(const char *const *bufs, const size_t *lens, size_t n);
void rb200_set_free(rb200_set_t *s);
/* Opt-in for sets made by rb200_set_upload: promise that the host bitmaps stay alive and unmodified
 * while results derived from the set are downloaded.  Pass-through containers of batch results
 * (unmatched keys of OR / XOR / ANDNOT) are then rebuilt on the host from the caller's own memory
 * instead of crossing PCIe again.  enable = 0 revokes the promise for later ops. */
int rb200_set_bind_host(rb200_set_t *s, int enable);
size_t rb200_set_count(const rb200_set_t *s);              /* number of bitmaps */
uint64_t rb200_set_container_count(const rb200_set_t *s);   /* total containers */
uint64_t rb200_set_payload_bytes(const rb200_set_t *s);     /* container_size_in_bytes summed */

/* Pairwise batch: result bitmap k = A[ia[k]] op B[ib[k]], k < npairs (ia/ib host arrays).
 * Returns a new device-resident set of npairs bitmaps (NULL on error).  A may equal B. */
rb200_set_t *rb200_batch_op(int op, const rb200_set_t *A, const rb200_set_t *B,
                            const uint32_t *ia, const uint32_t *ib, size_t npairs);

/* Batch ops return as soon as their kernels are queued on the library stream; the op's counters
 * (and a possible internal error) are collected when the result is first used.  This reads them:
 * device time of the whole op / of its compute kernel (CUDA events), algorithmic bytes. */
int rb200_set_op_stats(const rb200_set_t *s, float *device_ms, float *compute_ms, uint64_t *algorithmic_bytes);

/* Same with flags (the results are always new bitmaps):
 *   RB200_INPLACE_RULES    type rules of the in-place twins (roaring_bitmap_or_inplace ...)
 *   RB200_LAZY_RULES       OR / XOR only: the lazy variants (roaring.h:932-977); the result set is
 *                          in a LAZY state — feed it to further lazy ops, download it (the host
 *                          bitmaps carry the reference's lazy representation) or repair it with
 *                          rb200_set_repair_after_lazy; every other entry point refuses it.
 *                          | RB200_INPLACE_RULES = the lazy in-place twins
 *   RB200_LAZY_BITSET_CONVERSION   the `bitsetconversion` argument of the lazy OR functions
 *   RB200_LAZY_FROM_LAZY_INPUTS    with LAZY|INPLACE: no full-container short cut (the heap's
 *                          union of two temporaries, roaring_priority_queue.c:99) */
enum { RB200_INPLACE_RULES = 1, RB200_LAZY_RULES = 2, RB200_LAZY_BITSET_CONVERSION = 4,
       RB200_LAZY_FROM_LAZY_INPUTS = 8 };
rb200_set_t *rb200_batch_op_ex(int op, int flags, const rb200_set_t *A, const rb200_set_t *B,
                               const uint32_t *ia, const uint32_t *ib, size_t npairs);

/* out[k] = |A[ia[k]] AND B[ib[k]]|  (roaring_bitmap_and_cardinality per pair); 0 on success. */
int rb200_batch_and_cardinality(const rb200_set_t *A, const rb200_set_t *B, const uint32_t *ia,
                                const uint32_t *ib, size_t npairs, uint64_t *out);

/* out[k]: bit 0 = roaring_bitmap_equals, bit 1 = is_subset, bit 2 = is_strict_subset of
 * (A[ia[k]], B[ib[k]]); one cardinality sweep on the device.  0 on success. */
int rb200_batch_relations(const rb200_set_t *A, const rb200_set_t *B, const uint32_t *ia,
                          const uint32_t *ib, size_t npairs, uint8_t *out);

/* result[k] = roaring_bitmap_flip(S[idx[k]], range_start, range_end) (idx == NULL: every bitmap). */
rb200_set_t *rb200_batch_flip(const rb200_set_t *S, const uint32_t *idx, size_t n, uint64_t range_start,
                              uint64_t range_end);

/* 64-bit bitmaps (src/roaring64.c) through their portable format: result[k] =
 * roaring64_bitmap_{and,or,xor,andnot}(a[ia[k]], b[ib[k]]) — the same container grid per
 * high-32 bucket.  *out (pinned, owned by the library; blob k at *out + (*off)[k], (*len)[k]
 * bytes) is released with rb200_serialized_free.  Bytes in, bytes out; the in-memory form is
 * rb200_r64_batch_op below. */
int rb200_r64_batch_op_serialized(int op, const char *const *a, const size_t *alen, size_t na,
                                  const char *const *b, const size_t *blen, size_t nb,
                                  const uint32_t *ia, const uint32_t *ib, size_t npairs, char **out,
                                  uint64_t **off, uint64_t **len);
int rb200_r64_batch_and_cardinality_serialized(const char *const *a, const size_t *alen, size_t na,
                                               const char *const *b, const size_t *blen, size_t nb,
                                               const uint32_t *ia, const uint32_t *ib, size_t npairs,
                                               uint64_t *out);

/* In-memory 64-bit bitmaps of the HOST APPLICATION's CRoaring (the ART inside roaring64_bitmap_t is
 * private to that library): operands and results cross through its own
 * roaring64_bitmap_portable_serialize / _deserialize_safe, resolved in the running process.
 * out[k] = a[k] op b[k]; the caller frees out[k] with roaring64_bitmap_free.  0 on success. */
#ifndef ROARING64_H
typedef struct roaring64_bitmap_s roaring64_bitmap_t;
#endif
int rb200_r64_batch_op(int op, const roaring64_bitmap_t *const *a, const roaring64_bitmap_t *const *b,
                       size_t npairs, roaring64_bitmap_t **out);
int rb200_r64_batch_and_cardinality(const roaring64_bitmap_t *const *a, const roaring64_bitmap_t *const *b,
                                    size_t npairs, uint64_t *out);
/* Drop-in symbols of the 64-bit hot path, include/roaring/roaring64.h:423-522
 * (src/roaring64.c:1332, 1375, 1541, 1663, 1809 and the cardinality family). */
roaring64_bitmap_t *roaring64_bitmap_and(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2);
roaring64_bitmap_t *roaring64_bitmap_or(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2);
roaring64_bitmap_t *roaring64_bitmap_xor(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2);
roaring64_bitmap_t *roaring64_bitmap_andnot(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2);
uint64_t roaring64_bitmap_and_cardinality(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2);
uint64_t roaring64_bitmap_or_cardinality(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2);
uint64_t roaring64_bitmap_xor_cardinality(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2);
uint64_t roaring64_bitmap_andnot_cardinality(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2);
double roaring64_bitmap_jaccard_index(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2);
bool roaring64_bitmap_intersect(const roaring64_bitmap_t *r1, const roaring64_bitmap_t *r2);

/* roaring_bitmap_or_many over S[idx[0..n)] (idx == NULL: all bitmaps in order).
 * Returns a device-resident set holding ONE bitmap. */
rb200_set_t *rb200_or_many(const rb200_set_t *S, const uint32_t *idx, size_t n);

/* roaring_bitmap_xor_many over S[idx[0..n)] (idx == NULL: all bitmaps in order): ONE result bitmap. */
rb200_set_t *rb200_xor_many(const rb200_set_t *S, const uint32_t *idx, size_t n);

/* roaring_bitmap_or_many_heap over S[idx[0..n)]: ONE result bitmap.  Sequential by construction
 * (every union's operands depend on the sizes of the previous results): n-1 single-pair lazy ops. */
rb200_set_t *rb200_or_many_heap(const rb200_set_t *S, const uint32_t *idx, size_t n);

/* roaring_bitmap_repair_after_lazy on every bitmap of a set in a lazy state; returns a new set. */
rb200_set_t *rb200_set_repair_after_lazy(const rb200_set_t *S);

/* Key-sharded form used for multi-GPU aggregation: only containers whose high-16 key lies in
 * [key_lo, key_hi] take part; per-key result cardinalities are ADDED into card_per_key[65536]
 * when non-NULL (host array; the caller all-reduces it across ranks). */
rb200_set_t *rb200_or_many_keyrange(const rb200_set_t *S, const uint32_t *idx, size_t n,
                                    uint32_t key_lo, uint32_t key_hi, uint32_t *card_per_key);

/* ---------------------------------------------------------------------------------------
 * Multi-GPU (one process per GPU; SURVEY.md 8(e)).  Pairwise batches shard by PAIR (every rank
 * runs its own slice of the pair list, no data-path collective).  The many-way union shards the
 * HIGH-16 KEY SPACE: contiguous key ranges balanced by input bytes, rank g holds only the
 * containers of range g of every input, reduces them alone, and the ranks exchange ONE
 * ncclAllReduce(sum) of the per-key result cardinalities, uint32[K], K = keys of the span, on the
 * device.  The full result is the concatenation of the per-rank results in rank order.
 * libnccl is resolved at run time (dlopen), only when a communicator of more than one rank is made.
 * ------------------------------------------------------------------------------------- */
#define RB200_COMM_ID_BYTES 128
typedef struct rb200_comm rb200_comm_t;
/* rank 0: a fresh NCCL unique id (ncclGetUniqueId) to hand to every rank by any out-of-band means */
int rb200_comm_unique_id(char *id128);
/* every rank: ncclCommInitRank on the library's current device (nranks == 1: no NCCL at all) */
rb200_comm_t *rb200_comm_init_rank(const char *id128, int nranks, int rank);
/* or wrap an ncclComm_t the application already owns (not destroyed by rb200_comm_destroy) */
rb200_comm_t *rb200_comm_adopt(void *nccl_comm, int nranks, int rank);
int rb200_comm_size(const rb200_comm_t *c);
int rb200_comm_rank(const rb200_comm_t *c);
void rb200_comm_destroy(rb200_comm_t *c);
/* in-place all-reduce(sum) of `count` u64 words of DEVICE memory on the library stream */
int rb200_comm_allreduce_u64(rb200_comm_t *comm, uint64_t *d_buf, size_t count);
/* *d_acc (device u64) += sum of the cardinalities of every bitmap of the set, on the library stream */
int rb200_set_add_cardinality_device(const rb200_set_t *s, uint64_t *d_acc);

/* Host-side planning over portable-serialized inputs (no CUDA involved): nranks contiguous key
 * ranges [key_lo[g], key_hi[g]] covering 0..65535, balanced by container bytes per key;
 * span[0..1] = first / last key present in any input.  0 on success. */
int rb200_plan_key_ranges(const char *const *bufs, const size_t *lens, size_t n, int nranks,
                          uint32_t *key_lo, uint32_t *key_hi, uint32_t *span);
/* the bitmap restricted to keys [key_lo, key_hi] / the concatenation of bitmaps on disjoint
 * increasing key ranges, as new portable blobs (release with rb200_blob_free) */
int rb200_blob_slice_keys(const char *buf, size_t len, uint32_t key_lo, uint32_t key_hi, char **out, size_t *outlen);
int rb200_blobs_concat(const char *const *bufs, const size_t *lens, size_t n, char **out, size_t *outlen);
void rb200_blob_free(char *blob);
/* resident set holding only the containers with key in [key_lo, key_hi] of every input */
rb200_set_t *rb200_set_upload_serialized_keyrange(const char *const *bufs, const size_t *lens, size_t n,
                                                  uint32_t key_lo, uint32_t key_hi);
/* This rank's part of roaring_bitmap_or_many over S[idx[0..n)] (keys [key_lo, key_hi]) + the ONE
 * collective: per-key result cardinalities of [span_lo, span_hi] summed over the communicator on
 * the device; card_span (host, span_hi - span_lo + 1 entries) and *total_card (cardinality of the
 * whole union) are optional outputs, identical on every rank. */
rb200_set_t *rb200_or_many_sharded(const rb200_set_t *S, const uint32_t *idx, size_t n, uint32_t key_lo,
                                   uint32_t key_hi, uint32_t span_lo, uint32_t span_hi, rb200_comm_t *comm,
                                   uint32_t *card_span, uint64_t *total_card);
/* device time (ms) of the all-reduce of the last rb200_or_many_sharded call (CUDA events) */
float rb200_last_collective_ms(void);

/* Per-bitmap cardinalities of a set (host array of rb200_set_count entries); 0 on success. */
int rb200_set_cardinalities(const rb200_set_t *s, uint64_t *out);

/* Download (D2H) bitmap i / all bitmaps as host roaring_bitmap_t in the reference layout,
 * owned by the caller (free with roaring_bitmap_free or rb200_bitmap_free). */
roaring_bitmap_t *rb200_set_download(const rb200_set_t *s, size_t i);
int rb200_set_download_all(const rb200_set_t *s, roaring_bitmap_t **out);
/* Streaming download: the set is packed on the device once, then leaves it chunk by chunk
 * (<= chunk_bitmaps bitmaps / ~64 MB each, double-buffered pinned staging) while the caller
 * consumes and frees the previous chunk — bounded host memory, D2H overlapped with host work.
 *   st = rb200_download_begin(set, 1024);
 *   while ((n = rb200_download_next(st, out)) != 0 && n != (size_t)-1) { use(out, n); rb200_bitmaps_free(out, n); }
 *   rb200_download_end(st);                                                               */
typedef struct rb200_download_stream rb200_download_stream_t;
rb200_download_stream_t *rb200_download_begin(const rb200_set_t *s, size_t chunk_bitmaps);
size_t rb200_download_chunk_capacity(const rb200_download_stream_t *st);
size_t rb200_download_next(rb200_download_stream_t *st, roaring_bitmap_t **out);
void rb200_download_end(rb200_download_stream_t *st);

/* Visitor form: every bitmap of the set is materialised (reference layout) on a worker thread,
 * passed to fn(index, bitmap, ctx) and freed right after unless fn returns non-zero (callee then
 * owns it).  fn runs concurrently on several threads.  rb200_visit_sum_cardinality is a ready-made
 * visitor: *(uint64_t*)ctx += cardinality of the bitmap. */
typedef int (*rb200_visit_fn)(size_t index, roaring_bitmap_t *bitmap, void *ctx);
int rb200_download_foreach(const rb200_set_t *s, rb200_visit_fn fn, void *ctx);
/* The same over several result sets as ONE pipelined stream (all sets packed first, their chunks
 * cross PCIe back to back; the index passed to fn keeps running across the sets). */
int rb200_download_foreach_many(const rb200_set_t *const *sets, size_t nsets, rb200_visit_fn fn, void *ctx);
/* Asynchronous form: pack `s` now, stream and materialise it on a background thread (own CUDA
 * stream, 4-deep pinned ring) while the caller keeps uploading / launching ops; `s` may be freed
 * as soon as the call returns.  rb200_download_wait() drains every queued download (0 = ok). */
int rb200_download_foreach_async(const rb200_set_t *s, rb200_visit_fn fn, void *ctx);
int rb200_download_wait(void);
int rb200_visit_sum_cardinality(size_t index, roaring_bitmap_t *bitmap, void *ctx);

/* Device-side roaring_bitmap_portable_serialize of every bitmap of a set + one D2H copy:
 * blob i = *buf + (*off)[i], (*len)[i] bytes (blob starts are 16-byte aligned).  *buf is pinned
 * host memory owned by the library; release all three with rb200_serialized_free. */
int rb200_set_serialize(const rb200_set_t *s, char **buf, uint64_t **off, uint64_t **len);
void rb200_serialized_free(char *buf, uint64_t *off, uint64_t *len);
/* Frozen format (src/roaring.c:3180-3456) on the device, both directions: emit every bitmap of a
 * set as roaring_bitmap_frozen_serialize would (blob starts 32-byte aligned: frozen_view works on
 * them in place; release with rb200_serialized_free), and build a resident set from frozen blobs. */
int rb200_set_serialize_frozen(const rb200_set_t *s, char **buf, uint64_t **off, uint64_t **len);
rb200_set_t *rb200_set_upload_frozen(const char *const *bufs, const size_t *lens, size_t n);

/* Batch producers / consumers next to the path (device kernels over a whole set):
 * mode 1 = roaring_bitmap_run_optimize [src/roaring.c:1530], mode 0 = remove_run_compression, and
 * roaring_bitmap_to_uint32_array [src/roaring_array.c:426] for every bitmap of the set. */
rb200_set_t *rb200_set_run_optimize(const rb200_set_t *s, int mode);
int rb200_set_to_uint32(const rb200_set_t *s, uint32_t **vals, uint64_t **off);
void rb200_values_free(uint32_t *vals, uint64_t *off);

/* Free n host bitmaps (e.g. the results of rb200_set_download_all) using several threads. */
void rb200_bitmaps_free(roaring_bitmap_t **bitmaps, size_t n);

/* Host-to-host batch through the device (what the drop-in symbols do for one pair):
 * upload a[], b[] -> batch op -> download.  out[k] owned by the caller. 0 on success. */
int rb200_batch_op_host(int op, const roaring_bitmap_t *const *a, const roaring_bitmap_t *const *b,
                        size_t npairs, roaring_bitmap_t **out);

/* Algorithmic bytes of the last batch / many op as defined in SURVEY.md §8(d)
 * (container_size_in_bytes of matched inputs + outputs + 2x pass-through). */
uint64_t rb200_last_algorithmic_bytes(void);
/* Device time (ms) of the last batch / many op, measured with CUDA events on its stream. */
float rb200_last_device_ms(void);
/* Device time (ms) of the grid-cell kernel (k_compute_items / k_card_items / k_or_many2) alone. */
float rb200_last_compute_ms(void);
/* Bytes copied device->host by the last rb200_set_download* call (directory + payload slab). */
uint64_t rb200_last_download_bytes(void);

#ifdef __cplusplus
}
#endif
#endif /* ROARING_B200_H */
